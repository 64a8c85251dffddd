// indices.cuh -- sinks and host side of the index queries (gsb200_raster_indices, gsb200_surfel_indices): which
// gaussians each pixel composites, walking only the batches [range_start, range_end) of kIndexBatch records of its list.
//
// Two passes over the same workspace: the count pass writes the pair count of every pixel and their exclusive int64
// scan (sort.cu) and copies the total to the caller; the emit pass writes each pixel's pairs, front to back, at its
// scanned start.  The output is pixel-major over (image, row, col).
#pragma once

#include "common.cuh"

namespace gsb
{
constexpr int kIndexBatch = kTile * kTile; // records per batch of the range arguments (one per thread of a tile's CTA)

// workspace of P pixels: counts int32 [P + 1] (the last entry is 0) | starts int64 [P + 1] (starts[P] = total) | scan scratch
struct PixelCounts
{
    int32_t *counts;
    int64_t *starts;
    void *scratch;
    size_t scratch_bytes;
};
size_t pixel_counts_bytes(int64_t P);
PixelCounts carve_pixel_counts(void *workspace, int64_t P);
// exclusive scan of counts [P + 1] into starts, then total[0] = starts[P] (device to device)
int scan_pixel_counts(const PixelCounts &pc, int64_t P, int64_t *total, cudaStream_t st);

// What a pair-query walk (raster_indices_kernel of raster.cu, surfel_indices_kernel of surfel.cu) does with a pixel's
// pairs is its Sink's:
//   begin(live, pix, pix_in, image_id)  once per thread (pix: the output row, pix_in: the row-major pixel in its image)
//   pair(k, g, w)                        the pixel's k-th pair: flatten id g, weight w = alpha * T before the pair
//   end(pix, count, T)                   once per live pixel, after the walk
struct CountSink // rasterize_to_indices_in_range's count pass and rasterize_num_contributing_gaussians
{
    int32_t *counts; // [rows] pairs per pixel
    float *alphas;   // [rows] 1 - final T, or null
    __device__ __forceinline__ void begin(bool, int64_t, int64_t, int) {}
    __device__ __forceinline__ void pair(int32_t, int32_t, float) {}
    __device__ __forceinline__ void end(int64_t pix, int32_t count, float T) const
    {
        counts[pix] = count;
        if(alphas != nullptr)
            alphas[pix] = 1.0f - T;
    }
};

struct PairSink // rasterize_to_indices_in_range's emit pass: the pairs from the pixel's scanned start
{
    int64_t N;
    const int64_t *starts;
    int64_t *gaussian_ids, *pixel_ids, *image_ids;
    int64_t base, pix_in;
    int image_id;
    __device__ __forceinline__ void begin(bool live, int64_t pix, int64_t in_image, int image)
    {
        base     = live ? starts[pix] : 0;
        pix_in   = in_image;
        image_id = image;
    }
    __device__ __forceinline__ void pair(int32_t k, int32_t g, float) const
    {
        gaussian_ids[base + k] = (int64_t)g % N;
        pixel_ids[base + k]    = pix_in;
        image_ids[base + k]    = image_id;
    }
    __device__ __forceinline__ void end(int64_t, int32_t, float) const {}
};

// Argument checks and the pass sequence shared by both index queries.  `inputs_ok`: the gaussian rows, the
// transmittances, offsets and flatten_ids are given.  launch(n_tiles, b0, b1, sink) launches the pass's kernel with its
// sink: CountSink for the count pass (emit = 0), PairSink for the emit pass.
template<class Launch>
int run_index_pass(
    int64_t I, int64_t N, uint32_t W, uint32_t H, uint32_t tile_size, uint32_t tw, uint32_t th, int64_t n_isects,
    int64_t range_start, int64_t range_end, bool inputs_ok, int emit, void *workspace, size_t workspace_bytes, int64_t *total,
    int64_t *gaussian_ids, int64_t *pixel_ids, int64_t *image_ids, cudaStream_t st, Launch &&launch
)
{
    if(I < 0 || N < 0 || n_isects < 0 || range_start < 0 || range_end < 0)
        return GSB200_E_INVALID;
    if(tile_size != (uint32_t)kTile)
        return GSB200_E_UNSUPPORTED;
    if(!emit && total == nullptr)
        return GSB200_E_INVALID;
    const int64_t P = I * (int64_t)H * (int64_t)W;
    if(P == 0 || N == 0 || n_isects == 0 || range_end <= range_start)
    { // no pairs: nothing to launch
        if(!emit)
            GSB_CUDA_TRY(cudaMemsetAsync(total, 0, sizeof(int64_t), st));
        return GSB200_OK;
    }
    if(!inputs_ok || (emit && !(gaussian_ids && pixel_ids && image_ids)) || !tile_grid_covers(tw, th, W, H))
        return GSB200_E_INVALID;
    if(workspace == nullptr || workspace_bytes < pixel_counts_bytes(P))
        return GSB200_E_WORKSPACE;
    if((double)I * tw * th >= 2147483648.0 || n_isects >= 2147483648LL)
        return GSB200_E_UNSUPPORTED;
    // a range beyond the last batch of every list means "to the end" (no list has 2^31 batches)
    const int32_t b0 = (int32_t)(range_start < 0x7fffffffLL ? range_start : 0x7fffffffLL);
    const int32_t b1 = (int32_t)(range_end < 0x7fffffffLL ? range_end : 0x7fffffffLL);
    const unsigned n_tiles = (unsigned)(I * tw * th);
    const PixelCounts pc   = carve_pixel_counts(workspace, P);
    if(emit)
        return launch(n_tiles, b0, b1, PairSink{N, pc.starts, gaussian_ids, pixel_ids, image_ids});
    GSB_CUDA_TRY(cudaMemsetAsync(pc.counts + P, 0, sizeof(int32_t), st));
    if(int rc = launch(n_tiles, b0, b1, CountSink{pc.counts, nullptr}))
        return rc;
    return scan_pixel_counts(pc, P, total, st);
}
} // namespace gsb
