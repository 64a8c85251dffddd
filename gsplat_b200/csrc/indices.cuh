// indices.cuh -- sinks and host side of the index queries (gsb200_raster_indices, gsb200_surfel_indices,
// gsb200_eval3d_indices): which gaussians each pixel composites, walking only the batches [range_start, range_end) of
// kIndexBatch records of its list; and of the per-pixel contributor queries of the three walks (gsb200_contrib_*,
// gsb200_surfel_contrib_*, gsb200_eval3d_contrib_*).
//
// Two passes over the same workspace: the count pass writes the pair count of every pixel and their exclusive int64
// scan (sort.cu) and copies the total to the caller; the emit pass writes each pixel's pairs, front to back, at its
// scanned start.  The output is pixel-major over (image, row, col).
#pragma once

#include <algorithm>
#include <initializer_list>

#include "common.cuh"
#include "pixels.cuh"

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

// What a pair-query walk (raster_indices_kernel of raster.cu, pair_walk_kernel below with the models of surfel.cu and
// ut.cu) does with a pixel's pairs is its Sink's (every walk runs kIndexBatch threads per CTA, one pixel per thread):
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

// rasterize_contributing_gaussian_ids: the first K pairs of a pixel at [pix, k] (later ones are dropped, as the
// reference drops them), -1 / 0 after its last pair; nothing outside the pixel's row of K.
struct IdsSink
{
    int32_t N, K;
    int32_t *ids;   // [rows, K] g % N
    float *weights; // [rows, K] alpha * T before the pair
    int64_t row;
    __device__ __forceinline__ void begin(bool, int64_t pix, int64_t, int) { row = pix * K; }
    __device__ __forceinline__ void pair(int32_t k, int32_t g, float w) const
    {
        if(k < K)
        {
            ids[row + k]     = g % N;
            weights[row + k] = w;
        }
    }
    __device__ __forceinline__ void end(int64_t, int32_t count, float) const
    {
        for(int32_t k = count < K ? count : K; k < K; ++k)
        {
            ids[row + k]     = -1;
            weights[row + k] = 0.f;
        }
    }
};

// rasterize_top_contributing_gaussian_ids: K slots per pixel in dynamic shared memory ({id, weight, walk position},
// slot k of thread t at [k * kIndexBatch + t]: conflict-free).  The reference's rule: empty slots hold -1, 0, +inf; a
// pair replaces the lowest-weight slot (the first on ties) only when strictly heavier; at the end the slots are sorted
// by walk position (stable), i.e. front to back with the empty ones last.
struct TopSink
{
    static constexpr size_t kSlotBytes = sizeof(int32_t) + sizeof(float) + sizeof(uint32_t);
    int32_t N, K;
    int32_t *ids;   // [rows, K]
    float *weights; // [rows, K]
    int64_t row;
    int32_t *s_id;
    float *s_w;
    uint32_t *s_pos;
    __device__ __forceinline__ void begin(bool, int64_t pix, int64_t, int)
    {
        extern __shared__ __align__(16) int32_t s_top_slots[];
        const size_t plane = (size_t)K * kIndexBatch;
        s_id  = s_top_slots + threadIdx.x;
        s_w   = reinterpret_cast<float *>(s_top_slots + plane) + threadIdx.x;
        s_pos = reinterpret_cast<uint32_t *>(s_top_slots + 2 * plane) + threadIdx.x;
        row   = pix * K;
        for(int32_t k = 0; k < K; ++k)
        {
            s_id[k * kIndexBatch]  = -1;
            s_w[k * kIndexBatch]   = 0.f;
            s_pos[k * kIndexBatch] = 0xffffffffu;
        }
    }
    __device__ __forceinline__ void pair(int32_t k, int32_t g, float w) const
    {
        int32_t m = 0;
        float wm  = s_w[0];
        for(int32_t j = 1; j < K; ++j)
        {
            const float v = s_w[j * kIndexBatch];
            if(v < wm)
            {
                wm = v;
                m  = j;
            }
        }
        if(w > wm)
        {
            s_w[m * kIndexBatch]   = w;
            s_id[m * kIndexBatch]  = g % N;
            s_pos[m * kIndexBatch] = (uint32_t)k;
        }
    }
    __device__ __forceinline__ void end(int64_t, int32_t, float) const
    {
        for(int32_t i = 1; i < K; ++i)
        {
            const uint32_t p = s_pos[i * kIndexBatch];
            const float w    = s_w[i * kIndexBatch];
            const int32_t id = s_id[i * kIndexBatch];
            int32_t j        = i - 1;
            for(; j >= 0 && s_pos[j * kIndexBatch] > p; --j)
            {
                s_pos[(j + 1) * kIndexBatch] = s_pos[j * kIndexBatch];
                s_w[(j + 1) * kIndexBatch]   = s_w[j * kIndexBatch];
                s_id[(j + 1) * kIndexBatch]  = s_id[j * kIndexBatch];
            }
            s_pos[(j + 1) * kIndexBatch] = p;
            s_w[(j + 1) * kIndexBatch]   = w;
            s_id[(j + 1) * kIndexBatch]  = id;
        }
        for(int32_t k = 0; k < K; ++k)
        {
            ids[row + k]     = s_id[k * kIndexBatch];
            weights[row + k] = s_w[k * kIndexBatch];
        }
    }
};

// The pair-query walk of the 2DGS and 3DGUT queries: the (pixel, gaussian) pairs a family's compositing forward
// composites, walking only the batches [b0, b1) of each tile's list from the pixel's given transmittance (null: T = 1).
// One CTA per 16x16 tile of the pixel policy (DensePixels: every tile of the [I, th, tw] grid; SparsePixels: every
// active tile), one pixel per thread; a pixel is live when it has an output row.  The Model (SurfelModel of surfel.cu,
// Eval3dModel of ut.cu) is the forward's:
//   I, W, H, tw, th                           the tile grid
//   kMinBlocks                                the forward's minimum of resident CTAs (launch bounds; 0: none)
//   Rec, stage(rec, g)                        the staged record of flatten id g (one per thread of a batch)
//   Pixel, setup(img, i, j, live, px) -> bool  the pixel's state; whether it composites.  Called by every thread.
//   hit(rec, px) -> {ok, alpha}               the forward's evaluation of one record at the pixel
// A live pixel that does not composite still gets begin and end (count 0, T as given).  Every thread stages records and
// meets every barrier.  The stop rule is the forward's, so the alphas are its render_alphas bit for bit.
template<class Model, class Sink, class Pix = DensePixels>
__global__ void __launch_bounds__(kIndexBatch, Model::kMinBlocks) pair_walk_kernel(
    Model model, const float *__restrict__ transmittances, const int32_t *__restrict__ offsets,
    const int32_t *__restrict__ flatten_ids, int64_t n_isects, int32_t b0, int32_t b1, Sink sink, const Pix pixmap = Pix{}
)
{
    __shared__ typename Model::Rec rec[kIndexBatch];
    const uint32_t tile  = pixmap.tile(blockIdx.x); // image * th * tw + tile row * tw + tile col
    const uint32_t img   = tile / (model.tw * model.th);
    const uint32_t tin   = tile - img * model.tw * model.th;
    const uint32_t tr    = threadIdx.x;
    const uint32_t i     = (tin / model.tw) * kTile + tr / kTile;
    const uint32_t j     = (tin % model.tw) * kTile + tr % kTile;
    const int64_t pix_in = (int64_t)i * model.W + j;
    bool live;
    int64_t pix, start, end;
    if constexpr(Pix::kSparse)
    {
        pix   = pixmap.slot(blockIdx.x, (int)tr, live);
        start = offsets[blockIdx.x];
        end   = offsets[blockIdx.x + 1];
    }
    else
    {
        live  = i < model.H && j < model.W;
        pix   = (int64_t)img * model.H * model.W + pix_in;
        start = offsets[tile];
        end   = (tile + 1 == model.I * model.tw * model.th) ? n_isects : offsets[tile + 1];
    }
    const int64_t b_end = min((int64_t)b1, (end - start + kIndexBatch - 1) / kIndexBatch);
    typename Model::Pixel px;
    bool done   = !model.setup(img, i, j, live, px);
    float T     = (live && transmittances != nullptr) ? transmittances[pix] : 1.f;
    int32_t cnt = 0;
    sink.begin(live, pix, pix_in, img);
    for(int64_t b = b0; b < b_end; ++b)
    {
        if(__syncthreads_count(done) == kIndexBatch)
            break;
        const int64_t batch = start + b * kIndexBatch;
        if(batch + tr < end)
            model.stage(rec[tr], flatten_ids[batch + tr]);
        __syncthreads();
        const int n_b = (int)min((int64_t)kIndexBatch, end - batch);
        for(int t = 0; t < n_b && !done; ++t)
        {
            const auto h = model.hit(rec[t], px);
            if(!h.ok)
                continue;
            const float next_T = T * (1.f - h.alpha);
            if(next_T <= kTransmittanceThreshold)
            { // exclusive: this gaussian does not contribute
                done = true;
                break;
            }
            sink.pair(cnt, rec[t].id, h.alpha * T);
            ++cnt;
            T = next_T;
        }
    }
    if(live)
        sink.end(pix, cnt, T);
}

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

// ---- per-pixel contributor queries: the full walk from T = 1 with one sink, over every tile (dense) or over the active
// tiles of a sparse layout (active_tiles != null).  The checks run in run_index_pass's order with its return codes;
// every pixel is written, also when there are no intersections.
//
// The arguments of the C entries that do not depend on what a walk composites; the walk (below) carries the rest.
struct ContribArgs
{
    int64_t I, N;
    uint32_t W, H, tile_size, tw, th;
    const int32_t *offsets, *flatten_ids;
    int64_t n_isects, n_active;
    const int32_t *active_tiles;
    const uint64_t *tile_pixel_mask;
    const int64_t *tile_pixel_cumsum, *pixel_map;
};

// ContribArgs from the parameters of a contributor entry, named as gsb200_contrib_count's, over I images
#define GSB200_CONTRIB_ARGS(I)                                                                                          \
    gsb::ContribArgs                                                                                                    \
    {                                                                                                                   \
        I, N, image_width, image_height, tile_size, tile_width, tile_height, offsets, flatten_ids, n_isects, n_active,   \
            active_tiles, tile_pixel_mask, tile_pixel_cumsum, pixel_map                                                 \
    }

// The rows of the 2-D walks (raster.cu, surfel.cu): means2d [R, 2], conics [R, 3] or ray_transforms [R, 3, 3],
// opacities [R].  They are read only when there are intersections.
struct PlanarRows
{
    const float *means2d, *rows, *opacities;
    bool inputs_ok(int64_t n_isects) const { return n_isects == 0 || (means2d && rows && opacities); }
};

// A Walk is one unit's pair-query kernel with what it composites:
//   walk.inputs_ok(n_isects)                        whether what it reads is given
//   walk.launch(a, n_tiles, pixmap, sink, smem, st)  launches it over n_tiles CTAs from T = 1 through the whole lists
//   Walk::max_samples()                             the largest K of its TopSink on the current device (top_max_samples)
// launch_walk and top_max_samples are the steps every walk takes.
template<class... Params, class... Args>
int launch_walk(void (*kernel)(Params...), unsigned n_tiles, size_t smem, cudaStream_t st, const Args &...args)
{
    if(smem > 0) // TopSink's slots
        GSB_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<n_tiles, kIndexBatch, smem, st>>>(args...);
    return check_launch();
}

// largest K of a top-K walk on the current device: its opt-in shared memory per block, less the static shared memory
// (the staging arrays) of the largest of its TopSink instantiations, over the K slots of every thread
inline int top_max_samples(std::initializer_list<const void *> walks)
{
    int dev = 0, optin = 0;
    GSB_CUDA_TRY(cudaGetDevice(&dev));
    GSB_CUDA_TRY(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    size_t staging = 0;
    for(const void *k : walks)
    {
        cudaFuncAttributes a;
        GSB_CUDA_TRY(cudaFuncGetAttributes(&a, k));
        staging = std::max(staging, a.sharedSizeBytes);
    }
    if((size_t)optin <= staging)
        return 0;
    return (int)(((size_t)optin - staging) / ((size_t)kIndexBatch * TopSink::kSlotBytes));
}

template<class Walk, class Sink>
int run_contrib(const Walk &walk, const ContribArgs &a, bool outputs_ok, size_t smem, const Sink &sink, cudaStream_t st)
{
    const bool sparse = a.active_tiles != nullptr;
    if(a.I < 0 || a.N < 0 || a.n_isects < 0 || a.n_active < 0)
        return GSB200_E_INVALID;
    if(a.tile_size != (uint32_t)kTile)
        return GSB200_E_UNSUPPORTED;
    const int64_t n_tiles = sparse ? a.n_active : a.I * (int64_t)a.tw * a.th;
    if(n_tiles == 0 || a.W == 0 || a.H == 0)
        return GSB200_OK; // no pixels
    const bool inputs_ok = a.offsets && walk.inputs_ok(a.n_isects) && (a.n_isects == 0 || a.flatten_ids)
                        && (!sparse || (a.tile_pixel_mask && a.tile_pixel_cumsum && a.pixel_map));
    if(!inputs_ok || !outputs_ok || !tile_grid_covers(a.tw, a.th, a.W, a.H))
        return GSB200_E_INVALID;
    if(n_tiles >= 2147483648LL || a.n_isects >= 2147483648LL)
        return GSB200_E_UNSUPPORTED;
    if(sparse)
        return walk.launch(a, (unsigned)n_tiles, SparsePixels{a.active_tiles, a.tile_pixel_mask, a.tile_pixel_cumsum, a.pixel_map}, sink, smem, st);
    return walk.launch(a, (unsigned)n_tiles, DensePixels{}, sink, smem, st);
}

// count: CountSink
template<class Walk>
int contrib_count(const Walk &walk, const ContribArgs &a, int32_t *counts, float *alphas, cudaStream_t st)
{
    return run_contrib(walk, a, counts != nullptr, 0, CountSink{counts, alphas}, st);
}

// ids: IdsSink; max_samples = 0 writes nothing
template<class Walk>
int contrib_ids(const Walk &walk, const ContribArgs &a, int max_samples, int32_t *ids, float *weights, cudaStream_t st)
{
    if(max_samples < 0 || a.N > 0x7fffffffLL)
        return GSB200_E_INVALID;
    if(max_samples == 0)
        return GSB200_OK;
    return run_contrib(walk, a, ids && weights, 0, IdsSink{(int32_t)a.N, max_samples, ids, weights, 0}, st);
}

// top: TopSink, num_samples in [1, Walk::max_samples()]
template<class Walk>
int contrib_top(const Walk &walk, const ContribArgs &a, int num_samples, int32_t *ids, float *weights, cudaStream_t st)
{
    if(num_samples <= 0 || a.N > 0x7fffffffLL)
        return GSB200_E_INVALID;
    const int bound = Walk::max_samples();
    if(bound < 0)
        return bound;
    if(num_samples > bound)
        return GSB200_E_UNSUPPORTED;
    const TopSink sink{(int32_t)a.N, num_samples, ids, weights, 0, nullptr, nullptr, nullptr};
    const size_t smem = (size_t)num_samples * kIndexBatch * TopSink::kSlotBytes;
    return run_contrib(walk, a, ids && weights, smem, sink, st);
}
} // namespace gsb
