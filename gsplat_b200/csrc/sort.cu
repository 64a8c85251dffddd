// sort.cu -- the library-level functions (version, error strings, last CUDA error), the sparse pixel layout, a
// cub::DeviceRadixSort::SortPairs over one key per requested pixel, and the pixel-count scan of the index queries.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "indices.cuh"

namespace gsb
{
static thread_local cudaError_t g_last_error = cudaSuccess;
void set_last_cuda_error(cudaError_t e) { g_last_error = e; }
} // namespace gsb

extern "C" const char *gsb200_version(void) { return "gsplat_b200 0.1.0 (sm_90a)"; }

extern "C" const char *gsb200_error_string(int code)
{
    switch(code)
    {
    case GSB200_OK: return "ok";
    case GSB200_E_INVALID: return "invalid argument";
    case GSB200_E_UNSUPPORTED: return "unsupported configuration (camera model / channel count / tile size not built)";
    case GSB200_E_CUDA: return "CUDA error";
    case GSB200_E_WORKSPACE: return "workspace too small";
    case GSB200_E_KEYBITS: return "intersect_tile: (image, tile) id packing needs more than 32 bits";
    default: return "unknown error";
    }
}

extern "C" const char *gsb200_last_cuda_error(void) { return cudaGetErrorString(gsb::g_last_error); }

extern "C" uint32_t gsb200_bits_for_count(int64_t count) { return gsb::bits_for_count(count); }

// ---- sparse tile layout (build_sparse_tile_layout): which tiles hold requested pixels, which pixels of each tile, and
// where each pixel's output goes.  One key per pixel, dense tile id << 8 | in-tile raster position, sorted stably with
// its pixel index; the runs of equal tile ids are the active tiles (ascending), their bits the in-tile masks, their
// ends the inclusive pixel cumsum, and the sorted pixel indices the pixel map.  Two calls: the sort, after which the
// caller reads the number of active tiles (n_active, device int64) and sizes the outputs, then the finish.
namespace gsb
{
constexpr int kPosBits = 8; // in-tile position bits of a 16 x 16 tile

__global__ void __launch_bounds__(256) sparse_pixel_keys_kernel(
    int64_t P, const int32_t *__restrict__ pixels, const int32_t *__restrict__ image_ids, uint32_t tw, uint32_t th,
    int64_t *__restrict__ keys, int32_t *__restrict__ vals
)
{
    const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(p >= P)
        return;
    const int2 rc       = reinterpret_cast<const int2 *>(pixels)[p]; // (row, col)
    const int64_t tile  = ((int64_t)image_ids[p] * th + rc.x / kTile) * tw + rc.y / kTile;
    const int64_t pos   = (rc.x % kTile) * kTile + rc.y % kTile;
    keys[p]             = (tile << kPosBits) | pos;
    vals[p]             = (int32_t)p;
}

// heads[k] = 1 where a run of equal tile ids starts
__global__ void __launch_bounds__(256) sparse_run_heads_kernel(int64_t P, const int64_t *__restrict__ keys, int32_t *__restrict__ heads)
{
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(k >= P)
        return;
    heads[k] = (k == 0 || (keys[k] >> kPosBits) != (keys[k - 1] >> kPosBits)) ? 1 : 0;
}

__global__ void sparse_n_active_kernel(int64_t P, const int32_t *__restrict__ run, int64_t *__restrict__ n_active)
{
    n_active[0] = run[P - 1];
}

// run[k] = 1-based index of the active tile of sorted pixel k
__global__ void __launch_bounds__(256) sparse_layout_finish_kernel(
    int64_t P, const int64_t *__restrict__ keys, const int32_t *__restrict__ vals, const int32_t *__restrict__ run,
    int32_t *__restrict__ active_tiles, uint8_t *__restrict__ active_tile_mask, unsigned long long *__restrict__ tile_pixel_mask,
    int64_t *__restrict__ tile_pixel_cumsum, int64_t *__restrict__ pixel_map
)
{
    const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(k >= P)
        return;
    const int64_t key  = keys[k];
    const int64_t tile = key >> kPosBits;
    const int pos      = (int)(key & ((1 << kPosBits) - 1));
    const int32_t r    = run[k] - 1;
    pixel_map[k]       = vals[k];
    // duplicate pixels set the same bit: the rank of a bit then stays below the tile's pixel count
    atomicOr(tile_pixel_mask + (size_t)r * 4 + (pos >> 6), 1ull << (pos & 63));
    if(k == 0 || run[k - 1] != run[k])
    {
        active_tiles[r]        = (int32_t)tile;
        active_tile_mask[tile] = 1;
    }
    if(k == P - 1 || run[k + 1] != run[k])
        tile_pixel_cumsum[r] = k + 1;
}

struct SparseLayout
{
    size_t keys_in, keys_out, vals_in, vals_out, heads, run, cub, total;
};
static SparseLayout sparse_layout(int64_t P, int end_bit)
{
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    SparseLayout L;
    size_t scan = 0, sort = 0;
    cub::DeviceScan::InclusiveSum((void *)nullptr, scan, (const int32_t *)nullptr, (int32_t *)nullptr, P);
    cub::DeviceRadixSort::SortPairs(
        (void *)nullptr, sort, (const int64_t *)nullptr, (int64_t *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr, P, 0, end_bit
    );
    L.keys_in  = 0;
    L.keys_out = L.keys_in + al(sizeof(int64_t) * (size_t)P);
    L.vals_in  = L.keys_out + al(sizeof(int64_t) * (size_t)P);
    L.vals_out = L.vals_in + al(sizeof(int32_t) * (size_t)P);
    L.heads    = L.vals_out + al(sizeof(int32_t) * (size_t)P);
    L.run      = L.heads + al(sizeof(int32_t) * (size_t)P);
    L.cub      = L.run + al(sizeof(int32_t) * (size_t)P);
    L.total    = L.cub + al(scan > sort ? scan : sort) + 256;
    return L;
}

static int sparse_layout_args(int64_t P, int64_t n_images, uint32_t tile_size, uint32_t tw, uint32_t th, int &end_bit)
{
    if(tile_size != (uint32_t)kTile)
        return GSB200_E_UNSUPPORTED;
    if(P < 0 || P > 0x7fffffffLL || n_images < 0 || n_images * (int64_t)tw * th >= (1LL << 31))
        return GSB200_E_INVALID;
    end_bit = kPosBits + (int)bits_for_count(n_images * (int64_t)tw * th);
    return GSB200_OK;
}
} // namespace gsb

extern "C" size_t gsb200_sparse_layout_workspace_bytes(int64_t P, int64_t n_images, uint32_t tile_width, uint32_t tile_height)
{
    int end_bit = 0;
    if(P <= 0 || gsb::sparse_layout_args(P, n_images, (uint32_t)gsb::kTile, tile_width, tile_height, end_bit) != GSB200_OK)
        return 0;
    return gsb::sparse_layout(P, end_bit).total;
}

// pixels int32 [P, 2] (row, col) inside the tile grid, image_ids int32 [P] in [0, n_images) (checked by the caller)
extern "C" int gsb200_sparse_layout_sort(
    int64_t P, const int32_t *pixels, const int32_t *image_ids, int64_t n_images, uint32_t tile_size, uint32_t tile_width,
    uint32_t tile_height, void *workspace, size_t workspace_bytes, int64_t *n_active, void *stream
)
{
    int end_bit = 0;
    if(int rc = gsb::sparse_layout_args(P, n_images, tile_size, tile_width, tile_height, end_bit))
        return rc;
    if(!n_active)
        return GSB200_E_INVALID;
    cudaStream_t st = (cudaStream_t)stream;
    if(P == 0)
    {
        GSB_CUDA_TRY(cudaMemsetAsync(n_active, 0, sizeof(int64_t), st));
        return GSB200_OK;
    }
    if(!pixels || !image_ids || !workspace)
        return GSB200_E_INVALID;
    const auto L = gsb::sparse_layout(P, end_bit);
    if(L.total > workspace_bytes)
        return GSB200_E_WORKSPACE;
    char *ws         = static_cast<char *>(workspace);
    int64_t *k_in    = reinterpret_cast<int64_t *>(ws + L.keys_in), *k_out = reinterpret_cast<int64_t *>(ws + L.keys_out);
    int32_t *v_in    = reinterpret_cast<int32_t *>(ws + L.vals_in), *v_out = reinterpret_cast<int32_t *>(ws + L.vals_out);
    int32_t *heads   = reinterpret_cast<int32_t *>(ws + L.heads), *run = reinterpret_cast<int32_t *>(ws + L.run);
    const size_t cub_bytes = L.total - L.cub;
    gsb::sparse_pixel_keys_kernel<<<gsb::grid_for(P, 256), 256, 0, st>>>(P, pixels, image_ids, tile_width, tile_height, k_in, v_in);
    if(int rc = gsb::check_launch())
        return rc;
    size_t sort_bytes = cub_bytes;
    GSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + L.cub, sort_bytes, k_in, k_out, v_in, v_out, P, 0, end_bit, st));
    gsb::sparse_run_heads_kernel<<<gsb::grid_for(P, 256), 256, 0, st>>>(P, k_out, heads);
    if(int rc = gsb::check_launch())
        return rc;
    size_t scan_bytes = cub_bytes;
    GSB_CUDA_TRY(cub::DeviceScan::InclusiveSum(ws + L.cub, scan_bytes, heads, run, P, st));
    gsb::sparse_n_active_kernel<<<1, 1, 0, st>>>(P, run, n_active);
    return gsb::check_launch();
}

// outputs: active_tiles int32 [n_active], active_tile_mask bool bytes [n_images, th, tw], tile_pixel_mask uint64
// [n_active, 4], tile_pixel_cumsum int64 [n_active], pixel_map int64 [P]; n_active as read back after the sort
extern "C" int gsb200_sparse_layout_finish(
    int64_t P, int64_t n_images, uint32_t tile_width, uint32_t tile_height, int64_t n_active, const void *workspace,
    size_t workspace_bytes, int32_t *active_tiles, uint8_t *active_tile_mask, uint64_t *tile_pixel_mask,
    int64_t *tile_pixel_cumsum, int64_t *pixel_map, void *stream
)
{
    int end_bit = 0;
    if(int rc = gsb::sparse_layout_args(P, n_images, (uint32_t)gsb::kTile, tile_width, tile_height, end_bit))
        return rc;
    if(n_active < 0 || n_active > P || (n_images > 0 && !active_tile_mask))
        return GSB200_E_INVALID;
    cudaStream_t st = (cudaStream_t)stream;
    if(n_images > 0)
        GSB_CUDA_TRY(cudaMemsetAsync(active_tile_mask, 0, (size_t)n_images * tile_width * tile_height, st));
    if(P == 0)
        return GSB200_OK;
    if(!workspace || !active_tiles || !tile_pixel_mask || !tile_pixel_cumsum || !pixel_map || n_active == 0)
        return GSB200_E_INVALID;
    const auto L = gsb::sparse_layout(P, end_bit);
    if(L.total > workspace_bytes)
        return GSB200_E_WORKSPACE;
    const char *ws = static_cast<const char *>(workspace);
    GSB_CUDA_TRY(cudaMemsetAsync(tile_pixel_mask, 0, sizeof(uint64_t) * 4 * (size_t)n_active, st));
    gsb::sparse_layout_finish_kernel<<<gsb::grid_for(P, 256), 256, 0, st>>>(
        P, reinterpret_cast<const int64_t *>(ws + L.keys_out), reinterpret_cast<const int32_t *>(ws + L.vals_out),
        reinterpret_cast<const int32_t *>(ws + L.run), active_tiles, active_tile_mask,
        reinterpret_cast<unsigned long long *>(tile_pixel_mask), tile_pixel_cumsum, pixel_map
    );
    return gsb::check_launch();
}

// ---- per-pixel pair counts of the index queries (indices.cuh): exclusive int64 scan of int32 counts
namespace gsb
{
static size_t align256_bytes(size_t b) { return (b + 255) & ~(size_t)255; }

static size_t pixel_scan_scratch(int64_t P)
{
    size_t bytes = 0;
    cub::DeviceScan::ExclusiveScan(
        (void *)nullptr, bytes, (const int32_t *)nullptr, (int64_t *)nullptr, cuda::std::plus<int64_t>{}, (int64_t)0, P + 1
    );
    return bytes;
}

size_t pixel_counts_bytes(int64_t P)
{
    return align256_bytes(sizeof(int32_t) * (size_t)(P + 1)) + align256_bytes(sizeof(int64_t) * (size_t)(P + 1))
         + align256_bytes(pixel_scan_scratch(P));
}

PixelCounts carve_pixel_counts(void *workspace, int64_t P)
{
    char *p             = (char *)workspace;
    const size_t counts = align256_bytes(sizeof(int32_t) * (size_t)(P + 1));
    const size_t starts = align256_bytes(sizeof(int64_t) * (size_t)(P + 1));
    return {(int32_t *)p, (int64_t *)(p + counts), p + counts + starts, pixel_scan_scratch(P)};
}

int scan_pixel_counts(const PixelCounts &pc, int64_t P, int64_t *total, cudaStream_t st)
{
    size_t bytes = pc.scratch_bytes;
    GSB_CUDA_TRY(cub::DeviceScan::ExclusiveScan(
        pc.scratch, bytes, (const int32_t *)pc.counts, pc.starts, cuda::std::plus<int64_t>{}, (int64_t)0, P + 1, st
    ));
    GSB_CUDA_TRY(cudaMemcpyAsync(total, pc.starts + P, sizeof(int64_t), cudaMemcpyDeviceToDevice, st));
    return GSB200_OK;
}
} // namespace gsb

extern "C" size_t gsb200_indices_workspace_bytes(int64_t n_pixels)
{
    if(n_pixels < 0)
        return 0;
    return gsb::pixel_counts_bytes(n_pixels);
}
