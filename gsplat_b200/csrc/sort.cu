// sort.cu -- (isect_id, flatten_id) radix sort and library-level helpers.
//
// The sorts are cub::DeviceRadixSort::SortPairs (the library call the reference makes,
// csrc/IntersectTile.cu:1078-1121; its onesweep kernels are compiled here for sm_90a), used twice:
// once over the N projected rows on (image, depth) and once over the S intersections on the (image, tile)
// bits only -- see gsb200_isect_depth_order below.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include "common.cuh"

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

extern "C" size_t gsb200_sort_workspace_bytes(int64_t n_isects, int begin_bit, int end_bit)
{
    if(n_isects <= 0)
        return 0;
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(
        (void *)nullptr, bytes, (const int64_t *)nullptr, (int64_t *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr,
        n_isects, begin_bit, end_bit
    );
    return bytes + 256;
}

// Stable LSD radix sort of the (key, value) pairs on key bits [begin_bit, end_bit).
extern "C" int gsb200_sort_pairs(
    int64_t n_isects, int begin_bit, int end_bit, const int64_t *keys_in, const int32_t *vals_in, int64_t *keys_out,
    int32_t *vals_out, void *workspace, size_t workspace_bytes, void *stream
)
{
    if(n_isects < 0 || begin_bit < 0 || end_bit < begin_bit || end_bit > 64)
        return GSB200_E_INVALID;
    if(n_isects == 0)
        return GSB200_OK;
    if(!keys_in || !vals_in || !keys_out || !vals_out || !workspace)
        return GSB200_E_INVALID;
    cudaStream_t st = (cudaStream_t)stream;
    size_t need     = 0;
    cub::DeviceRadixSort::SortPairs((void *)nullptr, need, keys_in, keys_out, vals_in, vals_out, n_isects, begin_bit, end_bit, st);
    if(need > workspace_bytes)
        return GSB200_E_WORKSPACE;
    GSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(workspace, need, keys_in, keys_out, vals_in, vals_out, n_isects, begin_bit, end_bit, st));
    return GSB200_OK;
}

// Narrow variant for the (image, tile)-only sort of the depth-ordered intersections: 2- or 4-byte dense tile ids
// as keys, the row index as value -- 6 (8) instead of 12 bytes per intersection and direction in each radix pass.
namespace gsb
{
template<class KeyT>
static int sort_tile_pairs(
    int64_t n, int end_bit, const void *keys_in, const int32_t *vals_in, void *keys_out, int32_t *vals_out, void *workspace,
    size_t workspace_bytes, cudaStream_t st
)
{
    size_t need = 0;
    cub::DeviceRadixSort::SortPairs(
        (void *)nullptr, need, static_cast<const KeyT *>(keys_in), static_cast<KeyT *>(keys_out), vals_in, vals_out, n, 0, end_bit, st
    );
    if(need > workspace_bytes)
        return GSB200_E_WORKSPACE;
    GSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(
        workspace, need, static_cast<const KeyT *>(keys_in), static_cast<KeyT *>(keys_out), vals_in, vals_out, n, 0, end_bit, st
    ));
    return GSB200_OK;
}
} // namespace gsb

extern "C" size_t gsb200_sort_tile_pairs_workspace_bytes(int64_t n_isects, int key_bytes, int end_bit)
{
    if(n_isects <= 0)
        return 0;
    size_t bytes = 0;
    if(key_bytes == 2)
        cub::DeviceRadixSort::SortPairs(
            (void *)nullptr, bytes, (const uint16_t *)nullptr, (uint16_t *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr,
            n_isects, 0, end_bit
        );
    else
        cub::DeviceRadixSort::SortPairs(
            (void *)nullptr, bytes, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr,
            n_isects, 0, end_bit
        );
    return bytes + 256;
}

extern "C" int gsb200_sort_tile_pairs(
    int64_t n_isects, int key_bytes, int end_bit, const void *keys_in, const int32_t *vals_in, void *keys_out, int32_t *vals_out,
    void *workspace, size_t workspace_bytes, void *stream
)
{
    if(n_isects < 0 || (key_bytes != 2 && key_bytes != 4) || end_bit < 0 || end_bit > 8 * key_bytes)
        return GSB200_E_INVALID;
    if(n_isects == 0)
        return GSB200_OK;
    if(!keys_in || !vals_in || !keys_out || !vals_out || !workspace)
        return GSB200_E_INVALID;
    cudaStream_t st = (cudaStream_t)stream;
    if(key_bytes == 2)
        return gsb::sort_tile_pairs<uint16_t>(n_isects, end_bit, keys_in, vals_in, keys_out, vals_out, workspace, workspace_bytes, st);
    return gsb::sort_tile_pairs<uint32_t>(n_isects, end_bit, keys_in, vals_in, keys_out, vals_out, workspace, workspace_bytes, st);
}

// ---- depth order of the projected gaussians (pre-pass of the tile intersection)
// The reference sorts all S intersections on (image, tile, depth) = 45+ key bits.  Sorting the rows ONCE by
// (image, depth) and emitting the intersections in that order leaves only the (image, tile) bits for the
// S-sized sort: both sorts are stable, so inside a tile the result is (depth, then row index) -- exactly the
// order the reference's single stable sort produces (csrc/Intersect.cpp:283-326).
namespace gsb
{
__global__ void __launch_bounds__(256) depth_key_kernel(
    int64_t total, int64_t N, const int32_t *__restrict__ radii, const float *__restrict__ depths,
    const int64_t *__restrict__ image_ids, uint64_t *__restrict__ keys, int32_t *__restrict__ rows
)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= total)
        return;
    const int2 r = reinterpret_cast<const int2 *>(radii)[i];
    uint64_t k   = ~0ull; // culled rows go last
    if(r.x > 0 && r.y > 0)
        k = ((uint64_t)(image_ids ? image_ids[i] : i / N) << 32) | (uint64_t)__float_as_uint(depths[i]);
    keys[i] = k;
    rows[i] = (int32_t)i;
}

// single image: the key is the depth's bit pattern alone (culled rows 0xffffffff sort last; a visible depth is a
// positive finite float, never that pattern) -- 8 instead of 12 bytes per row and pass
__global__ void __launch_bounds__(256) depth_key32_kernel(
    int64_t total, const int32_t *__restrict__ radii, const float *__restrict__ depths, uint32_t *__restrict__ keys,
    int32_t *__restrict__ rows
)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= total)
        return;
    const int2 r = reinterpret_cast<const int2 *>(radii)[i];
    keys[i]      = (r.x > 0 && r.y > 0) ? __float_as_uint(depths[i]) : 0xffffffffu;
    rows[i]      = (int32_t)i;
}

struct DepthOrderLayout
{
    size_t keys_in, keys_out, rows_in, cub, total;
};
static DepthOrderLayout depth_order_layout(int64_t total, int end_bit)
{
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    DepthOrderLayout L;
    size_t cub_bytes = 0;
    cub::DeviceRadixSort::SortPairs(
        (void *)nullptr, cub_bytes, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr,
        total, 0, end_bit
    );
    L.keys_in  = 0;
    L.keys_out = L.keys_in + al(sizeof(uint64_t) * (size_t)total);
    L.rows_in  = L.keys_out + al(sizeof(uint64_t) * (size_t)total);
    L.cub      = L.rows_in + al(sizeof(int32_t) * (size_t)total);
    L.total    = L.cub + al(cub_bytes) + 256;
    return L;
}
} // namespace gsb

extern "C" size_t gsb200_isect_depth_order_workspace_bytes(int64_t I, int64_t total_rows)
{
    if(total_rows <= 0 || I <= 0)
        return 0;
    return gsb::depth_order_layout(total_rows, 32 + (int)gsb::bits_for_count(I)).total;
}

extern "C" int gsb200_isect_depth_order(
    int64_t I, int64_t N, const int32_t *radii, const float *depths, const int64_t *image_ids, int32_t *order,
    void *workspace, size_t workspace_bytes, void *stream
)
{
    if(I < 0 || N < 0)
        return GSB200_E_INVALID;
    const int64_t total = image_ids ? N : I * N; // packed: N rows in total
    if(total == 0)
        return GSB200_OK;
    if(!radii || !depths || !order || !workspace || total > 0x7fffffffLL)
        return GSB200_E_INVALID;
    const int end_bit = 32 + (int)gsb::bits_for_count(I);
    const auto L      = gsb::depth_order_layout(total, end_bit);
    if(L.total > workspace_bytes)
        return GSB200_E_WORKSPACE;
    char *ws         = static_cast<char *>(workspace);
    uint64_t *k_in   = reinterpret_cast<uint64_t *>(ws + L.keys_in), *k_out = reinterpret_cast<uint64_t *>(ws + L.keys_out);
    int32_t *rows_in = reinterpret_cast<int32_t *>(ws + L.rows_in);
    cudaStream_t st  = (cudaStream_t)stream;
    size_t cub_bytes = L.total - L.cub;
    if(I == 1 && image_ids == nullptr)
    { // 32-bit keys in the (larger) 64-bit key buffers; the CUB temp storage sized for 64-bit keys is ample
        uint32_t *k32_in = reinterpret_cast<uint32_t *>(k_in), *k32_out = reinterpret_cast<uint32_t *>(k_out);
        gsb::depth_key32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(total, radii, depths, k32_in, rows_in);
        if(int rc = gsb::check_launch())
            return rc;
        size_t need = 0;
        cub::DeviceRadixSort::SortPairs((void *)nullptr, need, k32_in, k32_out, rows_in, order, total, 0, 32, st);
        if(need > cub_bytes)
            return GSB200_E_WORKSPACE;
        GSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + L.cub, need, k32_in, k32_out, rows_in, order, total, 0, 32, st));
        return GSB200_OK;
    }
    gsb::depth_key_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(total, N, radii, depths, image_ids, k_in, rows_in);
    if(int rc = gsb::check_launch())
        return rc;
    GSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, k_in, k_out, rows_in, order, total, 0, end_bit, st));
    return GSB200_OK;
}


// ---- depth order of the rows that HAVE tiles (round 2).  gsb200_isect_depth_order sorts every projected row, culled
// ones included (71 % at BASELINE configs[2]; in a trainer with 3 M gaussians that is 2 M dead rows through four radix
// passes).  Once the per-row tile counts are known (gsb200_isect_count_totals) and the host has read the two totals,
// the rows with tiles are compacted (stable: ascending row index), only those are sorted by (image, depth), and the
// counts are scanned in that order -- same final order as before (both steps are stable), a third of the rows.
namespace gsb
{
struct HasTiles
{
    const int32_t *tiles;
    __host__ __device__ bool operator()(const int32_t &i) const { return tiles[i] > 0; }
};
struct CountOf
{
    const int32_t *tiles;
    __host__ __device__ int64_t operator()(const int32_t &row) const { return (int64_t)tiles[row]; }
};

__global__ void __launch_bounds__(256) depth_key_rows_kernel(
    int64_t n_rows, int64_t N, const int32_t *__restrict__ rows, const float *__restrict__ depths,
    const int64_t *__restrict__ image_ids, bool single_image, void *__restrict__ keys
)
{
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(j >= n_rows)
        return;
    const int64_t i  = rows[j];
    const uint32_t d = __float_as_uint(depths[i]);
    if(single_image)
        static_cast<uint32_t *>(keys)[j] = d;
    else
        static_cast<uint64_t *>(keys)[j] = ((uint64_t)(image_ids ? image_ids[i] : i / N) << 32) | (uint64_t)d;
}

struct VisibleOrderLayout
{
    size_t rows_in, keys_in, keys_out, n_sel, cub, total;
};
static VisibleOrderLayout visible_order_layout(int64_t total_rows, int64_t n_vis, int end_bit)
{
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    VisibleOrderLayout L;
    size_t a = 0, b = 0, c = 0;
    cub::DeviceSelect::If((void *)nullptr, a, cub::CountingInputIterator<int32_t>(0), (int32_t *)nullptr, (int32_t *)nullptr, total_rows, HasTiles{nullptr});
    cub::DeviceRadixSort::SortPairs(
        (void *)nullptr, b, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr, n_vis, 0, end_bit
    );
    cub::TransformInputIterator<int64_t, CountOf, const int32_t *> it((const int32_t *)nullptr, CountOf{nullptr});
    cub::DeviceScan::InclusiveSum((void *)nullptr, c, it, (int64_t *)nullptr, n_vis);
    const size_t cub_bytes = a > b ? (a > c ? a : c) : (b > c ? b : c);
    L.rows_in  = 0;
    L.keys_in  = L.rows_in + al(sizeof(int32_t) * (size_t)n_vis);
    L.keys_out = L.keys_in + al(sizeof(uint64_t) * (size_t)n_vis);
    L.n_sel    = L.keys_out + al(sizeof(uint64_t) * (size_t)n_vis);
    L.cub      = L.n_sel + 256;
    L.total    = L.cub + al(cub_bytes) + 256;
    return L;
}
} // namespace gsb

extern "C" size_t gsb200_isect_order_visible_workspace_bytes(int64_t I, int64_t total_rows, int64_t n_vis)
{
    if(total_rows <= 0 || I <= 0 || n_vis <= 0)
        return 0;
    return gsb::visible_order_layout(total_rows, n_vis, 32 + (int)gsb::bits_for_count(I)).total;
}

extern "C" int gsb200_isect_order_visible(
    int64_t I, int64_t N, int64_t n_vis, const int32_t *tiles_per_gauss, const float *depths, const int64_t *image_ids,
    int32_t *order, int64_t *cum_tiles, void *workspace, size_t workspace_bytes, void *stream
)
{
    if(I < 0 || N < 0 || n_vis < 0)
        return GSB200_E_INVALID;
    const int64_t total = image_ids ? N : I * N;
    if(total == 0 || n_vis == 0)
        return GSB200_OK;
    if(!tiles_per_gauss || !depths || !order || !cum_tiles || !workspace || total > 0x7fffffffLL || n_vis > total)
        return GSB200_E_INVALID;
    const bool single = (I == 1 && image_ids == nullptr);
    const int end_bit = single ? 32 : 32 + (int)gsb::bits_for_count(I);
    const auto L      = gsb::visible_order_layout(total, n_vis, 32 + (int)gsb::bits_for_count(I));
    if(L.total > workspace_bytes)
        return GSB200_E_WORKSPACE;
    char *ws         = static_cast<char *>(workspace);
    int32_t *rows_in = reinterpret_cast<int32_t *>(ws + L.rows_in);
    void *k_in = ws + L.keys_in, *k_out = ws + L.keys_out;
    int32_t *n_sel   = reinterpret_cast<int32_t *>(ws + L.n_sel);
    cudaStream_t st  = (cudaStream_t)stream;
    size_t cub_bytes = L.total - L.cub;
    // 1. rows with tiles, ascending (n_vis of them: the caller read that total from gsb200_isect_count_totals)
    GSB_CUDA_TRY(cub::DeviceSelect::If(
        ws + L.cub, cub_bytes, cub::CountingInputIterator<int32_t>(0), rows_in, n_sel, total, gsb::HasTiles{tiles_per_gauss}, st
    ));
    // 2. (image, depth) keys of those rows, stable sort
    gsb::depth_key_rows_kernel<<<(unsigned)((n_vis + 255) / 256), 256, 0, st>>>(n_vis, N, rows_in, depths, image_ids, single, k_in);
    if(int rc = gsb::check_launch())
        return rc;
    cub_bytes = L.total - L.cub;
    if(single)
        GSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(
            ws + L.cub, cub_bytes, static_cast<const uint32_t *>(k_in), static_cast<uint32_t *>(k_out), rows_in, order, n_vis, 0, 32, st
        ));
    else
        GSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(
            ws + L.cub, cub_bytes, static_cast<const uint64_t *>(k_in), static_cast<uint64_t *>(k_out), rows_in, order, n_vis, 0, end_bit, st
        ));
    // 3. inclusive scan of the tile counts taken in that order
    cub::TransformInputIterator<int64_t, gsb::CountOf, const int32_t *> it(order, gsb::CountOf{tiles_per_gauss});
    cub_bytes = L.total - L.cub;
    GSB_CUDA_TRY(cub::DeviceScan::InclusiveSum(ws + L.cub, cub_bytes, it, cum_tiles, n_vis, st));
    return GSB200_OK;
}

// ---- the whole sorted dense intersection stage in one call, sized by CAPACITIES (round 2).
// rasterization() used to read the totals of the count pass on the host before it could size and launch anything else:
// the GPU idled for the round trip and for the host's launch latency behind it (40 us per step at BASELINE configs[2],
// 100 us when a PCIe upload was in flight).  Here every launch is sized by host-side capacities (cap_vis rows with
// tiles, cap_isects intersections) while the REAL counts stay in device memory (`totals`, from gsb200_isect_count_totals
// or gsb200_project_sh_fwd_rows): slots beyond the real counts are padding that sorts last, and nothing is ever written
// past a capacity.  The caller launches this with capacities predicted from earlier calls, reads the totals afterwards
// (by then this work is queued behind them), takes the first totals[0] entries if both counts fit, and otherwise calls
// again with exact capacities.  With capacities equal to the totals the padding is empty and this is the plain pipeline.
namespace gsb
{
struct CountOfBounded
{
    const int32_t *tiles, *order;
    const int64_t *totals;
    int64_t cap;
    __host__ __device__ int64_t operator()(const int32_t &j) const
    {
        const int64_t n = totals[1] < cap ? totals[1] : cap;
        return (int64_t)j < n ? (int64_t)tiles[order[j]] : 0;
    }
};

__global__ void __launch_bounds__(256) depth_key_rows_bounded_kernel(
    int64_t cap_vis, int64_t N, const int32_t *__restrict__ rows, const float *__restrict__ depths, bool single_image,
    const int64_t *__restrict__ totals, void *__restrict__ keys
)
{
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(j >= cap_vis)
        return;
    const bool real  = j < totals[1];
    const int64_t i  = real ? rows[j] : 0;
    const uint32_t d = real ? __float_as_uint(depths[i]) : 0xffffffffu;
    if(single_image)
        static_cast<uint32_t *>(keys)[j] = d;
    else
        static_cast<uint64_t *>(keys)[j] = real ? (((uint64_t)(i / N) << 32) | (uint64_t)d) : ~0ull;
}

struct SortedLayout
{
    size_t rows_in, keys_in, keys_out, order, cum, n_sel, tkeys, tvals, cub, total;
};
static SortedLayout sorted_layout(int64_t total_rows, int64_t cap_vis, int64_t cap_isects, int key_bytes, int depth_end_bit, int tile_end_bit)
{
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    SortedLayout L;
    size_t a = 0, b = 0, c = 0, d = 0;
    cub::DeviceSelect::If((void *)nullptr, a, cub::CountingInputIterator<int32_t>(0), (int32_t *)nullptr, (int32_t *)nullptr, total_rows, HasTiles{nullptr});
    cub::DeviceRadixSort::SortPairs(
        (void *)nullptr, b, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr, cap_vis, 0, depth_end_bit
    );
    cub::TransformInputIterator<int64_t, CountOfBounded, cub::CountingInputIterator<int32_t>> it(
        cub::CountingInputIterator<int32_t>(0), CountOfBounded{nullptr, nullptr, nullptr, 0}
    );
    cub::DeviceScan::InclusiveSum((void *)nullptr, c, it, (int64_t *)nullptr, cap_vis);
    if(key_bytes == 2)
        cub::DeviceRadixSort::SortPairs(
            (void *)nullptr, d, (const uint16_t *)nullptr, (uint16_t *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr, cap_isects, 0, tile_end_bit
        );
    else
        cub::DeviceRadixSort::SortPairs(
            (void *)nullptr, d, (const uint32_t *)nullptr, (uint32_t *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr, cap_isects, 0, tile_end_bit
        );
    size_t cub_bytes = a > b ? a : b;
    cub_bytes        = cub_bytes > c ? cub_bytes : c;
    cub_bytes        = cub_bytes > d ? cub_bytes : d;
    L.rows_in  = 0; // the compaction writes every row that has tiles, however many: sized for all rows
    L.keys_in  = L.rows_in + al(sizeof(int32_t) * (size_t)total_rows);
    L.keys_out = L.keys_in + al(sizeof(uint64_t) * (size_t)cap_vis);
    L.order    = L.keys_out + al(sizeof(uint64_t) * (size_t)cap_vis);
    L.cum      = L.order + al(sizeof(int32_t) * (size_t)cap_vis);
    L.n_sel    = L.cum + al(sizeof(int64_t) * (size_t)cap_vis);
    L.tkeys    = L.n_sel + 256;
    L.tvals    = L.tkeys + al((size_t)key_bytes * (size_t)cap_isects);
    L.cub      = L.tvals + al(sizeof(int32_t) * (size_t)cap_isects);
    L.total    = L.cub + al(cub_bytes) + 256;
    return L;
}
} // namespace gsb

extern "C" size_t gsb200_isect_sorted_workspace_bytes(
    int64_t I, int64_t N, int64_t cap_vis, int64_t cap_isects, int key_bytes, uint32_t tile_width, uint32_t tile_height
)
{
    if(I <= 0 || N <= 0 || cap_vis <= 0 || cap_isects <= 0 || (key_bytes != 2 && key_bytes != 4))
        return 0;
    const int tile_end = (int)gsb::bits_for_count(I * (int64_t)tile_width * tile_height);
    return gsb::sorted_layout(I * N, cap_vis, cap_isects, key_bytes, 32 + (int)gsb::bits_for_count(I), tile_end > 0 ? tile_end : 1).total;
}

extern "C" int gsb200_isect_sorted(
    int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *depths, const float *conics,
    const float *opacities, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, const int32_t *tiles_per_gauss,
    const int64_t *totals, int64_t cap_vis, int64_t cap_isects, int64_t max_tiles_hint, int key_bytes, void *tile_keys,
    int32_t *flatten_ids, int32_t *offsets, void *workspace, size_t workspace_bytes, void *stream
)
{
    if(I <= 0 || N <= 0 || cap_vis <= 0 || cap_isects <= 0 || tile_size == 0 || (key_bytes != 2 && key_bytes != 4))
        return GSB200_E_INVALID;
    const int64_t total = I * N, total_tiles = I * (int64_t)tile_width * tile_height;
    if(!means2d || !radii || !depths || !tiles_per_gauss || !totals || !tile_keys || !flatten_ids || !offsets || !workspace
       || total > 0x7fffffffLL || cap_vis > total || cap_isects > 0x7fffffffLL)
        return GSB200_E_INVALID;
    if((int)gsb::bits_for_count(total_tiles) > 8 * key_bytes)
        return GSB200_E_KEYBITS;
    const bool single  = I == 1;
    const int depth_end = single ? 32 : 32 + (int)gsb::bits_for_count(I);
    int tile_end        = (int)gsb::bits_for_count(total_tiles);
    tile_end            = tile_end > 0 ? tile_end : 1;
    const auto L        = gsb::sorted_layout(total, cap_vis, cap_isects, key_bytes, 32 + (int)gsb::bits_for_count(I), tile_end);
    if(L.total > workspace_bytes)
        return GSB200_E_WORKSPACE;
    char *ws         = static_cast<char *>(workspace);
    int32_t *rows_in = reinterpret_cast<int32_t *>(ws + L.rows_in), *order = reinterpret_cast<int32_t *>(ws + L.order);
    void *k_in = ws + L.keys_in, *k_out = ws + L.keys_out;
    int64_t *cum     = reinterpret_cast<int64_t *>(ws + L.cum);
    int32_t *n_sel   = reinterpret_cast<int32_t *>(ws + L.n_sel);
    void *tkeys      = ws + L.tkeys;
    int32_t *tvals   = reinterpret_cast<int32_t *>(ws + L.tvals);
    cudaStream_t st  = (cudaStream_t)stream;
    const size_t cub_cap = L.total - L.cub;
    size_t cub_bytes     = cub_cap;
    // 1. rows with tiles, ascending
    GSB_CUDA_TRY(cub::DeviceSelect::If(
        ws + L.cub, cub_bytes, cub::CountingInputIterator<int32_t>(0), rows_in, n_sel, total, gsb::HasTiles{tiles_per_gauss}, st
    ));
    // 2. their (image, depth) keys -- padding slots get the largest key -- and a stable sort of the cap_vis slots
    gsb::depth_key_rows_bounded_kernel<<<(unsigned)((cap_vis + 255) / 256), 256, 0, st>>>(cap_vis, N, rows_in, depths, single, totals, k_in);
    if(int rc = gsb::check_launch())
        return rc;
    cub_bytes = cub_cap;
    if(single)
        GSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(
            ws + L.cub, cub_bytes, static_cast<const uint32_t *>(k_in), static_cast<uint32_t *>(k_out), rows_in, order, cap_vis, 0, 32, st
        ));
    else
        GSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(
            ws + L.cub, cub_bytes, static_cast<const uint64_t *>(k_in), static_cast<uint64_t *>(k_out), rows_in, order, cap_vis, 0, depth_end, st
        ));
    // 3. inclusive scan of the tile counts in that order (0 for padding slots)
    cub::TransformInputIterator<int64_t, gsb::CountOfBounded, cub::CountingInputIterator<int32_t>> it(
        cub::CountingInputIterator<int32_t>(0), gsb::CountOfBounded{tiles_per_gauss, order, totals, cap_vis}
    );
    cub_bytes = cub_cap;
    GSB_CUDA_TRY(cub::DeviceScan::InclusiveSum(ws + L.cub, cub_bytes, it, cum, cap_vis, st));
    // 4. emission in depth order, (dense tile id, row) pairs; 5. stable sort on the tile id; 6. offsets
    if(int rc = gsb::emit_tilekeys_bounded(
           I, N, cap_vis, max_tiles_hint, means2d, radii, depths, conics, opacities, cum, order, tile_size, tile_width, tile_height,
           key_bytes, tkeys, tvals, totals, cap_isects, st
       ))
        return rc;
    if(key_bytes == 2)
    {
        if(int rc = gsb::sort_tile_pairs<uint16_t>(cap_isects, tile_end, tkeys, tvals, tile_keys, flatten_ids, ws + L.cub, cub_cap, st))
            return rc;
    }
    else if(int rc = gsb::sort_tile_pairs<uint32_t>(cap_isects, tile_end, tkeys, tvals, tile_keys, flatten_ids, ws + L.cub, cub_cap, st))
        return rc;
    return gsb::offsets_tilekeys_bounded(cap_isects, key_bytes, tile_keys, total_tiles, offsets, totals, st);
}

// ---- the totals, published straight into pinned host memory.  A cudaMemcpyAsync of 24 bytes takes a copy engine and,
// on a box whose PCIe link is busy with an image upload, arrives late; a handful of system-scope stores from a kernel do
// not.  host_mapped: int64 [4] in pinned (mapped) host memory; the host polls host_mapped[3] for `seq`.
namespace gsb
{
__global__ void publish_totals_kernel(const int64_t *__restrict__ totals, volatile int64_t *host, int64_t seq)
{
    if(threadIdx.x < 3)
        host[threadIdx.x] = totals[threadIdx.x];
    __threadfence_system();
    __syncwarp();
    if(threadIdx.x == 0)
        host[3] = seq;
}
} // namespace gsb

extern "C" int gsb200_publish_totals(const int64_t *totals, int64_t *host_mapped, int64_t seq, void *stream)
{
    if(!totals || !host_mapped)
        return GSB200_E_INVALID;
    void *dptr = nullptr;
    if(cudaHostGetDevicePointer(&dptr, host_mapped, 0) != cudaSuccess || dptr == nullptr)
    {
        (void)cudaGetLastError(); // not mapped for this device: clear the error, the caller falls back to a copy
        return GSB200_E_UNSUPPORTED;
    }
    gsb::publish_totals_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(totals, static_cast<volatile int64_t *>(dptr), seq);
    return gsb::check_launch();
}
