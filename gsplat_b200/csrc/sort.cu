// sort.cu -- the sorted tile intersection (gsb200_isect_sorted), the sparse pixel layout and library-level helpers.
//
// The sorts are cub::DeviceRadixSort::SortPairs (the library call the reference makes,
// csrc/IntersectTile.cu:1078-1121; its onesweep kernels are compiled here for sm_90a), used twice:
// once over the rows that have tiles on (image, depth) and once over the S intersections on the dense
// (image, tile) id only -- see gsb200_isect_sorted below.
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

// The (image, tile)-only sort of the depth-ordered intersections: 2- or 4-byte dense tile ids as keys, the row index
// as value -- 6 (8) instead of the reference's 12 bytes per intersection and direction in each radix pass.
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

// ---- depth order of every projected row (pre-pass of the masked tile intersection, gsb200_isect_sparse_count)
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

size_t depth_order_workspace_bytes(int64_t I, int64_t total_rows)
{
    if(total_rows <= 0 || I <= 0)
        return 0;
    return depth_order_layout(total_rows, 32 + (int)bits_for_count(I)).total;
}

// order int32 [rows] = the projected rows in ascending (image, depth bits, row) order, culled rows (radii <= 0) last.
// rows = I * N, or N when image_ids (packed layout) is given.
int depth_order(
    int64_t I, int64_t N, const int32_t *radii, const float *depths, const int64_t *image_ids, int32_t *order,
    void *workspace, size_t workspace_bytes, cudaStream_t st
)
{
    if(I < 0 || N < 0)
        return GSB200_E_INVALID;
    const int64_t total = image_ids ? N : I * N; // packed: N rows in total
    if(total == 0)
        return GSB200_OK;
    if(!radii || !depths || !order || !workspace || total > 0x7fffffffLL)
        return GSB200_E_INVALID;
    const int end_bit = 32 + (int)bits_for_count(I);
    const auto L      = depth_order_layout(total, end_bit);
    if(L.total > workspace_bytes)
        return GSB200_E_WORKSPACE;
    char *ws         = static_cast<char *>(workspace);
    uint64_t *k_in   = reinterpret_cast<uint64_t *>(ws + L.keys_in), *k_out = reinterpret_cast<uint64_t *>(ws + L.keys_out);
    int32_t *rows_in = reinterpret_cast<int32_t *>(ws + L.rows_in);
    size_t cub_bytes = L.total - L.cub;
    if(I == 1 && image_ids == nullptr)
    { // 32-bit keys in the (larger) 64-bit key buffers; the CUB temp storage sized for 64-bit keys is ample
        uint32_t *k32_in = reinterpret_cast<uint32_t *>(k_in), *k32_out = reinterpret_cast<uint32_t *>(k_out);
        depth_key32_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(total, radii, depths, k32_in, rows_in);
        if(int rc = check_launch())
            return rc;
        size_t need = 0;
        cub::DeviceRadixSort::SortPairs((void *)nullptr, need, k32_in, k32_out, rows_in, order, total, 0, 32, st);
        if(need > cub_bytes)
            return GSB200_E_WORKSPACE;
        GSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + L.cub, need, k32_in, k32_out, rows_in, order, total, 0, 32, st));
        return GSB200_OK;
    }
    depth_key_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(total, N, radii, depths, image_ids, k_in, rows_in);
    if(int rc = check_launch())
        return rc;
    GSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(ws + L.cub, cub_bytes, k_in, k_out, rows_in, order, total, 0, end_bit, st));
    return GSB200_OK;
}
} // namespace gsb

// ---- the whole sorted intersection stage in one call, sized by CAPACITIES (round 2).
// Sorting every projected row by depth would put the culled ones (71 % at BASELINE configs[2]; in a trainer with 3 M
// gaussians that is 2 M dead rows) through four radix passes: the rows with tiles are compacted first (stable:
// ascending row index), only those are sorted by (image, depth), and the counts are scanned in that order -- the same
// final order, both steps being stable, for a third of the rows.
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
struct HasTiles
{
    const int32_t *tiles;
    __host__ __device__ bool operator()(const int32_t &i) const { return tiles[i] > 0; }
};
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
    int64_t cap_vis, int64_t N, const int32_t *__restrict__ rows, const float *__restrict__ depths,
    const int64_t *__restrict__ image_ids, bool single_image, const int64_t *__restrict__ totals, void *__restrict__ keys
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
        static_cast<uint64_t *>(keys)[j] = real ? (((uint64_t)(image_ids ? image_ids[i] : i / N) << 32) | (uint64_t)d) : ~0ull;
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
    int64_t I, int64_t total_rows, int64_t cap_vis, int64_t cap_isects, int key_bytes, uint32_t tile_width, uint32_t tile_height
)
{
    if(I <= 0 || total_rows <= 0 || cap_vis <= 0 || cap_isects <= 0 || (key_bytes != 2 && key_bytes != 4))
        return 0;
    const int tile_end = (int)gsb::bits_for_count(I * (int64_t)tile_width * tile_height);
    return gsb::sorted_layout(total_rows, cap_vis, cap_isects, key_bytes, 32 + (int)gsb::bits_for_count(I), tile_end > 0 ? tile_end : 1).total;
}

extern "C" int gsb200_isect_sorted(
    int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *depths, const float *conics,
    const float *opacities, const int64_t *image_ids, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
    const int32_t *tiles_per_gauss, const int64_t *totals, int64_t cap_vis, int64_t cap_isects, int64_t max_tiles_hint,
    int key_bytes, void *tile_keys, int32_t *flatten_ids, int32_t *offsets, void *workspace, size_t workspace_bytes,
    void *stream
)
{
    if(I <= 0 || N <= 0 || cap_vis <= 0 || cap_isects <= 0 || tile_size == 0 || (key_bytes != 2 && key_bytes != 4))
        return GSB200_E_INVALID;
    // packed layout: N rows in total (image_ids given), I only sizes the keys and the offsets; dense: I * N rows
    const int64_t total = image_ids ? N : I * N, total_tiles = I * (int64_t)tile_width * tile_height;
    if(!means2d || !radii || !depths || !tiles_per_gauss || !totals || !tile_keys || !flatten_ids || !offsets || !workspace
       || total > 0x7fffffffLL || cap_vis > total || cap_isects > 0x7fffffffLL)
        return GSB200_E_INVALID;
    if(gsb::bits_for_count(I) + gsb::bits_for_count((int64_t)tile_width * tile_height) > 32
       || (int)gsb::bits_for_count(total_tiles) > 8 * key_bytes)
        return GSB200_E_KEYBITS;
    const bool single  = I == 1; // one image: the depth bits alone are the key, whatever the row layout
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
    gsb::depth_key_rows_bounded_kernel<<<(unsigned)((cap_vis + 255) / 256), 256, 0, st>>>(
        cap_vis, N, rows_in, depths, image_ids, single, totals, k_in
    );
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
           N, cap_vis, max_tiles_hint, means2d, radii, depths, conics, opacities, cum, image_ids, order, tile_size, tile_width,
           tile_height, key_bytes, tkeys, tvals, totals, cap_isects, st
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
