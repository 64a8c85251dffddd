// isect.cu -- the tile intersection: which tiles every projected gaussian touches, as per-tile lists in depth order.
// Compiled with -fmad=false: the fused projection (pergauss.cu) counts tiles with the same tiles_of_gaussian
// (isect.cuh), and the counts of the two units must agree bit for bit.
//
// In pipeline order: the per-row tile count, the depth order of the rows, the scan of the counts in that order, the
// emission of (tile id, row) pairs, their stable sort on the tile id and the per-tile offsets.  gsb200_isect_sorted runs
// the stages after the count in one call.  Given a tile mask (isect_tiles_sparse), the count and the emission see only
// the tiles the mask sets, and gsb200_isect_active_offsets picks the offsets of the active tiles.
// The sorts are cub::DeviceRadixSort::SortPairs (the library call the reference makes, csrc/IntersectTile.cu:1078-1121;
// its onesweep kernels are compiled here for sm_90a), used twice: once over the rows that have tiles on (image, depth)
// and once over the S intersections on the dense (image, tile) id only.
//
// Reference kernels replaced: csrc/IntersectTile.cu:83-464,925-988.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include "isect.cuh"

namespace gsb
{
constexpr int kThreads = 256;

// ------------------------------------------------------------------ tile rows
// The tiles of one gaussian row by row, each row's tile interval in closed form: how a warp shares the rows of a
// gaussian with many tiles (the masked count, isect_emit_coop_kernel).
constexpr int kSmallTiles = 64; // measured: below ~2 warps' worth of tiles the per-gaussian warp hand-over costs more than it saves

struct AccuGauss
{
    float mx, my, A, Bc, Cc, disc, t, ts;
    float bminu, bmaxu, bminv, bmaxv, amin_v, amax_v, pu, pv, coeff;
    int ru0, ru1, rv0, rv1;
    bool isY, accu, empty;
    int x0, x1; // AABB path
};

__device__ __forceinline__ AccuGauss accu_setup(
    float mx, float my, int rx, int ry, bool accu, float A, float Bc, float Cc, float opacity, uint32_t tile_size,
    uint32_t tw, uint32_t th
)
{
    AccuGauss g;
    g.mx = mx, g.my = my, g.A = A, g.Bc = Bc, g.Cc = Cc, g.accu = accu, g.ts = (float)tile_size;
    g.empty     = rx <= 0 || ry <= 0;
    g.ru0 = g.ru1 = g.rv0 = g.rv1 = g.x0 = g.x1 = 0;
    g.isY                                        = false;
    auto clampi = [](int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); };
    if(g.empty)
        return g;
    const float ts = g.ts;
    if(accu)
    {
        g.disc          = Bc * Bc - A * Cc;
        float t         = 2.f * exact_log(opacity / kAlphaThreshold);
        const float cap = kGaussianExtend * kGaussianExtend;
        g.t             = t < cap ? t : cap;
        const float ntd = -g.t / g.disc;
        const float xe = sqrtf(ntd * Cc), ye = sqrtf(ntd * A);
        const float bminx = mx - xe, bminy = my - ye, bmaxx = mx + xe, bmaxy = my + ye;
        const float BxC = Bc * xe / Cc, ByA = Bc * ye / A;
        const float argminx = my + BxC, argminy = mx + ByA, argmaxx = my - BxC, argmaxy = mx - ByA;
        const int rminx = clampi((int)(bminx / ts), 0, (int)tw), rminy = clampi((int)(bminy / ts), 0, (int)th);
        const int rmaxx = clampi((int)(bmaxx / ts + 1.f), 0, (int)tw), rmaxy = clampi((int)(bmaxy / ts + 1.f), 0, (int)th);
        const int ys = rmaxy - rminy, xs = rmaxx - rminx;
        if(ys * xs == 0)
        {
            g.empty = true;
            return g;
        }
        g.isY = ys < xs;
        g.ru0 = g.isY ? rminy : rminx, g.ru1 = g.isY ? rmaxy : rmaxx, g.rv0 = g.isY ? rminx : rminy, g.rv1 = g.isY ? rmaxx : rmaxy;
        g.bminu = g.isY ? bminy : bminx, g.bmaxu = g.isY ? bmaxy : bmaxx;
        g.bminv = g.isY ? bminx : bminy, g.bmaxv = g.isY ? bmaxx : bmaxy;
        g.amin_v = g.isY ? argminx : argminy, g.amax_v = g.isY ? argmaxx : argmaxy;
        g.pu = g.isY ? my : mx, g.pv = g.isY ? mx : my, g.coeff = g.isY ? A : Cc;
    }
    else
    {
        const float trx = (float)rx / ts, try_ = (float)ry / ts, tx = mx / ts, ty = my / ts;
        g.x0 = clampi((int)floorf(tx - trx), 0, (int)tw), g.ru0 = clampi((int)floorf(ty - try_), 0, (int)th);
        g.x1 = clampi((int)ceilf(tx + trx), 0, (int)tw), g.ru1 = clampi((int)ceilf(ty + try_), 0, (int)th);
        g.isY = true; // rows are tile rows
        if(g.ru1 <= g.ru0 || g.x1 <= g.x0)
            g.empty = true;
    }
    return g;
}

// tile interval [v0, v1) of row u (ru0 <= u < ru1); identical, bit for bit, to what tiles_of_gaussian enumerates
__device__ __forceinline__ void accu_row(const AccuGauss &g, int u, int &v0, int &v1)
{
    if(!g.accu)
    {
        v0 = g.x0, v1 = g.x1;
        return;
    }
    const float ts = g.ts;
    auto line = [&](float coord, float &lo, float &hi) {
        const float h  = coord - g.pu;
        const float sq = sqrtf(g.disc * h * h + g.t * g.coeff);
        lo             = (-g.Bc * h - sq) / g.coeff + g.pv;
        hi             = (-g.Bc * h + sq) / g.coeff + g.pv;
    };
    const float min_line = (float)u * ts, max_line = min_line + ts;
    float minlo = g.bmaxv, minhi = g.bminv; // the sequential scheme's initial values
    if(u > g.ru0 || g.bminu <= min_line)
        line(min_line, minlo, minhi);
    float maxlo, maxhi;
    if(max_line <= g.bmaxu)
        line(max_line, maxlo, maxhi);
    else if(u > g.ru0)
        maxlo = minlo, maxhi = minhi; // the far line was not computed: the previous one is kept
    else
        maxlo = g.bmaxv, maxhi = g.bminv;
    const float emin = (min_line <= g.amin_v && g.amin_v < max_line) ? g.bminv : (minlo < maxlo ? minlo : maxlo);
    const float emax = (min_line <= g.amax_v && g.amax_v < max_line) ? g.bmaxv : (minhi > maxhi ? minhi : maxhi);
    const int e0 = (int)(emin / ts), e1 = (int)(emax / ts + 1.f);
    v0 = e0 < g.rv1 ? e0 : g.rv1;
    v0 = v0 > g.rv0 ? v0 : g.rv0;
    v1 = e1 > g.rv0 ? e1 : g.rv0;
    v1 = v1 < g.rv1 ? v1 : g.rv1;
    if(v1 < v0)
        v1 = v0;
}

// ------------------------------------------------------------------ count
// A masked row with more tiles than this is counted by its whole warp.  Measured on an H100 80GB HBM3 at 700 W, bench.py's
// scene (1M rows, one 1080p view): handing over rows above 64 tiles, the masked count of the 3DGS rows took 29 us, above
// 256 tiles 23 us (the same up to 1024); that of the surfel rows takes 100 us either way, 230 us without any hand-over.
constexpr int kManyMaskedTiles = 256;

// Row-order tile count of every row.  TOTALS: also the totals the host reads once (block_tile_totals); without them
// this is the first pass of the unsorted intersection.  MASKED: only the tiles whose byte in tile_mask [I, th, tw] is
// set count; row i belongs to image image_ids[i], or i / N without image_ids.
template<bool TOTALS, bool MASKED = false>
__global__ void __launch_bounds__(kThreads) isect_count_kernel(
    int64_t total, const float *__restrict__ means2d, const int32_t *__restrict__ radii, const float *__restrict__ conics,
    const float *__restrict__ opacities, uint32_t tile_size, uint32_t tw, uint32_t th, int32_t *__restrict__ tiles_per_gauss,
    unsigned long long *__restrict__ totals, int64_t N = 0, int64_t I = 0, const int64_t *__restrict__ image_ids = nullptr,
    const uint8_t *__restrict__ tile_mask = nullptr
)
{
    unsigned long long *s_tot = nullptr;
    if constexpr(TOTALS)
        s_tot = block_tile_totals_begin();
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    int cnt         = 0;
    bool many       = false; // MASKED: a row of more than kManyMaskedTiles tiles
    if(i < total)
    {
        const int2 r = reinterpret_cast<const int2 *>(radii)[i];
        if(r.x > 0 && r.y > 0)
        {
            const float2 m = reinterpret_cast<const float2 *>(means2d)[i];
            float cn[3] = {0.f, 0.f, 0.f}, op = 0.f;
            const bool accu = conics != nullptr && opacities != nullptr;
            if(accu)
                cn[0] = conics[i * 3], cn[1] = conics[i * 3 + 1], cn[2] = conics[i * 3 + 2], op = opacities[i];
            if constexpr(MASKED)
            {
                // the mask has no bytes for an image outside [0, I): such a row counts no tile, so the compaction drops
                // it and no later pass reads its image
                const int64_t img = image_ids ? image_ids[i] : i / N;
                if(img >= 0 && img < I)
                {
                    const uint8_t *tm = tile_mask + img * (int64_t)tw * th;
                    many = tiles_of_gaussian(m.x, m.y, r.x, r.y, accu ? cn : nullptr, accu ? &op : nullptr, tile_size, tw, th, [](int64_t) {})
                           > kManyMaskedTiles;
                    if(!many)
                        tiles_of_gaussian(m.x, m.y, r.x, r.y, accu ? cn : nullptr, accu ? &op : nullptr, tile_size, tw, th, [&](int64_t t) {
                            cnt += tm[t] != 0;
                        });
                }
            }
            else
                cnt = tiles_of_gaussian(m.x, m.y, r.x, r.y, accu ? cn : nullptr, accu ? &op : nullptr, tile_size, tw, th, [](int64_t) {});
        }
        if constexpr(!MASKED)
            tiles_per_gauss[i] = cnt;
    }
    if constexpr(MASKED)
    {
        // Rows with many tiles (large gaussians near the camera) lie scattered over the row order: one lane looping over
        // all the tiles of such a row would hold its warp for each of them.  Here the warp counts the row, one tile row per
        // lane, with the row intervals of accu_row (the tiles of tiles_of_gaussian).
        const unsigned lane = threadIdx.x & 31;
        for(uint32_t big = __ballot_sync(0xffffffffu, many); big; big &= big - 1)
        {
            const int src      = __ffs(big) - 1;
            const int64_t b    = i - (int64_t)lane + src;
            const int2 r       = reinterpret_cast<const int2 *>(radii)[b];
            const float2 m     = reinterpret_cast<const float2 *>(means2d)[b];
            const bool accu    = conics != nullptr && opacities != nullptr;
            const AccuGauss g  = accu_setup(
                m.x, m.y, r.x, r.y, accu, accu ? conics[b * 3] : 0.f, accu ? conics[b * 3 + 1] : 0.f,
                accu ? conics[b * 3 + 2] : 0.f, accu ? opacities[b] : 0.f, tile_size, tw, th
            );
            const uint8_t *tm = tile_mask + (image_ids ? image_ids[b] : b / N) * (int64_t)tw * th;
            int c             = 0;
            for(int u = g.ru0 + (int)lane; u < g.ru1; u += 32)
            {
                int v0 = 0, v1 = 0;
                accu_row(g, u, v0, v1);
                for(int v = v0; v < v1; ++v)
                    c += tm[g.isY ? (int64_t)u * tw + v : (int64_t)v * tw + u] != 0;
            }
            c = __reduce_add_sync(0xffffffffu, c);
            if((int)lane == src)
                cnt = c;
        }
        if(i < total)
            tiles_per_gauss[i] = cnt;
    }
    if constexpr(TOTALS)
        block_tile_totals(cnt, s_tot, totals);
}

// ------------------------------------------------------------------ depth order
// The reference sorts all S intersections on (image, tile, depth) = 45+ key bits.  Sorting the rows ONCE by
// (image, depth) and emitting the intersections in that order leaves only the (image, tile) bits for the
// S-sized sort: both sorts are stable, so inside a tile the result is (depth, then row index) -- exactly the
// order the reference's single stable sort produces (csrc/Intersect.cpp:283-326).
// gsb200_isect_sorted sorts only the rows that have tiles: their compaction, keys and counts
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

// ------------------------------------------------------------------ emission
// Key of one (gaussian, tile) intersection.  int64_t: the reference's isect id, (image | tile) << 32 | depth bits
// (csrc/IntersectTile.cu:925-988).  uint16_t / uint32_t: the dense tile id image * n_tiles + tile alone -- the rows are
// emitted in depth order already, so the S-sized sort only needs those bits, and moving 2 + 4 instead of 8 + 4 bytes per
// intersection and pass halves its traffic (the 64-bit ids are rebuilt on demand: isect_ids_from_tilekeys_kernel).
template<class KeyT>
struct IsectKey
{
    uint32_t base;
    __device__ __forceinline__ IsectKey(int64_t image, uint32_t, uint32_t, int64_t n_tiles) : base((uint32_t)(image * n_tiles)) {}
    __device__ __forceinline__ KeyT operator()(int64_t tile) const { return (KeyT)(base + (uint32_t)tile); }
};
template<>
struct IsectKey<int64_t>
{
    int64_t hi_db;
    __device__ __forceinline__ IsectKey(int64_t image, uint32_t dbits, uint32_t tile_n_bits, int64_t)
        : hi_db((image << (32 + tile_n_bits)) | (int64_t)dbits)
    {
    }
    __device__ __forceinline__ int64_t operator()(int64_t tile) const { return hi_db | (tile << 32); }
};

// Capacity-bounded emission (gsb200_isect_sorted): the launch covers `total` = capacity row slots and writes into
// capacity-sized outputs, while the real counts sit in device memory (totals[0] intersections, totals[1] rows with
// tiles).  Returns the number of real row slots; the slots between the real intersections and the capacity get padding
// pairs (largest key: the stable sort leaves them behind every real pair; row 0: any valid row).
template<class KeyT>
__device__ __forceinline__ int64_t emit_bounded_rows(
    int64_t j, int64_t n_threads, int64_t total, const int64_t *__restrict__ totals, int64_t cap_isects,
    KeyT *__restrict__ isect_ids, int32_t *__restrict__ flatten_ids
)
{
    const int64_t n_real = totals[0] < cap_isects ? totals[0] : cap_isects;
    for(int64_t s = n_real + j; s < cap_isects; s += n_threads)
    {
        isect_ids[s]   = (KeyT)~(KeyT)0;
        flatten_ids[s] = 0;
    }
    return totals[1] < total ? totals[1] : total;
}

// MASKED: only the tiles whose byte in tile_mask [I, th, tw] is set are emitted, as the masked count counted them.
template<class KeyT, bool MASKED = false>
__global__ void __launch_bounds__(kThreads) isect_emit_kernel(
    int64_t total, int64_t N, const float *__restrict__ means2d, const int32_t *__restrict__ radii,
    const float *__restrict__ depths, const float *__restrict__ conics, const float *__restrict__ opacities,
    const int64_t *__restrict__ cum_tiles, const int64_t *__restrict__ image_ids, const int32_t *__restrict__ order,
    uint32_t tile_size, uint32_t tw, uint32_t th, uint32_t tile_n_bits, KeyT *__restrict__ isect_ids,
    int32_t *__restrict__ flatten_ids, const int64_t *__restrict__ totals = nullptr, int64_t cap_isects = 0,
    const uint8_t *__restrict__ tile_mask = nullptr
)
{
    const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(totals != nullptr)
        total = emit_bounded_rows<KeyT>(j, (int64_t)gridDim.x * blockDim.x, total, totals, cap_isects, isect_ids, flatten_ids);
    if(j >= total)
        return;
    if(totals != nullptr && cum_tiles[j] > cap_isects)
        return; // beyond the speculative capacity: the host sees totals[0] > capacity and redoes the stage
    const int64_t i = order ? (int64_t)order[j] : j;
    const int2 r    = reinterpret_cast<const int2 *>(radii)[i];
    if(r.x <= 0 || r.y <= 0)
        return;
    const float2 m = reinterpret_cast<const float2 *>(means2d)[i];
    float cn[3] = {0.f, 0.f, 0.f}, op = 0.f;
    const bool accu = conics != nullptr && opacities != nullptr;
    if(accu)
        cn[0] = conics[i * 3], cn[1] = conics[i * 3 + 1], cn[2] = conics[i * 3 + 2], op = opacities[i];
    int64_t cur         = (j == 0) ? 0 : cum_tiles[j - 1];
    // packed rows carry their image id
    const int64_t img = image_ids ? image_ids[i] : (i / N);
    const IsectKey<KeyT> key(img, __float_as_uint(depths[i]), tile_n_bits, (int64_t)tw * th);
    const uint8_t *tm = MASKED ? tile_mask + img * (int64_t)tw * th : nullptr;
    tiles_of_gaussian(m.x, m.y, r.x, r.y, accu ? cn : nullptr, accu ? &op : nullptr, tile_size, tw, th, [&](int64_t tile) {
        if(MASKED && tm[tile] == 0)
            return;
        isect_ids[cur]   = key(tile);
        flatten_ids[cur] = (int32_t)i;
        ++cur;
    });
}

// ---- warp-cooperative emit.  One thread per gaussian with a loop over ITS tiles (isect_emit_kernel) leaves a warp
// waiting for its largest gaussian and writes 8 + 4 byte records at lane-dependent strides: at S = 20 M (large
// screen-space gaussians) it took 444 us for 240 MB of output.  Here a gaussian with more than kSmallTiles tiles is
// handed to its whole warp: the tile interval of every tile row is a closed form of the row index (the incremental
// scheme of tiles_of_gaussian only carries the previous row's far line over as the next row's near line), so lane r
// computes row ru0 + r, a warp scan places the rows, and the lanes then write the tiles round-robin -- consecutive
// lanes, consecutive addresses -- in the same order as the sequential enumeration.
template<class KeyT>
__global__ void __launch_bounds__(kThreads) isect_emit_coop_kernel(
    int64_t total, int64_t N, const float *__restrict__ means2d, const int32_t *__restrict__ radii,
    const float *__restrict__ depths, const float *__restrict__ conics, const float *__restrict__ opacities,
    const int64_t *__restrict__ cum_tiles, const int64_t *__restrict__ image_ids, const int32_t *__restrict__ order,
    uint32_t tile_size, uint32_t tw, uint32_t th, uint32_t tile_n_bits, KeyT *__restrict__ isect_ids,
    int32_t *__restrict__ flatten_ids, const int64_t *__restrict__ totals = nullptr, int64_t cap_isects = 0
)
{
    const int64_t j     = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned lane = threadIdx.x & 31;
    if(totals != nullptr)
        total = emit_bounded_rows<KeyT>(j, (int64_t)gridDim.x * blockDim.x, total, totals, cap_isects, isect_ids, flatten_ids);
    const bool active   = j < total && !(totals != nullptr && cum_tiles[j] > cap_isects);
    const int64_t i     = active ? (order ? (int64_t)order[j] : j) : 0;
    int2 r              = make_int2(0, 0);
    float2 m            = make_float2(0.f, 0.f);
    float cn0 = 0.f, cn1 = 0.f, cn2 = 0.f, op = 0.f;
    const bool accu = conics != nullptr && opacities != nullptr;
    int64_t cur = 0, img = 0;
    uint32_t dbits = 0;
    int cnt = 0;
    if(active)
    {
        r = reinterpret_cast<const int2 *>(radii)[i];
        if(r.x > 0 && r.y > 0)
        {
            m = reinterpret_cast<const float2 *>(means2d)[i];
            if(accu)
                cn0 = conics[i * 3], cn1 = conics[i * 3 + 1], cn2 = conics[i * 3 + 2], op = opacities[i];
            cur   = (j == 0) ? 0 : cum_tiles[j - 1];
            cnt   = (int)(cum_tiles[j] - cur);
            img   = image_ids ? image_ids[i] : (i / N);
            dbits = __float_as_uint(depths[i]);
        }
    }
    // small gaussians: the owning lane writes its few tiles
    if(cnt > 0 && cnt <= kSmallTiles)
    {
        float cn[3] = {cn0, cn1, cn2};
        const IsectKey<KeyT> key(img, dbits, tile_n_bits, (int64_t)tw * th);
        tiles_of_gaussian(m.x, m.y, r.x, r.y, accu ? cn : nullptr, accu ? &op : nullptr, tile_size, tw, th, [&](int64_t tile) {
            isect_ids[cur]   = key(tile);
            flatten_ids[cur] = (int32_t)i;
            ++cur;
        });
    }
    // large gaussians: one at a time, the whole warp
    uint32_t big = __ballot_sync(0xffffffffu, cnt > kSmallTiles);
    while(big)
    {
        const int src = __ffs(big) - 1;
        big &= big - 1;
        const float bmx = __shfl_sync(0xffffffffu, m.x, src), bmy = __shfl_sync(0xffffffffu, m.y, src);
        const int brx = __shfl_sync(0xffffffffu, r.x, src), bry = __shfl_sync(0xffffffffu, r.y, src);
        const float b0 = __shfl_sync(0xffffffffu, cn0, src), b1 = __shfl_sync(0xffffffffu, cn1, src);
        const float b2 = __shfl_sync(0xffffffffu, cn2, src), bop = __shfl_sync(0xffffffffu, op, src);
        const int64_t bcur = __shfl_sync(0xffffffffu, cur, src), bimg = __shfl_sync(0xffffffffu, img, src);
        const uint32_t bdb = __shfl_sync(0xffffffffu, dbits, src);
        const IsectKey<KeyT> bkey(bimg, bdb, tile_n_bits, (int64_t)tw * th);
        const int32_t bi  = (int32_t)__shfl_sync(0xffffffffu, i, src);
        const AccuGauss g = accu_setup(bmx, bmy, brx, bry, accu, b0, b1, b2, bop, tile_size, tw, th);
        if(g.empty)
            continue;
        int64_t base = bcur;
        for(int u0 = g.ru0; u0 < g.ru1; u0 += 32)
        {
            const int u = u0 + (int)lane;
            int v0 = 0, v1 = 0;
            if(u < g.ru1)
                accu_row(g, u, v0, v1);
            const int len = v1 - v0;
            int incl      = len;
#pragma unroll
            for(int o = 1; o < 32; o <<= 1)
            {
                const int up = __shfl_up_sync(0xffffffffu, incl, o);
                if((int)lane >= o)
                    incl += up;
            }
            const int excl  = incl - len;
            const int chunk = __shfl_sync(0xffffffffu, incl, 31);
            // tile k of this 32-row chunk: row = the last row with excl <= k (binary search over the lanes; the loop is
            // warp-uniform so that every shuffle sees all 32 lanes, only the stores are predicated)
            for(int k0 = 0; k0 < chunk; k0 += 32)
            {
                const int k = k0 + (int)lane;
                int row     = 0;
#pragma unroll
                for(int step = 16; step > 0; step >>= 1)
                {
                    const int probe = row + step; // <= 31
                    const int pe    = __shfl_sync(0xffffffffu, excl, probe);
                    if(pe <= k)
                        row = probe;
                }
                const int rex = __shfl_sync(0xffffffffu, excl, row);
                const int rv0 = __shfl_sync(0xffffffffu, v0, row);
                if(k < chunk)
                {
                    const int v        = rv0 + (k - rex);
                    const int uu       = u0 + row;
                    const int64_t tile = g.isY ? (int64_t)uu * tw + v : (int64_t)v * tw + uu;
                    isect_ids[base + k]   = bkey(tile);
                    flatten_ids[base + k] = bi;
                }
            }
            base += chunk;
        }
    }
}

// Dense tile ids are key_bytes wide, 2 or 4 (the caller checked): calls f with a uint16_t or a uint32_t, whose type
// is the key type.
template<class F>
static auto with_key_type(int key_bytes, F &&f)
{
    return key_bytes == 2 ? f(uint16_t{}) : f(uint32_t{});
}

// stage of gsb200_isect_sorted, which checked the arguments: emission of the cap_vis depth-ordered row slots into
// capacity-sized outputs, real counts in `totals` (device)
static int emit_tilekeys_bounded(
    int64_t N, int64_t cap_vis, int64_t max_tiles_hint, const float *means2d, const int32_t *radii, const float *depths,
    const float *conics, const float *opacities, const int64_t *cum_tiles, const int64_t *image_ids, const uint8_t *tile_mask,
    const int32_t *order, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, int key_bytes, void *keys,
    int32_t *flatten_ids, const int64_t *totals, int64_t cap_isects, cudaStream_t st
)
{
    const uint32_t tile_bits = bits_for_count((int64_t)tile_width * tile_height);
    // the cooperative kernel pays off when SOME gaussian covers many tiles (one lane looping over thousands of tiles is the
    // tail of the whole launch); when even the largest row has few, the plain one-thread-per-gaussian kernel is leaner
    // (38 vs 45 us at cfg3)
    const bool serial = max_tiles_hint > 0 && max_tiles_hint <= 96;
    return with_key_type(key_bytes, [&](auto key) {
        using KeyT = decltype(key);
        // a mask breaks the contiguous per-row tile intervals the cooperative kernel places: one thread per row
        if(tile_mask != nullptr)
            isect_emit_kernel<KeyT, true><<<grid_for(cap_vis, kThreads), kThreads, 0, st>>>(
                cap_vis, N, means2d, radii, depths, conics, opacities, cum_tiles, image_ids, order, tile_size, tile_width,
                tile_height, tile_bits, static_cast<KeyT *>(keys), flatten_ids, totals, cap_isects, tile_mask
            );
        else if(serial)
            isect_emit_kernel<KeyT><<<grid_for(cap_vis, kThreads), kThreads, 0, st>>>(
                cap_vis, N, means2d, radii, depths, conics, opacities, cum_tiles, image_ids, order, tile_size, tile_width,
                tile_height, tile_bits, static_cast<KeyT *>(keys), flatten_ids, totals, cap_isects
            );
        else
            isect_emit_coop_kernel<KeyT><<<grid_for(cap_vis, kThreads), kThreads, 0, st>>>(
                cap_vis, N, means2d, radii, depths, conics, opacities, cum_tiles, image_ids, order, tile_size, tile_width,
                tile_height, tile_bits, static_cast<KeyT *>(keys), flatten_ids, totals, cap_isects
            );
        return check_launch();
    });
}

// ------------------------------------------------------------------ tile sort
// The (image, tile)-only sort of the depth-ordered intersections: 2- or 4-byte dense tile ids as keys, the row index
// as value -- 6 (8) instead of the reference's 12 bytes per intersection and direction in each radix pass.
template<class KeyT>
static size_t sort_tile_pairs_workspace_bytes(int64_t n, int end_bit)
{
    size_t bytes = 0;
    cub::DeviceRadixSort::SortPairs(
        (void *)nullptr, bytes, (const KeyT *)nullptr, (KeyT *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr, n, 0, end_bit
    );
    return bytes;
}

template<class KeyT>
static int sort_tile_pairs(
    int64_t n, int end_bit, const void *keys_in, const int32_t *vals_in, void *keys_out, int32_t *vals_out, void *workspace,
    size_t workspace_bytes, cudaStream_t st
)
{
    size_t need = sort_tile_pairs_workspace_bytes<KeyT>(n, end_bit);
    if(need > workspace_bytes)
        return GSB200_E_WORKSPACE;
    GSB_CUDA_TRY(cub::DeviceRadixSort::SortPairs(
        workspace, need, static_cast<const KeyT *>(keys_in), static_cast<KeyT *>(keys_out), vals_in, vals_out, n, 0, end_bit, st
    ));
    return GSB200_OK;
}

// ------------------------------------------------------------------ offsets
// offsets[(image, tile)] = first sorted index of that tile's run.  One thread per sorted
// intersection; a thread that starts a new run also fills the empty tiles before it.
__global__ void __launch_bounds__(kThreads) isect_offsets_kernel(
    int64_t n_isects, const int64_t *__restrict__ isect_ids, int64_t total_tiles, int64_t n_tiles, uint32_t tile_n_bits,
    int32_t *__restrict__ offsets
)
{
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(s >= n_isects)
        return;
    const int64_t mask = ((int64_t)1 << tile_n_bits) - 1;
    const int64_t hi   = isect_ids[s] >> 32;
    const int64_t id   = (hi >> tile_n_bits) * n_tiles + (hi & mask);
    int64_t prev       = -1;
    if(s > 0)
    {
        const int64_t hp = isect_ids[s - 1] >> 32;
        prev             = (hp >> tile_n_bits) * n_tiles + (hp & mask);
    }
    for(int64_t k = prev + 1; k <= id; ++k)
        offsets[k] = (int32_t)s;
    if(s == n_isects - 1)
        for(int64_t k = id + 1; k < total_tiles; ++k)
            offsets[k] = (int32_t)n_isects;
}

// offsets[(image, tile)] from sorted dense tile ids (narrow keys): same contract as isect_offsets_kernel
template<class KeyT>
__global__ void __launch_bounds__(kThreads) isect_offsets_tilekeys_kernel(
    int64_t n_isects, const KeyT *__restrict__ keys, int64_t total_tiles, int32_t *__restrict__ offsets,
    const int64_t *__restrict__ totals = nullptr
)
{
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(totals != nullptr && totals[0] < n_isects)
        n_isects = totals[0]; // capacity-sized launch: the pairs past the real count are padding
    if(s >= n_isects)
        return;
    // Real keys are < total_tiles.  After a capacity miss (gsb200_isect_sorted with a count above its capacity) some
    // slots hold uninitialised pairs: the result is discarded by the caller, but no write may leave the array.
    int64_t id         = (int64_t)keys[s];
    const int64_t prev = s > 0 ? (int64_t)keys[s - 1] : -1;
    id                 = id < total_tiles ? id : total_tiles - 1;
    for(int64_t k = prev + 1; k <= id; ++k)
        offsets[k] = (int32_t)s;
    if(s == n_isects - 1)
        for(int64_t k = id + 1; k < total_tiles; ++k)
            offsets[k] = (int32_t)n_isects;
}

static int offsets_tilekeys_bounded(
    int64_t cap_isects, int key_bytes, const void *keys, int64_t total_tiles, int32_t *offsets, const int64_t *totals, cudaStream_t st
)
{
    // no thread writes anything when the real count is 0: start from zeros
    GSB_CUDA_TRY(cudaMemsetAsync(offsets, 0, sizeof(int32_t) * (size_t)total_tiles, st));
    if(cap_isects == 0)
        return GSB200_OK;
    return with_key_type(key_bytes, [&](auto key) {
        using KeyT = decltype(key);
        isect_offsets_tilekeys_kernel<KeyT><<<grid_for(cap_isects, kThreads), kThreads, 0, st>>>(
            cap_isects, static_cast<const KeyT *>(keys), total_tiles, offsets, totals
        );
        return check_launch();
    });
}

// tile_offsets[a] = offsets[active_tiles[a]] for a < n_active, tile_offsets[n_active] = n_isects.  The ids come from the
// caller unchecked: one outside [0, total_tiles) gets n_isects, as if it were a tile past the last one.
__global__ void __launch_bounds__(kThreads) isect_active_offsets_kernel(
    int64_t n_active, const int32_t *__restrict__ active_tiles, int64_t total_tiles, const int32_t *__restrict__ offsets,
    int64_t n_isects, int32_t *__restrict__ tile_offsets
)
{
    const int64_t a = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(a > n_active)
        return;
    const int64_t t = a < n_active ? (int64_t)active_tiles[a] : -1;
    tile_offsets[a] = t >= 0 && t < total_tiles ? offsets[t] : (int32_t)n_isects;
}

// the reference's 64-bit intersection ids, rebuilt from the sorted tile ids and the rows' depths
template<class KeyT>
__global__ void __launch_bounds__(kThreads) isect_ids_from_tilekeys_kernel(
    int64_t n_isects, const KeyT *__restrict__ keys, const int32_t *__restrict__ flatten_ids, const float *__restrict__ depths,
    int64_t n_tiles, uint32_t tile_n_bits, int64_t *__restrict__ isect_ids
)
{
    const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(s >= n_isects)
        return;
    const int64_t id = (int64_t)keys[s];
    const int64_t image = id / n_tiles, tile = id - image * n_tiles;
    isect_ids[s] = (((image << tile_n_bits) | tile) << 32) | (int64_t)__float_as_uint(depths[flatten_ids[s]]);
}

// ------------------------------------------------------------------ workspace of gsb200_isect_sorted
struct SortedLayout
{
    size_t rows_in, keys_in, keys_out, order, cum, n_sel, tkeys, tvals, cub, total;
};
static SortedLayout sorted_layout(int64_t total_rows, int64_t cap_vis, int64_t cap_isects, int key_bytes, int depth_end_bit, int tile_end_bit)
{
    auto al = [](size_t b) { return (b + 255) & ~(size_t)255; };
    SortedLayout L;
    size_t a = 0, b = 0, c = 0;
    cub::DeviceSelect::If((void *)nullptr, a, cub::CountingInputIterator<int32_t>(0), (int32_t *)nullptr, (int32_t *)nullptr, total_rows, HasTiles{nullptr});
    cub::DeviceRadixSort::SortPairs(
        (void *)nullptr, b, (const uint64_t *)nullptr, (uint64_t *)nullptr, (const int32_t *)nullptr, (int32_t *)nullptr, cap_vis, 0, depth_end_bit
    );
    cub::TransformInputIterator<int64_t, CountOfBounded, cub::CountingInputIterator<int32_t>> it(
        cub::CountingInputIterator<int32_t>(0), CountOfBounded{nullptr, nullptr, nullptr, 0}
    );
    cub::DeviceScan::InclusiveSum((void *)nullptr, c, it, (int64_t *)nullptr, cap_vis);
    const size_t d = with_key_type(key_bytes, [&](auto key) {
        return sort_tile_pairs_workspace_bytes<decltype(key)>(cap_isects, tile_end_bit);
    });
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

// ------------------------------------------------------------------ totals to the host
// The totals, published straight into pinned host memory.  A cudaMemcpyAsync of 24 bytes takes a copy engine and,
// on a box whose PCIe link is busy with an image upload, arrives late; a handful of system-scope stores from a kernel do
// not.  host_mapped: int64 [4] in pinned (mapped) host memory; the host polls host_mapped[3] for `seq`.
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

// =====================================================================================================
// C ABI
using namespace gsb;

extern "C" size_t gsb200_isect_scan_workspace_bytes(int64_t n_elements)
{
    size_t bytes = 0;
    if(n_elements <= 0)
        return 0;
    cub::DeviceScan::InclusiveSum((void *)nullptr, bytes, (const int32_t *)nullptr, (int64_t *)nullptr, n_elements);
    return bytes + 256;
}

extern "C" int gsb200_isect_count(
    int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *conics, const float *opacities,
    uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, int32_t *tiles_per_gauss, int64_t *cum_tiles,
    void *workspace, size_t workspace_bytes, void *stream
)
{
    if(I < 0 || N < 0 || tile_size == 0)
        return GSB200_E_INVALID;
    const int64_t total = I * N;
    if(total == 0)
        return GSB200_OK;
    if(!means2d || !radii || !tiles_per_gauss || !cum_tiles || !workspace || total > 0x7fffffffLL)
        return GSB200_E_INVALID;
    if(bits_for_count(I) + bits_for_count((int64_t)tile_width * tile_height) > 32)
        return GSB200_E_KEYBITS;
    cudaStream_t st = (cudaStream_t)stream;
    size_t need     = 0;
    cub::DeviceScan::InclusiveSum((void *)nullptr, need, tiles_per_gauss, cum_tiles, total, st);
    if(need > workspace_bytes)
        return GSB200_E_WORKSPACE;
    isect_count_kernel<false><<<grid_for(total, kThreads), kThreads, 0, st>>>(
        total, means2d, radii, conics, opacities, tile_size, tile_width, tile_height, tiles_per_gauss, nullptr
    );
    if(int rc = check_launch())
        return rc;
    GSB_CUDA_TRY(cub::DeviceScan::InclusiveSum(workspace, need, tiles_per_gauss, cum_tiles, total, st));
    return GSB200_OK;
}

extern "C" int gsb200_isect_emit(
    int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *depths, const float *conics,
    const float *opacities, const int64_t *cum_tiles, const int64_t *image_ids, uint32_t tile_size, uint32_t tile_width,
    uint32_t tile_height, int64_t *isect_ids, int32_t *flatten_ids, void *stream
)
{
    if(I < 0 || N < 0 || tile_size == 0)
        return GSB200_E_INVALID;
    // packed layout: N rows in total (image_ids given), I only sizes the key; dense: I * N rows
    const int64_t total = image_ids ? N : I * N;
    if(total == 0)
        return GSB200_OK;
    if(!means2d || !radii || !depths || !cum_tiles || !isect_ids || !flatten_ids)
        return GSB200_E_INVALID;
    const uint32_t tile_bits = bits_for_count((int64_t)tile_width * tile_height);
    if(bits_for_count(I) + tile_bits > 32)
        return GSB200_E_KEYBITS;
    isect_emit_coop_kernel<int64_t><<<grid_for(total, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
        total, N, means2d, radii, depths, conics, opacities, cum_tiles, image_ids, nullptr, tile_size, tile_width, tile_height,
        tile_bits, isect_ids, flatten_ids
    );
    return check_launch();
}

extern "C" int gsb200_isect_count_totals(
    int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *conics, const float *opacities,
    const int64_t *image_ids, const uint8_t *tile_mask, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
    int32_t *tiles_per_gauss, int64_t *totals, void *stream
)
{
    if(I < 0 || N < 0 || tile_size == 0 || !totals)
        return GSB200_E_INVALID;
    cudaStream_t st = (cudaStream_t)stream;
    GSB_CUDA_TRY(cudaMemsetAsync(totals, 0, 3 * sizeof(int64_t), st));
    // the rows of gsb200_isect_sorted: N rows in total when image_ids is given, else I * N
    const int64_t total = image_ids ? N : I * N;
    if(total == 0)
        return GSB200_OK;
    if(!means2d || !radii || !tiles_per_gauss || total > 0x7fffffffLL)
        return GSB200_E_INVALID;
    if(bits_for_count(I) + bits_for_count((int64_t)tile_width * tile_height) > 32)
        return GSB200_E_KEYBITS;
    unsigned long long *tot = reinterpret_cast<unsigned long long *>(totals);
    if(tile_mask != nullptr)
        isect_count_kernel<true, true><<<grid_for(total, kThreads), kThreads, 0, st>>>(
            total, means2d, radii, conics, opacities, tile_size, tile_width, tile_height, tiles_per_gauss, tot, N, I, image_ids,
            tile_mask
        );
    else
        isect_count_kernel<true><<<grid_for(total, kThreads), kThreads, 0, st>>>(
            total, means2d, radii, conics, opacities, tile_size, tile_width, tile_height, tiles_per_gauss, tot
        );
    return check_launch();
}

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
extern "C" size_t gsb200_isect_sorted_workspace_bytes(
    int64_t I, int64_t total_rows, int64_t cap_vis, int64_t cap_isects, int key_bytes, uint32_t tile_width, uint32_t tile_height
)
{
    if(I <= 0 || total_rows <= 0 || cap_vis <= 0 || cap_isects <= 0 || (key_bytes != 2 && key_bytes != 4))
        return 0;
    const int tile_end = (int)bits_for_count(I * (int64_t)tile_width * tile_height);
    return sorted_layout(total_rows, cap_vis, cap_isects, key_bytes, 32 + (int)bits_for_count(I), tile_end > 0 ? tile_end : 1).total;
}

extern "C" int gsb200_isect_sorted(
    int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *depths, const float *conics,
    const float *opacities, const int64_t *image_ids, const uint8_t *tile_mask, uint32_t tile_size, uint32_t tile_width,
    uint32_t tile_height, const int32_t *tiles_per_gauss, const int64_t *totals, int64_t cap_vis, int64_t cap_isects,
    int64_t max_tiles_hint, int key_bytes, void *tile_keys, int32_t *flatten_ids, int32_t *offsets, void *workspace,
    size_t workspace_bytes, void *stream
)
{
    if(I <= 0 || N <= 0 || cap_vis <= 0 || cap_isects <= 0 || tile_size == 0 || (key_bytes != 2 && key_bytes != 4))
        return GSB200_E_INVALID;
    // packed layout: N rows in total (image_ids given), I only sizes the keys and the offsets; dense: I * N rows
    const int64_t total = image_ids ? N : I * N, total_tiles = I * (int64_t)tile_width * tile_height;
    if(!means2d || !radii || !depths || !tiles_per_gauss || !totals || !tile_keys || !flatten_ids || !offsets || !workspace
       || total > 0x7fffffffLL || cap_vis > total || cap_isects > 0x7fffffffLL)
        return GSB200_E_INVALID;
    if(bits_for_count(I) + bits_for_count((int64_t)tile_width * tile_height) > 32
       || (int)bits_for_count(total_tiles) > 8 * key_bytes)
        return GSB200_E_KEYBITS;
    const bool single  = I == 1; // one image: the depth bits alone are the key, whatever the row layout
    const int depth_end = single ? 32 : 32 + (int)bits_for_count(I);
    int tile_end        = (int)bits_for_count(total_tiles);
    tile_end            = tile_end > 0 ? tile_end : 1;
    const auto L        = sorted_layout(total, cap_vis, cap_isects, key_bytes, 32 + (int)bits_for_count(I), tile_end);
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
        ws + L.cub, cub_bytes, cub::CountingInputIterator<int32_t>(0), rows_in, n_sel, total, HasTiles{tiles_per_gauss}, st
    ));
    // 2. their (image, depth) keys -- padding slots get the largest key -- and a stable sort of the cap_vis slots
    depth_key_rows_bounded_kernel<<<(unsigned)((cap_vis + 255) / 256), 256, 0, st>>>(
        cap_vis, N, rows_in, depths, image_ids, single, totals, k_in
    );
    if(int rc = check_launch())
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
    cub::TransformInputIterator<int64_t, CountOfBounded, cub::CountingInputIterator<int32_t>> it(
        cub::CountingInputIterator<int32_t>(0), CountOfBounded{tiles_per_gauss, order, totals, cap_vis}
    );
    cub_bytes = cub_cap;
    GSB_CUDA_TRY(cub::DeviceScan::InclusiveSum(ws + L.cub, cub_bytes, it, cum, cap_vis, st));
    // 4. emission in depth order, (dense tile id, row) pairs; 5. stable sort on the tile id; 6. offsets
    if(int rc = emit_tilekeys_bounded(
           N, cap_vis, max_tiles_hint, means2d, radii, depths, conics, opacities, cum, image_ids, tile_mask, order, tile_size,
           tile_width, tile_height, key_bytes, tkeys, tvals, totals, cap_isects, st
       ))
        return rc;
    if(int rc = with_key_type(key_bytes, [&](auto key) {
           return sort_tile_pairs<decltype(key)>(cap_isects, tile_end, tkeys, tvals, tile_keys, flatten_ids, ws + L.cub, cub_cap, st);
       }))
        return rc;
    return offsets_tilekeys_bounded(cap_isects, key_bytes, tile_keys, total_tiles, offsets, totals, st);
}

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
    publish_totals_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(totals, static_cast<volatile int64_t *>(dptr), seq);
    return check_launch();
}

extern "C" int gsb200_isect_ids_from_tilekeys(
    int64_t n_isects, int key_bytes, const void *tile_keys, const int32_t *flatten_ids, const float *depths, int64_t I,
    uint32_t tile_width, uint32_t tile_height, int64_t *isect_ids, void *stream
)
{
    if(n_isects < 0 || I < 0 || (key_bytes != 2 && key_bytes != 4))
        return GSB200_E_INVALID;
    if(n_isects == 0)
        return GSB200_OK;
    if(!tile_keys || !flatten_ids || !depths || !isect_ids)
        return GSB200_E_INVALID;
    const int64_t n_tiles = (int64_t)tile_width * tile_height;
    cudaStream_t st       = (cudaStream_t)stream;
    return with_key_type(key_bytes, [&](auto key) {
        using KeyT = decltype(key);
        isect_ids_from_tilekeys_kernel<KeyT><<<grid_for(n_isects, kThreads), kThreads, 0, st>>>(
            n_isects, static_cast<const KeyT *>(tile_keys), flatten_ids, depths, n_tiles, bits_for_count(n_tiles), isect_ids
        );
        return check_launch();
    });
}

extern "C" int gsb200_isect_offsets(
    int64_t n_isects, const int64_t *isect_ids, int64_t I, uint32_t tile_width, uint32_t tile_height, int32_t *offsets,
    void *stream
)
{
    if(n_isects < 0 || I < 0)
        return GSB200_E_INVALID;
    const int64_t n_tiles = (int64_t)tile_width * tile_height;
    const int64_t total   = I * n_tiles;
    if(total == 0)
        return GSB200_OK;
    if(!offsets)
        return GSB200_E_INVALID;
    cudaStream_t st = (cudaStream_t)stream;
    if(n_isects == 0)
    {
        GSB_CUDA_TRY(cudaMemsetAsync(offsets, 0, sizeof(int32_t) * (size_t)total, st));
        return GSB200_OK;
    }
    if(!isect_ids)
        return GSB200_E_INVALID;
    isect_offsets_kernel<<<grid_for(n_isects, kThreads), kThreads, 0, st>>>(
        n_isects, isect_ids, total, n_tiles, bits_for_count(n_tiles), offsets
    );
    return check_launch();
}

extern "C" int gsb200_isect_active_offsets(
    int64_t n_active, const int32_t *active_tiles, int64_t I, uint32_t tile_width, uint32_t tile_height,
    const int32_t *offsets, int64_t n_isects, int32_t *tile_offsets, void *stream
)
{
    const int64_t total_tiles = I * (int64_t)tile_width * tile_height;
    if(n_active < 0 || I < 0 || n_isects < 0 || n_isects > 0x7fffffffLL || !tile_offsets || (n_active > 0 && !active_tiles)
       || (total_tiles > 0 && !offsets))
        return GSB200_E_INVALID;
    isect_active_offsets_kernel<<<grid_for(n_active + 1, kThreads), kThreads, 0, (cudaStream_t)stream>>>(
        n_active, active_tiles, total_tiles, offsets, n_isects, tile_offsets
    );
    return check_launch();
}
