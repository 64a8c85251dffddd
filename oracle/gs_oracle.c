/*
 * gs_oracle.c -- CPU oracle for the gsplat rasterization() hot path.
 *
 * TEST INFRASTRUCTURE ONLY (see gso_impl.h header).  Plain C restatement of the
 * reference algorithms (nerfstudio-project/gsplat v1.6.0, /root/reference/gsplat/cuda);
 * each function cites the file:line it follows.  Parity status: pinned against the
 * reference's own Python twins (_torch_impl.py / _math.py) through the committed
 * fixtures in tests/golden/ (generator: tests/golden/make_golden.py).
 *
 * Built by oracle/Makefile into oracle/libgs_oracle.so:
 *     gcc -O2 -fopenmp -ffp-contract=off -shared -fPIC gs_oracle.c -lm
 * -ffp-contract=off keeps every float op individually rounded so the CUDA kernels that
 * are compiled with -fmad=false can be compared bit for bit.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* ---- float32 instantiation: *_f32 ---- */
#define REAL float
#define SUF _f32
#define R_SQRT sqrtf
#define R_EXP expf
#define R_CEIL ceilf
#define R_FLOOR floorf
#define R_FREXP frexpf
#define R_ATAN2 atan2f
#include "gso_impl.h"
#undef REAL
#undef SUF
#undef R_SQRT
#undef R_EXP
#undef R_CEIL
#undef R_FLOOR
#undef R_FREXP
#undef R_ATAN2

/* ---- float64 instantiation: *_f64 ---- */
#define REAL double
#define SUF _f64
#define R_SQRT sqrt
#define R_EXP exp
#define R_CEIL ceil
#define R_FLOOR floor
#define R_FREXP frexp
#define R_ATAN2 atan2
#include "gso_impl.h"
#undef REAL
#undef SUF

/* Bits needed to index `count` items as 0..count-1 (0 when count <= 1).
 * Reference: csrc/MathUtils.h:26-36 (bits_for_count). */
uint32_t gso_bits_for_count(int64_t count)
{
    if(count <= 1)
        return 0;
    uint64_t v = (uint64_t)count - 1u;
    uint32_t b = 0;
    while(v)
    {
        ++b;
        v >>= 1;
    }
    return b;
}

/* Stable LSD radix sort of (int64 key, int32 value) pairs over key bits [0, end_bit).
 * Reference: cub::DeviceRadixSort::SortPairs call, csrc/IntersectTile.cu:1078-1121 -- a stable
 * sort on the low `32 + tile_bits + image_bits` key bits. */
int gso_sort_pairs(int64_t n, int end_bit, const int64_t *keys_in, const int32_t *vals_in, int64_t *keys_out, int32_t *vals_out)
{
    if(n <= 0)
        return 0;
    int64_t *k0 = (int64_t *)malloc(sizeof(int64_t) * (size_t)n), *k1 = (int64_t *)malloc(sizeof(int64_t) * (size_t)n);
    int32_t *v0 = (int32_t *)malloc(sizeof(int32_t) * (size_t)n), *v1 = (int32_t *)malloc(sizeof(int32_t) * (size_t)n);
    if(!k0 || !k1 || !v0 || !v1)
        return -1;
    memcpy(k0, keys_in, sizeof(int64_t) * (size_t)n);
    memcpy(v0, vals_in, sizeof(int32_t) * (size_t)n);
    for(int shift = 0; shift < end_bit; shift += 8)
    {
        int64_t hist[257];
        memset(hist, 0, sizeof(hist));
        int bits      = end_bit - shift < 8 ? end_bit - shift : 8;
        uint64_t mask = (1ull << bits) - 1ull;
        for(int64_t i = 0; i < n; ++i)
            hist[(((uint64_t)k0[i]) >> shift & mask) + 1]++;
        for(int b = 0; b < 256; ++b)
            hist[b + 1] += hist[b];
        for(int64_t i = 0; i < n; ++i)
        {
            int64_t d = hist[((uint64_t)k0[i]) >> shift & mask]++;
            k1[d]     = k0[i];
            v1[d]     = v0[i];
        }
        int64_t *tk = k0; k0 = k1; k1 = tk;
        int32_t *tv = v0; v0 = v1; v1 = tv;
    }
    memcpy(keys_out, k0, sizeof(int64_t) * (size_t)n);
    memcpy(vals_out, v0, sizeof(int32_t) * (size_t)n);
    free(k0); free(k1); free(v0); free(v1);
    return 0;
}

/* offsets[I, th, tw]: exclusive start of each (image, tile) run in the sorted keys.
 * Reference: csrc/IntersectTile.cu:925-988 (intersect_offset_kernel); n_isects == 0 -> zeros
 * (:1003-1007). */
int gso_isect_offsets(int64_t n_isects, const int64_t *isect_ids, int64_t I, uint32_t tw, uint32_t th, int32_t *offsets)
{
    int64_t n_tiles    = (int64_t)tw * th;
    uint32_t tile_bits = gso_bits_for_count(n_tiles);
    int64_t total      = I * n_tiles;
    if(n_isects == 0)
    {
        memset(offsets, 0, sizeof(int32_t) * (size_t)total);
        return 0;
    }
    int64_t next = 0; /* next (image,tile) slot whose offset is still unwritten */
    for(int64_t s = 0; s < n_isects; ++s)
    {
        int64_t hi  = isect_ids[s] >> 32;
        int64_t img = hi >> tile_bits, tid = hi & ((1ll << tile_bits) - 1);
        int64_t id  = img * n_tiles + tid;
        while(next <= id)
            offsets[next++] = (int32_t)s;
    }
    while(next < total)
        offsets[next++] = (int32_t)n_isects;
    return 0;
}
