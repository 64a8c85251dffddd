// isect.cuh -- the device code of the tile intersection that more than one unit runs: the tile enumeration of one
// gaussian and the block reduction of the three totals.  The fused projection (pergauss.cu) counts tiles with the same
// functions as the count and emit kernels (isect.cu); both units are compiled with -fmad=false, so the counts agree
// bit for bit.
#pragma once
#include "gaussmath.cuh"

namespace gsb
{
// Enumerates the tiles of one gaussian in the reference's emit order, calling f(tile_id).
// AccuTile / SNUGBOX (csrc/IntersectTile.cu:83-207, 288-373) or the radius AABB (:374-463).
template<class F>
__device__ __forceinline__ int tiles_of_gaussian(
    float mx, float my, int rx, int ry, const float *conic, const float *opacity, uint32_t tile_size, uint32_t tw,
    uint32_t th, F &&f
)
{
    if(rx <= 0 || ry <= 0)
        return 0;
    int count      = 0;
    const float ts = (float)tile_size;
    auto clampi    = [](int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); };
    if(conic != nullptr && opacity != nullptr)
    {
        const float A = conic[0], Bc = conic[1], Cc = conic[2];
        const float disc = Bc * Bc - A * Cc;
        float t          = 2.f * exact_log(*opacity / kAlphaThreshold);
        const float cap  = kGaussianExtend * kGaussianExtend;
        t                = t < cap ? t : cap;
        const float ntd  = -t / disc;
        const float xe = sqrtf(ntd * Cc), ye = sqrtf(ntd * A);
        const float bminx = mx - xe, bminy = my - ye, bmaxx = mx + xe, bmaxy = my + ye;
        const float BxC = Bc * xe / Cc, ByA = Bc * ye / A;
        const float argminx = my + BxC, argminy = mx + ByA, argmaxx = my - BxC, argmaxy = mx - ByA;
        const int rminx = clampi((int)(bminx / ts), 0, (int)tw), rminy = clampi((int)(bminy / ts), 0, (int)th);
        const int rmaxx = clampi((int)(bmaxx / ts + 1.f), 0, (int)tw), rmaxy = clampi((int)(bmaxy / ts + 1.f), 0, (int)th);
        const int ys = rmaxy - rminy, xs = rmaxx - rminx;
        if(ys * xs == 0)
            return 0;
        const bool isY = ys < xs;
        const int ru0 = isY ? rminy : rminx, ru1 = isY ? rmaxy : rmaxx, rv0 = isY ? rminx : rminy, rv1 = isY ? rmaxx : rmaxy;
        const float bminu = isY ? bminy : bminx, bmaxu = isY ? bmaxy : bmaxx;
        const float bminv = isY ? bminx : bminy, bmaxv = isY ? bmaxx : bmaxy;
        const float amin_v = isY ? argminx : argminy, amax_v = isY ? argmaxx : argmaxy;
        const float pu = isY ? my : mx, pv = isY ? mx : my, coeff = isY ? A : Cc;
        auto line = [&](float coord, float &lo, float &hi) {
            const float h  = coord - pu;
            const float sq = sqrtf(disc * h * h + t * coeff);
            lo             = (-Bc * h - sq) / coeff + pv;
            hi             = (-Bc * h + sq) / coeff + pv;
        };
        float maxlo = bmaxv, maxhi = bminv, minlo, minhi;
        float min_line = (float)ru0 * ts;
        if(bminu <= min_line)
            line(min_line, minlo, minhi);
        else
            minlo = maxlo, minhi = maxhi;
        for(int u = ru0; u < ru1; ++u)
        {
            const float max_line = min_line + ts;
            if(max_line <= bmaxu)
                line(max_line, maxlo, maxhi);
            const float emin = (min_line <= amin_v && amin_v < max_line) ? bminv : (minlo < maxlo ? minlo : maxlo);
            const float emax = (min_line <= amax_v && amax_v < max_line) ? bmaxv : (minhi > maxhi ? minhi : maxhi);
            const int e0 = (int)(emin / ts), e1 = (int)(emax / ts + 1.f);
            int v0 = e0 < rv1 ? e0 : rv1;
            v0     = v0 > rv0 ? v0 : rv0;
            int v1 = e1 > rv0 ? e1 : rv0;
            v1     = v1 < rv1 ? v1 : rv1;
            for(int v = v0; v < v1; ++v)
            {
                ++count;
                f(isY ? (int64_t)u * tw + v : (int64_t)v * tw + u);
            }
            minlo = maxlo, minhi = maxhi, min_line = max_line;
        }
    }
    else
    {
        const float trx = (float)rx / ts, try_ = (float)ry / ts, tx = mx / ts, ty = my / ts;
        const int x0 = clampi((int)floorf(tx - trx), 0, (int)tw), y0 = clampi((int)floorf(ty - try_), 0, (int)th);
        const int x1 = clampi((int)ceilf(tx + trx), 0, (int)tw), y1 = clampi((int)ceilf(ty + try_), 0, (int)th);
        for(int i = y0; i < y1; ++i)
            for(int j = x0; j < x1; ++j)
            {
                ++count;
                f((int64_t)i * tw + j);
            }
    }
    return count;
}

// The totals of a launch that counts tiles, accumulated over its blocks into totals (int64 [3], zeroed by the host):
// [0] = number of intersections, [1] = rows with tiles, [2] = the largest tile count of a row (picks the emit kernel).
// block_tile_totals_begin() is the first thing every thread of the block does; block_tile_totals() the last, with the
// thread's tile count (0 for a thread without a row).
__device__ __forceinline__ unsigned long long *block_tile_totals_begin()
{
    __shared__ unsigned long long s_tot[3];
    if(threadIdx.x < 3)
        s_tot[threadIdx.x] = 0ull;
    __syncthreads();
    return s_tot;
}
__device__ __forceinline__ void block_tile_totals(int cnt, unsigned long long *s_tot, unsigned long long *__restrict__ totals)
{
    const int wsum         = __reduce_add_sync(0xffffffffu, cnt);
    const int wmax         = __reduce_max_sync(0xffffffffu, cnt);
    const unsigned nonzero = __ballot_sync(0xffffffffu, cnt > 0);
    if((threadIdx.x & 31) == 0 && nonzero != 0u)
    {
        atomicAdd(&s_tot[0], (unsigned long long)wsum);
        atomicAdd(&s_tot[1], (unsigned long long)__popc(nonzero));
        atomicMax(&s_tot[2], (unsigned long long)wmax);
    }
    __syncthreads();
    if(threadIdx.x < 2 && s_tot[threadIdx.x] != 0ull)
        atomicAdd(&totals[threadIdx.x], s_tot[threadIdx.x]);
    if(threadIdx.x == 2 && s_tot[2] != 0ull)
        atomicMax(&totals[2], s_tot[2]);
}
} // namespace gsb
