// common.cuh -- shared device/host helpers for libgsplat_b200 (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "../../include/gsplat_b200.h"

namespace gsb
{
// ---- constants of the path (reference: include/Common.h:97-114, gsplat/cuda/_constants.py:16-27)
constexpr float kAlphaThreshold        = 1.f / 255.f;
constexpr float kGaussianExtend        = 3.33f;
constexpr float kMaxAlpha              = 0.99f;
constexpr float kTransmittanceThreshold = 1e-4f;
constexpr float kMinCompensation       = 0.005f;
constexpr float kMinOneMinusAlpha      = 1e-6f;
constexpr int kTile                    = 16; // the only tile size the rasterizer is built for

// ---- error plumbing
void set_last_cuda_error(cudaError_t e);

inline int check_launch()
{
    cudaError_t e = cudaGetLastError();
    if(e != cudaSuccess)
    {
        set_last_cuda_error(e);
        return GSB200_E_CUDA;
    }
    return GSB200_OK;
}

#define GSB_CUDA_TRY(expr)                \
    do                                    \
    {                                     \
        cudaError_t e__ = (expr);         \
        if(e__ != cudaSuccess)            \
        {                                 \
            gsb::set_last_cuda_error(e__); \
            return GSB200_E_CUDA;         \
        }                                 \
    } while(0)

inline uint32_t bits_for_count(int64_t count)
{
    if(count <= 1)
        return 0u;
    uint64_t v = (uint64_t)count - 1u;
    uint32_t b = 0;
    while(v)
    {
        ++b;
        v >>= 1;
    }
    return b;
}

inline unsigned grid_for(int64_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

// The colour channel counts the compositing kernels are built for: f(std::integral_constant<int, D>{}) for one of them,
// GSB200_E_UNSUPPORTED for any other D.
template<class F>
inline int with_channels(int D, F &&f)
{
    switch(D)
    {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 3: return f(std::integral_constant<int, 3>{});
    case 4: return f(std::integral_constant<int, 4>{});
    case 5: return f(std::integral_constant<int, 5>{});
    case 8: return f(std::integral_constant<int, 8>{});
    case 16: return f(std::integral_constant<int, 16>{});
    case 32: return f(std::integral_constant<int, 32>{});
    default: return GSB200_E_UNSUPPORTED;
    }
}

// does a tw x th grid of kTile-pixel tiles cover a W x H image?
inline bool tile_grid_covers(uint32_t tw, uint32_t th, uint32_t W, uint32_t H)
{
    return (uint64_t)tw * kTile >= W && (uint64_t)th * kTile >= H;
}

#ifdef __CUDACC__
// ---- mbarrier / bulk-copy (TMA 1-D, SASS UBLKCP) wrappers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// make mbarrier.init visible to the async (TMA) proxy
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// order prior generic-proxy smem accesses before later async-proxy writes to the same smem
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t *bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory"
    );
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    while(!mbar_try_wait(bar, parity))
    {
    }
}
// 1-D bulk async copy global -> shared, completion counted in bytes on `bar`.
// dst, src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar)
{
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory"
    );
}

__device__ __forceinline__ float4 ldg_nc_f4(const float4 *p)
{
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
                 : "l"(p));
    return r;
}

// ex2 / rcp exactly as the reference evaluates them (it is built with -use_fast_math, so its __expf is
// ex2.approx.ftz(x * log2e) and its 1.0f / x is rcp.approx.ftz): one MUFU each, no range fix-up code.
__device__ __forceinline__ float fast_exp(float x)
{
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x * 1.4426950408889634f));
    return y;
}
__device__ __forceinline__ float fast_ex2(float x)
{
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ float fast_rcp(float x)
{
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// Butterfly ("transpose") warp reduction of M per-lane values: after the call, lane L holds in v[0]
// the full 32-lane sum of slot butterfly_slot<M>(L) (if that slot is < M).  Costs
// ceil(M/2)+ceil(M/4)+... shuffles instead of 5*M.
template<int M, int OFF>
struct Butterfly
{
    static __device__ __forceinline__ void run(float *v, const unsigned lane)
    {
        if constexpr(OFF >= 1)
        {
            if constexpr(M > 1)
            {
                constexpr int H = (M + 1) / 2;
                const bool up   = (lane & OFF) != 0;
#pragma unroll
                for(int i = 0; i < H; ++i)
                {
                    const float hi   = (i + H < M) ? v[i + H] : 0.f;
                    const float send = up ? v[i] : hi;
                    const float keep = up ? hi : v[i];
                    v[i]             = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
                }
                Butterfly<H, OFF / 2>::run(v, lane);
            }
            else
            {
                v[0] += __shfl_xor_sync(0xffffffffu, v[0], OFF);
                Butterfly<1, OFF / 2>::run(v, lane);
            }
        }
    }
};

// Slot owned by `lane` after Butterfly<M,16>::run, or -1 when the lane holds padding or a
// duplicate (once a group is down to one value the remaining steps are plain all-reduces, so
// several lanes end up with the same sum; only the one with those lane bits clear owns it).
template<int M>
__device__ __forceinline__ int butterfly_slot(unsigned lane)
{
    int mt = M; // padded size carried by the template recursion
    int mr = M; // real entries among them
    int slot = 0;
    bool primary = true;
#pragma unroll
    for(int off = 16; off >= 1; off >>= 1)
    {
        if(mt > 1)
        {
            const int h = (mt + 1) / 2;
            if(lane & off)
            {
                slot += h;
                mr = mr > h ? mr - h : 0; // the upper half keeps the entries past h (zero-padded)
            }
            else
                mr = mr < h ? mr : h;
            mt = h;
        }
        else if(lane & off)
            primary = false;
    }
    return (mr >= 1 && primary) ? slot : -1;
}

// The compositing backwards' gradient emit (surfel.cu, ut.cu): butterfly-reduces gv[OFF, OFF + 32) across the warp, adds
// each owned nonzero slot of record r with dst.add(slot, r, sum, CDIM); recurses over the remaining 32-value chunks.
template<int OFF, int NV, class Rec, class Dst>
__device__ __forceinline__ void reduce_emit(const float *gv, unsigned lane, const Rec &r, const Dst &dst, int CDIM)
{
    constexpr int M = (NV - OFF) < 32 ? (NV - OFF) : 32;
    float v[M];
#pragma unroll
    for(int k = 0; k < M; ++k)
        v[k] = gv[OFF + k];
    Butterfly<M, 16>::run(v, lane);
    const int s = butterfly_slot<M>(lane);
    if(s >= 0 && v[0] != 0.f)
        dst.add(OFF + s, r, v[0], CDIM);
    if constexpr(OFF + 32 < NV)
        reduce_emit<OFF + 32, NV>(gv, lane, r, dst, CDIM);
}
#endif // __CUDACC__
} // namespace gsb
