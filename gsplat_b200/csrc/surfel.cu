// surfel.cu -- 2DGS (surfel splatting): the dense ray-transform projection and its VJP, and the per-tile compositing of
// colours, normals, L1 depth distortion and median depth with its backward.  Compiled with -fmad=false: the forward and
// the backward evaluate alpha with the same individually rounded operations, so both passes take the same threshold
// decisions for every (pixel, gaussian) pair.
//
// Reference semantics: csrc/Projection2DGSFused.cu (projection and VJP), csrc/Projection2DGS.cuh (ray-transform VJP),
// csrc/RasterizeToPixels2DGSSerialBatchFwd.cu / Bwd.cu (compositing), include/Common.h and csrc/Rasterization.h (constants).
#include "gaussmath.cuh"
#include "indices.cuh"
#include "pixels.cuh"

namespace gsb
{
namespace
{
constexpr int kSurfThreads       = 256;
constexpr float kSurfFilterInvSq = 2.f; // FILTER_INV_SQUARE_2DGS: weight of the screen-space (2-D) kernel

// ------------------------------------------------------------------ projection
// Camera-frame quantities of one (camera, gaussian): the two scaled tangent axes, the normal axis and the centre.
struct SurfelCam
{
    float ca[3], cb[3], cn[3], mc[3];
};

__device__ __forceinline__ void rot_apply(const M3 &R, const float *v, float *o)
{
#pragma unroll
    for(int i = 0; i < 3; ++i)
        o[i] = R.m[i * 3 + 0] * v[0] + R.m[i * 3 + 1] * v[1] + R.m[i * 3 + 2] * v[2];
}
__device__ __forceinline__ void rot_apply_t(const M3 &R, const float *v, float *o)
{
#pragma unroll
    for(int i = 0; i < 3; ++i)
        o[i] = R.m[0 * 3 + i] * v[0] + R.m[1 * 3 + i] * v[1] + R.m[2 * 3 + i] * v[2];
}

__device__ __forceinline__ SurfelCam surfel_to_camera(const Cam &cam, const M3 &Rq, const float *s, const float *mean)
{
    SurfelCam o;
    const float a[3] = {Rq.m[0] * s[0], Rq.m[3] * s[0], Rq.m[6] * s[0]};
    const float b[3] = {Rq.m[1] * s[1], Rq.m[4] * s[1], Rq.m[7] * s[1]};
    const float n[3] = {Rq.m[2], Rq.m[5], Rq.m[8]};
    rot_apply(cam.R, a, o.ca);
    rot_apply(cam.R, b, o.cb);
    rot_apply(cam.R, n, o.cn);
    rot_apply(cam.R, mean, o.mc);
#pragma unroll
    for(int i = 0; i < 3; ++i)
        o.mc[i] = o.mc[i] + cam.t[i];
    return o;
}

// One thread per (b, c, n).  Culled rows get radii 0 and zero float outputs.
__global__ void __launch_bounds__(kSurfThreads) surfel_project_fwd_kernel(
    int64_t B, int64_t C, int64_t N, const float *__restrict__ means, const float *__restrict__ quats,
    const float *__restrict__ scales, const float *__restrict__ viewmats, const float *__restrict__ Ks, uint32_t W, uint32_t H,
    float near_plane, float far_plane, float radius_clip, int32_t *__restrict__ radii, float *__restrict__ means2d,
    float *__restrict__ depths, float *__restrict__ ray_transforms, float *__restrict__ normals
)
{
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(idx >= B * C * N)
        return;
    const int64_t b = idx / (C * N), c = (idx / N) % C, n = idx % N;
    const int64_t bn = b * N + n;
    const Cam cam    = load_cam(viewmats + (b * C + c) * 16, Ks + (b * C + c) * 9);
    const float mean[3] = {means[bn * 3], means[bn * 3 + 1], means[bn * 3 + 2]};
    const float q[4]    = {quats[bn * 4], quats[bn * 4 + 1], quats[bn * 4 + 2], quats[bn * 4 + 3]};
    const float s[2]    = {scales[bn * 3], scales[bn * 3 + 1]};

    int rx = 0, ry = 0;
    float M[9], mx = 0.f, my = 0.f, nrm[3] = {0.f, 0.f, 0.f}, depth = 0.f;
#pragma unroll
    for(int k = 0; k < 9; ++k)
        M[k] = 0.f;
    {
        const M3 Rq         = quat_to_rotmat(q);
        const SurfelCam sc  = surfel_to_camera(cam, Rq, s, mean);
        const float z       = sc.mc[2];
        if(!(z <= near_plane || z >= far_plane))
        {
            // rows of K * [ca cb mc]
            const float T0[3] = {cam.fx * sc.ca[0] + cam.cx * sc.ca[2], cam.fx * sc.cb[0] + cam.cx * sc.cb[2], cam.fx * sc.mc[0] + cam.cx * sc.mc[2]};
            const float T1[3] = {cam.fy * sc.ca[1] + cam.cy * sc.ca[2], cam.fy * sc.cb[1] + cam.cy * sc.cb[2], cam.fy * sc.mc[1] + cam.cy * sc.mc[2]};
            const float T2[3] = {sc.ca[2], sc.cb[2], sc.mc[2]};
            const float dist  = T2[0] * T2[0] + T2[1] * T2[1] - T2[2] * T2[2];
            if(dist != 0.f)
            {
                // f = (1, 1, -1) / dist: the [1, 1, -1] construction of the screen mean and half extent
                const float inv = 1.f / dist;
                const float f0 = inv, f1 = inv, f2 = -inv;
                const float m2x = f0 * T0[0] * T2[0] + f1 * T0[1] * T2[1] + f2 * T0[2] * T2[2];
                const float m2y = f0 * T1[0] * T2[0] + f1 * T1[1] * T2[1] + f2 * T1[2] * T2[2];
                const float ex  = m2x * m2x - (f0 * T0[0] * T0[0] + f1 * T0[1] * T0[1] + f2 * T0[2] * T0[2]);
                const float ey  = m2y * m2y - (f0 * T1[0] * T1[0] + f1 * T1[1] * T1[1] + f2 * T1[2] * T1[2]);
                const float fr_x = ceilf(kGaussianExtend * sqrtf(fmaxf(1e-4f, ex)));
                const float fr_y = ceilf(kGaussianExtend * sqrtf(fmaxf(1e-4f, ey)));
                const bool clipped = fr_x <= radius_clip && fr_y <= radius_clip;
                const bool off     = m2x + fr_x <= 0.f || m2x - fr_x >= (float)W || m2y + fr_y <= 0.f || m2y - fr_y >= (float)H;
                // finite inputs can overflow here (fx * scale beyond FLT_MAX): a NaN screen mean passes every off-screen
                // test and composites at alpha 0.99 wherever it is listed, so such a row is culled
                bool finite = isfinite(m2x) && isfinite(m2y) && isfinite(z);
#pragma unroll
                for(int k = 0; k < 3; ++k)
                    finite = finite && isfinite(T0[k]) && isfinite(T1[k]) && isfinite(T2[k]);
                if(!clipped && !off && finite)
                {
                    rx = (int)fr_x, ry = (int)fr_y;
                    mx = m2x, my = m2y, depth = z;
#pragma unroll
                    for(int k = 0; k < 3; ++k)
                        M[k] = T0[k], M[3 + k] = T1[k], M[6 + k] = T2[k];
                    // the normal faces the camera
                    const float cosv = -(sc.cn[0] * sc.mc[0] + sc.cn[1] * sc.mc[1] + sc.cn[2] * sc.mc[2]);
                    const float mult = cosv > 0.f ? 1.f : -1.f;
#pragma unroll
                    for(int k = 0; k < 3; ++k)
                        nrm[k] = sc.cn[k] * mult;
                }
            }
        }
    }
    reinterpret_cast<int2 *>(radii)[idx]     = make_int2(rx, ry);
    reinterpret_cast<float2 *>(means2d)[idx] = make_float2(mx, my);
    depths[idx] = depth;
#pragma unroll
    for(int k = 0; k < 9; ++k)
        ray_transforms[idx * 9 + k] = M[k];
#pragma unroll
    for(int k = 0; k < 3; ++k)
        normals[idx * 3 + k] = nrm[k];
}

// One thread per (b, n), looping over the C cameras (as projection_bwd_kernel of pergauss.cu): the per-gaussian sums stay
// in registers, every v_means / v_quats / v_scales row is written once; v_viewmats is warp-reduced, then atomically added.
__global__ void __launch_bounds__(kSurfThreads) surfel_project_bwd_kernel(
    int64_t B, int64_t C, int64_t N, const float *__restrict__ means, const float *__restrict__ quats,
    const float *__restrict__ scales, const float *__restrict__ viewmats, const float *__restrict__ Ks,
    const int32_t *__restrict__ radii, const float *__restrict__ ray_transforms, const float *__restrict__ v_means2d,
    const float *__restrict__ v_depths, const float *__restrict__ v_ray_transforms, const float *__restrict__ v_normals,
    float *__restrict__ v_means, float *__restrict__ v_quats, float *__restrict__ v_scales, float *__restrict__ v_viewmats
)
{
    const int64_t bn    = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active   = bn < B * N;
    const int64_t b     = active ? bn / N : 0, n = active ? bn % N : 0;
    const unsigned lane = threadIdx.x & 31;
    float mean[3] = {0.f, 0.f, 0.f}, q[4] = {1.f, 0.f, 0.f, 0.f}, s[2] = {1.f, 1.f};
    if(active)
    {
#pragma unroll
        for(int k = 0; k < 3; ++k)
            mean[k] = means[bn * 3 + k];
#pragma unroll
        for(int k = 0; k < 4; ++k)
            q[k] = quats[bn * 4 + k];
        s[0] = scales[bn * 3], s[1] = scales[bn * 3 + 1];
    }
    const M3 Rq = quat_to_rotmat(q);
    // world-frame gradients of the two scaled tangent axes, the normal axis and the centre, summed over cameras
    float v_a[3] = {0.f, 0.f, 0.f}, v_b[3] = {0.f, 0.f, 0.f}, v_n[3] = {0.f, 0.f, 0.f}, v_mean[3] = {0.f, 0.f, 0.f};
    bool seen = false;
    for(int64_t c = 0; c < C; ++c)
    {
        const int64_t idx = (b * C + c) * N + n;
        const bool vis    = active && radii[idx * 2] > 0 && radii[idx * 2 + 1] > 0;
        seen |= vis;
        float vm_part[12];
#pragma unroll
        for(int k = 0; k < 12; ++k)
            vm_part[k] = 0.f;
        if(vis)
        {
            const Cam cam = load_cam(viewmats + (b * C + c) * 16, Ks + (b * C + c) * 9);
            const SurfelCam sc = surfel_to_camera(cam, Rq, s, mean);
            float M[9], vM[9];
#pragma unroll
            for(int k = 0; k < 9; ++k)
                M[k] = ray_transforms[idx * 9 + k], vM[k] = v_ray_transforms[idx * 9 + k];
            vM[8] = vM[8] + v_depths[idx]; // depth = M[2][2]
            const float vmx = v_means2d[idx * 2], vmy = v_means2d[idx * 2 + 1];
            if(vmx != 0.f || vmy != 0.f)
            {
                const float t2[3] = {M[6], M[7], -M[8]}; // (1, 1, -1) * M2
                const float inv   = 1.f / (M[6] * t2[0] + M[7] * t2[1] + M[8] * t2[2]);
                const float m2x   = (M[0] * t2[0] + M[1] * t2[1] + M[2] * t2[2]) * inv;
                const float m2y   = (M[3] * t2[0] + M[4] * t2[1] + M[5] * t2[2]) * inv;
                const float sgn[3] = {1.f, 1.f, -1.f};
#pragma unroll
                for(int k = 0; k < 3; ++k)
                {
                    vM[k]     = vM[k] + vmx * inv * t2[k];
                    vM[3 + k] = vM[3 + k] + vmy * inv * t2[k];
                    vM[6 + k] = vM[6 + k] + vmx * inv * (sgn[k] * M[k] - 2.f * m2x * t2[k])
                              + vmy * inv * (sgn[k] * M[3 + k] - 2.f * m2y * t2[k]);
                }
            }
            // M = K * [ca cb mc]: v_[ca cb mc] = K^T vM
            float vT[9];
#pragma unroll
            for(int j = 0; j < 3; ++j)
            {
                vT[j]     = cam.fx * vM[j];
                vT[3 + j] = cam.fy * vM[3 + j];
                vT[6 + j] = cam.cx * vM[j] + cam.cy * vM[3 + j] + vM[6 + j];
            }
            const float v_ca[3] = {vT[0], vT[3], vT[6]}, v_cb[3] = {vT[1], vT[4], vT[7]}, v_mc[3] = {vT[2], vT[5], vT[8]};
            const float cosv = -(sc.cn[0] * sc.mc[0] + sc.cn[1] * sc.mc[1] + sc.cn[2] * sc.mc[2]);
            const float mult = cosv > 0.f ? 1.f : -1.f;
            const float v_cn[3] = {v_normals[idx * 3] * mult, v_normals[idx * 3 + 1] * mult, v_normals[idx * 3 + 2] * mult};
            float w[3];
            rot_apply_t(cam.R, v_ca, w);
#pragma unroll
            for(int k = 0; k < 3; ++k)
                v_a[k] += w[k];
            rot_apply_t(cam.R, v_cb, w);
#pragma unroll
            for(int k = 0; k < 3; ++k)
                v_b[k] += w[k];
            rot_apply_t(cam.R, v_cn, w);
#pragma unroll
            for(int k = 0; k < 3; ++k)
                v_n[k] += w[k];
            rot_apply_t(cam.R, v_mc, w);
#pragma unroll
            for(int k = 0; k < 3; ++k)
                v_mean[k] += w[k];
            if(v_viewmats)
            { // v_R = v_ca a^T + v_cb b^T + v_cn n^T + v_mc mean^T ; v_t = v_mc  (a, b, n: world-frame axes)
                const float a[3]  = {Rq.m[0] * s[0], Rq.m[3] * s[0], Rq.m[6] * s[0]};
                const float bb[3] = {Rq.m[1] * s[1], Rq.m[4] * s[1], Rq.m[7] * s[1]};
                const float nn[3] = {Rq.m[2], Rq.m[5], Rq.m[8]};
#pragma unroll
                for(int i = 0; i < 3; ++i)
                {
#pragma unroll
                    for(int j = 0; j < 3; ++j)
                        vm_part[i * 4 + j] = v_ca[i] * a[j] + v_cb[i] * bb[j] + v_cn[i] * nn[j] + v_mc[i] * mean[j];
                    vm_part[i * 4 + 3] = v_mc[i];
                }
            }
        }
        if(v_viewmats)
        {
            // one warp reduction when the whole warp belongs to one batch element, else per-lane atomics
            const int64_t b0  = __shfl_sync(0xffffffffu, b, 0);
            const bool same_b = __all_sync(0xffffffffu, !active || b == b0);
            if(same_b)
            {
                Butterfly<12, 16>::run(vm_part, lane);
                const int slot = butterfly_slot<12>(lane);
                if(slot >= 0 && vm_part[0] != 0.f)
                    atomicAdd(v_viewmats + (b0 * C + c) * 16 + slot, vm_part[0]);
            }
            else if(vis)
            {
#pragma unroll
                for(int k = 0; k < 12; ++k)
                    atomicAdd(v_viewmats + (b * C + c) * 16 + k, vm_part[k]);
            }
        }
    }
    if(!active)
        return;
#pragma unroll
    for(int k = 0; k < 3; ++k)
        v_means[bn * 3 + k] = v_mean[k];
    // a gaussian no camera sees gets zero (its quaternion may be zero: the normalisation VJP would give NaN)
    float vq[4] = {0.f, 0.f, 0.f, 0.f}, vs0 = 0.f, vs1 = 0.f;
    if(seen)
    {
        M3 G; // dL/dRq: columns s0 * v_a, s1 * v_b, v_n
#pragma unroll
        for(int i = 0; i < 3; ++i)
        {
            G.m[i * 3 + 0] = s[0] * v_a[i];
            G.m[i * 3 + 1] = s[1] * v_b[i];
            G.m[i * 3 + 2] = v_n[i];
        }
        quat_to_rotmat_vjp(q, G, vq);
        vs0 = Rq.m[0] * v_a[0] + Rq.m[3] * v_a[1] + Rq.m[6] * v_a[2];
        vs1 = Rq.m[1] * v_b[0] + Rq.m[4] * v_b[1] + Rq.m[7] * v_b[2];
    }
#pragma unroll
    for(int k = 0; k < 4; ++k)
        v_quats[bn * 4 + k] = vq[k];
    v_scales[bn * 3]     = vs0;
    v_scales[bn * 3 + 1] = vs1;
    v_scales[bn * 3 + 2] = 0.f;
}

// ------------------------------------------------------------------ compositing
// One staged gaussian of a tile: screen mean, opacity, the three rows of the ray transform, its row index.
struct SurfRec
{
    float x, y, o;
    float m[9];
    int32_t id;
};

__device__ __forceinline__ void stage(SurfRec &r, int32_t g, const float *means2d, const float *opacities, const float *rt)
{
    r.id = g;
    r.x  = means2d[(int64_t)g * 2];
    r.y  = means2d[(int64_t)g * 2 + 1];
    r.o  = opacities[g];
#pragma unroll
    for(int k = 0; k < 9; ++k)
        r.m[k] = rt[(int64_t)g * 9 + k];
}

// Kernel value of one gaussian at pixel centre (px, py).  ok = false: the ray is parallel to the splat (s.z == 0).
struct SurfHit
{
    float hu[3], hv[3], cz, u, v, g3, g2, dx, dy, vis, alpha;
    bool ok;
};

__device__ __forceinline__ SurfHit surf_eval(const SurfRec &r, float px, float py)
{
    SurfHit h;
#pragma unroll
    for(int k = 0; k < 3; ++k)
    {
        h.hu[k] = px * r.m[6 + k] - r.m[k];
        h.hv[k] = py * r.m[6 + k] - r.m[3 + k];
    }
    const float sx = h.hu[1] * h.hv[2] - h.hu[2] * h.hv[1];
    const float sy = h.hu[2] * h.hv[0] - h.hu[0] * h.hv[2];
    h.cz           = h.hu[0] * h.hv[1] - h.hu[1] * h.hv[0];
    h.ok           = h.cz != 0.f;
    h.u            = sx / h.cz;
    h.v            = sy / h.cz;
    h.g3           = h.u * h.u + h.v * h.v;
    h.dx           = r.x - px;
    h.dy           = r.y - py;
    h.g2           = kSurfFilterInvSq * (h.dx * h.dx + h.dy * h.dy);
    const float sigma = 0.5f * fminf(h.g3, h.g2);
    h.vis          = fast_exp(-sigma);
    h.alpha        = fminf(kMaxAlpha, r.o * h.vis);
    h.ok           = h.ok && !(sigma < 0.f) && !(h.alpha < kAlphaThreshold);
    return h;
}

// One CTA per tile of the pixel policy (pixels.cuh): every tile of the [I, th, tw] grid (DensePixels), or every active
// tile with its requested pixels only (SparsePixels).  A pixel that is not live stages records and meets every barrier
// but composites and writes nothing.
template<int CDIM, class Pix = DensePixels>
__global__ void __launch_bounds__(kSurfThreads) surfel_raster_fwd_kernel(
    uint32_t I, const float *__restrict__ means2d, const float *__restrict__ rt, const float *__restrict__ colors,
    const float *__restrict__ opacities, const float *__restrict__ normals, const float *__restrict__ backgrounds,
    const uint8_t *__restrict__ masks, uint32_t W, uint32_t H, uint32_t tw, uint32_t th, const int32_t *__restrict__ offsets,
    const int32_t *__restrict__ flatten_ids, int64_t n_isects, float *__restrict__ render_colors, float *__restrict__ render_alphas,
    float *__restrict__ render_normals, float *__restrict__ render_distort, float *__restrict__ render_median,
    int32_t *__restrict__ last_ids, int32_t *__restrict__ median_ids, const Pix pixmap = Pix{}
)
{
    __shared__ SurfRec rec[kSurfThreads];
    const uint32_t tile = pixmap.tile(blockIdx.x); // image * th * tw + tile row * tw + tile col
    const uint32_t img  = tile / (tw * th);
    const uint32_t tin  = tile - img * tw * th;
    const uint32_t tr   = threadIdx.x;
    const uint32_t i    = (tin / tw) * kTile + tr / kTile;
    const uint32_t j    = (tin % tw) * kTile + tr % kTile;
    bool inside;
    int64_t pix;
    if constexpr(Pix::kSparse)
        pix = pixmap.slot(blockIdx.x, (int)tr, inside);
    else
    {
        inside = i < H && j < W;
        pix    = (int64_t)img * H * W + (int64_t)i * W + j;
    }
    const float *bg     = backgrounds ? backgrounds + (int64_t)img * CDIM : nullptr;

    if(masks && !masks[tile])
    {
        if(inside)
        {
#pragma unroll
            for(int k = 0; k < CDIM; ++k)
                render_colors[pix * CDIM + k] = bg ? bg[k] : 0.f;
            render_alphas[pix] = 0.f;
#pragma unroll
            for(int k = 0; k < 3; ++k)
                render_normals[pix * 3 + k] = 0.f;
            render_distort[pix] = 0.f;
            render_median[pix]  = 0.f;
            last_ids[pix]       = 0;
            median_ids[pix]     = 0;
        }
        return;
    }
    int64_t start, end;
    if constexpr(Pix::kSparse)
    {
        start = offsets[blockIdx.x];
        end   = offsets[blockIdx.x + 1];
    }
    else
    {
        start = offsets[tile];
        end   = (tile + 1 == I * tw * th) ? n_isects : offsets[tile + 1];
    }
    const float px = (float)j + 0.5f, py = (float)i + 0.5f;

    float T = 1.f, distort = 0.f, accum_vis_depth = 0.f, median_depth = 0.f;
    int32_t cur_idx = 0, median_idx = 0;
    float pix_out[CDIM], nrm_out[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for(int k = 0; k < CDIM; ++k)
        pix_out[k] = 0.f;
    bool done = !inside;
    for(int64_t batch = start; batch < end; batch += kSurfThreads)
    {
        if(__syncthreads_count(done) == kSurfThreads)
            break;
        if(batch + tr < end)
            stage(rec[tr], flatten_ids[batch + tr], means2d, opacities, rt);
        __syncthreads();
        const int n_b = (int)min((int64_t)kSurfThreads, end - batch);
        for(int t = 0; t < n_b && !done; ++t)
        {
            const SurfRec &r = rec[t];
            const SurfHit h  = surf_eval(r, px, py);
            if(!h.ok)
                continue;
            const float next_T = T * (1.f - h.alpha);
            if(next_T <= kTransmittanceThreshold)
            { // exclusive: this gaussian does not contribute
                done = true;
                break;
            }
            const float vis = h.alpha * T;
            const float *c  = colors + (int64_t)r.id * CDIM;
#pragma unroll
            for(int k = 0; k < CDIM; ++k)
                pix_out[k] += c[k] * vis;
            const float *nn = normals + (int64_t)r.id * 3;
#pragma unroll
            for(int k = 0; k < 3; ++k)
                nrm_out[k] += nn[k] * vis;
            // L1 distortion (Mip-NeRF 360 / nerfacc): the depth is the last channel
            const float depth = c[CDIM - 1];
            distort += 2.f * (vis * depth * (1.f - T) - vis * accum_vis_depth);
            accum_vis_depth += vis * depth;
            if(T > 0.5f)
            {
                median_depth = depth;
                median_idx   = (int32_t)(batch + t);
            }
            cur_idx = (int32_t)(batch + t);
            T       = next_T;
        }
    }
    if(!inside)
        return;
    if constexpr(Pix::kSparse)
        pix = pixmap.slot(blockIdx.x, (int)tr, inside); // looked up again: the row is not held across the walk
    render_alphas[pix] = 1.f - T;
#pragma unroll
    for(int k = 0; k < CDIM; ++k)
        render_colors[pix * CDIM + k] = bg ? pix_out[k] + T * bg[k] : pix_out[k];
#pragma unroll
    for(int k = 0; k < 3; ++k)
        render_normals[pix * 3 + k] = nrm_out[k];
    render_distort[pix] = distort;
    render_median[pix]  = median_depth;
    last_ids[pix]       = cur_idx;
    median_ids[pix]     = median_idx;
}

// The 2DGS model of pair_walk_kernel (indices.cuh), the pair query and contributor queries of
// rasterize_to_indices_in_range_2dgs and rasterize_*_contributing_gaussian*_2dgs: surfel_raster_fwd_kernel's staging
// and surf_eval at the pixel centre.  Every live pixel composites, margin pixels of a sparse tile included.
struct SurfelModel
{
    uint32_t I, W, H, tw, th;
    const float *means2d, *rt, *opacities;
    static constexpr int kMinBlocks = 0; // the forward's launch bounds: no minimum
    using Rec   = SurfRec;
    using Pixel = float2; // the pixel centre
    __device__ __forceinline__ void stage(SurfRec &r, int32_t g) const { gsb::stage(r, g, means2d, opacities, rt); }
    __device__ __forceinline__ bool setup(uint32_t, uint32_t i, uint32_t j, bool live, float2 &p) const
    {
        p = make_float2((float)j + 0.5f, (float)i + 0.5f);
        return live;
    }
    __device__ __forceinline__ SurfHit hit(const SurfRec &r, float2 p) const { return surf_eval(r, p.x, p.y); }
};

struct SurfGradDst
{
    float *means2d, *rt, *colors, *opacities, *normals, *densify, *abs;

    // reduce_emit's routing (common.cuh): slot of the gradient vector of surfel_raster_bwd_kernel to its row
    __device__ __forceinline__ void add(int slot, const SurfRec &r, float val, int CDIM) const
    {
        const int64_t g = r.id;
        if(slot < CDIM)
            atomicAdd(colors + g * CDIM + slot, val);
        else if(slot < CDIM + 3)
            atomicAdd(normals + g * 3 + (slot - CDIM), val);
        else if(slot < CDIM + 12)
        {
            const int e = slot - CDIM - 3;
            atomicAdd(rt + g * 9 + e, val);
            if(e == 2 || e == 5)
                atomicAdd(densify + g * 2 + (e == 5), val * r.m[8]);
        }
        else if(slot < CDIM + 14)
            atomicAdd(means2d + g * 2 + (slot - CDIM - 12), val);
        else if(slot == CDIM + 14)
            atomicAdd(opacities + g, val);
        else if(abs)
            atomicAdd(abs + g * 2 + (slot - CDIM - 15), val);
    }
};

// Back to front over each tile's list.  Per gaussian, the warp's per-pixel gradients (colours, normals, ray transform,
// screen mean, opacity, |screen mean|) are butterfly-reduced and added with one atomic per value; v_densify is the
// z-column of the ray-transform gradient times M[2][2], the same for every pixel of the gaussian.
template<int CDIM, class Pix = DensePixels>
__global__ void __launch_bounds__(kSurfThreads) surfel_raster_bwd_kernel(
    uint32_t I, const float *__restrict__ means2d, const float *__restrict__ rt, const float *__restrict__ colors,
    const float *__restrict__ opacities, const float *__restrict__ normals, const float *__restrict__ backgrounds,
    const uint8_t *__restrict__ masks, uint32_t W, uint32_t H, uint32_t tw, uint32_t th, const int32_t *__restrict__ offsets,
    const int32_t *__restrict__ flatten_ids, int64_t n_isects, const float *__restrict__ render_colors,
    const float *__restrict__ render_alphas, const int32_t *__restrict__ last_ids, const int32_t *__restrict__ median_ids,
    const float *__restrict__ v_render_colors, const float *__restrict__ v_render_alphas,
    const float *__restrict__ v_render_normals, const float *__restrict__ v_render_distort,
    const float *__restrict__ v_render_median, SurfGradDst dst, const Pix pixmap = Pix{}
)
{
    constexpr int NV = CDIM + 17; // colours | normals 3 | ray transform 9 | xy 2 | opacity 1 | abs xy 2
    __shared__ SurfRec rec[kSurfThreads];
    __shared__ float s_col[kSurfThreads * CDIM];
    __shared__ float s_nrm[kSurfThreads * 3];
    const uint32_t tile = pixmap.tile(blockIdx.x);
    if(masks && !masks[tile])
        return;
    const uint32_t img  = tile / (tw * th);
    const uint32_t tin  = tile - img * tw * th;
    const uint32_t tr   = threadIdx.x;
    const unsigned lane = tr & 31;
    const uint32_t i    = (tin / tw) * kTile + tr / kTile;
    const uint32_t j    = (tin % tw) * kTile + tr % kTile;
    // a pixel that is not live reads the row of a live one (the image's first pixel; sparse: row 0) and adds nothing
    bool inside;
    int64_t pix;
    if constexpr(Pix::kSparse)
        pix = pixmap.slot(blockIdx.x, (int)tr, inside);
    else
    {
        inside = i < H && j < W;
        pix    = inside ? (int64_t)img * H * W + (int64_t)i * W + j : (int64_t)img * H * W;
    }
    // the list range after bg, as before the pixel policy: read in the other order, the dense kernel's code changes
    const float *bg = backgrounds ? backgrounds + (int64_t)img * CDIM : nullptr;
    int64_t start, end;
    if constexpr(Pix::kSparse)
    {
        start = offsets[blockIdx.x];
        end   = offsets[blockIdx.x + 1];
    }
    else
    {
        start = offsets[tile];
        end   = (tile + 1 == I * tw * th) ? n_isects : offsets[tile + 1];
    }
    const float px = (float)j + 0.5f, py = (float)i + 0.5f;

    const float T_final = 1.f - render_alphas[pix];
    float T             = T_final;
    float buf[CDIM], buf_n[3] = {0.f, 0.f, 0.f}, v_rc[CDIM], v_rn[3];
#pragma unroll
    for(int k = 0; k < CDIM; ++k)
    {
        buf[k]  = 0.f;
        v_rc[k] = v_render_colors[pix * CDIM + k];
    }
#pragma unroll
    for(int k = 0; k < 3; ++k)
        v_rn[k] = v_render_normals ? v_render_normals[pix * 3 + k] : 0.f;
    const float v_ra     = v_render_alphas ? v_render_alphas[pix] : 0.f;
    const float v_dist   = v_render_distort ? v_render_distort[pix] : 0.f;
    const float v_median = v_render_median ? v_render_median[pix] : 0.f;
    const int64_t bin_final  = inside ? last_ids[pix] : -1;
    const int64_t median_idx = inside ? median_ids[pix] : -1;
    // distortion: accumulated weight and weighted depth (the forward's, without the background term)
    const float accum_w = 1.f - T_final;
    const float accum_d = render_colors[pix * CDIM + CDIM - 1] - (bg ? T_final * bg[CDIM - 1] : 0.f);
    float accum_w_buf = accum_w, accum_d_buf = accum_d, distort_buf = 0.f;
    float bg_dot = 0.f;
    if(bg)
    {
#pragma unroll
        for(int k = 0; k < CDIM; ++k)
            bg_dot += bg[k] * v_rc[k];
    }
    int64_t warp_bin_final = bin_final;
#pragma unroll
    for(int off = 16; off >= 1; off >>= 1)
        warp_bin_final = max(warp_bin_final, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)warp_bin_final, off));

    for(int64_t batch_end = end - 1; batch_end >= start; batch_end -= kSurfThreads)
    {
        __syncthreads();
        const int64_t idx = batch_end - tr;
        if(idx >= start)
        {
            const int32_t g = flatten_ids[idx];
            stage(rec[tr], g, means2d, opacities, rt);
#pragma unroll
            for(int k = 0; k < CDIM; ++k)
                s_col[tr * CDIM + k] = colors[(int64_t)g * CDIM + k];
#pragma unroll
            for(int k = 0; k < 3; ++k)
                s_nrm[tr * 3 + k] = normals[(int64_t)g * 3 + k];
        }
        __syncthreads();
        const int n_b = (int)min((int64_t)kSurfThreads, batch_end + 1 - start);
        const int t0  = (int)max((int64_t)0, batch_end - warp_bin_final);
        for(int t = t0; t < n_b; ++t)
        {
            const SurfRec &r = rec[t];
            const int64_t gi = batch_end - t;
            bool valid       = inside && gi <= bin_final;
            SurfHit h;
            if(valid)
            {
                h     = surf_eval(r, px, py);
                valid = h.ok;
            }
            if(!__any_sync(0xffffffffu, valid))
                continue;
            float gv[NV];
#pragma unroll
            for(int k = 0; k < NV; ++k)
                gv[k] = 0.f;
            if(valid)
            {
                const float *c  = s_col + t * CDIM;
                const float *nn = s_nrm + t * 3;
                const float ra  = 1.f / fmaxf(kMinOneMinusAlpha, 1.f - h.alpha);
                T               = T * ra;
                const float fac = h.alpha * T;
                float v_alpha   = 0.f;
#pragma unroll
                for(int k = 0; k < CDIM; ++k)
                {
                    gv[k] = fac * v_rc[k];
                    v_alpha += (c[k] * T - buf[k] * ra) * v_rc[k];
                }
                if(gi == median_idx)
                    gv[CDIM - 1] += v_median;
#pragma unroll
                for(int k = 0; k < 3; ++k)
                {
                    gv[CDIM + k] = fac * v_rn[k];
                    v_alpha += (nn[k] * T - buf_n[k] * ra) * v_rn[k];
                }
                v_alpha += T_final * ra * v_ra;
                v_alpha += -T_final * ra * bg_dot;
                {
                    const float depth = c[CDIM - 1];
                    const float dl_dw = 2.f * (2.f * (depth * accum_w_buf - accum_d_buf) + (accum_d - depth * accum_w));
                    v_alpha += (dl_dw * T - distort_buf * ra) * v_dist;
                    accum_d_buf -= fac * depth;
                    accum_w_buf -= fac;
                    distort_buf += dl_dw * fac;
                    gv[CDIM - 1] += 2.f * fac * (2.f - 2.f * T - accum_w + fac) * v_dist;
                }
                if(r.o * h.vis <= kMaxAlpha)
                {
                    const float v_G = r.o * v_alpha;
                    if(h.g3 <= h.g2)
                    { // ray-splat intersection kernel
                        const float v_u = v_G * -h.vis * h.u, v_v = v_G * -h.vis * h.v;
                        const float ax = v_u / h.cz, ay = v_v / h.cz;
                        const float vc[3] = {ax, ay, -(ax * h.u + ay * h.v)};
                        // s = hu x hv:  v_hu = hv x vc,  v_hv = vc x hu
                        const float vhu[3] = {h.hv[1] * vc[2] - h.hv[2] * vc[1], h.hv[2] * vc[0] - h.hv[0] * vc[2], h.hv[0] * vc[1] - h.hv[1] * vc[0]};
                        const float vhv[3] = {vc[1] * h.hu[2] - vc[2] * h.hu[1], vc[2] * h.hu[0] - vc[0] * h.hu[2], vc[0] * h.hu[1] - vc[1] * h.hu[0]};
#pragma unroll
                        for(int k = 0; k < 3; ++k)
                        {
                            gv[CDIM + 3 + k]     = -vhu[k];
                            gv[CDIM + 3 + 3 + k] = -vhv[k];
                            gv[CDIM + 3 + 6 + k] = px * vhu[k] + py * vhv[k];
                        }
                    }
                    else
                    { // screen-space kernel
                        gv[CDIM + 12] = v_G * (-h.vis * kSurfFilterInvSq * h.dx);
                        gv[CDIM + 13] = v_G * (-h.vis * kSurfFilterInvSq * h.dy);
                        gv[CDIM + 15] = fabsf(gv[CDIM + 12]);
                        gv[CDIM + 16] = fabsf(gv[CDIM + 13]);
                    }
                    gv[CDIM + 14] = h.vis * v_alpha;
                }
#pragma unroll
                for(int k = 0; k < CDIM; ++k)
                    buf[k] += c[k] * fac;
#pragma unroll
                for(int k = 0; k < 3; ++k)
                    buf_n[k] += nn[k] * fac;
            }
            reduce_emit<0, NV>(gv, lane, r, dst, CDIM);
        }
    }
}

// The checks both compositing entries make last, in this order: the tile grid covers the image, and the flattened
// row and tile indices fit in int32.
int surfel_raster_limits(int64_t I, int64_t N, uint32_t W, uint32_t H, uint32_t tw, uint32_t th)
{
    if(!tile_grid_covers(tw, th, W, H))
        return GSB200_E_INVALID;
    if((double)I * (double)N * 9.0 >= 2147483648.0 || (double)I * tw * th >= 2147483648.0)
        return GSB200_E_UNSUPPORTED;
    return GSB200_OK;
}

// The compositing launches of the dense and sparse entries, after each entry's own checks: n_ctas CTAs over the tiles
// of the pixel policy pm, with the kernel's arguments before pm.
template<class Pix, class... Args>
int surfel_raster_fwd(int D, unsigned n_ctas, const Pix &pm, cudaStream_t st, const Args &...args)
{
    return with_channels(D, [&](auto C) {
        surfel_raster_fwd_kernel<C, Pix><<<n_ctas, kSurfThreads, 0, st>>>(args..., pm);
        return check_launch();
    });
}

template<class Pix, class... Args>
int surfel_raster_bwd(int D, unsigned n_ctas, const Pix &pm, cudaStream_t st, const Args &...args)
{
    return with_channels(D, [&](auto C) {
        surfel_raster_bwd_kernel<C, Pix><<<n_ctas, kSurfThreads, 0, st>>>(args..., pm);
        return check_launch();
    });
}
} // namespace
} // namespace gsb

// ---------------------------------------------------------------------------------------------
// C ABI
extern "C" int gsb200_surfel_projection_fwd(
    int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales, const float *viewmats,
    const float *Ks, uint32_t image_width, uint32_t image_height, float near_plane, float far_plane, float radius_clip,
    int32_t *radii, float *means2d, float *depths, float *ray_transforms, float *normals, void *stream
)
{
    if(B < 0 || C < 0 || N < 0)
        return GSB200_E_INVALID;
    const int64_t n = B * C * N;
    if(n == 0)
        return GSB200_OK;
    if(!means || !quats || !scales || !viewmats || !Ks || !radii || !means2d || !depths || !ray_transforms || !normals)
        return GSB200_E_INVALID;
    gsb::surfel_project_fwd_kernel<<<gsb::grid_for(n, gsb::kSurfThreads), gsb::kSurfThreads, 0, (cudaStream_t)stream>>>(
        B, C, N, means, quats, scales, viewmats, Ks, image_width, image_height, near_plane, far_plane, radius_clip, radii,
        means2d, depths, ray_transforms, normals
    );
    return gsb::check_launch();
}

extern "C" int gsb200_surfel_projection_bwd(
    int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales, const float *viewmats,
    const float *Ks, const int32_t *radii, const float *ray_transforms, const float *v_means2d, const float *v_depths,
    const float *v_ray_transforms, const float *v_normals, float *v_means, float *v_quats, float *v_scales, float *v_viewmats,
    void *stream
)
{
    if(B < 0 || C < 0 || N < 0)
        return GSB200_E_INVALID;
    if(B * N == 0)
        return GSB200_OK;
    if(!means || !quats || !scales || !viewmats || !Ks || !radii || !ray_transforms || !v_means2d || !v_depths
       || !v_ray_transforms || !v_normals || !v_means || !v_quats || !v_scales)
        return GSB200_E_INVALID;
    cudaStream_t st = (cudaStream_t)stream;
    if(v_viewmats)
        GSB_CUDA_TRY(cudaMemsetAsync(v_viewmats, 0, sizeof(float) * 16 * B * C, st));
    gsb::surfel_project_bwd_kernel<<<gsb::grid_for(B * N, gsb::kSurfThreads), gsb::kSurfThreads, 0, st>>>(
        B, C, N, means, quats, scales, viewmats, Ks, radii, ray_transforms, v_means2d, v_depths, v_ray_transforms, v_normals,
        v_means, v_quats, v_scales, v_viewmats
    );
    return gsb::check_launch();
}

extern "C" int gsb200_surfel_raster_fwd(
    int64_t I, int64_t N, int D, const float *means2d, const float *ray_transforms, const float *colors,
    const float *opacities, const float *normals, const float *backgrounds, const uint8_t *masks, uint32_t image_width,
    uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, const int32_t *offsets,
    const int32_t *flatten_ids, int64_t n_isects, float *render_colors, float *render_alphas, float *render_normals,
    float *render_distort, float *render_median, int32_t *last_ids, int32_t *median_ids, void *stream
)
{
    if(I < 0 || N < 0 || n_isects < 0 || !offsets || !render_colors || !render_alphas || !render_normals || !render_distort
       || !render_median || !last_ids || !median_ids)
        return GSB200_E_INVALID;
    if(n_isects > 0 && (!means2d || !ray_transforms || !colors || !opacities || !normals || !flatten_ids))
        return GSB200_E_INVALID;
    if(tile_size != (uint32_t)gsb::kTile)
        return GSB200_E_UNSUPPORTED;
    if(I == 0 || image_width == 0 || image_height == 0)
        return GSB200_OK;
    if(int rc = gsb::surfel_raster_limits(I, N, image_width, image_height, tile_width, tile_height))
        return rc;
    return gsb::surfel_raster_fwd(
        D, (uint32_t)I * tile_width * tile_height, gsb::DensePixels{}, (cudaStream_t)stream, (uint32_t)I, means2d,
        ray_transforms, colors, opacities, normals, backgrounds, masks, image_width, image_height, tile_width, tile_height,
        offsets, flatten_ids, n_isects, render_colors, render_alphas, render_normals, render_distort, render_median,
        last_ids, median_ids
    );
}

extern "C" int gsb200_surfel_raster_bwd(
    int64_t I, int64_t N, int D, const float *means2d, const float *ray_transforms, const float *colors,
    const float *opacities, const float *normals, const float *backgrounds, const uint8_t *masks, uint32_t image_width,
    uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, const int32_t *offsets,
    const int32_t *flatten_ids, int64_t n_isects, const float *render_colors, const float *render_alphas,
    const int32_t *last_ids, const int32_t *median_ids, const float *v_render_colors, const float *v_render_alphas,
    const float *v_render_normals, const float *v_render_distort, const float *v_render_median, float *v_means2d,
    float *v_ray_transforms, float *v_colors, float *v_opacities, float *v_normals, float *v_densify, float *v_means2d_abs,
    void *stream
)
{
    if(I < 0 || N < 0 || n_isects < 0)
        return GSB200_E_INVALID;
    if(tile_size != (uint32_t)gsb::kTile)
        return GSB200_E_UNSUPPORTED;
    if(n_isects == 0 || I == 0 || image_width == 0 || image_height == 0)
        return GSB200_OK;
    if(!means2d || !ray_transforms || !colors || !opacities || !normals || !offsets || !flatten_ids || !render_colors
       || !render_alphas || !last_ids || !median_ids || !v_render_colors || !v_means2d || !v_ray_transforms || !v_colors
       || !v_opacities || !v_normals || !v_densify)
        return GSB200_E_INVALID;
    if(int rc = gsb::surfel_raster_limits(I, N, image_width, image_height, tile_width, tile_height))
        return rc;
    const gsb::SurfGradDst dst{v_means2d, v_ray_transforms, v_colors, v_opacities, v_normals, v_densify, v_means2d_abs};
    return gsb::surfel_raster_bwd(
        D, (uint32_t)I * tile_width * tile_height, gsb::DensePixels{}, (cudaStream_t)stream, (uint32_t)I, means2d,
        ray_transforms, colors, opacities, normals, backgrounds, masks, image_width, image_height, tile_width, tile_height,
        offsets, flatten_ids, n_isects, render_colors, render_alphas, last_ids, median_ids, v_render_colors,
        v_render_alphas, v_render_normals, v_render_distort, v_render_median, dst
    );
}

// ---- sparse pixels (rasterize_to_pixels_2dgs_sparse): one CTA per active tile of the layout of gsb200_sparse_layout_*,
// outputs [P, *] in the original pixel order.  The checks run in the order of gsb200_raster_sparse_fwd / _bwd, then the
// row limit of the dense entries.
static int surfel_rows_ok(int64_t n_rows)
{
    return (double)n_rows * 9.0 >= 2147483648.0 ? GSB200_E_UNSUPPORTED : GSB200_OK;
}

extern "C" int gsb200_surfel_raster_sparse_fwd(
    int64_t n_rows, int D, const float *means2d, const float *ray_transforms, const float *colors, const float *opacities,
    const float *normals, const float *backgrounds, const uint8_t *masks, uint32_t image_width, uint32_t image_height,
    uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, int64_t n_active, const int32_t *active_tiles,
    const int32_t *tile_offsets, const int32_t *flatten_ids, int64_t n_isects, const uint64_t *tile_pixel_mask,
    const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, float *render_colors, float *render_alphas,
    float *render_normals, float *render_distort, float *render_median, int32_t *last_ids, int32_t *median_ids, void *stream
)
{
    if(tile_size != (uint32_t)gsb::kTile)
        return GSB200_E_UNSUPPORTED;
    if(n_rows < 0 || n_isects < 0)
        return GSB200_E_INVALID;
    if(int rc = gsb::sparse_args_ok(n_active, active_tiles, tile_offsets, tile_pixel_mask, tile_pixel_cumsum, pixel_map, image_width, image_height, tile_width, tile_height))
        return rc;
    if(n_active == 0)
        return GSB200_OK;
    if(!render_colors || !render_alphas || !render_normals || !render_distort || !render_median || !last_ids || !median_ids)
        return GSB200_E_INVALID;
    if(n_isects > 0 && (!means2d || !ray_transforms || !colors || !opacities || !normals || !flatten_ids))
        return GSB200_E_INVALID;
    if(int rc = surfel_rows_ok(n_rows))
        return rc;
    const gsb::SparsePixels pm{active_tiles, tile_pixel_mask, tile_pixel_cumsum, pixel_map};
    return gsb::surfel_raster_fwd(
        D, (uint32_t)n_active, pm, (cudaStream_t)stream, 1u, means2d, ray_transforms, colors, opacities, normals,
        backgrounds, masks, image_width, image_height, tile_width, tile_height, tile_offsets, flatten_ids, n_isects,
        render_colors, render_alphas, render_normals, render_distort, render_median, last_ids, median_ids
    );
}

extern "C" int gsb200_surfel_raster_sparse_bwd(
    int64_t n_rows, int D, const float *means2d, const float *ray_transforms, const float *colors, const float *opacities,
    const float *normals, const float *backgrounds, const uint8_t *masks, uint32_t image_width, uint32_t image_height,
    uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, int64_t n_active, const int32_t *active_tiles,
    const int32_t *tile_offsets, const int32_t *flatten_ids, int64_t n_isects, const uint64_t *tile_pixel_mask,
    const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, const float *render_colors, const float *render_alphas,
    const int32_t *last_ids, const int32_t *median_ids, const float *v_render_colors, const float *v_render_alphas,
    const float *v_render_normals, const float *v_render_distort, const float *v_render_median, float *v_means2d,
    float *v_ray_transforms, float *v_colors, float *v_opacities, float *v_normals, float *v_densify, float *v_means2d_abs,
    void *stream
)
{
    if(tile_size != (uint32_t)gsb::kTile)
        return GSB200_E_UNSUPPORTED;
    if(n_rows < 0 || n_isects < 0)
        return GSB200_E_INVALID;
    if(int rc = gsb::sparse_args_ok(n_active, active_tiles, tile_offsets, tile_pixel_mask, tile_pixel_cumsum, pixel_map, image_width, image_height, tile_width, tile_height))
        return rc;
    if(n_isects == 0 || n_active == 0)
        return GSB200_OK;
    if(!means2d || !ray_transforms || !colors || !opacities || !normals || !flatten_ids || !render_colors || !render_alphas
       || !last_ids || !median_ids || !v_render_colors || !v_means2d || !v_ray_transforms || !v_colors || !v_opacities
       || !v_normals || !v_densify)
        return GSB200_E_INVALID;
    if(int rc = surfel_rows_ok(n_rows))
        return rc;
    const gsb::SparsePixels pm{active_tiles, tile_pixel_mask, tile_pixel_cumsum, pixel_map};
    const gsb::SurfGradDst dst{v_means2d, v_ray_transforms, v_colors, v_opacities, v_normals, v_densify, v_means2d_abs};
    return gsb::surfel_raster_bwd(
        D, (uint32_t)n_active, pm, (cudaStream_t)stream, 1u, means2d, ray_transforms, colors, opacities, normals,
        backgrounds, masks, image_width, image_height, tile_width, tile_height, tile_offsets, flatten_ids, n_isects,
        render_colors, render_alphas, last_ids, median_ids, v_render_colors, v_render_alphas, v_render_normals,
        v_render_distort, v_render_median, dst
    );
}

// ---- rasterize_to_indices_in_range_2dgs: count pass (emit = 0) and emit pass (emit = 1) over one workspace (indices.cuh)
extern "C" int gsb200_surfel_indices(
    int64_t I, int64_t N, const float *means2d, const float *ray_transforms, const float *opacities,
    const float *transmittances, uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width,
    uint32_t tile_height, const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t range_start,
    int64_t range_end, int emit, void *workspace, size_t workspace_bytes, int64_t *total, int64_t *gaussian_ids,
    int64_t *pixel_ids, int64_t *image_ids, void *stream
)
{
    const cudaStream_t st = (cudaStream_t)stream;
    const bool inputs_ok  = means2d && ray_transforms && opacities && transmittances && offsets && flatten_ids;
    return gsb::run_index_pass(
        I, N, image_width, image_height, tile_size, tile_width, tile_height, n_isects, range_start, range_end, inputs_ok, emit,
        workspace, workspace_bytes, total, gaussian_ids, pixel_ids, image_ids, st,
        [&](unsigned n_tiles, int32_t b0, int32_t b1, auto sink) {
            const gsb::SurfelModel model{(uint32_t)I, image_width, image_height, tile_width, tile_height, means2d,
                                         ray_transforms, opacities};
            gsb::pair_walk_kernel<<<n_tiles, gsb::kIndexBatch, 0, st>>>(
                model, transmittances, offsets, flatten_ids, n_isects, b0, b1, sink
            );
            return gsb::check_launch();
        }
    );
}

// ---- 2DGS per-pixel contributor queries over the pair walk of SurfelModel (indices.cuh: run_contrib and its checks, in
// the order and with the return codes of gsb200_contrib_*)
namespace gsb
{
struct SurfelWalk : PlanarRows
{
    template<class Pix, class Sink>
    int launch(const ContribArgs &a, unsigned n_tiles, const Pix &pm, const Sink &sink, size_t smem, cudaStream_t st) const
    {
        return launch_walk(
            pair_walk_kernel<SurfelModel, Sink, Pix>, n_tiles, smem, st,
            SurfelModel{(uint32_t)a.I, a.W, a.H, a.tw, a.th, means2d, rows, opacities}, (const float *)nullptr, a.offsets,
            a.flatten_ids, a.n_isects, (int32_t)0, (int32_t)0x7fffffff, sink, pm
        );
    }
    static int max_samples()
    {
        return top_max_samples({
            (const void *)pair_walk_kernel<SurfelModel, TopSink, DensePixels>,
            (const void *)pair_walk_kernel<SurfelModel, TopSink, SparsePixels>
        });
    }
};
} // namespace gsb

extern "C" int gsb200_surfel_contrib_max_samples(void)
{
    return gsb::SurfelWalk::max_samples();
}

extern "C" int gsb200_surfel_contrib_count(
    int64_t I, int64_t N, const float *means2d, const float *ray_transforms, const float *opacities, uint32_t image_width,
    uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, const int32_t *offsets,
    const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
    const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int32_t *counts,
    float *alphas, void *stream
)
{
    return gsb::contrib_count(
        gsb::SurfelWalk{{means2d, ray_transforms, opacities}}, GSB200_CONTRIB_ARGS(I), counts, alphas, (cudaStream_t)stream
    );
}

extern "C" int gsb200_surfel_contrib_ids(
    int64_t I, int64_t N, const float *means2d, const float *ray_transforms, const float *opacities, uint32_t image_width,
    uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, const int32_t *offsets,
    const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
    const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int max_samples,
    int32_t *ids, float *weights, void *stream
)
{
    return gsb::contrib_ids(
        gsb::SurfelWalk{{means2d, ray_transforms, opacities}}, GSB200_CONTRIB_ARGS(I), max_samples, ids, weights, (cudaStream_t)stream
    );
}

extern "C" int gsb200_surfel_contrib_top(
    int64_t I, int64_t N, const float *means2d, const float *ray_transforms, const float *opacities, uint32_t image_width,
    uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, const int32_t *offsets,
    const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
    const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int num_samples,
    int32_t *ids, float *weights, void *stream
)
{
    return gsb::contrib_top(
        gsb::SurfelWalk{{means2d, ray_transforms, opacities}}, GSB200_CONTRIB_ARGS(I), num_samples, ids, weights, (cudaStream_t)stream
    );
}
