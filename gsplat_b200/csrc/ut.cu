// ut.cu -- 3DGUT: the unscented-transform projection through a distorted camera (fully_fused_projection_with_ut) and
// the compositing that evaluates every gaussian in 3-D along each pixel's ray (rasterize_to_pixels_eval3d), with its
// backward.  Compiled with -fmad=false: the forward and the backward evaluate each (pixel, gaussian) response with the
// same individually rounded operations, so both passes take the same alpha and transmittance decisions.
//
// Reference semantics: csrc/ProjectionUT3DGSFused.cu and include/Cameras.cuh (sigma points, weights, the UT validity
// rule, the culling tail), csrc/RasterizeToPixelsFromWorld3DGS.cuh (the maximum response of a gaussian along a ray and
// the compositing thresholds).  The reference's backward gives no gradient to viewmats, and neither does this one.
#include "camera.cuh"
#include "gaussmath.cuh"
#include "indices.cuh"
#include "pixels.cuh"

namespace gsb
{
namespace
{
constexpr int kUtThreads = 256;

struct UtParams
{
    float alpha, beta, kappa, margin;
    int require_all;
};

// Each camera's two poses for the threads of one projection CTA: the images its rows fall in, one thread per image.
// Called by every thread of the CTA.
__device__ __forceinline__ RsPoses cta_rs_poses(RsPoses *s_poses, int64_t total, int64_t N, const float *viewmats, const float *viewmats_rs)
{
    const int64_t lo    = (int64_t)blockIdx.x * kUtThreads;
    const int64_t first = lo / N, last = (min(lo + kUtThreads, total) - 1) / N;
    for(int64_t img = first + threadIdx.x; img <= last; img += kUtThreads)
        s_poses[img - first] = load_rs_poses(viewmats + img * 16, viewmats_rs + img * 16);
    __syncthreads();
    const int64_t idx = lo + threadIdx.x;
    return s_poses[(idx < total ? idx / N : first) - first];
}

// One thread per (b, c, n).  Culled rows get radii 0 and zero float outputs.  Rolling shutter: each sigma point is
// projected at the pose of the row or column it lands in (cam_project_rs); the depth and the near / far cull take the
// mid-frame pose.  FTheta without the global z order: the near / far cull and the depth take the distance |mean_c|
// from the camera centre, as the lens images points behind the camera plane.
template<class Shutter, class Lens>
__global__ void __launch_bounds__(kUtThreads) ut_project_kernel(
    int64_t B, int64_t C, int64_t N, const float *__restrict__ means, const float *__restrict__ quats,
    const float *__restrict__ scales, const float *__restrict__ opacities, const float *__restrict__ viewmats,
    const float *__restrict__ Ks, int cam_kind, const float *__restrict__ radial, const float *__restrict__ tangential,
    const float *__restrict__ thin, uint32_t W, uint32_t H, float eps2d, float near_plane, float far_plane,
    float radius_clip, UtParams ut, int32_t *__restrict__ radii, float *__restrict__ means2d, float *__restrict__ depths,
    float *__restrict__ conics, float *__restrict__ compensations, Shutter shutter, Lens lens
)
{
    const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    [[maybe_unused]] RsPoses poses;
    if constexpr(Shutter::kRolling)
    {
        // at most one image per row of the CTA, plus the one its first row starts in
        __shared__ RsPoses s_poses[kUtThreads + 1];
        poses = cta_rs_poses(s_poses, B * C * N, N, viewmats, shutter.viewmats_rs);
    }
    if(idx >= B * C * N)
        return;
    const int64_t b = idx / (C * N), c = (idx / N) % C, n = idx % N;
    const int64_t bn = b * N + n, bc = b * C + c;
    const float mean[3] = {means[bn * 3], means[bn * 3 + 1], means[bn * 3 + 2]};
    const float q[4]    = {quats[bn * 4], quats[bn * 4 + 1], quats[bn * 4 + 2], quats[bn * 4 + 3]};
    const float s[3]    = {scales[bn * 3], scales[bn * 3 + 1], scales[bn * 3 + 2]};

    int rx = 0, ry = 0;
    float mx = 0.f, my = 0.f, depth = 0.f, ca = 0.f, cb = 0.f, cc = 0.f, comp = 0.f;
    const float qn2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    const Cam cam   = Shutter::kRolling ? pose_at(poses, 0.5f) : load_cam(viewmats + bc * 16, Ks + bc * 9);
    float pc[3];
#pragma unroll
    for(int i = 0; i < 3; ++i)
        pc[i] = cam.R.m[i * 3 + 0] * mean[0] + cam.R.m[i * 3 + 1] * mean[1] + cam.R.m[i * 3 + 2] * mean[2] + cam.t[i];
    // a zero quaternion or a zero scale axis has no 3-D precision matrix to evaluate along a ray
    const bool degenerate = fabsf(qn2) < FLT_EPSILON || fabsf(s[0]) < FLT_EPSILON || fabsf(s[1]) < FLT_EPSILON
                         || fabsf(s[2]) < FLT_EPSILON;
    float zc = pc[2];
    if constexpr(Lens::kFTheta)
    {
        if(!lens.global_z_order)
            zc = sqrtf(pc[0] * pc[0] + pc[1] * pc[1] + pc[2] * pc[2]);
    }
    if(!degenerate && !(zc < near_plane || zc > far_plane))
    {
        const auto cm = lens.model(cam_kind, Ks, radial, tangential, thin, bc, W, H);
        const M3 Rq       = quat_to_rotmat(q);
        const float lam   = ut.alpha * ut.alpha * (3.f + ut.kappa) - 3.f;
        const float spread = sqrtf(3.f + lam);
        const float w_mean0 = lam / (3.f + lam);
        const float w_cov0  = w_mean0 + (1.f - ut.alpha * ut.alpha + ut.beta);
        const float w_rest  = 1.f / (2.f * (3.f + lam));
        float pu[7], pv[7];
        bool any = false, all = true;
        float m2x = 0.f, m2y = 0.f;
#pragma unroll
        for(int k = 0; k < 7; ++k)
        {
            // sigma point k: the mean, then mean +- spread * s_i * (column i of the rotation)
            float x[3] = {mean[0], mean[1], mean[2]};
            if(k > 0)
            {
                const int ax    = (k - 1) % 3;
                const float sg  = k <= 3 ? 1.f : -1.f;
                const float mag = spread * s[ax];
#pragma unroll
                for(int i = 0; i < 3; ++i)
                    x[i] = sg > 0.f ? x[i] + mag * Rq.m[i * 3 + ax] : x[i] - mag * Rq.m[i * 3 + ax];
            }
            bool ok;
            if constexpr(Shutter::kRolling)
                ok = cam_project_rs(cm, poses, shutter.type, x, ut.margin, pu[k], pv[k]);
            else
            {
                float xc[3];
#pragma unroll
                for(int i = 0; i < 3; ++i)
                    xc[i] = cam.R.m[i * 3 + 0] * x[0] + cam.R.m[i * 3 + 1] * x[1] + cam.R.m[i * 3 + 2] * x[2] + cam.t[i];
                ok = cam_project(cm, xc, ut.margin, pu[k], pv[k]);
            }
            any = any || ok;
            all = all && ok;
            // with every point required, the first invalid one ends the transform (the row is culled)
            const float w = k == 0 ? w_mean0 : w_rest;
            m2x = m2x + w * pu[k];
            m2y = m2y + w * pv[k];
        }
        if(ut.require_all ? all : any)
        {
            float c00 = 0.f, c01 = 0.f, c11 = 0.f;
#pragma unroll
            for(int k = 0; k < 7; ++k)
            {
                const float w  = k == 0 ? w_cov0 : w_rest;
                const float du = pu[k] - m2x, dv = pv[k] - m2y;
                c00 = c00 + w * (du * du);
                c01 = c01 + w * (du * dv);
                c11 = c11 + w * (dv * dv);
            }
            const float det_orig = c00 * c11 - c01 * c01;
            c00 += eps2d;
            c11 += eps2d;
            const float det      = c00 * c11 - c01 * c01;
            const float ratio    = det_orig / det;
            const float floor_   = kMinCompensation * kMinCompensation;
            const float compensation = sqrtf(ratio > floor_ ? ratio : floor_);
            // the centre covariance weight is negative, so the UT covariance need not be positive semi-definite
            bool keep = det > 0.f && !(c00 < 0.f || c11 < 0.f);
            float extend = kGaussianExtend;
            if(keep && opacities != nullptr)
            {
                const float op = opacities[bn] * compensation;
                keep = !(op < kAlphaThreshold);
                if(keep)
                {
                    const float e2 = sqrtf(2.f * exact_log(op / kAlphaThreshold));
                    extend = e2 < extend ? e2 : extend;
                }
            }
            if(keep)
            {
                // tight box: the smaller of the axis extent and the larger eigenvalue's
                const float hb  = 0.5f * (c00 + c11);
                const float tmp = sqrtf(fmaxf(0.01f, hb * hb - det));
                const float r1  = extend * sqrtf(hb + tmp);
                const float fr_x = ceilf(fminf(extend * sqrtf(c00), r1));
                const float fr_y = ceilf(fminf(extend * sqrtf(c11), r1));
                const float ood  = 1.f / det;
                const bool clipped = fr_x <= radius_clip && fr_y <= radius_clip;
                const bool off = m2x + fr_x <= 0.f || m2x - fr_x >= (float)W || m2y + fr_y <= 0.f || m2y - fr_y >= (float)H;
                const float k0 = c11 * ood, k1 = -c01 * ood, k2 = c00 * ood;
                // finite inputs can overflow (a far sigma point through a strong distortion): a NaN row would pass every
                // off-screen test, so it is culled
                const bool finite = isfinite(m2x) && isfinite(m2y) && isfinite(k0) && isfinite(k1) && isfinite(k2)
                                 && isfinite(fr_x) && isfinite(fr_y) && isfinite(zc);
                if(!clipped && !off && finite)
                {
                    rx = (int)fr_x, ry = (int)fr_y;
                    mx = m2x, my = m2y, depth = zc;
                    ca = k0, cb = k1, cc = k2;
                    comp = compensation;
                }
            }
        }
    }
    reinterpret_cast<int2 *>(radii)[idx]     = make_int2(rx, ry);
    reinterpret_cast<float2 *>(means2d)[idx] = make_float2(mx, my);
    depths[idx]         = depth;
    conics[idx * 3 + 0] = ca;
    conics[idx * 3 + 1] = cb;
    conics[idx * 3 + 2] = cc;
    if(compensations)
        compensations[idx] = comp;
}

// ------------------------------------------------------------------ compositing
// One staged gaussian of a tile: world mean, opacity of its (image, gaussian) row, the world-to-unit-sphere map
// M = S^-1 R^T, its row id in [I * N] and its gaussian id in [B * N].
struct EvalRec
{
    float mu[3], o;
    float m[9];
    int32_t id, bn;
};

__device__ __forceinline__ void stage(
    EvalRec &r, int32_t g, int64_t C, int64_t N, const float *means, const float *quats, const float *scales,
    const float *opacities
)
{
    const int64_t bn = (g / (C * N)) * N + g % N;
    r.id             = g;
    r.bn             = (int32_t)bn;
    r.o              = opacities[g];
#pragma unroll
    for(int k = 0; k < 3; ++k)
        r.mu[k] = means[bn * 3 + k];
    const float q[4] = {quats[bn * 4], quats[bn * 4 + 1], quats[bn * 4 + 2], quats[bn * 4 + 3]};
    const M3 R       = quat_to_rotmat(q);
#pragma unroll
    for(int i = 0; i < 3; ++i)
    {
        const float inv = 1.f / scales[bn * 3 + i];
#pragma unroll
        for(int j = 0; j < 3; ++j)
            r.m[i * 3 + j] = R.m[j * 3 + i] * inv;
    }
}

// The world ray of pixel (i, j) of one camera: origin, unit direction.  false: the camera model cannot unproject it.
template<class Model>
__device__ __forceinline__ bool pixel_ray(const float *vm, const Model &cm, uint32_t i, uint32_t j, float *ro, float *rd)
{
    float dc[3];
    const bool ok = cam_unproject(cm, (float)j + 0.5f, (float)i + 0.5f, dc);
    const float R[9] = {vm[0], vm[1], vm[2], vm[4], vm[5], vm[6], vm[8], vm[9], vm[10]};
    const float t[3] = {vm[3], vm[7], vm[11]};
#pragma unroll
    for(int k = 0; k < 3; ++k)
    {
        ro[k] = -(R[0 * 3 + k] * t[0] + R[1 * 3 + k] * t[1] + R[2 * 3 + k] * t[2]);
        rd[k] = R[0 * 3 + k] * dc[0] + R[1 * 3 + k] * dc[1] + R[2 * 3 + k] * dc[2];
    }
    return ok;
}

// Rolling shutter: the same ray, carried to the world by the pose at the frame time of the pixel centre's row or column.
// The forward and the backward build it alike, so both take the same alpha and transmittance decisions.
template<class Model>
__device__ __forceinline__ bool pixel_ray(
    const RsPoses &P, int type, const Model &cm, uint32_t i, uint32_t j, float *ro, float *rd
)
{
    float dc[3];
    const float u = (float)j + 0.5f, v = (float)i + 0.5f;
    const bool ok   = cam_unproject(cm, u, v, dc);
    const Cam pose  = pose_at(P, shutter_time(type, cm.W, cm.H, u, v));
    const float *R  = pose.R.m;
#pragma unroll
    for(int k = 0; k < 3; ++k)
    {
        ro[k] = -(R[0 * 3 + k] * pose.t[0] + R[1 * 3 + k] * pose.t[1] + R[2 * 3 + k] * pose.t[2]);
        rd[k] = R[0 * 3 + k] * dc[0] + R[1 * 3 + k] * dc[1] + R[2 * 3 + k] * dc[2];
    }
    return ok;
}

// The pixel's ray under either shutter.  Rolling: the image's two poses are loaded once per CTA (one image per CTA);
// every thread of the CTA calls this.
template<class Shutter, class Model>
__device__ __forceinline__ bool shutter_pixel_ray(
    const Shutter &shutter, const float *viewmats, uint32_t img, bool inside, const Model &cm, uint32_t i, uint32_t j,
    float *ro, float *rd
)
{
    __shared__ RsPoses s_poses;
    if(threadIdx.x == 0)
        s_poses = load_rs_poses(viewmats + (int64_t)img * 16, shutter.viewmats_rs + (int64_t)img * 16);
    __syncthreads();
    return inside && pixel_ray(s_poses, shutter.type, cm, i, j, ro, rd);
}

// Maximum response of one gaussian along a ray: a = M (o - mu), g = normalize(M d); the closest approach to the
// gaussian's centre in its own frame is |g x a|.  ok = false: the approach lies behind the ray origin, or alpha < 1/255.
struct EvalHit
{
    float w[3], a[3], b[3], bl, g[3], c[3], resp, alpha;
    bool ok;
};

__device__ __forceinline__ EvalHit eval_hit(const EvalRec &r, const float *ro, const float *rd)
{
    EvalHit h;
#pragma unroll
    for(int k = 0; k < 3; ++k)
        h.w[k] = ro[k] - r.mu[k];
#pragma unroll
    for(int i = 0; i < 3; ++i)
    {
        h.a[i] = r.m[i * 3 + 0] * h.w[0] + r.m[i * 3 + 1] * h.w[1] + r.m[i * 3 + 2] * h.w[2];
        h.b[i] = r.m[i * 3 + 0] * rd[0] + r.m[i * 3 + 1] * rd[1] + r.m[i * 3 + 2] * rd[2];
    }
    const float l2 = h.b[0] * h.b[0] + h.b[1] * h.b[1] + h.b[2] * h.b[2];
    h.bl           = sqrtf(l2);
    const float inv = l2 > 0.f ? 1.f / h.bl : 1.f;
#pragma unroll
    for(int k = 0; k < 3; ++k)
        h.g[k] = h.b[k] * inv;
    const float hit_t = -(h.g[0] * h.a[0] + h.g[1] * h.a[1] + h.g[2] * h.a[2]);
    h.c[0]  = h.g[1] * h.a[2] - h.g[2] * h.a[1];
    h.c[1]  = h.g[2] * h.a[0] - h.g[0] * h.a[2];
    h.c[2]  = h.g[0] * h.a[1] - h.g[1] * h.a[0];
    const float dist = h.c[0] * h.c[0] + h.c[1] * h.c[1] + h.c[2] * h.c[2];
    h.resp  = fast_exp(-0.5f * dist);
    h.alpha = fminf(kMaxAlpha, r.o * h.resp);
    // Ordered comparisons: a NaN hit_t or response (a zero, sub-1/FLT_MAX or infinite scale, a non-finite mean) makes
    // no contribution.  fminf would turn a NaN response into alpha 0.99.
    h.ok    = hit_t >= 0.f && r.o * h.resp >= kAlphaThreshold && l2 > 0.f;
    return h;
}

struct EvalGeom
{
    uint32_t I, C, N, W, H, tw, th;
    int cam_kind;
    const float *viewmats, *Ks, *radial, *tangential, *thin;
};

// One CTA per 16x16 tile of the pixel policy (pixels.cuh), one pixel per thread: every tile of the [I, th, tw] grid
// (DensePixels), or every active tile with its requested pixels only (SparsePixels).  A pixel is composited when it has
// an output row (live) and lies inside the W x H image: its ray and its rolling-shutter frame time are defined there
// only, so a live margin pixel of a partial sparse tile gets the background and alpha 0.  Every other thread stages
// records and meets every barrier but composites nothing.  last_ids: the list index of the pixel's last composited
// gaussian, -1 for none.
template<int CDIM, class Shutter, class Lens, class Pix = DensePixels>
__global__ void __launch_bounds__(kUtThreads, 1) eval3d_fwd_kernel(
    EvalGeom geo, const float *__restrict__ means, const float *__restrict__ quats, const float *__restrict__ scales,
    const float *__restrict__ colors, const float *__restrict__ opacities, const float *__restrict__ backgrounds,
    const uint8_t *__restrict__ masks, const int32_t *__restrict__ offsets, const int32_t *__restrict__ flatten_ids,
    int64_t n_isects, float *__restrict__ render_colors, float *__restrict__ render_alphas, int32_t *__restrict__ last_ids,
    Shutter shutter, Lens lens, const Pix pixmap = Pix{}
)
{
    __shared__ EvalRec rec[kUtThreads];
    const uint32_t tile = pixmap.tile(blockIdx.x); // image * th * tw + tile row * tw + tile col
    const uint32_t img  = tile / (geo.tw * geo.th);
    const uint32_t tin  = tile - img * geo.tw * geo.th;
    const uint32_t tr   = threadIdx.x;
    const uint32_t i    = (tin / geo.tw) * kTile + tr / kTile;
    const uint32_t j    = (tin % geo.tw) * kTile + tr % kTile;
    bool live, inside = i < geo.H && j < geo.W;
    int64_t pix;
    if constexpr(Pix::kSparse)
    {
        pix    = pixmap.slot(blockIdx.x, (int)tr, live);
        inside = inside && live;
    }
    else
    {
        live = inside;
        pix  = (int64_t)img * geo.H * geo.W + (int64_t)i * geo.W + j;
    }
    const float *bg     = backgrounds ? backgrounds + (int64_t)img * CDIM : nullptr;
    if(masks && !masks[tile])
    {
        if(live)
        {
#pragma unroll
            for(int k = 0; k < CDIM; ++k)
                render_colors[pix * CDIM + k] = bg ? bg[k] : 0.f;
            render_alphas[pix] = 0.f;
            last_ids[pix]      = -1;
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
        end   = (tile + 1 == geo.I * geo.tw * geo.th) ? n_isects : offsets[tile + 1];
    }
    float ro[3] = {0.f, 0.f, 0.f}, rd[3] = {0.f, 0.f, 1.f};
    bool done = !inside;
    if constexpr(Shutter::kRolling)
    {
        const auto cm = lens.model(geo.cam_kind, geo.Ks, geo.radial, geo.tangential, geo.thin, img, geo.W, geo.H);
        done          = !shutter_pixel_ray(shutter, geo.viewmats, img, inside, cm, i, j, ro, rd);
    }
    else if(inside)
    {
        const auto cm = lens.model(geo.cam_kind, geo.Ks, geo.radial, geo.tangential, geo.thin, img, geo.W, geo.H);
        done          = !pixel_ray(geo.viewmats + (int64_t)img * 16, cm, i, j, ro, rd);
    }
    float T = 1.f, pix_out[CDIM];
#pragma unroll
    for(int k = 0; k < CDIM; ++k)
        pix_out[k] = 0.f;
    int32_t cur_idx = -1;
    for(int64_t batch = start; batch < end; batch += kUtThreads)
    {
        if(__syncthreads_count(done) == kUtThreads)
            break;
        if(batch + tr < end)
            stage(rec[tr], flatten_ids[batch + tr], geo.C, geo.N, means, quats, scales, opacities);
        __syncthreads();
        const int n_b = (int)min((int64_t)kUtThreads, end - batch);
        for(int t = 0; t < n_b && !done; ++t)
        {
            const EvalRec &r = rec[t];
            const EvalHit h  = eval_hit(r, ro, rd);
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
            cur_idx = (int32_t)(batch + t);
            T       = next_T;
        }
    }
    if(!live)
        return;
    render_alphas[pix] = 1.f - T;
#pragma unroll
    for(int k = 0; k < CDIM; ++k)
        render_colors[pix * CDIM + k] = bg ? pix_out[k] + T * bg[k] : pix_out[k];
    last_ids[pix] = cur_idx;
}

// The 3DGUT model of pair_walk_kernel (indices.cuh), the pair query and contributor queries of the _eval3d ops:
// eval3d_fwd_kernel's staging, ray (camera model, rolling-shutter pose) and eval_hit.  As in the forward, a pixel
// composites only when it is live, lies inside the W x H image and has a ray.
template<class Shutter, class Lens>
struct Eval3dModel : EvalGeom
{
    const float *means, *quats, *scales, *opacities;
    Shutter shutter;
    Lens lens;
    static constexpr int kMinBlocks = 1; // the forward's launch bounds
    using Rec = EvalRec;
    struct Pixel
    {
        float ro[3], rd[3];
    };
    __device__ __forceinline__ void stage(EvalRec &r, int32_t g) const { gsb::stage(r, g, C, N, means, quats, scales, opacities); }
    __device__ __forceinline__ bool setup(uint32_t img, uint32_t i, uint32_t j, bool live, Pixel &p) const
    {
        const bool inside = i < H && j < W && live;
        p                 = {{0.f, 0.f, 0.f}, {0.f, 0.f, 1.f}};
        if constexpr(Shutter::kRolling)
        {
            const auto cm = lens.model(cam_kind, Ks, radial, tangential, thin, img, W, H);
            return shutter_pixel_ray(shutter, viewmats, img, inside, cm, i, j, p.ro, p.rd);
        }
        else if(inside)
        {
            const auto cm = lens.model(cam_kind, Ks, radial, tangential, thin, img, W, H);
            return pixel_ray(viewmats + (int64_t)img * 16, cm, i, j, p.ro, p.rd);
        }
        return false;
    }
    __device__ __forceinline__ EvalHit hit(const EvalRec &r, const Pixel &p) const { return eval_hit(r, p.ro, p.rd); }
};

struct EvalGradDst
{
    float *colors, *opacities, *rec; // rec: [B * N, 12] = v_mean 3 | v_M 9

    // reduce_emit's routing (common.cuh): slot of the gradient vector of eval3d_bwd_kernel to its row
    __device__ __forceinline__ void add(int slot, const EvalRec &r, float val, int CDIM) const
    {
        if(slot < CDIM)
            atomicAdd(colors + (int64_t)r.id * CDIM + slot, val);
        else if(slot == CDIM)
            atomicAdd(opacities + r.id, val);
        else
            atomicAdd(rec + (int64_t)r.bn * 12 + (slot - CDIM - 1), val);
    }
};

// Back to front over each tile's list.  Per gaussian, the warp's per-pixel gradients (colours, opacity, mean, M) are
// butterfly-reduced and added with one atomic per value.  The tiles and the pixels that composite are the forward's
// (eval3d_fwd_kernel, same pixel policy).
template<int CDIM, class Shutter, class Lens, class Pix = DensePixels>
__global__ void __launch_bounds__(kUtThreads, 1) eval3d_bwd_kernel(
    EvalGeom geo, const float *__restrict__ means, const float *__restrict__ quats, const float *__restrict__ scales,
    const float *__restrict__ colors, const float *__restrict__ opacities, const float *__restrict__ backgrounds,
    const uint8_t *__restrict__ masks, const int32_t *__restrict__ offsets, const int32_t *__restrict__ flatten_ids,
    int64_t n_isects, const float *__restrict__ render_alphas, const int32_t *__restrict__ last_ids,
    const float *__restrict__ v_render_colors, const float *__restrict__ v_render_alphas, EvalGradDst dst, Shutter shutter,
    Lens lens, const Pix pixmap = Pix{}
)
{
    constexpr int NV = CDIM + 13; // colours | opacity 1 | mean 3 | M 9
    __shared__ EvalRec rec[kUtThreads];
    __shared__ float s_col[kUtThreads * CDIM];
    const uint32_t tile = pixmap.tile(blockIdx.x);
    if(masks && !masks[tile])
        return;
    const uint32_t img  = tile / (geo.tw * geo.th);
    const uint32_t tin  = tile - img * geo.tw * geo.th;
    const uint32_t tr   = threadIdx.x;
    const unsigned lane = tr & 31;
    const uint32_t i    = (tin / geo.tw) * kTile + tr / kTile;
    const uint32_t j    = (tin % geo.tw) * kTile + tr % kTile;
    // a pixel that does not composite reads the row of a live one (the image's first pixel; sparse: its own row, or row
    // 0 when it has none) and adds nothing
    bool inside = i < geo.H && j < geo.W;
    int64_t pix;
    if constexpr(Pix::kSparse)
    {
        bool live;
        pix    = pixmap.slot(blockIdx.x, (int)tr, live);
        inside = inside && live;
    }
    else
        pix = inside ? (int64_t)img * geo.H * geo.W + (int64_t)i * geo.W + j : (int64_t)img * geo.H * geo.W;
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
        end   = (tile + 1 == geo.I * geo.tw * geo.th) ? n_isects : offsets[tile + 1];
    }
    float ro[3] = {0.f, 0.f, 0.f}, rd[3] = {0.f, 0.f, 1.f};
    if constexpr(Shutter::kRolling)
    {
        const auto cm = lens.model(geo.cam_kind, geo.Ks, geo.radial, geo.tangential, geo.thin, img, geo.W, geo.H);
        inside        = shutter_pixel_ray(shutter, geo.viewmats, img, inside, cm, i, j, ro, rd);
    }
    else if(inside)
    {
        const auto cm = lens.model(geo.cam_kind, geo.Ks, geo.radial, geo.tangential, geo.thin, img, geo.W, geo.H);
        inside        = pixel_ray(geo.viewmats + (int64_t)img * 16, cm, i, j, ro, rd);
    }

    const float T_final = 1.f - render_alphas[pix];
    float T             = T_final;
    float buf[CDIM], v_rc[CDIM];
#pragma unroll
    for(int k = 0; k < CDIM; ++k)
    {
        buf[k]  = 0.f;
        v_rc[k] = v_render_colors[pix * CDIM + k];
    }
    const float v_ra = v_render_alphas ? v_render_alphas[pix] : 0.f;
    float bg_dot     = 0.f;
    if(bg)
    {
#pragma unroll
        for(int k = 0; k < CDIM; ++k)
            bg_dot += bg[k] * v_rc[k];
    }
    const int64_t bin_final = inside ? last_ids[pix] : -1;
    int64_t warp_bin_final  = bin_final;
#pragma unroll
    for(int off = 16; off >= 1; off >>= 1)
        warp_bin_final = max(warp_bin_final, (int64_t)__shfl_xor_sync(0xffffffffu, (long long)warp_bin_final, off));

    for(int64_t batch_end = end - 1; batch_end >= start; batch_end -= kUtThreads)
    {
        __syncthreads();
        const int64_t idx = batch_end - tr;
        if(idx >= start)
        {
            const int32_t g = flatten_ids[idx];
            stage(rec[tr], g, geo.C, geo.N, means, quats, scales, opacities);
#pragma unroll
            for(int k = 0; k < CDIM; ++k)
                s_col[tr * CDIM + k] = colors[(int64_t)g * CDIM + k];
        }
        __syncthreads();
        const int n_b = (int)min((int64_t)kUtThreads, batch_end + 1 - start);
        const int t0  = (int)max((int64_t)0, batch_end - warp_bin_final);
        for(int t = t0; t < n_b; ++t)
        {
            const EvalRec &r = rec[t];
            const int64_t gi = batch_end - t;
            bool valid       = inside && gi <= bin_final;
            EvalHit h;
            if(valid)
            {
                h     = eval_hit(r, ro, rd);
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
                v_alpha += T_final * ra * v_ra;
                v_alpha += -T_final * ra * bg_dot;
                if(r.o * h.resp <= kMaxAlpha)
                {
                    gv[CDIM] = h.resp * v_alpha;
                    // d resp / d dist = -resp / 2, dist = |c|^2, c = g x a
                    const float v_dist = -0.5f * h.resp * (r.o * v_alpha);
                    float vc[3];
#pragma unroll
                    for(int k = 0; k < 3; ++k)
                        vc[k] = 2.f * v_dist * h.c[k];
                    // c = g x a:  v_g = a x vc,  v_a = vc x g
                    const float vg[3] = {h.a[1] * vc[2] - h.a[2] * vc[1], h.a[2] * vc[0] - h.a[0] * vc[2], h.a[0] * vc[1] - h.a[1] * vc[0]};
                    const float va[3] = {vc[1] * h.g[2] - vc[2] * h.g[1], vc[2] * h.g[0] - vc[0] * h.g[2], vc[0] * h.g[1] - vc[1] * h.g[0]};
                    // g = b / |b|
                    const float gd = h.g[0] * vg[0] + h.g[1] * vg[1] + h.g[2] * vg[2];
                    float vb[3];
#pragma unroll
                    for(int k = 0; k < 3; ++k)
                        vb[k] = (vg[k] - h.g[k] * gd) / h.bl;
                    // a = M (o - mu), b = M d
#pragma unroll
                    for(int k = 0; k < 3; ++k)
                        gv[CDIM + 1 + k] = -(r.m[0 * 3 + k] * va[0] + r.m[1 * 3 + k] * va[1] + r.m[2 * 3 + k] * va[2]);
#pragma unroll
                    for(int p = 0; p < 3; ++p)
#pragma unroll
                        for(int q = 0; q < 3; ++q)
                            gv[CDIM + 4 + p * 3 + q] = va[p] * h.w[q] + vb[p] * rd[q];
                }
#pragma unroll
                for(int k = 0; k < CDIM; ++k)
                    buf[k] += c[k] * fac;
            }
            reduce_emit<0, NV>(gv, lane, r, dst, CDIM);
        }
    }
}

// Per gaussian: the accumulated record (v_mean, v_M) to v_means, v_quats, v_scales through M = S^-1 R^T.
__global__ void __launch_bounds__(kUtThreads) eval3d_finish_kernel(
    int64_t BN, const float *__restrict__ quats, const float *__restrict__ scales, const float *__restrict__ rec,
    float *__restrict__ v_means, float *__restrict__ v_quats, float *__restrict__ v_scales
)
{
    const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(g >= BN)
        return;
    const float *rg = rec + g * 12;
#pragma unroll
    for(int k = 0; k < 3; ++k)
        v_means[g * 3 + k] = rg[k];
    const float q[4] = {quats[g * 4], quats[g * 4 + 1], quats[g * 4 + 2], quats[g * 4 + 3]};
    const M3 R       = quat_to_rotmat(q);
    // a gaussian with no v_M gets zero v_scales and v_quats, also when its scale or quaternion makes M non-finite (such
    // a gaussian never contributes)
    const bool any_vm = rg[3] != 0.f || rg[4] != 0.f || rg[5] != 0.f || rg[6] != 0.f || rg[7] != 0.f || rg[8] != 0.f
                        || rg[9] != 0.f || rg[10] != 0.f || rg[11] != 0.f;
    M3 vR;
#pragma unroll
    for(int i = 0; i < 3; ++i)
    {
        const float s   = scales[g * 3 + i];
        const float inv = 1.f / s;
        float acc       = 0.f;
#pragma unroll
        for(int j = 0; j < 3; ++j)
        {
            const float vm     = rg[3 + i * 3 + j];
            vR.m[j * 3 + i]    = vm * inv;
            acc               += vm * R.m[j * 3 + i];
        }
        v_scales[g * 3 + i] = any_vm ? -acc * inv * inv : 0.f;
    }
    float vq[4] = {0.f, 0.f, 0.f, 0.f};
    if(any_vm)
        quat_to_rotmat_vjp(q, vR, vq);
#pragma unroll
    for(int k = 0; k < 4; ++k)
        v_quats[g * 4 + k] = vq[k];
}

// The camera model and its coefficients: pinhole / fisheye take the per-camera arrays, FTheta the shared parameters
// alone (reference_poly 0 or 1, finite values).  A rolling shutter takes an end pose, the global shutter none; the frame
// time divides by the rows (or columns) - 1.
int camera_checks(
    int cam_kind, const float *radial, const float *tangential, const float *thin, const gsb200_ftheta_params *ft,
    const float *viewmats_rs, int rolling_shutter, uint32_t W, uint32_t H
)
{
    if(cam_kind != kUtPinhole && cam_kind != kUtFisheye && cam_kind != kUtFTheta)
        return GSB200_E_UNSUPPORTED;
    if((cam_kind == kUtFTheta) != (ft != nullptr))
        return GSB200_E_INVALID;
    if(cam_kind == kUtFTheta)
    {
        if(radial || tangential || thin)
            return GSB200_E_INVALID;
        if(ft->reference_poly != kFThetaPixelToAngle && ft->reference_poly != kFThetaAngleToPixel)
            return GSB200_E_INVALID;
        bool finite = isfinite(ft->max_angle);
        for(int i = 0; i < 6; ++i)
            finite = finite && isfinite(ft->pixeldist_to_angle_poly[i]) && isfinite(ft->angle_to_pixeldist_poly[i]);
        for(int i = 0; i < 3; ++i)
            finite = finite && isfinite(ft->linear_cde[i]);
        if(!finite)
            return GSB200_E_INVALID;
    }
    if(rolling_shutter < 0 || rolling_shutter > kShutterGlobal)
        return GSB200_E_INVALID;
    if((viewmats_rs != nullptr) != (rolling_shutter != kShutterGlobal))
        return GSB200_E_INVALID;
    const bool rows = rolling_shutter == kShutterTopToBottom || rolling_shutter == kShutterBottomToTop;
    const bool cols = rolling_shutter == kShutterLeftToRight || rolling_shutter == kShutterRightToLeft;
    if((rows && H < 2) || (cols && W < 2))
        return GSB200_E_INVALID;
    return GSB200_OK;
}

int eval3d_checks(
    int64_t B, int64_t C, int64_t N, uint32_t W, uint32_t H, uint32_t tile_size, uint32_t tw, uint32_t th
)
{
    if(B < 0 || C < 0 || N < 0)
        return GSB200_E_INVALID;
    if(tile_size != (uint32_t)kTile)
        return GSB200_E_UNSUPPORTED;
    if(B * C > 0 && W > 0 && H > 0 && !tile_grid_covers(tw, th, W, H))
        return GSB200_E_INVALID;
    if((double)B * C * N >= 2147483648.0 || (double)B * C * tw * th >= 2147483648.0)
        return GSB200_E_UNSUPPORTED;
    return GSB200_OK;
}

// Runs f with the kernels' shutter policy: the global shutter for no end pose.
template<class F>
int with_shutter(const float *viewmats_rs, int rolling_shutter, F &&f)
{
    if(viewmats_rs)
        return f(RollingShutter{viewmats_rs, rolling_shutter});
    return f(GlobalShutter{});
}

// Runs f with the kernels' shutter and lens policies: FThetaLens, its parameters copied by value, for FTheta parameters;
// CamLens (the runtime pinhole / fisheye model) otherwise.
template<class F>
int with_policies(const float *viewmats_rs, int rolling_shutter, const gsb200_ftheta_params *ft, int global_z_order, F &&f)
{
    return with_shutter(viewmats_rs, rolling_shutter, [&](auto shutter) {
        if(ft)
            return f(shutter, FThetaLens{*ft, global_z_order});
        return f(shutter, CamLens{});
    });
}

// The tiles and the camera of the compositing and query entries, from their parameters.
EvalGeom eval_geom(
    int64_t B, int64_t C, int64_t N, uint32_t W, uint32_t H, uint32_t tw, uint32_t th, int cam_kind, const float *viewmats,
    const float *Ks, const float *radial, const float *tangential, const float *thin
)
{
    return {(uint32_t)(B * C), (uint32_t)C, (uint32_t)N, W, H, tw, th, cam_kind, viewmats, Ks, radial, tangential, thin};
}

// The compositing launches of the dense and sparse entries, after each entry's own checks: n_ctas CTAs over the tiles
// of the pixel policy pm, with the kernel's arguments between geo and the policies.
template<class Pix, class... Args>
int eval3d_fwd(
    const EvalGeom &geo, unsigned n_ctas, const Pix &pm, int D, const gsb200_ftheta_params *ft, const float *viewmats_rs,
    int rolling_shutter, cudaStream_t st, const Args &...args
)
{
    return with_policies(viewmats_rs, rolling_shutter, ft, 1, [&](auto shutter, auto lens) {
        return with_channels(D, [&](auto CH) {
            eval3d_fwd_kernel<CH, decltype(shutter), decltype(lens), Pix><<<n_ctas, kUtThreads, 0, st>>>(
                geo, args..., shutter, lens, pm
            );
            return check_launch();
        });
    });
}

// composite: whether the compositing backward runs (args: its arguments between scales and dst) before the finish
// kernel, which turns the B * N records of dst into v_means, v_quats and v_scales
template<class Pix, class... Args>
int eval3d_bwd(
    const EvalGeom &geo, unsigned n_ctas, const Pix &pm, bool composite, int D, const gsb200_ftheta_params *ft,
    const float *viewmats_rs, int rolling_shutter, cudaStream_t st, int64_t BN, const float *means, const float *quats,
    const float *scales, const EvalGradDst &dst, float *v_means, float *v_quats, float *v_scales, const Args &...args
)
{
    const int rc = !composite ? GSB200_OK : with_policies(viewmats_rs, rolling_shutter, ft, 1, [&](auto shutter, auto lens) {
        return with_channels(D, [&](auto CH) {
            eval3d_bwd_kernel<CH, decltype(shutter), decltype(lens), Pix><<<n_ctas, kUtThreads, 0, st>>>(
                geo, means, quats, scales, args..., dst, shutter, lens, pm
            );
            return check_launch();
        });
    });
    if(rc)
        return rc;
    eval3d_finish_kernel<<<grid_for(BN, kUtThreads), kUtThreads, 0, st>>>(BN, quats, scales, dst.rec, v_means, v_quats, v_scales);
    return check_launch();
}

// The contributor queries' walk (indices.cuh: run_contrib): pair_walk_kernel of Eval3dModel over the rows and the
// camera of gsb200_eval3d_fwd, from T = 1 through the whole lists.  Its inputs are the camera (every pixel's ray reads
// it) and, when there are intersections, the gaussians; a sparse layout needs at least one image for its tiles to lie in.
struct Eval3dWalk
{
    EvalGeom geo;
    const float *means, *quats, *scales, *opacities;
    const gsb200_ftheta_params *ft;
    const float *viewmats_rs;
    int rolling_shutter;

    bool inputs_ok(int64_t n_isects) const
    {
        return geo.I > 0 && geo.viewmats && geo.Ks && (n_isects == 0 || (means && quats && scales && opacities));
    }
    // runs f with the Eval3dModel of the walk's shutter and lens
    template<class F>
    int with_model(F &&f) const
    {
        return with_policies(viewmats_rs, rolling_shutter, ft, 1, [&](auto shutter, auto lens) {
            return f(Eval3dModel<decltype(shutter), decltype(lens)>{geo, means, quats, scales, opacities, shutter, lens});
        });
    }
    template<class Pix, class Sink>
    int launch(const ContribArgs &a, unsigned n_tiles, const Pix &pm, const Sink &sink, size_t smem, cudaStream_t st) const
    {
        return with_model([&](const auto &model) {
            return launch_walk(
                pair_walk_kernel<std::decay_t<decltype(model)>, Sink, Pix>, n_tiles, smem, st, model, (const float *)nullptr,
                a.offsets, a.flatten_ids, a.n_isects, (int32_t)0, (int32_t)0x7fffffff, sink, pm
            );
        });
    }
    // one bound for every camera and shutter: the largest staging of the eight top-K instantiations (the rolling ones
    // also hold the image's two poses)
    static int max_samples()
    {
        return top_max_samples({
            (const void *)pair_walk_kernel<Eval3dModel<GlobalShutter, CamLens>, TopSink, DensePixels>,
            (const void *)pair_walk_kernel<Eval3dModel<GlobalShutter, FThetaLens>, TopSink, DensePixels>,
            (const void *)pair_walk_kernel<Eval3dModel<RollingShutter, CamLens>, TopSink, DensePixels>,
            (const void *)pair_walk_kernel<Eval3dModel<RollingShutter, FThetaLens>, TopSink, DensePixels>,
            (const void *)pair_walk_kernel<Eval3dModel<GlobalShutter, CamLens>, TopSink, SparsePixels>,
            (const void *)pair_walk_kernel<Eval3dModel<GlobalShutter, FThetaLens>, TopSink, SparsePixels>,
            (const void *)pair_walk_kernel<Eval3dModel<RollingShutter, CamLens>, TopSink, SparsePixels>,
            (const void *)pair_walk_kernel<Eval3dModel<RollingShutter, FThetaLens>, TopSink, SparsePixels>,
        });
    }
};

// The checks of every 3DGUT query entry before its own: sizes, the walk's camera, then the sparse layout if any.
int eval3d_query_checks(
    int64_t B, int64_t C, int64_t N, const Eval3dWalk &w, uint32_t tile_size, int64_t n_active,
    const int32_t *active_tiles, const int32_t *offsets, const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum,
    const int64_t *pixel_map
)
{
    const EvalGeom &g = w.geo;
    if(int rc = eval3d_checks(B, C, N, g.W, g.H, tile_size, g.tw, g.th))
        return rc;
    if(int rc = camera_checks(g.cam_kind, g.radial, g.tangential, g.thin, w.ft, w.viewmats_rs, w.rolling_shutter, g.W, g.H))
        return rc;
    if(active_tiles != nullptr)
        return sparse_args_ok(n_active, active_tiles, offsets, tile_pixel_mask, tile_pixel_cumsum, pixel_map, g.W, g.H, g.tw, g.th);
    return GSB200_OK;
}
} // namespace
} // namespace gsb

// ---------------------------------------------------------------------------------------------
// C ABI
extern "C" int gsb200_ut_projection_fwd(
    int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales, const float *opacities,
    const float *viewmats, const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
    const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
    int global_z_order, uint32_t image_width, uint32_t image_height, float eps2d, float near_plane, float far_plane,
    float radius_clip, float ut_alpha, float ut_beta, float ut_kappa, float ut_in_image_margin_factor,
    int ut_require_all_sigma_points_valid, int32_t *radii, float *means2d, float *depths, float *conics,
    float *compensations, void *stream
)
{
    if(B < 0 || C < 0 || N < 0)
        return GSB200_E_INVALID;
    if(int rc = gsb::camera_checks(camera_model, radial_coeffs, tangential_coeffs, thin_prism_coeffs, ftheta, viewmats_rs,
                                   rolling_shutter, image_width, image_height))
        return rc;
    if(camera_model == gsb::kUtFisheye && (tangential_coeffs || thin_prism_coeffs))
        return GSB200_E_INVALID;
    if(!global_z_order && camera_model != gsb::kUtFTheta)
        return GSB200_E_UNSUPPORTED;
    if(!(ut_alpha * ut_alpha * (3.f + ut_kappa) > 0.f))
        return GSB200_E_INVALID;
    const int64_t n = B * C * N;
    if(n == 0)
        return GSB200_OK;
    if(!means || !quats || !scales || !viewmats || !Ks || !radii || !means2d || !depths || !conics)
        return GSB200_E_INVALID;
    const gsb::UtParams ut{ut_alpha, ut_beta, ut_kappa, ut_in_image_margin_factor, ut_require_all_sigma_points_valid};
    return gsb::with_policies(viewmats_rs, rolling_shutter, ftheta, global_z_order, [&](auto shutter, auto lens) {
        gsb::ut_project_kernel<<<gsb::grid_for(n, gsb::kUtThreads), gsb::kUtThreads, 0, (cudaStream_t)stream>>>(
            B, C, N, means, quats, scales, opacities, viewmats, Ks, camera_model, radial_coeffs, tangential_coeffs,
            thin_prism_coeffs, image_width, image_height, eps2d, near_plane, far_plane, radius_clip, ut, radii, means2d,
            depths, conics, compensations, shutter, lens
        );
        return gsb::check_launch();
    });
}

extern "C" int gsb200_eval3d_fwd(
    int64_t B, int64_t C, int64_t N, int D, const float *means, const float *quats, const float *scales,
    const float *colors, const float *opacities, const float *backgrounds, const uint8_t *masks, const float *viewmats,
    const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
    const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
    const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, float *render_colors, float *render_alphas, int32_t *last_ids,
    void *stream
)
{
    if(n_isects < 0)
        return GSB200_E_INVALID;
    if(int rc = gsb::eval3d_checks(B, C, N, image_width, image_height, tile_size, tile_width, tile_height))
        return rc;
    if(int rc = gsb::camera_checks(camera_model, radial_coeffs, tangential_coeffs, thin_prism_coeffs, ftheta, viewmats_rs,
                                   rolling_shutter, image_width, image_height))
        return rc;
    if(B * C == 0 || image_width == 0 || image_height == 0)
        return GSB200_OK;
    if(!viewmats || !Ks || !offsets || !render_colors || !render_alphas || !last_ids)
        return GSB200_E_INVALID;
    if(n_isects > 0 && (!means || !quats || !scales || !colors || !opacities || !flatten_ids))
        return GSB200_E_INVALID;
    const gsb::EvalGeom geo = gsb::eval_geom(B, C, N, image_width, image_height, tile_width, tile_height, camera_model,
                                             viewmats, Ks, radial_coeffs, tangential_coeffs, thin_prism_coeffs);
    return gsb::eval3d_fwd(
        geo, geo.I * tile_width * tile_height, gsb::DensePixels{}, D, ftheta, viewmats_rs, rolling_shutter,
        (cudaStream_t)stream, means, quats, scales, colors, opacities, backgrounds, masks, offsets, flatten_ids, n_isects,
        render_colors, render_alphas, last_ids
    );
}

extern "C" int gsb200_eval3d_bwd(
    int64_t B, int64_t C, int64_t N, int D, const float *means, const float *quats, const float *scales,
    const float *colors, const float *opacities, const float *backgrounds, const uint8_t *masks, const float *viewmats,
    const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
    const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
    const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, const float *render_alphas, const int32_t *last_ids,
    const float *v_render_colors, const float *v_render_alphas, float *grad_records, float *v_colors, float *v_opacities,
    float *v_means, float *v_quats, float *v_scales, void *stream
)
{
    if(n_isects < 0)
        return GSB200_E_INVALID;
    if(int rc = gsb::eval3d_checks(B, C, N, image_width, image_height, tile_size, tile_width, tile_height))
        return rc;
    if(int rc = gsb::camera_checks(camera_model, radial_coeffs, tangential_coeffs, thin_prism_coeffs, ftheta, viewmats_rs,
                                   rolling_shutter, image_width, image_height))
        return rc;
    if(B * N == 0)
        return GSB200_OK;
    if(!quats || !scales || !grad_records || !v_means || !v_quats || !v_scales)
        return GSB200_E_INVALID;
    const bool composite = n_isects > 0 && B * C > 0 && image_width > 0 && image_height > 0;
    if(composite
       && (!means || !colors || !opacities || !viewmats || !Ks || !offsets || !flatten_ids || !render_alphas || !last_ids
           || !v_render_colors || !v_colors || !v_opacities))
        return GSB200_E_INVALID;
    const gsb::EvalGeom geo = gsb::eval_geom(B, C, N, image_width, image_height, tile_width, tile_height, camera_model,
                                             viewmats, Ks, radial_coeffs, tangential_coeffs, thin_prism_coeffs);
    return gsb::eval3d_bwd(
        geo, geo.I * tile_width * tile_height, gsb::DensePixels{}, composite, D, ftheta, viewmats_rs, rolling_shutter,
        (cudaStream_t)stream, B * N, means, quats, scales, gsb::EvalGradDst{v_colors, v_opacities, grad_records}, v_means,
        v_quats, v_scales, colors, opacities, backgrounds, masks, offsets, flatten_ids, n_isects, render_alphas, last_ids,
        v_render_colors, v_render_alphas
    );
}

// ---- sparse pixels (rasterize_to_pixels_eval3d_sparse): one CTA per active tile of the layout of gsb200_sparse_layout_*,
// outputs [P, *] in the original pixel order.  Every check of the dense entries and of the sparse layout runs before
// any launch.
extern "C" int gsb200_eval3d_sparse_fwd(
    int64_t B, int64_t C, int64_t N, int D, const float *means, const float *quats, const float *scales,
    const float *colors, const float *opacities, const float *backgrounds, const uint8_t *masks, const float *viewmats,
    const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
    const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
    int64_t n_active, const int32_t *active_tiles, const int32_t *tile_offsets, const int32_t *flatten_ids,
    int64_t n_isects, const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map,
    float *render_colors, float *render_alphas, int32_t *last_ids, void *stream
)
{
    if(n_isects < 0)
        return GSB200_E_INVALID;
    if(int rc = gsb::eval3d_checks(B, C, N, image_width, image_height, tile_size, tile_width, tile_height))
        return rc;
    if(int rc = gsb::camera_checks(camera_model, radial_coeffs, tangential_coeffs, thin_prism_coeffs, ftheta, viewmats_rs,
                                   rolling_shutter, image_width, image_height))
        return rc;
    if(int rc = gsb::sparse_args_ok(n_active, active_tiles, tile_offsets, tile_pixel_mask, tile_pixel_cumsum, pixel_map,
                                    image_width, image_height, tile_width, tile_height))
        return rc;
    if(n_active == 0)
        return GSB200_OK;
    if(B * C == 0 || !viewmats || !Ks || !render_colors || !render_alphas || !last_ids)
        return GSB200_E_INVALID;
    if(n_isects > 0 && (!means || !quats || !scales || !colors || !opacities || !flatten_ids))
        return GSB200_E_INVALID;
    const gsb::SparsePixels pm{active_tiles, tile_pixel_mask, tile_pixel_cumsum, pixel_map};
    return gsb::eval3d_fwd(
        gsb::eval_geom(B, C, N, image_width, image_height, tile_width, tile_height, camera_model, viewmats, Ks,
                       radial_coeffs, tangential_coeffs, thin_prism_coeffs),
        (uint32_t)n_active, pm, D, ftheta, viewmats_rs, rolling_shutter, (cudaStream_t)stream, means, quats, scales,
        colors, opacities, backgrounds, masks, tile_offsets, flatten_ids, n_isects, render_colors, render_alphas, last_ids
    );
}

extern "C" int gsb200_eval3d_sparse_bwd(
    int64_t B, int64_t C, int64_t N, int D, const float *means, const float *quats, const float *scales,
    const float *colors, const float *opacities, const float *backgrounds, const uint8_t *masks, const float *viewmats,
    const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
    const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
    int64_t n_active, const int32_t *active_tiles, const int32_t *tile_offsets, const int32_t *flatten_ids,
    int64_t n_isects, const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map,
    const float *render_alphas, const int32_t *last_ids, const float *v_render_colors, const float *v_render_alphas,
    float *grad_records, float *v_colors, float *v_opacities, float *v_means, float *v_quats, float *v_scales, void *stream
)
{
    if(n_isects < 0)
        return GSB200_E_INVALID;
    if(int rc = gsb::eval3d_checks(B, C, N, image_width, image_height, tile_size, tile_width, tile_height))
        return rc;
    if(int rc = gsb::camera_checks(camera_model, radial_coeffs, tangential_coeffs, thin_prism_coeffs, ftheta, viewmats_rs,
                                   rolling_shutter, image_width, image_height))
        return rc;
    if(int rc = gsb::sparse_args_ok(n_active, active_tiles, tile_offsets, tile_pixel_mask, tile_pixel_cumsum, pixel_map,
                                    image_width, image_height, tile_width, tile_height))
        return rc;
    if(B * N == 0)
        return GSB200_OK;
    if(!quats || !scales || !grad_records || !v_means || !v_quats || !v_scales)
        return GSB200_E_INVALID;
    // the finish kernel runs without the compositing: an unsupported channel count is refused before either
    if(gsb::with_channels(D, [](auto) { return GSB200_OK; }))
        return GSB200_E_UNSUPPORTED;
    const bool composite = n_isects > 0 && n_active > 0;
    if(composite
       && (B * C == 0 || !means || !colors || !opacities || !viewmats || !Ks || !flatten_ids || !render_alphas || !last_ids
           || !v_render_colors || !v_colors || !v_opacities))
        return GSB200_E_INVALID;
    const gsb::SparsePixels pm{active_tiles, tile_pixel_mask, tile_pixel_cumsum, pixel_map};
    return gsb::eval3d_bwd(
        gsb::eval_geom(B, C, N, image_width, image_height, tile_width, tile_height, camera_model, viewmats, Ks,
                       radial_coeffs, tangential_coeffs, thin_prism_coeffs),
        (uint32_t)n_active, pm, composite, D, ftheta, viewmats_rs, rolling_shutter, (cudaStream_t)stream, B * N, means,
        quats, scales, gsb::EvalGradDst{v_colors, v_opacities, grad_records}, v_means, v_quats, v_scales, colors, opacities,
        backgrounds, masks, tile_offsets, flatten_ids, n_isects, render_alphas, last_ids, v_render_colors, v_render_alphas
    );
}

// ---- rasterize_to_indices_in_range_eval3d: count pass (emit = 0) and emit pass (emit = 1) over one workspace
// (indices.cuh), after the size and camera checks of gsb200_eval3d_fwd
extern "C" int gsb200_eval3d_indices(
    int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales, const float *opacities,
    const float *viewmats, const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
    const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
    const float *transmittances, uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width,
    uint32_t tile_height, const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t range_start,
    int64_t range_end, int emit, void *workspace, size_t workspace_bytes, int64_t *total, int64_t *gaussian_ids,
    int64_t *pixel_ids, int64_t *image_ids, void *stream
)
{
    const gsb::Eval3dWalk walk{gsb::eval_geom(B, C, N, image_width, image_height, tile_width, tile_height, camera_model,
                                              viewmats, Ks, radial_coeffs, tangential_coeffs, thin_prism_coeffs),
                               means, quats, scales, opacities, ftheta, viewmats_rs, rolling_shutter};
    if(int rc = gsb::eval3d_query_checks(B, C, N, walk, tile_size, 0, nullptr, nullptr, nullptr, nullptr, nullptr))
        return rc;
    const cudaStream_t st = (cudaStream_t)stream;
    const bool inputs_ok  = means && quats && scales && opacities && viewmats && Ks && transmittances && offsets && flatten_ids;
    return gsb::run_index_pass(
        B * C, N, image_width, image_height, tile_size, tile_width, tile_height, n_isects, range_start, range_end, inputs_ok,
        emit, workspace, workspace_bytes, total, gaussian_ids, pixel_ids, image_ids, st,
        [&](unsigned n_tiles, int32_t b0, int32_t b1, auto sink) {
            return walk.with_model([&](const auto &model) {
                gsb::pair_walk_kernel<<<n_tiles, gsb::kIndexBatch, 0, st>>>(
                    model, transmittances, offsets, flatten_ids, n_isects, b0, b1, sink
                );
                return gsb::check_launch();
            });
        }
    );
}

// ---- 3DGUT per-pixel contributor queries over Eval3dWalk: the size, camera and (sparse) layout checks of
// gsb200_eval3d_sparse_fwd, then run_contrib's (indices.cuh), in the order and with the return codes of gsb200_contrib_*
extern "C" int gsb200_eval3d_contrib_max_samples(void)
{
    return gsb::Eval3dWalk::max_samples();
}

extern "C" int gsb200_eval3d_contrib_count(
    int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales, const float *opacities,
    const float *viewmats, const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
    const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
    const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
    const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int32_t *counts,
    float *alphas, void *stream
)
{
    const gsb::Eval3dWalk walk{gsb::eval_geom(B, C, N, image_width, image_height, tile_width, tile_height, camera_model,
                                              viewmats, Ks, radial_coeffs, tangential_coeffs, thin_prism_coeffs),
                               means, quats, scales, opacities, ftheta, viewmats_rs, rolling_shutter};
    if(int rc = gsb::eval3d_query_checks(B, C, N, walk, tile_size, n_active, active_tiles, offsets, tile_pixel_mask,
                                         tile_pixel_cumsum, pixel_map))
        return rc;
    return gsb::contrib_count(walk, GSB200_CONTRIB_ARGS(B * C), counts, alphas, (cudaStream_t)stream);
}

extern "C" int gsb200_eval3d_contrib_ids(
    int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales, const float *opacities,
    const float *viewmats, const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
    const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
    const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
    const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int max_samples,
    int32_t *ids, float *weights, void *stream
)
{
    const gsb::Eval3dWalk walk{gsb::eval_geom(B, C, N, image_width, image_height, tile_width, tile_height, camera_model,
                                              viewmats, Ks, radial_coeffs, tangential_coeffs, thin_prism_coeffs),
                               means, quats, scales, opacities, ftheta, viewmats_rs, rolling_shutter};
    if(int rc = gsb::eval3d_query_checks(B, C, N, walk, tile_size, n_active, active_tiles, offsets, tile_pixel_mask,
                                         tile_pixel_cumsum, pixel_map))
        return rc;
    return gsb::contrib_ids(walk, GSB200_CONTRIB_ARGS(B * C), max_samples, ids, weights, (cudaStream_t)stream);
}

extern "C" int gsb200_eval3d_contrib_top(
    int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales, const float *opacities,
    const float *viewmats, const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
    const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
    uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
    const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
    const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int num_samples,
    int32_t *ids, float *weights, void *stream
)
{
    const gsb::Eval3dWalk walk{gsb::eval_geom(B, C, N, image_width, image_height, tile_width, tile_height, camera_model,
                                              viewmats, Ks, radial_coeffs, tangential_coeffs, thin_prism_coeffs),
                               means, quats, scales, opacities, ftheta, viewmats_rs, rolling_shutter};
    if(int rc = gsb::eval3d_query_checks(B, C, N, walk, tile_size, n_active, active_tiles, offsets, tile_pixel_mask,
                                         tile_pixel_cumsum, pixel_map))
        return rc;
    return gsb::contrib_top(walk, GSB200_CONTRIB_ARGS(B * C), num_samples, ids, weights, (cudaStream_t)stream);
}
