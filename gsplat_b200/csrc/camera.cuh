// camera.cuh -- the distorted camera models of the 3DGUT operators: OpenCV pinhole (radial 6 as a rational k1..k6,
// tangential 2, thin prism 4) and OpenCV fisheye (odd polynomial theta + k1 theta^3 + .. + k4 theta^9), forward
// projection of a camera-frame point and unprojection of an image point to a unit camera ray.
//
// Reference semantics: include/Cameras.cuh (PerfectPinholeCameraModel, OpenCVPinholeCameraModel with 5 Newton
// undistortion steps, OpenCVFisheyeCameraModel with 20 Newton steps on the angle, the validity margin and the fisheye
// maximum angle).  A pinhole camera given no coefficient group at all is the perfect pinhole: no radial validity test
// and a closed-form ray.
#pragma once
#include <float.h>

#include "common.cuh"
#include "gaussmath.cuh"

namespace gsb
{
constexpr int kUtPinhole = 0;
constexpr int kUtFisheye = 2; // ids as in ops._camera_model_id

struct CamModel
{
    float fx, fy, cx, cy;
    float k[6], p[2], s[4]; // fisheye: k[0..3]
    uint32_t W, H;
    int kind;
    bool distorted;   // pinhole with any coefficient group given
    float max_angle;  // fisheye
    float inv_slope;  // fisheye: first guess of theta per unit normalised radius
};

// polynomials in theta^2 of the fisheye model: f(t) = t * P(t^2), f'(t) = Q(t^2)
__device__ __forceinline__ float fe_f(const float *k, float t)
{
    const float t2 = t * t;
    return t * (1.f + t2 * (k[0] + t2 * (k[1] + t2 * (k[2] + t2 * k[3]))));
}
__device__ __forceinline__ float fe_df(const float *k, float t)
{
    const float t2 = t * t;
    return 1.f + t2 * (3.f * k[0] + t2 * (5.f * k[1] + t2 * (7.f * k[2] + t2 * (9.f * k[3]))));
}

__device__ __forceinline__ CamModel load_cam_model(
    int kind, const float *K, const float *radial, const float *tangential, const float *thin, int64_t cam, uint32_t W,
    uint32_t H
)
{
    CamModel m;
    m.kind = kind;
    m.W = W, m.H = H;
    m.fx = K[cam * 9 + 0], m.fy = K[cam * 9 + 4], m.cx = K[cam * 9 + 2], m.cy = K[cam * 9 + 5];
#pragma unroll
    for(int i = 0; i < 6; ++i)
        m.k[i] = 0.f;
#pragma unroll
    for(int i = 0; i < 2; ++i)
        m.p[i] = 0.f;
#pragma unroll
    for(int i = 0; i < 4; ++i)
        m.s[i] = 0.f;
    m.max_angle = FLT_MAX, m.inv_slope = 0.f;
    m.distorted = false;
    if(kind == kUtPinhole)
    {
        m.distorted = radial || tangential || thin;
#pragma unroll
        for(int i = 0; i < 6; ++i)
            m.k[i] = radial ? radial[cam * 6 + i] : 0.f;
#pragma unroll
        for(int i = 0; i < 2; ++i)
            m.p[i] = tangential ? tangential[cam * 2 + i] : 0.f;
#pragma unroll
        for(int i = 0; i < 4; ++i)
            m.s[i] = thin ? thin[cam * 4 + i] : 0.f;
        return m;
    }
#pragma unroll
    for(int i = 0; i < 4; ++i)
        m.k[i] = radial ? radial[cam * 4 + i] : 0.f;
    // The model is trusted while the image radius grows with the angle: up to the first zero of f' or, past the
    // image's far corner, the angle of that corner.  f' is sampled on [0, bound] and its first sign change bisected.
    const float mdx = fmaxf((float)W - m.cx, m.cx), mdy = fmaxf((float)H - m.cy, m.cy);
    const float max_r = sqrtf(mdx * mdx + mdy * mdy);
    const float bound = fmaxf(max_r / m.fx, max_r / m.fy);
    m.max_angle = bound;
    constexpr int kSamples = 64;
    float lo = 0.f;
    for(int i = 1; i <= kSamples; ++i)
    {
        const float hi = bound * (float)i / (float)kSamples;
        if(fe_df(m.k, hi) <= 0.f)
        {
            float a = lo, b = hi;
            for(int it = 0; it < 32; ++it)
            {
                const float mid = 0.5f * (a + b);
                if(fe_df(m.k, mid) > 0.f)
                    a = mid;
                else
                    b = mid;
            }
            m.max_angle = a;
            break;
        }
        lo = hi;
    }
    const float max_nd = fmaxf((float)W / 2.f / m.fx, (float)H / 2.f / m.fy);
    m.inv_slope = m.max_angle / max_nd;
    return m;
}

template<class Model>
__device__ __forceinline__ bool in_margin(const Model &m, float u, float v, float margin)
{
    const float mx = (float)m.W * margin, my = (float)m.H * margin;
    return -mx <= u && u < (float)m.W + mx && -my <= v && v < (float)m.H + my;
}

// OpenCV pinhole distortion at normalised (x, y): radial factor icD and the tangential + thin-prism offset
__device__ __forceinline__ float pinhole_distort(const CamModel &m, float x, float y, float &dx, float &dy)
{
    const float x2 = x * x, y2 = y * y, r2 = x2 + y2;
    const float num = 1.f + r2 * (m.k[0] + r2 * (m.k[1] + r2 * m.k[2]));
    const float den = 1.f + r2 * (m.k[3] + r2 * (m.k[4] + r2 * m.k[5]));
    const float a1 = 2.f * x * y;
    dx = m.p[0] * a1 + m.p[1] * (r2 + 2.f * x2) + r2 * (m.s[0] + r2 * m.s[1]);
    dy = m.p[0] * (r2 + 2.f * y2) + m.p[1] * a1 + r2 * (m.s[2] + r2 * m.s[3]);
    return fabsf(den) > 1e-8f ? num / den : 0.f;
}

// The distortion map D(x, y) = icD (x, y) + offset and its Jacobian J (row-major d(Dx, Dy)/d(x, y)).  false: icD <= 0,
// where the map folds the image over and has no inverse.
__device__ __forceinline__ bool pinhole_distort_jacobian(const CamModel &m, float x, float y, float *D, float *J)
{
    const float r2  = x * x + y * y;
    const float num = 1.f + r2 * (m.k[0] + r2 * (m.k[1] + r2 * m.k[2]));
    const float den = 1.f + r2 * (m.k[3] + r2 * (m.k[4] + r2 * m.k[5]));
    const float icd = num / den;
    if(!(icd > 0.f))
        return false;
    // d icD / d r2, and the thin-prism slopes d(s0 r2 + s1 r2^2) / d r2
    const float dnum = m.k[0] + r2 * (2.f * m.k[1] + 3.f * r2 * m.k[2]);
    const float dden = m.k[3] + r2 * (2.f * m.k[4] + 3.f * r2 * m.k[5]);
    const float dicd = (dnum - icd * dden) / den;
    const float gx = m.s[0] + 2.f * m.s[1] * r2, gy = m.s[2] + 2.f * m.s[3] * r2;
    const float p0 = m.p[0], p1 = m.p[1];
    D[0] = icd * x + p0 * 2.f * x * y + p1 * (r2 + 2.f * x * x) + r2 * (m.s[0] + r2 * m.s[1]);
    D[1] = icd * y + p0 * (r2 + 2.f * y * y) + p1 * 2.f * x * y + r2 * (m.s[2] + r2 * m.s[3]);
    J[0] = icd + 2.f * x * x * dicd + 2.f * p0 * y + 6.f * p1 * x + 2.f * x * gx;
    J[1] = 2.f * x * y * dicd + 2.f * p0 * x + 2.f * p1 * y + 2.f * y * gx;
    J[2] = 2.f * x * y * dicd + 2.f * p0 * x + 2.f * p1 * y + 2.f * x * gy;
    J[3] = icd + 2.f * y * y * dicd + 6.f * p0 * y + 2.f * p1 * x + 2.f * y * gy;
    return true;
}

// Camera-frame point -> image point.  Returns validity; (u, v) is set also for an invalid point, as the unscented
// transform averages every sigma point: (0, 0) behind the camera.
__device__ __forceinline__ bool cam_project(const CamModel &m, const float *pc, float margin, float &u, float &v)
{
    u = 0.f, v = 0.f;
    if(pc[2] <= 0.f)
        return false;
    if(m.kind == kUtPinhole)
    {
        const float x = pc[0] / pc[2], y = pc[1] / pc[2];
        if(!m.distorted)
        {
            u = x * m.fx + m.cx, v = y * m.fy + m.cy;
            return in_margin(m, u, v, margin);
        }
        float dx, dy;
        const float icD = pinhole_distort(m, x, y, dx, dy);
        u = (icD * x + dx) * m.fx + m.cx;
        v = (icD * y + dy) * m.fy + m.cy;
        return icD > 0.8f && in_margin(m, u, v, margin);
    }
    const float ax = fabsf(pc[0]), ay = fabsf(pc[1]);
    const float lo = fminf(ax, ay), hi = fmaxf(ax, ay);
    float rxy = 0.f;
    if(hi > 0.f)
    {
        const float q = lo / hi;
        rxy = hi * sqrtf(1.f + q * q);
    }
    if(rxy <= 0.f)
        rxy = FLT_EPSILON;
    const float th_full = atan2f(rxy, pc[2]);
    const float th = th_full < m.max_angle ? th_full : m.max_angle;
    const float delta = fe_f(m.k, th) / rxy;
    if(delta <= 0.f)
        return false;
    u = m.fx * delta * pc[0] + m.cx;
    v = m.fy * delta * pc[1] + m.cy;
    return in_margin(m, u, v, margin) && th_full < m.max_angle;
}

// Image point -> unit camera ray.  false: the model cannot invert at this point (the Newton iteration did not converge
// or left the valid range); such a pixel composites nothing.
__device__ __forceinline__ bool cam_unproject(const CamModel &m, float u, float v, float *d)
{
    const float x0 = (u - m.cx) / m.fx, y0 = (v - m.cy) / m.fy;
    if(m.kind == kUtPinhole)
    {
        float x = x0, y = y0;
        bool ok = !m.distorted;
        // Newton on D(x, y) = (x0, y0), D the distortion map, from the distorted point itself
        for(int it = 0; it < 5 && m.distorted; ++it)
        {
            float D[2], J[4];
            if(!pinhole_distort_jacobian(m, x, y, D, J))
                break;
            const float det = J[0] * J[3] - J[1] * J[2];
            if(fabsf(det) < 1e-6f)
                break;
            const float ex = x0 - D[0], ey = y0 - D[1];
            const float sx = (J[3] * ex - J[1] * ey) / det;
            const float sy = (J[0] * ey - J[2] * ex) / det;
            x += sx, y += sy;
            if(fabsf(sx) < 1e-6f && fabsf(sy) < 1e-6f)
            {
                ok = true;
                break;
            }
        }
        const float inv = 1.f / sqrtf(x * x + y * y + 1.f);
        d[0] = x * inv, d[1] = y * inv, d[2] = inv;
        return ok;
    }
    const float delta = sqrtf(x0 * x0 + y0 * y0);
    float t = m.inv_slope * delta;
    bool conv = false;
    for(int it = 0; it < 20; ++it)
    {
        const float dx = (fe_f(m.k, t) - delta) / fe_df(m.k, t);
        t -= dx;
        if(fabsf(dx) < 1e-6f)
        {
            conv = true;
            break;
        }
    }
    d[0] = 0.f, d[1] = 0.f, d[2] = 1.f;
    if(t < 0.f || t >= m.max_angle || !conv)
        return false;
    if(delta >= 1e-6f)
    {
        const float sc = sinf(t) / delta;
        d[0] = sc * x0, d[1] = sc * y0, d[2] = cosf(t);
    }
    return true;
}

// ------------------------------------------------------------------ FTheta
// Reference semantics: include/Cameras.cuh (FThetaCameraModel with 3 Newton steps).  The image radius delta of a ray at
// angle theta from the optical axis is given by two polynomials of degree 5 calibrated together: the forward one
// (angle to pixel distance) and the backward one (pixel distance to angle).  The reference polynomial is evaluated
// directly, the other direction inverts it by Newton steps that start from the other polynomial.  A linear map
// [[c, d], [e, 1]] takes the radial offset to the image, about the principal point Ks (cx, cy) + 0.5: FTheta's image
// origin is the centre of the first pixel.  The parameters are shared by every camera of a call.
constexpr int kUtFTheta           = 3;
constexpr int kFThetaPixelToAngle = 0; // reference_poly: the backward polynomial is the reference
constexpr int kFThetaAngleToPixel = 1; // the forward one is
constexpr int kFThetaNewtonSteps  = 3;

struct FThetaModel
{
    float bw[6], fw[6]; // backward (pixel distance -> angle), forward (angle -> pixel distance)
    float dref[5];      // derivative of the reference polynomial
    float max_angle, c, d, e, cx, cy;
    uint32_t W, H;
    int reference_poly;
};

__device__ __forceinline__ float poly6(const float *k, float x)
{
    return k[0] + x * (k[1] + x * (k[2] + x * (k[3] + x * (k[4] + x * k[5]))));
}
__device__ __forceinline__ float poly5(const float *k, float x)
{
    return k[0] + x * (k[1] + x * (k[2] + x * (k[3] + x * k[4])));
}

// x with ref(x) = y: kFThetaNewtonSteps Newton steps on the reference polynomial from approx(y), stopping early once a
// step is below 1e-6 (converged).
__device__ __forceinline__ float ftheta_newton(const float *ref, const float *dref, const float *approx, float y, bool &converged)
{
    float x   = poly6(approx, y);
    converged = false;
#pragma unroll
    for(int it = 0; it < kFThetaNewtonSteps; ++it)
    {
        const float dx = (poly6(ref, x) - y) / poly5(dref, x);
        x -= dx;
        if(fabsf(dx) < 1e-6f)
        {
            converged = true;
            break;
        }
    }
    return x;
}

// Camera-frame point -> image point.  No z <= 0 guard: a calibration with max_angle > pi/2 images points behind the
// camera plane.  Beyond max_angle the angle is clamped and the point is invalid; its image point is still set.  The
// forward direction ignores the Newton convergence flag: float32 rounding keeps the last step near 1e-5 pixel for
// typical calibrations, while delta is accurate.
__device__ __forceinline__ bool cam_project(const FThetaModel &m, const float *pc, float margin, float &u, float &v)
{
    const float ax = fabsf(pc[0]), ay = fabsf(pc[1]);
    const float lo = fminf(ax, ay), hi = fmaxf(ax, ay);
    float rxy = 0.f;
    if(hi > 0.f)
    {
        const float q = lo / hi;
        rxy = hi * sqrtf(1.f + q * q);
    }
    if(rxy <= 0.f)
        rxy = FLT_EPSILON;
    const float th_full = atan2f(rxy, pc[2]);
    const float th      = th_full < m.max_angle ? th_full : m.max_angle;
    bool converged;
    const float delta = m.reference_poly == kFThetaAngleToPixel ? poly6(m.fw, th) : ftheta_newton(m.bw, m.dref, m.fw, th, converged);
    const float ix = delta * (pc[0] / rxy), iy = delta * (pc[1] / rxy);
    u = m.c * ix + m.d * iy + m.cx;
    v = m.e * ix + iy + m.cy;
    return in_margin(m, u, v, margin) && th_full < m.max_angle;
}

// Image point -> unit camera ray.  false: the linear map is singular, or the Newton inversion of the forward polynomial
// did not converge; such a pixel composites nothing.
__device__ __forceinline__ bool cam_unproject(const FThetaModel &m, float u, float v, float *dir)
{
    dir[0] = 0.f, dir[1] = 0.f, dir[2] = 1.f;
    const float x = u - m.cx, y = v - m.cy;
    const float det = m.c - m.e * m.d;
    if(fabsf(det) < 1e-8f)
        return false;
    const float ux = (x - m.d * y) / det, uy = (-m.e * x + m.c * y) / det;
    const float delta = sqrtf(ux * ux + uy * uy);
    float theta;
    if(m.reference_poly == kFThetaPixelToAngle)
        theta = poly6(m.bw, delta);
    else
    {
        bool converged;
        theta = ftheta_newton(m.fw, m.dref, m.bw, delta, converged);
        if(!converged)
            return false;
    }
    if(delta >= 1e-6f)
    {
        const float sc = sinf(theta) / delta;
        dir[0] = sc * ux, dir[1] = sc * uy, dir[2] = cosf(theta);
    }
    return true;
}

// ------------------------------------------------------------------ lens policies
// The kernels' camera model is a compile-time policy: CamLens is the runtime OpenCV pinhole / fisheye CamModel (loaded
// from the per-camera coefficient arrays), FThetaLens carries the shared FTheta parameters by value.
struct CamLens
{
    static constexpr bool kFTheta = false;
    __device__ __forceinline__ CamModel model(
        int kind, const float *K, const float *radial, const float *tangential, const float *thin, int64_t cam, uint32_t W,
        uint32_t H
    ) const
    {
        return load_cam_model(kind, K, radial, tangential, thin, cam, W, H);
    }
};
struct FThetaLens
{
    static constexpr bool kFTheta = true;
    gsb200_ftheta_params p;
    int global_z_order; // 0: the projection culls and orders on the distance |mean_c|, not on z
    __device__ __forceinline__ FThetaModel model(
        int, const float *K, const float *, const float *, const float *, int64_t cam, uint32_t W, uint32_t H
    ) const
    {
        FThetaModel m;
#pragma unroll
        for(int i = 0; i < 6; ++i)
            m.bw[i] = p.pixeldist_to_angle_poly[i], m.fw[i] = p.angle_to_pixeldist_poly[i];
        const bool bw_ref = p.reference_poly == kFThetaPixelToAngle;
#pragma unroll
        for(int i = 0; i < 5; ++i)
            m.dref[i] = (float)(i + 1) * (bw_ref ? m.bw[i + 1] : m.fw[i + 1]);
        m.max_angle = p.max_angle;
        m.c = p.linear_cde[0], m.d = p.linear_cde[1], m.e = p.linear_cde[2];
        m.cx = K[cam * 9 + 2] + 0.5f, m.cy = K[cam * 9 + 5] + 0.5f;
        m.W = W, m.H = H;
        m.reference_poly = p.reference_poly;
        return m;
    }
};

// ------------------------------------------------------------------ rolling shutter
// Reference semantics: include/Cameras.cuh (RollingShutterParameters, interpolate_shutter_pose,
// shutter_relative_frame_time, world_point_to_image_point_shutter_pose).  Each image row or column is exposed at its
// own pose, interpolated between the start pose (viewmats) and the end pose (viewmats_rs) at the frame time of that row
// or column.  Ids as the reference's RollingShutterType.
constexpr int kShutterTopToBottom = 0;
constexpr int kShutterLeftToRight = 1;
constexpr int kShutterBottomToTop = 2;
constexpr int kShutterRightToLeft = 3;
constexpr int kShutterGlobal      = 4;
constexpr int kShutterIterations  = 10;

// Kernel policies: the global shutter takes the pose of viewmats; the rolling one interpolates each camera's two poses.
struct GlobalShutter
{
    static constexpr bool kRolling = false;
};
struct RollingShutter
{
    static constexpr bool kRolling = true;
    const float *viewmats_rs;
    int type;
};

// The two poses of one camera, rotations as quaternions (w, x, y, z) with q1 on q0's short arc, and the slerp's
// constant angle between them (0: near-parallel, interpolated component-wise).
struct RsPoses
{
    float q0[4], q1[4], t0[3], t1[3], angle, sin_angle;
};

// Unit quaternion of the rotation block of a row-major 4x4 pose, from its largest component (as glm::quat_cast).
__device__ __forceinline__ void quat_from_pose(const float *vm, float *q)
{
    const float r00 = vm[0], r01 = vm[1], r02 = vm[2];
    const float r10 = vm[4], r11 = vm[5], r12 = vm[6];
    const float r20 = vm[8], r21 = vm[9], r22 = vm[10];
    const float f[4] = {r00 + r11 + r22, r00 - r11 - r22, r11 - r00 - r22, r22 - r00 - r11}; // 4 c^2 - 1, c = w, x, y, z
    int big = 0;
#pragma unroll
    for(int k = 1; k < 4; ++k)
        big = f[k] > f[big] ? k : big;
    const float v    = sqrtf(f[big] + 1.f) * 0.5f;
    const float mult = 0.25f / v;
    const float a = (r21 - r12) * mult, b = (r02 - r20) * mult, c = (r10 - r01) * mult; // w x, w y, w z
    const float d = (r10 + r01) * mult, e = (r02 + r20) * mult, g = (r21 + r12) * mult; // x y, x z, y z
    switch(big)
    {
    case 0: q[0] = v, q[1] = a, q[2] = b, q[3] = c; break;
    case 1: q[0] = a, q[1] = v, q[2] = d, q[3] = e; break;
    case 2: q[0] = b, q[1] = d, q[2] = v, q[3] = g; break;
    default: q[0] = c, q[1] = e, q[2] = g, q[3] = v; break;
    }
}

__device__ __forceinline__ RsPoses load_rs_poses(const float *vm0, const float *vm1)
{
    RsPoses P;
    quat_from_pose(vm0, P.q0);
    quat_from_pose(vm1, P.q1);
    P.t0[0] = vm0[3], P.t0[1] = vm0[7], P.t0[2] = vm0[11];
    P.t1[0] = vm1[3], P.t1[1] = vm1[7], P.t1[2] = vm1[11];
    float c = P.q0[0] * P.q1[0] + P.q0[1] * P.q1[1] + P.q0[2] * P.q1[2] + P.q0[3] * P.q1[3];
    if(c < 0.f)
    {
#pragma unroll
        for(int k = 0; k < 4; ++k)
            P.q1[k] = -P.q1[k];
        c = -c;
    }
    P.angle = 0.f, P.sin_angle = 0.f;
    if(!(c > 1.f - FLT_EPSILON))
    {
        P.angle     = acosf(c);
        P.sin_angle = sinf(P.angle);
    }
    return P;
}

// The pose at relative frame time a (not clamped: points in the margin have times outside [0, 1]): translation
// (1 - a) t0 + a t1, rotation the normalised slerp of the two quaternions.
__device__ __forceinline__ Cam pose_at(const RsPoses &P, float a)
{
    float q[4];
    if(P.angle == 0.f)
    {
#pragma unroll
        for(int k = 0; k < 4; ++k)
            q[k] = P.q0[k] * (1.f - a) + P.q1[k] * a;
    }
    else
    {
        const float s0 = sinf((1.f - a) * P.angle), s1 = sinf(a * P.angle);
#pragma unroll
        for(int k = 0; k < 4; ++k)
            q[k] = (s0 * P.q0[k] + s1 * P.q1[k]) / P.sin_angle;
    }
    Cam c;
    c.R = quat_to_rotmat(q); // normalises q
#pragma unroll
    for(int k = 0; k < 3; ++k)
        c.t[k] = (1.f - a) * P.t0[k] + a * P.t1[k];
    c.fx = c.fy = c.cx = c.cy = 0.f;
    return c;
}

// Relative frame time of image point (u, v): the exposure time of its row or column, 0 at the first, 1 at the last.
// The caller guarantees H > 1 (rows) or W > 1 (columns).
__device__ __forceinline__ float shutter_time(int type, uint32_t W, uint32_t H, float u, float v)
{
    switch(type)
    {
    case kShutterTopToBottom: return floorf(v) / (float)(H - 1);
    case kShutterLeftToRight: return floorf(u) / (float)(W - 1);
    case kShutterBottomToTop: return ((float)H - ceilf(v)) / (float)(H - 1);
    default: return ((float)W - ceilf(u)) / (float)(W - 1);
    }
}

template<class Model>
__device__ __forceinline__ bool cam_project_at(const Model &m, const Cam &pose, const float *x, float margin, float &u, float &v)
{
    float xc[3];
#pragma unroll
    for(int i = 0; i < 3; ++i)
        xc[i] = pose.R.m[i * 3 + 0] * x[0] + pose.R.m[i * 3 + 1] * x[1] + pose.R.m[i * 3 + 2] * x[2] + pose.t[i];
    return cam_project(m, xc, margin, u, v);
}

// World point -> image point through a rolling shutter: start from the start pose's projection if it is valid, else
// the end pose's (neither valid: the point is invalid, at the end pose's image point), then re-project at the frame
// time of the current point until that time repeats, at most kShutterIterations times.  The point and its validity are
// those of the last projection.
template<class Model>
__device__ __forceinline__ bool cam_project_rs(
    const Model &m, const RsPoses &P, int type, const float *x, float margin, float &u, float &v
)
{
    float u0, v0, u1, v1;
    const bool ok0 = cam_project_at(m, pose_at(P, 0.f), x, margin, u0, v0);
    const bool ok1 = cam_project_at(m, pose_at(P, 1.f), x, margin, u1, v1);
    u = ok0 ? u0 : u1, v = ok0 ? v0 : v1;
    if(!ok0 && !ok1)
        return false;
    bool ok = true;
    float prev = -FLT_MAX;
    for(int it = 0; it < kShutterIterations; ++it)
    {
        const float a = shutter_time(type, m.W, m.H, u, v);
        if(a == prev)
            break;
        prev = a;
        ok   = cam_project_at(m, pose_at(P, a), x, margin, u, v);
    }
    return ok;
}
} // namespace gsb
