/*
 * gso_impl.h -- body of the CPU oracle, instantiated twice by gs_oracle.c
 * (REAL=float -> *_f32, REAL=double -> *_f64).
 *
 * TEST INFRASTRUCTURE ONLY.  This is a plain-C restatement of the reference
 * (nerfstudio-project/gsplat v1.6.0) algorithms for the rasterization() hot
 * path.  Nothing under gsplat_b200/ may import, link or call it; only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
 *
 * Every function cites the reference file:line it follows (paths relative to
 * /root/reference/gsplat/cuda).  Layouts are the reference's: row-major
 * tensors, quaternions wxyz, conics (a,b,c) = upper triangle of Sigma2d^-1.
 */

#define CAT_(a, b) a##b
#define CAT(a, b) CAT_(a, b)
#define FN(name) CAT(name, SUF)

/* -------- small dense helpers (row-major 3x3) -------- */

/* float -> int32 with the GPU's conversion (cvt.rzi.s32: truncate toward zero, saturate at the int32 range, NaN -> 0).
 * A plain C cast is undefined outside the int32 range (x86 returns INT32_MIN, which would turn a huge radius into a
 * culled row and a far tile bound into the wrong end of the grid). */
static inline int32_t FN(f2i)(REAL v)
{
    if(v != v)
        return 0;
    if(v >= (REAL)2147483647.0)
        return INT32_MAX;
    if(v <= (REAL)-2147483648.0)
        return INT32_MIN;
    return (int32_t)v;
}

static inline void FN(mat3_mul)(const REAL *A, const REAL *B, REAL *C_)
{
    for(int i = 0; i < 3; ++i)
        for(int j = 0; j < 3; ++j)
            C_[i * 3 + j] = A[i * 3 + 0] * B[0 * 3 + j] + A[i * 3 + 1] * B[1 * 3 + j] + A[i * 3 + 2] * B[2 * 3 + j];
}

static inline void FN(mat3_mul_bt)(const REAL *A, const REAL *B, REAL *C_)
{ /* C = A * B^T */
    for(int i = 0; i < 3; ++i)
        for(int j = 0; j < 3; ++j)
            C_[i * 3 + j] = A[i * 3 + 0] * B[j * 3 + 0] + A[i * 3 + 1] * B[j * 3 + 1] + A[i * 3 + 2] * B[j * 3 + 2];
}

static inline void FN(mat3_mul_at)(const REAL *A, const REAL *B, REAL *C_)
{ /* C = A^T * B */
    for(int i = 0; i < 3; ++i)
        for(int j = 0; j < 3; ++j)
            C_[i * 3 + j] = A[0 * 3 + i] * B[0 * 3 + j] + A[1 * 3 + i] * B[1 * 3 + j] + A[2 * 3 + i] * B[2 * 3 + j];
}

/* natural log built from exactly-rounded float ops only, so that the CUDA
 * kernels (compiled with -fmad=false) reproduce it bit for bit.  Used where
 * the reference calls __logf(opacity / ALPHA_THRESHOLD)
 * (csrc/ProjectionEWA3DGSFused.cu:180, csrc/IntersectTile.cu:302). */
static inline REAL FN(gs_log)(REAL x)
{
    int e;
    REAL m = R_FREXP(x, &e); /* exact: m in [0.5,1) */
    if(m < (REAL)0.70710678118654752)
    {
        m = m * (REAL)2;
        e -= 1;
    }
    REAL f = m - (REAL)1;
    REAL s = f / ((REAL)2 + f);
    REAL z = s * s;
    REAL p = z
           * ((REAL)0.33333333333333333
              + z
                    * ((REAL)0.2
                       + z * ((REAL)0.14285714285714285 + z * ((REAL)0.11111111111111111 + z * (REAL)0.09090909090909091))));
    REAL two_s = (REAL)2 * s;
    return (REAL)e * (REAL)0.69314718055994531 + (two_s + two_s * p);
}

/* quaternion (wxyz, un-normalised) -> rotation matrix, row-major.
 * Reference: include/Utils.cuh:228-251 (quat_to_rotmat). */
static inline void FN(quat_to_rotmat)(const REAL *q, REAL *R, REAL *inv_norm_out)
{
    REAL w = q[0], x = q[1], y = q[2], z = q[3];
    REAL inv_norm = (REAL)1 / R_SQRT(x * x + y * y + z * z + w * w);
    x *= inv_norm;
    y *= inv_norm;
    z *= inv_norm;
    w *= inv_norm;
    REAL x2 = x * x, y2 = y * y, z2 = z * z;
    REAL xy = x * y, xz = x * z, yz = y * z;
    REAL wx = w * x, wy = w * y, wz = w * z;
    R[0] = (REAL)1 - (REAL)2 * (y2 + z2);
    R[1] = (REAL)2 * (xy - wz);
    R[2] = (REAL)2 * (xz + wy);
    R[3] = (REAL)2 * (xy + wz);
    R[4] = (REAL)1 - (REAL)2 * (x2 + z2);
    R[5] = (REAL)2 * (yz - wx);
    R[6] = (REAL)2 * (xz - wy);
    R[7] = (REAL)2 * (yz + wx);
    R[8] = (REAL)1 - (REAL)2 * (x2 + y2);
    if(inv_norm_out)
        *inv_norm_out = inv_norm;
}

/* VJP of quat_to_rotmat.  G = dL/dR row-major.  Reference: Utils.cuh:253-283. */
static inline void FN(quat_to_rotmat_vjp)(const REAL *q, const REAL *G, REAL *v_q)
{
    REAL w = q[0], x = q[1], y = q[2], z = q[3];
    REAL inv_norm = (REAL)1 / R_SQRT(x * x + y * y + z * z + w * w);
    x *= inv_norm;
    y *= inv_norm;
    z *= inv_norm;
    w *= inv_norm;
    /* G[r*3+c] */
    REAL vw = (REAL)2 * (x * (G[7] - G[5]) + y * (G[2] - G[6]) + z * (G[3] - G[1]));
    REAL vx = (REAL)2 * ((REAL)-2 * x * (G[4] + G[8]) + y * (G[3] + G[1]) + z * (G[6] + G[2]) + w * (G[7] - G[5]));
    REAL vy = (REAL)2 * (x * (G[3] + G[1]) - (REAL)2 * y * (G[0] + G[8]) + z * (G[7] + G[5]) + w * (G[2] - G[6]));
    REAL vz = (REAL)2 * (x * (G[6] + G[2]) + y * (G[7] + G[5]) - (REAL)2 * z * (G[0] + G[4]) + w * (G[3] - G[1]));
    REAL dot = vw * w + vx * x + vy * y + vz * z;
    v_q[0] += (vw - dot * w) * inv_norm;
    v_q[1] += (vx - dot * x) * inv_norm;
    v_q[2] += (vy - dot * y) * inv_norm;
    v_q[3] += (vz - dot * z) * inv_norm;
}

/* covar = (R S)(R S)^T and/or preci = (R S^-1)(R S^-1)^T.
 * Reference: Utils.cuh:285-311 (quat_scale_to_covar_preci). */
static inline void FN(quat_scale_to_covar_preci_one)(const REAL *q, const REAL *s, REAL *covar, REAL *preci)
{
    REAL R[9];
    FN(quat_to_rotmat)(q, R, NULL);
    if(covar)
    {
        REAL M[9];
        for(int i = 0; i < 3; ++i)
            for(int j = 0; j < 3; ++j)
                M[i * 3 + j] = R[i * 3 + j] * s[j];
        FN(mat3_mul_bt)(M, M, covar);
    }
    if(preci)
    {
        REAL M[9];
        for(int i = 0; i < 3; ++i)
            for(int j = 0; j < 3; ++j)
                M[i * 3 + j] = R[i * 3 + j] * ((REAL)1 / s[j]);
        FN(mat3_mul_bt)(M, M, preci);
    }
}

/* Reference: Utils.cuh:313-347 (quat_scale_to_covar_vjp). v_covar row-major (full 3x3). */
static inline void FN(quat_scale_to_covar_vjp)(const REAL *q, const REAL *s, const REAL *v_covar, REAL *v_q, REAL *v_s)
{
    REAL R[9], M[9], Gs[9], v_M[9], v_R[9];
    FN(quat_to_rotmat)(q, R, NULL);
    for(int i = 0; i < 3; ++i)
        for(int j = 0; j < 3; ++j)
        {
            M[i * 3 + j]  = R[i * 3 + j] * s[j];
            Gs[i * 3 + j] = v_covar[i * 3 + j] + v_covar[j * 3 + i];
        }
    FN(mat3_mul)(Gs, M, v_M);
    for(int i = 0; i < 3; ++i)
        for(int j = 0; j < 3; ++j)
            v_R[i * 3 + j] = v_M[i * 3 + j] * s[j];
    FN(quat_to_rotmat_vjp)(q, v_R, v_q);
    for(int j = 0; j < 3; ++j)
        v_s[j] += R[0 * 3 + j] * v_M[0 * 3 + j] + R[1 * 3 + j] * v_M[1 * 3 + j] + R[2 * 3 + j] * v_M[2 * 3 + j];
}

/* Reference: Utils.cuh:349-385 (quat_scale_to_preci_vjp). */
static inline void FN(quat_scale_to_preci_vjp)(const REAL *q, const REAL *s, const REAL *v_preci, REAL *v_q, REAL *v_s)
{
    REAL R[9], M[9], Gs[9], v_M[9], v_R[9], is[3];
    FN(quat_to_rotmat)(q, R, NULL);
    for(int j = 0; j < 3; ++j)
        is[j] = (REAL)1 / s[j];
    for(int i = 0; i < 3; ++i)
        for(int j = 0; j < 3; ++j)
        {
            M[i * 3 + j]  = R[i * 3 + j] * is[j];
            Gs[i * 3 + j] = v_preci[i * 3 + j] + v_preci[j * 3 + i];
        }
    FN(mat3_mul)(Gs, M, v_M);
    for(int i = 0; i < 3; ++i)
        for(int j = 0; j < 3; ++j)
            v_R[i * 3 + j] = v_M[i * 3 + j] * is[j];
    FN(quat_to_rotmat_vjp)(q, v_R, v_q);
    for(int j = 0; j < 3; ++j)
        v_s[j] += -is[j] * is[j]
                * (R[0 * 3 + j] * v_M[0 * 3 + j] + R[1 * 3 + j] * v_M[1 * 3 + j] + R[2 * 3 + j] * v_M[2 * 3 + j]);
}

/* ---------------------------------------------------------------------- */
/* quat_scale_to_covar_preci op.  Reference: csrc/QuatScaleToCovarCUDA.cu:37-110 (fwd),
 * :211-300 (bwd).  covars/precis: [N,3,3] or [N,6] (triu); either may be NULL. */
int FN(gso_quat_scale_to_covar_preci)(int64_t N, const REAL *quats, const REAL *scales, int triu, REAL *covars, REAL *precis)
{
    for(int64_t n = 0; n < N; ++n)
    {
        REAL cv[9], pr[9];
        FN(quat_scale_to_covar_preci_one)(quats + n * 4, scales + n * 3, covars ? cv : NULL, precis ? pr : NULL);
        const int tri[6] = {0, 1, 2, 4, 5, 8};
        if(covars)
        {
            if(triu)
                for(int k = 0; k < 6; ++k)
                    covars[n * 6 + k] = cv[tri[k]];
            else
                for(int k = 0; k < 9; ++k)
                    covars[n * 9 + k] = cv[k];
        }
        if(precis)
        {
            if(triu)
                for(int k = 0; k < 6; ++k)
                    precis[n * 6 + k] = pr[tri[k]];
            else
                for(int k = 0; k < 9; ++k)
                    precis[n * 9 + k] = pr[k];
        }
    }
    return 0;
}

static inline void FN(expand_sym_grad)(const REAL *v, int triu, REAL *G)
{
    if(triu)
    { /* off-diagonals appear once in the triu vector: split evenly */
        G[0] = v[0];
        G[1] = G[3] = v[1] * (REAL)0.5;
        G[2] = G[6] = v[2] * (REAL)0.5;
        G[4] = v[3];
        G[5] = G[7] = v[4] * (REAL)0.5;
        G[8] = v[5];
    }
    else
        for(int k = 0; k < 9; ++k)
            G[k] = v[k];
}

int FN(gso_quat_scale_to_covar_preci_bwd)(
    int64_t N, const REAL *quats, const REAL *scales, int triu, const REAL *v_covars, const REAL *v_precis, REAL *v_quats,
    REAL *v_scales
)
{
    const int stride = triu ? 6 : 9;
    for(int64_t n = 0; n < N; ++n)
    {
        REAL vq[4] = {0, 0, 0, 0}, vs[3] = {0, 0, 0}, G[9];
        if(v_covars)
        {
            FN(expand_sym_grad)(v_covars + n * stride, triu, G);
            FN(quat_scale_to_covar_vjp)(quats + n * 4, scales + n * 3, G, vq, vs);
        }
        if(v_precis)
        {
            FN(expand_sym_grad)(v_precis + n * stride, triu, G);
            FN(quat_scale_to_preci_vjp)(quats + n * 4, scales + n * 3, G, vq, vs);
        }
        for(int k = 0; k < 4; ++k)
            v_quats[n * 4 + k] = vq[k];
        for(int k = 0; k < 3; ++k)
            v_scales[n * 3 + k] = vs[k];
    }
    return 0;
}

/* ---------------------------------------------------------------------- */
/* Perspective projection pieces shared by fwd and bwd.
 * Reference: include/Utils.cuh:567-607 (persp_proj). */
typedef struct
{
    REAL J00, J11, J02, J12; /* 2x3 Jacobian non-zeros */
    REAL tx, ty, rz, rz2;
    int x_in, y_in; /* inside the 1.3x FOV clamp */
} FN(PerspJ);

static inline FN(PerspJ) FN(persp_jacobian)(const REAL *pc, REAL fx, REAL fy, REAL cx, REAL cy, uint32_t W, uint32_t H)
{
    FN(PerspJ) o;
    REAL x = pc[0], y = pc[1], z = pc[2];
    REAL tan_fovx  = (REAL)0.5 * (REAL)W / fx;
    REAL tan_fovy  = (REAL)0.5 * (REAL)H / fy;
    REAL lim_x_pos = ((REAL)W - cx) / fx + (REAL)0.3 * tan_fovx;
    REAL lim_x_neg = cx / fx + (REAL)0.3 * tan_fovx;
    REAL lim_y_pos = ((REAL)H - cy) / fy + (REAL)0.3 * tan_fovy;
    REAL lim_y_neg = cy / fy + (REAL)0.3 * tan_fovy;
    o.rz           = (REAL)1 / z;
    o.rz2          = o.rz * o.rz;
    REAL xz = x * o.rz, yz = y * o.rz;
    REAL cxz = xz > -lim_x_neg ? xz : -lim_x_neg; /* max(-lim_neg, x/z) */
    cxz      = cxz < lim_x_pos ? cxz : lim_x_pos; /* min(lim_pos, .)    */
    REAL cyz = yz > -lim_y_neg ? yz : -lim_y_neg;
    cyz      = cyz < lim_y_pos ? cyz : lim_y_pos;
    o.tx     = z * cxz;
    o.ty     = z * cyz;
    o.J00    = fx * o.rz;
    o.J11    = fy * o.rz;
    o.J02    = -fx * o.tx * o.rz2;
    o.J12    = -fy * o.ty * o.rz2;
    o.x_in   = (xz <= lim_x_pos && xz >= -lim_x_neg);
    o.y_in   = (yz <= lim_y_pos && yz >= -lim_y_neg);
    return o;
}

/* Orthographic and fisheye camera models: dense 2x3 Jacobian J (row-major) + projected mean.
 * Reference: include/Utils.cuh:498-526 (ortho_proj), :692-731 (fisheye_proj).  camera_model ids follow
 * the reference's CameraModelType (ext.cpp:58-64): 0 pinhole, 1 ortho, 2 fisheye. */
static inline void FN(ortho_fisheye_jacobian)(int camera_model, const REAL *pc, REAL fx, REAL fy, REAL cx, REAL cy, REAL *J, REAL *m2)
{
    REAL x = pc[0], y = pc[1], z = pc[2];
    if(camera_model == 1)
    {
        J[0] = fx; J[1] = 0; J[2] = 0;
        J[3] = 0; J[4] = fy; J[5] = 0;
        m2[0] = fx * x + cx;
        m2[1] = fy * y + cy;
        return;
    }
    const REAL eps = (REAL)0.0000001;
    REAL xy_len = R_SQRT(x * x + y * y) + eps;
    REAL theta  = R_ATAN2(xy_len, z + eps);
    m2[0]       = x * fx * theta / xy_len + cx;
    m2[1]       = y * fy * theta / xy_len + cy;
    REAL x2 = x * x + eps, y2 = y * y, xy = x * y;
    REAL x2y2 = x2 + y2;
    REAL inv  = (REAL)1 / (x2y2 + z * z);
    REAL b    = R_ATAN2(xy_len, z) / xy_len / x2y2;
    REAL a    = z * inv / x2y2;
    J[0] = fx * (x2 * a + y2 * b);
    J[1] = fx * xy * (a - b);
    J[2] = -fx * x * inv;
    J[3] = fy * xy * (a - b);
    J[4] = fy * (y2 * a + x2 * b);
    J[5] = -fy * y * inv;
}

/* v_pc (camera-space mean gradient) of the two models given v_mean2d and v_J (2x3, row-major).
 * Reference: Utils.cuh:528-565 (ortho_proj_vjp), :733-846 (fisheye_proj_vjp: the closed-form dJ/d{x,y,z}). */
static inline void FN(ortho_fisheye_vjp)(
    int camera_model, const REAL *pc, REAL fx, REAL fy, const REAL *J, const REAL *vm2, const REAL *v_J, REAL *v_pc
)
{
    for(int j = 0; j < 3; ++j)
        v_pc[j] = J[0 * 3 + j] * vm2[0] + J[1 * 3 + j] * vm2[1];
    if(camera_model == 1)
        return;
    REAL x = pc[0], y = pc[1], z = pc[2];
    const REAL eps = (REAL)0.0000001;
    REAL x2 = x * x + eps, y2 = y * y, xy = x * y;
    REAL x2y2 = x2 + y2;
    REAL len  = R_SQRT(x * x + y * y) + eps;
    REAL r2   = x2y2 + z * z; /* squared distance */
    REAL ir2  = (REAL)1 / r2;
    REAL theta = R_ATAN2(len, z);
    REAL l4 = r2 * r2;
    REAL E  = -l4 * x2y2 * theta + r2 * x2y2 * len * z;
    REAL F  = (REAL)3 * l4 * theta - (REAL)3 * r2 * len * z - (REAL)2 * x2y2 * len * z;
    REAL pA = x * ((REAL)3 * E + x2 * F), pB = y * (E + x2 * F), pC = x * (E + y2 * F), pD = y * ((REAL)3 * E + y2 * F);
    REAL S1 = x2 - y2 - z * z, S2 = y2 - x2 - z * z;
    REAL inv1 = ir2 * ir2;
    REAL inv2 = inv1 / (x2y2 * x2y2 * len);
    /* d J[r][c] / d {x, y, z}, rows r = 0 (fx) and 1 (fy) */
    REAL dx[6] = {fx * pA * inv2, fx * pB * inv2, fx * S1 * inv1, fy * pB * inv2, fy * pC * inv2, (REAL)2 * fy * xy * inv1};
    REAL dy[6] = {dx[1], fx * pC * inv2, (REAL)2 * fx * xy * inv1, dx[4], fy * pD * inv2, fy * S2 * inv1};
    REAL dz[6] = {dx[2], dy[2], (REAL)2 * fx * x * z * inv1, dx[5], dy[5], (REAL)2 * fy * y * z * inv1};
    REAL gx = 0, gy = 0, gz = 0;
    for(int k = 0; k < 6; ++k)
    {
        gx += dx[k] * v_J[k];
        gy += dy[k] * v_J[k];
        gz += dz[k] * v_J[k];
    }
    v_pc[0] += gx;
    v_pc[1] += gy;
    v_pc[2] += gz;
}

/* Forward of one (camera, gaussian).  Returns 0 if culled (radii = 0).
 * Reference: csrc/ProjectionEWA3DGSFused.cu:38-219. */
static inline int FN(project_one)(
    const REAL *mean, const REAL *covar6, const REAL *quat, const REAL *scale, const REAL *opacity, const REAL *vm,
    const REAL *K, uint32_t W, uint32_t H, REAL eps2d, REAL near_plane, REAL far_plane, REAL radius_clip, int want_comp,
    int camera_model, int32_t *radii, REAL *mean2d, REAL *depth, REAL *conic, REAL *comp
)
{
    REAL Rv[9] = {vm[0], vm[1], vm[2], vm[4], vm[5], vm[6], vm[8], vm[9], vm[10]};
    REAL t[3]  = {vm[3], vm[7], vm[11]};
    REAL pc[3];
    for(int i = 0; i < 3; ++i)
        pc[i] = Rv[i * 3 + 0] * mean[0] + Rv[i * 3 + 1] * mean[1] + Rv[i * 3 + 2] * mean[2] + t[i];
    radii[0] = radii[1] = 0;
    if(pc[2] < near_plane || pc[2] > far_plane)
        return 0;

    REAL cov[9];
    if(covar6)
    {
        cov[0] = covar6[0];
        cov[1] = cov[3] = covar6[1];
        cov[2] = cov[6] = covar6[2];
        cov[4] = covar6[3];
        cov[5] = cov[7] = covar6[4];
        cov[8] = covar6[5];
    }
    else
        FN(quat_scale_to_covar_preci_one)(quat, scale, cov, NULL);
    REAL T[9], covc[9];
    FN(mat3_mul)(Rv, cov, T);        /* Include/Utils.cuh:112-123 covarW2C: R * cov * R^T */
    FN(mat3_mul_bt)(T, Rv, covc);

    REAL fx = K[0], fy = K[4], cx = K[2], cy = K[5];
    REAL c00, c01, c10, c11, m2x, m2y;
    if(camera_model == 0)
    {
        FN(PerspJ) pj = FN(persp_jacobian)(pc, fx, fy, cx, cy, W, H);
        /* T2 = J * covc (2x3) ; cov2d = T2 * J^T */
        REAL T2[6];
        for(int j = 0; j < 3; ++j)
        {
            T2[0 * 3 + j] = pj.J00 * covc[0 * 3 + j] + pj.J02 * covc[2 * 3 + j];
            T2[1 * 3 + j] = pj.J11 * covc[1 * 3 + j] + pj.J12 * covc[2 * 3 + j];
        }
        c00 = T2[0] * pj.J00 + T2[2] * pj.J02;
        c01 = T2[1] * pj.J11 + T2[2] * pj.J12;
        c10 = T2[3] * pj.J00 + T2[5] * pj.J02;
        c11 = T2[4] * pj.J11 + T2[5] * pj.J12;
        m2x = fx * pc[0] * pj.rz + cx;
        m2y = fy * pc[1] * pj.rz + cy;
    }
    else
    {
        REAL J[6], m2[2], T2[6];
        FN(ortho_fisheye_jacobian)(camera_model, pc, fx, fy, cx, cy, J, m2);
        for(int i = 0; i < 2; ++i)
            for(int j = 0; j < 3; ++j)
                T2[i * 3 + j] = J[i * 3 + 0] * covc[0 * 3 + j] + J[i * 3 + 1] * covc[1 * 3 + j] + J[i * 3 + 2] * covc[2 * 3 + j];
        c00 = T2[0] * J[0] + T2[1] * J[1] + T2[2] * J[2];
        c01 = T2[0] * J[3] + T2[1] * J[4] + T2[2] * J[5];
        c10 = T2[3] * J[0] + T2[4] * J[1] + T2[5] * J[2];
        c11 = T2[3] * J[3] + T2[4] * J[4] + T2[5] * J[5];
        m2x = m2[0];
        m2y = m2[1];
    }

    /* add_blur: Utils.cuh:455-463 */
    REAL det_orig = c00 * c11 - c01 * c10;
    c00 += eps2d;
    c11 += eps2d;
    REAL det_blur = c00 * c11 - c01 * c10;
    REAL ratio    = det_orig / det_blur;
    REAL floor_   = (REAL)0.005 * (REAL)0.005;
    REAL compensation = R_SQRT(ratio > floor_ ? ratio : floor_);
    if(!(det_blur > (REAL)0))
        return 0;

    REAL ood = (REAL)1 / det_blur;
    REAL ia = c11 * ood, ib = -c01 * ood, ic = c00 * ood;

    REAL extend = (REAL)3.33;
    if(opacity)
    {
        REAL op = *opacity;
        if(want_comp)
            op *= compensation;
        if(op < (REAL)(1.0 / 255.0))
            return 0;
        REAL arg = (REAL)2 * FN(gs_log)(op / (REAL)(1.0 / 255.0));
        REAL e2 = R_SQRT(arg);
        extend = e2 < extend ? e2 : extend;
    }
    REAL rx = R_CEIL(extend * R_SQRT(c00));
    REAL ry = R_CEIL(extend * R_SQRT(c11));
    if(rx <= radius_clip && ry <= radius_clip)
        return 0;
    if(m2x + rx <= (REAL)0 || m2x - rx >= (REAL)W || m2y + ry <= (REAL)0 || m2y - ry >= (REAL)H)
        return 0;
    radii[0]  = FN(f2i)(rx); /* rx >= 2^31 saturates to INT32_MAX like the kernels' conversion */
    radii[1]  = FN(f2i)(ry);
    mean2d[0] = m2x;
    mean2d[1] = m2y;
    *depth    = pc[2];
    conic[0]  = ia;
    conic[1]  = ib;
    conic[2]  = ic;
    if(comp)
        *comp = compensation;
    return 1;
}

/* projection_ewa_3dgs_fused forward.  means [B,N,3], covars [B,N,6] or NULL,
 * quats [B,N,4], scales [B,N,3], opacities [B,N] or NULL, viewmats [B,C,4,4],
 * Ks [B,C,3,3]; outputs [B,C,N,*]; culled rows of the float outputs are set to 0
 * (the reference leaves them uninitialised, csrc/Projection.cpp:395-404).
 * camera_model: 0 pinhole, 1 ortho, 2 fisheye. */
int FN(gso_projection_fwd)(
    int64_t B, int64_t C, int64_t N, const REAL *means, const REAL *covars, const REAL *quats, const REAL *scales,
    const REAL *opacities, const REAL *viewmats, const REAL *Ks, uint32_t W, uint32_t H, REAL eps2d, REAL near_plane,
    REAL far_plane, REAL radius_clip, int camera_model, int32_t *radii, REAL *means2d, REAL *depths, REAL *conics,
    REAL *compensations
)
{
    if(camera_model < 0 || camera_model > 2)
        return -1;
#pragma omp parallel for schedule(static)
    for(int64_t idx = 0; idx < B * C * N; ++idx)
    {
        int64_t b = idx / (C * N), c = (idx / N) % C, n = idx % N;
        REAL m2[2] = {0, 0}, d = 0, cn[3] = {0, 0, 0}, cp = 0;
        FN(project_one)(
            means + (b * N + n) * 3, covars ? covars + (b * N + n) * 6 : NULL, quats ? quats + (b * N + n) * 4 : NULL,
            scales ? scales + (b * N + n) * 3 : NULL, opacities ? opacities + (b * N + n) : NULL,
            viewmats + (b * C + c) * 16, Ks + (b * C + c) * 9, W, H, eps2d, near_plane, far_plane, radius_clip,
            compensations != NULL, camera_model, radii + idx * 2, m2, &d, cn, &cp
        );
        means2d[idx * 2] = m2[0];
        means2d[idx * 2 + 1] = m2[1];
        depths[idx] = d;
        conics[idx * 3] = cn[0];
        conics[idx * 3 + 1] = cn[1];
        conics[idx * 3 + 2] = cn[2];
        if(compensations)
            compensations[idx] = cp;
    }
    return 0;
}

/* projection backward.  Reference: csrc/ProjectionEWA3DGSFused.cu:376-638 with the
 * VJPs of Utils.cuh:94-146 (posW2C/covarW2C), :448-492 (inverse, add_blur), :609-690
 * (persp_proj_vjp).  Gradient outputs are accumulated over cameras (zero-initialised here).
 * v_covars [B,N,6] (when covars given) else v_quats/v_scales.  v_viewmats optional [B,C,4,4]. */
int FN(gso_projection_bwd)(
    int64_t B, int64_t C, int64_t N, const REAL *means, const REAL *covars, const REAL *quats, const REAL *scales,
    const REAL *viewmats, const REAL *Ks, uint32_t W, uint32_t H, REAL eps2d, int camera_model, const int32_t *radii,
    const REAL *conics, const REAL *compensations, const REAL *v_means2d, const REAL *v_depths, const REAL *v_conics,
    const REAL *v_compensations, REAL *v_means, REAL *v_covars, REAL *v_quats, REAL *v_scales, REAL *v_viewmats
)
{
    if(camera_model < 0 || camera_model > 2)
        return -1;
    memset(v_means, 0, sizeof(REAL) * (size_t)(B * N * 3));
    if(v_covars)
        memset(v_covars, 0, sizeof(REAL) * (size_t)(B * N * 6));
    if(v_quats)
        memset(v_quats, 0, sizeof(REAL) * (size_t)(B * N * 4));
    if(v_scales)
        memset(v_scales, 0, sizeof(REAL) * (size_t)(B * N * 3));
    if(v_viewmats)
        memset(v_viewmats, 0, sizeof(REAL) * (size_t)(B * C * 16));
    for(int64_t idx = 0; idx < B * C * N; ++idx)
    {
        int64_t b = idx / (C * N), c = (idx / N) % C, n = idx % N;
        if(radii[idx * 2] <= 0 || radii[idx * 2 + 1] <= 0)
            continue;
        const REAL *mean = means + (b * N + n) * 3;
        const REAL *vm   = viewmats + (b * C + c) * 16;
        const REAL *K    = Ks + (b * C + c) * 9;
        REAL Rv[9]       = {vm[0], vm[1], vm[2], vm[4], vm[5], vm[6], vm[8], vm[9], vm[10]};
        REAL t[3]        = {vm[3], vm[7], vm[11]};

        /* d conic -> d cov2d :  v_Sigma = -P * v_P * P  (Utils.cuh:448-453) */
        REAL a = conics[idx * 3], bb = conics[idx * 3 + 1], cc = conics[idx * 3 + 2];
        REAL P[4]  = {a, bb, bb, cc};
        REAL vP[4] = {v_conics[idx * 3], v_conics[idx * 3 + 1] * (REAL)0.5, v_conics[idx * 3 + 1] * (REAL)0.5,
                      v_conics[idx * 3 + 2]};
        REAL tmp[4], vS[4];
        tmp[0] = P[0] * vP[0] + P[1] * vP[2];
        tmp[1] = P[0] * vP[1] + P[1] * vP[3];
        tmp[2] = P[2] * vP[0] + P[3] * vP[2];
        tmp[3] = P[2] * vP[1] + P[3] * vP[3];
        vS[0]  = -(tmp[0] * P[0] + tmp[1] * P[2]);
        vS[1]  = -(tmp[0] * P[1] + tmp[1] * P[3]);
        vS[2]  = -(tmp[2] * P[0] + tmp[3] * P[2]);
        vS[3]  = -(tmp[2] * P[1] + tmp[3] * P[3]);
        if(v_compensations)
        { /* add_blur_vjp, Utils.cuh:465-492 */
            REAL comp = compensations[idx], v_comp = v_compensations[idx];
            REAL det_conic = P[0] * P[3] - P[1] * P[2];
            REAL v_sqr = v_comp * (REAL)0.5 / (comp + (REAL)1e-6);
            REAL om    = (REAL)1 - comp * comp;
            vS[0] += v_sqr * (om * P[0] - eps2d * det_conic);
            vS[1] += v_sqr * (om * P[1]);
            vS[2] += v_sqr * (om * P[2]);
            vS[3] += v_sqr * (om * P[3] - eps2d * det_conic);
        }

        REAL cov[9];
        if(covars)
        {
            const REAL *c6 = covars + (b * N + n) * 6;
            cov[0] = c6[0]; cov[1] = cov[3] = c6[1]; cov[2] = cov[6] = c6[2];
            cov[4] = c6[3]; cov[5] = cov[7] = c6[4]; cov[8] = c6[5];
        }
        else
            FN(quat_scale_to_covar_preci_one)(quats + (b * N + n) * 4, scales + (b * N + n) * 3, cov, NULL);
        REAL pc[3];
        for(int i = 0; i < 3; ++i)
            pc[i] = Rv[i * 3 + 0] * mean[0] + Rv[i * 3 + 1] * mean[1] + Rv[i * 3 + 2] * mean[2] + t[i];
        REAL T[9], covc[9];
        FN(mat3_mul)(Rv, cov, T);
        FN(mat3_mul_bt)(T, Rv, covc);

        REAL fx = K[0], fy = K[4], cx = K[2], cy = K[5];
        FN(PerspJ) pj;
        REAL J[6], m2_unused[2];
        if(camera_model == 0)
        {
            pj   = FN(persp_jacobian)(pc, fx, fy, cx, cy, W, H);
            J[0] = pj.J00; J[1] = 0; J[2] = pj.J02;
            J[3] = 0; J[4] = pj.J11; J[5] = pj.J12;
        }
        else
        {
            memset(&pj, 0, sizeof(pj));
            FN(ortho_fisheye_jacobian)(camera_model, pc, fx, fy, cx, cy, J, m2_unused);
        }
        /* v_covc = J^T vS J */
        REAL JtG[6]; /* 3x2 = J^T (3x2) * vS (2x2) */
        for(int i = 0; i < 3; ++i)
            for(int j = 0; j < 2; ++j)
                JtG[i * 2 + j] = J[0 * 3 + i] * vS[0 * 2 + j] + J[1 * 3 + i] * vS[1 * 2 + j];
        REAL v_covc[9];
        for(int i = 0; i < 3; ++i)
            for(int j = 0; j < 3; ++j)
                v_covc[i * 3 + j] = JtG[i * 2 + 0] * J[0 * 3 + j] + JtG[i * 2 + 1] * J[1 * 3 + j];
        /* v_J = vS * J * covc^T + vS^T * J * covc  (2x3) */
        REAL GJ[6], GtJ[6], v_J[6];
        for(int i = 0; i < 2; ++i)
            for(int j = 0; j < 3; ++j)
            {
                GJ[i * 3 + j]  = vS[i * 2 + 0] * J[0 * 3 + j] + vS[i * 2 + 1] * J[1 * 3 + j];
                GtJ[i * 3 + j] = vS[0 * 2 + i] * J[0 * 3 + j] + vS[1 * 2 + i] * J[1 * 3 + j];
            }
        for(int i = 0; i < 2; ++i)
            for(int j = 0; j < 3; ++j)
                v_J[i * 3 + j] = (GJ[i * 3 + 0] * covc[j * 3 + 0] + GJ[i * 3 + 1] * covc[j * 3 + 1] + GJ[i * 3 + 2] * covc[j * 3 + 2])
                               + (GtJ[i * 3 + 0] * covc[0 * 3 + j] + GtJ[i * 3 + 1] * covc[1 * 3 + j] + GtJ[i * 3 + 2] * covc[2 * 3 + j]);
        REAL vm2x = v_means2d[idx * 2], vm2y = v_means2d[idx * 2 + 1];
        REAL v_pc[3];
        if(camera_model == 0)
        {
            REAL x = pc[0], y = pc[1];
            REAL rz = pj.rz, rz2 = pj.rz2, rz3 = rz2 * rz;
            v_pc[0] = fx * rz * vm2x;
            v_pc[1] = fy * rz * vm2y;
            v_pc[2] = -(fx * x * vm2x + fy * y * vm2y) * rz2;
            if(pj.x_in)
                v_pc[0] += -fx * rz2 * v_J[0 * 3 + 2];
            else
                v_pc[2] += -fx * rz3 * v_J[0 * 3 + 2] * pj.tx;
            if(pj.y_in)
                v_pc[1] += -fy * rz2 * v_J[1 * 3 + 2];
            else
                v_pc[2] += -fy * rz3 * v_J[1 * 3 + 2] * pj.ty;
            v_pc[2] += -fx * rz2 * v_J[0] - fy * rz2 * v_J[1 * 3 + 1] + (REAL)2 * fx * pj.tx * rz3 * v_J[0 * 3 + 2]
                     + (REAL)2 * fy * pj.ty * rz3 * v_J[1 * 3 + 2];
        }
        else
        {
            REAL vm2[2] = {vm2x, vm2y};
            FN(ortho_fisheye_vjp)(camera_model, pc, fx, fy, J, vm2, v_J, v_pc);
        }
        v_pc[2] += v_depths[idx];

        /* world: v_mean = R^T v_pc ; v_cov = R^T v_covc R */
        for(int j = 0; j < 3; ++j)
            v_means[(b * N + n) * 3 + j] += Rv[0 * 3 + j] * v_pc[0] + Rv[1 * 3 + j] * v_pc[1] + Rv[2 * 3 + j] * v_pc[2];
        REAL T3[9], v_cov[9];
        FN(mat3_mul_at)(Rv, v_covc, T3);
        FN(mat3_mul)(T3, Rv, v_cov);
        if(covars)
        {
            REAL *o = v_covars + (b * N + n) * 6;
            o[0] += v_cov[0];
            o[1] += v_cov[1] + v_cov[3];
            o[2] += v_cov[2] + v_cov[6];
            o[3] += v_cov[4];
            o[4] += v_cov[5] + v_cov[7];
            o[5] += v_cov[8];
        }
        else
            FN(quat_scale_to_covar_vjp)(
                quats + (b * N + n) * 4, scales + (b * N + n) * 3, v_cov, v_quats + (b * N + n) * 4, v_scales + (b * N + n) * 3
            );
        if(v_viewmats)
        { /* v_R = v_pc mean^T + v_covc R cov^T + v_covc^T R cov ; v_t = v_pc */
            REAL A1[9], A2[9], B1[9], B2[9];
            FN(mat3_mul)(v_covc, Rv, A1);
            FN(mat3_mul_bt)(A1, cov, A2);
            FN(mat3_mul_at)(v_covc, Rv, B1);
            FN(mat3_mul)(B1, cov, B2);
            REAL *o = v_viewmats + (b * C + c) * 16;
            for(int i = 0; i < 3; ++i)
            {
                for(int j = 0; j < 3; ++j)
                    o[i * 4 + j] += v_pc[i] * mean[j] + A2[i * 3 + j] + B2[i * 3 + j];
                o[i * 4 + 3] += v_pc[i];
            }
        }
    }
    return 0;
}

/* ---------------------------------------------------------------------- */
/* Spherical harmonics (real basis, P-P. Sloan, "Efficient Spherical Harmonic Evaluation",
 * JCGT 2013).  Reference: csrc/SphericalHarmonicsCUDA.cu:48-146 (fwd), :148-439 (vjp),
 * view direction dir = mean + R^T t, csrc/SphericalHarmonics.cuh:40-78.
 * The basis and its gradient are evaluated with 4-wide dual numbers (value, d/dx, d/dy, d/dz). */
typedef struct
{
    REAL v, x, y, z;
} FN(D4);
static inline FN(D4) FN(d4)(REAL v, REAL x, REAL y, REAL z)
{
    FN(D4) r = {v, x, y, z};
    return r;
}
static inline FN(D4) FN(d4_mul)(FN(D4) a, FN(D4) b)
{
    return FN(d4)(a.v * b.v, a.v * b.x + a.x * b.v, a.v * b.y + a.y * b.v, a.v * b.z + a.z * b.v);
}
static inline FN(D4) FN(d4_add)(FN(D4) a, FN(D4) b) { return FN(d4)(a.v + b.v, a.x + b.x, a.y + b.y, a.z + b.z); }
static inline FN(D4) FN(d4_sub)(FN(D4) a, FN(D4) b) { return FN(d4)(a.v - b.v, a.x - b.x, a.y - b.y, a.z - b.z); }
static inline FN(D4) FN(d4_s)(REAL s, FN(D4) a) { return FN(d4)(s * a.v, s * a.x, s * a.y, s * a.z); }
static inline FN(D4) FN(d4_sadd)(REAL s, FN(D4) a, REAL c) { return FN(d4)(s * a.v + c, s * a.x, s * a.y, s * a.z); }

/* Y[k], k < (deg+1)^2, for unit vector (x,y,z). */
static void FN(sh_basis)(int deg, REAL ux, REAL uy, REAL uz, FN(D4) *Y)
{
    FN(D4) x = FN(d4)(ux, 1, 0, 0), y = FN(d4)(uy, 0, 1, 0), z = FN(d4)(uz, 0, 0, 1);
    Y[0] = FN(d4)((REAL)0.2820947917738781, 0, 0, 0);
    if(deg < 1)
        return;
    Y[1] = FN(d4_s)((REAL)-0.48860251190292, y);
    Y[2] = FN(d4_s)((REAL)0.48860251190292, z);
    Y[3] = FN(d4_s)((REAL)-0.48860251190292, x);
    if(deg < 2)
        return;
    FN(D4) z2     = FN(d4_mul)(z, z);
    FN(D4) fTmp0B = FN(d4_s)((REAL)-1.092548430592079, z);
    FN(D4) fC1    = FN(d4_sub)(FN(d4_mul)(x, x), FN(d4_mul)(y, y));
    FN(D4) fS1    = FN(d4_s)((REAL)2, FN(d4_mul)(x, y));
    Y[4]          = FN(d4_s)((REAL)0.5462742152960395, fS1);
    Y[5]          = FN(d4_mul)(fTmp0B, y);
    Y[6]          = FN(d4_sadd)((REAL)0.9461746957575601, z2, (REAL)-0.3153915652525201);
    Y[7]          = FN(d4_mul)(fTmp0B, x);
    Y[8]          = FN(d4_s)((REAL)0.5462742152960395, fC1);
    if(deg < 3)
        return;
    FN(D4) fTmp0C = FN(d4_sadd)((REAL)-2.285228997322329, z2, (REAL)0.4570457994644658);
    FN(D4) fTmp1B = FN(d4_s)((REAL)1.445305721320277, z);
    FN(D4) fC2    = FN(d4_sub)(FN(d4_mul)(x, fC1), FN(d4_mul)(y, fS1));
    FN(D4) fS2    = FN(d4_add)(FN(d4_mul)(x, fS1), FN(d4_mul)(y, fC1));
    Y[9]          = FN(d4_s)((REAL)-0.5900435899266435, fS2);
    Y[10]         = FN(d4_mul)(fTmp1B, fS1);
    Y[11]         = FN(d4_mul)(fTmp0C, y);
    Y[12]         = FN(d4_mul)(z, FN(d4_sadd)((REAL)1.865881662950577, z2, (REAL)-1.119528997770346));
    Y[13]         = FN(d4_mul)(fTmp0C, x);
    Y[14]         = FN(d4_mul)(fTmp1B, fC1);
    Y[15]         = FN(d4_s)((REAL)-0.5900435899266435, fC2);
    if(deg < 4)
        return;
    FN(D4) fTmp0D = FN(d4_mul)(z, FN(d4_sadd)((REAL)-4.683325804901025, z2, (REAL)2.007139630671868));
    FN(D4) fTmp1C = FN(d4_sadd)((REAL)3.31161143515146, z2, (REAL)-0.47308734787878);
    FN(D4) fTmp2B = FN(d4_s)((REAL)-1.770130769779931, z);
    FN(D4) fC3    = FN(d4_sub)(FN(d4_mul)(x, fC2), FN(d4_mul)(y, fS2));
    FN(D4) fS3    = FN(d4_add)(FN(d4_mul)(x, fS2), FN(d4_mul)(y, fC2));
    Y[16]         = FN(d4_s)((REAL)0.6258357354491763, fS3);
    Y[17]         = FN(d4_mul)(fTmp2B, fS2);
    Y[18]         = FN(d4_mul)(fTmp1C, fS1);
    Y[19]         = FN(d4_mul)(fTmp0D, y);
    Y[20] = FN(d4_sub)(FN(d4_s)((REAL)1.984313483298443, FN(d4_mul)(z, Y[12])), FN(d4_s)((REAL)1.006230589874905, Y[6]));
    Y[21]         = FN(d4_mul)(fTmp0D, x);
    Y[22]         = FN(d4_mul)(fTmp1C, fC1);
    Y[23]         = FN(d4_mul)(fTmp2B, fC2);
    Y[24]         = FN(d4_s)((REAL)0.6258357354491763, fC3);
}

static inline void FN(sh_view_dir)(const REAL *mean, const REAL *vm, REAL *dir)
{
    REAL tx = vm[3], ty = vm[7], tz = vm[11];
    dir[0] = mean[0] + (vm[0] * tx + vm[4] * ty + vm[8] * tz);
    dir[1] = mean[1] + (vm[1] * tx + vm[5] * ty + vm[9] * tz);
    dir[2] = mean[2] + (vm[2] * tx + vm[6] * ty + vm[10] * tz);
}

/* spherical_harmonics forward, dense layout.  means [B,N,3], viewmats [B,C,4,4],
 * coeffs [N,K,D], masks [B,C,N] (uint8) or NULL -> colors [B,C,N,D]; masked rows = 0
 * (the reference leaves them uninitialised: csrc/SphericalHarmonics.cpp:244).
 * Reference kernel: csrc/SphericalHarmonicsCUDA.cu:443-488. */
int FN(gso_sh_fwd)(
    int64_t B, int64_t C, int64_t N, int64_t K, int64_t D, int degree, const REAL *means, const REAL *viewmats,
    const REAL *coeffs, const uint8_t *masks, REAL *colors
)
{
    if(degree < 0 || degree > 4 || (degree + 1) * (degree + 1) > K)
        return -1;
    const int nb = (degree + 1) * (degree + 1);
#pragma omp parallel for schedule(static)
    for(int64_t idx = 0; idx < B * C * N; ++idx)
    {
        int64_t b = idx / (C * N), c = (idx / N) % C, n = idx % N;
        REAL *out = colors + idx * D;
        for(int64_t d = 0; d < D; ++d)
            out[d] = 0;
        if(masks && !masks[idx])
            continue;
        REAL dir[3];
        FN(sh_view_dir)(means + (b * N + n) * 3, viewmats + (b * C + c) * 16, dir);
        REAL inorm = (REAL)1 / R_SQRT(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
        FN(D4) Y[25];
        FN(sh_basis)(degree, dir[0] * inorm, dir[1] * inorm, dir[2] * inorm, Y);
        const REAL *cf = coeffs + n * K * D;
        for(int64_t d = 0; d < D; ++d)
        {
            REAL acc = 0;
            for(int k = 0; k < nb; ++k)
                acc += Y[k].v * cf[k * D + d];
            out[d] = acc;
        }
    }
    return 0;
}

/* spherical_harmonics backward: v_coeffs [N,K,D] (summed over images, zero for k >= nb),
 * v_means [B,N,3] (optional).  Reference: csrc/SphericalHarmonicsCUDA.cu:785-890. */
int FN(gso_sh_bwd)(
    int64_t B, int64_t C, int64_t N, int64_t K, int64_t D, int degree, const REAL *means, const REAL *viewmats,
    const REAL *coeffs, const uint8_t *masks, const REAL *v_colors, REAL *v_coeffs, REAL *v_means
)
{
    if(degree < 0 || degree > 4 || (degree + 1) * (degree + 1) > K)
        return -1;
    const int nb = (degree + 1) * (degree + 1);
    memset(v_coeffs, 0, sizeof(REAL) * (size_t)(N * K * D));
    if(v_means)
        memset(v_means, 0, sizeof(REAL) * (size_t)(B * N * 3));
    for(int64_t idx = 0; idx < B * C * N; ++idx)
    {
        int64_t b = idx / (C * N), c = (idx / N) % C, n = idx % N;
        if(masks && !masks[idx])
            continue;
        REAL dir[3];
        FN(sh_view_dir)(means + (b * N + n) * 3, viewmats + (b * C + c) * 16, dir);
        REAL inorm = (REAL)1 / R_SQRT(dir[0] * dir[0] + dir[1] * dir[1] + dir[2] * dir[2]);
        REAL u[3] = {dir[0] * inorm, dir[1] * inorm, dir[2] * inorm};
        FN(D4) Y[25];
        FN(sh_basis)(degree, u[0], u[1], u[2], Y);
        const REAL *cf = coeffs + n * K * D;
        const REAL *vc = v_colors + idx * D;
        REAL vu[3]     = {0, 0, 0};
        for(int k = 0; k < nb; ++k)
        {
            REAL g = 0;
            for(int64_t d = 0; d < D; ++d)
            {
                v_coeffs[(n * K + k) * D + d] += Y[k].v * vc[d];
                g += cf[k * D + d] * vc[d];
            }
            vu[0] += g * Y[k].x;
            vu[1] += g * Y[k].y;
            vu[2] += g * Y[k].z;
        }
        if(v_means && degree >= 1)
        { /* through the normalisation: (I - u u^T) vu / |dir| */
            REAL dot = vu[0] * u[0] + vu[1] * u[1] + vu[2] * u[2];
            for(int j = 0; j < 3; ++j)
                v_means[(b * N + n) * 3 + j] += (vu[j] - dot * u[j]) * inorm;
        }
    }
    return 0;
}

/* ---------------------------------------------------------------------- */
/* Tile intersection.  Reference: csrc/IntersectTile.cu:83-207 (AccuTile/SNUGBOX helpers),
 * :213-464 (kernel), host csrc/Intersect.cpp:170-329, key layout
 * image << (32+tile_bits) | tile << 32 | float_bits(depth), bits_for_count csrc/MathUtils.h:26-36. */
typedef void (*FN(tile_cb))(void *ctx, int64_t tile_id);

static inline void FN(ellipse_line)(REAL A_, REAL B_, REAL C_, REAL disc, REAL t, REAL pu, REAL pv, REAL coeff, REAL coord, REAL *lo, REAL *hi)
{
    REAL h = coord - pu;
    REAL sq = R_SQRT(disc * h * h + t * coeff);
    (void)A_; (void)C_;
    *lo = (-B_ * h - sq) / coeff + pv;
    *hi = (-B_ * h + sq) / coeff + pv;
}

static inline int FN(clampi)(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

/* Enumerate the tiles one gaussian touches; returns the count and calls cb (if not NULL) per tile
 * in the reference's emit order. */
static int FN(tiles_of_gaussian)(
    REAL mx, REAL my, int32_t rx, int32_t ry, const REAL *conic, const REAL *opacity, uint32_t tile_size, uint32_t tw,
    uint32_t th, FN(tile_cb) cb, void *ctx
)
{
    if(rx <= 0 || ry <= 0)
        return 0;
    int count = 0;
    REAL ts   = (REAL)tile_size;
    if(conic && opacity)
    {
        REAL A_ = conic[0], B_ = conic[1], C_ = conic[2];
        REAL disc = B_ * B_ - A_ * C_;
        REAL t    = (REAL)2 * FN(gs_log)(*opacity / (REAL)(1.0 / 255.0));
        REAL cap  = (REAL)3.33 * (REAL)3.33;
        t         = t < cap ? t : cap;
        REAL ntd  = -t / disc;
        REAL xe = R_SQRT(ntd * C_), ye = R_SQRT(ntd * A_);
        REAL bminx = mx - xe, bminy = my - ye, bmaxx = mx + xe, bmaxy = my + ye;
        REAL BxC = B_ * xe / C_, ByA = B_ * ye / A_;
        /* argmin.x = y where x is minimal ; argmin.y = x where y is minimal */
        REAL argminx = my + BxC, argminy = mx + ByA, argmaxx = my - BxC, argmaxy = mx - ByA;
        int rminx = FN(clampi)(FN(f2i)(bminx / ts), 0, (int)tw), rminy = FN(clampi)(FN(f2i)(bminy / ts), 0, (int)th);
        int rmaxx = FN(clampi)(FN(f2i)(bmaxx / ts + (REAL)1), 0, (int)tw), rmaxy = FN(clampi)(FN(f2i)(bmaxy / ts + (REAL)1), 0, (int)th);
        int ys = rmaxy - rminy, xs = rmaxx - rminx;
        if(ys * xs == 0)
            return 0;
        int isY = ys < xs;
        /* u = iterated axis, v = swept axis */
        int ru0 = isY ? rminy : rminx, ru1 = isY ? rmaxy : rmaxx, rv0 = isY ? rminx : rminy, rv1 = isY ? rmaxx : rmaxy;
        REAL bminu = isY ? bminy : bminx, bmaxu = isY ? bmaxy : bmaxx, bminv = isY ? bminx : bminy, bmaxv = isY ? bmaxx : bmaxy;
        REAL amin_v = isY ? argminx : argminy; /* u-coordinate at which v is minimal */
        REAL amax_v = isY ? argmaxx : argmaxy;
        REAL pu = isY ? my : mx, pv = isY ? mx : my, coeff = isY ? A_ : C_;
        REAL maxlo = bmaxv, maxhi = bminv; /* "empty" interval, reversed */
        REAL minlo, minhi;
        REAL min_line = (REAL)ru0 * ts;
        if(bminu <= min_line)
            FN(ellipse_line)(A_, B_, C_, disc, t, pu, pv, coeff, min_line, &minlo, &minhi);
        else
        {
            minlo = maxlo;
            minhi = maxhi;
        }
        for(int u = ru0; u < ru1; ++u)
        {
            REAL max_line = min_line + ts;
            if(max_line <= bmaxu)
                FN(ellipse_line)(A_, B_, C_, disc, t, pu, pv, coeff, max_line, &maxlo, &maxhi);
            REAL emin, emax;
            if(min_line <= amin_v && amin_v < max_line)
                emin = bminv;
            else
                emin = minlo < maxlo ? minlo : maxlo;
            if(min_line <= amax_v && amax_v < max_line)
                emax = bmaxv;
            else
                emax = minhi > maxhi ? minhi : maxhi;
            int e0 = FN(f2i)(emin / ts), e1 = FN(f2i)(emax / ts + (REAL)1);
            int v0 = e0 < rv1 ? e0 : rv1; /* max(rv0, min(rv1, e0)) */
            v0     = v0 > rv0 ? v0 : rv0;
            int v1 = e1 > rv0 ? e1 : rv0; /* min(rv1, max(rv0, e1)) */
            v1     = v1 < rv1 ? v1 : rv1;
            for(int v = v0; v < v1; ++v)
            {
                ++count;
                if(cb)
                    cb(ctx, isY ? (int64_t)u * tw + v : (int64_t)v * tw + u);
            }
            minlo    = maxlo;
            minhi    = maxhi;
            min_line = max_line;
        }
    }
    else
    { /* AABB from radii: IntersectTile.cu:374-463 */
        REAL trx = (REAL)rx / ts, try_ = (REAL)ry / ts, tx = mx / ts, ty = my / ts;
        int x0 = FN(f2i)(R_FLOOR(tx - trx)), y0 = FN(f2i)(R_FLOOR(ty - try_)), x1 = FN(f2i)(R_CEIL(tx + trx)), y1 = FN(f2i)(R_CEIL(ty + try_));
        x0 = FN(clampi)(x0, 0, (int)tw); y0 = FN(clampi)(y0, 0, (int)th);
        x1 = FN(clampi)(x1, 0, (int)tw); y1 = FN(clampi)(y1, 0, (int)th);
        for(int i = y0; i < y1; ++i)
            for(int j = x0; j < x1; ++j)
            {
                ++count;
                if(cb)
                    cb(ctx, (int64_t)i * tw + j);
            }
    }
    return count;
}

typedef struct
{
    int64_t *isect_ids;
    int32_t *flatten_ids;
    int64_t cur;
    int64_t hi_bits;
    int64_t depth_bits;
    int32_t flat;
} FN(EmitCtx);

static void FN(emit_cb)(void *p, int64_t tile_id)
{
    FN(EmitCtx) *c            = (FN(EmitCtx) *)p;
    c->isect_ids[c->cur]   = c->hi_bits | (tile_id << 32) | c->depth_bits;
    c->flatten_ids[c->cur] = c->flat;
    c->cur++;
}

/* Pass 1: tiles_per_gauss [I,N]; returns total. */
int64_t FN(gso_isect_count)(
    int64_t I, int64_t N, const REAL *means2d, const int32_t *radii, const REAL *conics, const REAL *opacities,
    uint32_t tile_size, uint32_t tw, uint32_t th, int32_t *tiles_per_gauss
)
{
    int64_t total = 0;
#pragma omp parallel for schedule(static) reduction(+ : total)
    for(int64_t i = 0; i < I * N; ++i)
    {
        int cnt = FN(tiles_of_gaussian)(
            means2d[i * 2], means2d[i * 2 + 1], radii[i * 2], radii[i * 2 + 1], conics ? conics + i * 3 : NULL,
            opacities ? opacities + i : NULL, tile_size, tw, th, NULL, NULL
        );
        tiles_per_gauss[i] = cnt;
        total += cnt;
    }
    return total;
}

/* Pass 2: emit unsorted isect_ids / flatten_ids (caller sized them with pass 1). */
int FN(gso_isect_emit)(
    int64_t I, int64_t N, const REAL *means2d, const int32_t *radii, const REAL *depths, const REAL *conics,
    const REAL *opacities, uint32_t tile_size, uint32_t tw, uint32_t th, uint32_t tile_n_bits, int64_t *isect_ids,
    int32_t *flatten_ids
)
{
    FN(EmitCtx) ctx;
    ctx.isect_ids   = isect_ids;
    ctx.flatten_ids = flatten_ids;
    ctx.cur         = 0;
    for(int64_t i = 0; i < I * N; ++i)
    {
        float df        = (float)depths[i];
        uint32_t dbits;
        memcpy(&dbits, &df, 4);
        ctx.hi_bits    = (i / N) << (32 + tile_n_bits);
        ctx.depth_bits = (int64_t)dbits;
        ctx.flat       = (int32_t)i;
        FN(tiles_of_gaussian)(
            means2d[i * 2], means2d[i * 2 + 1], radii[i * 2], radii[i * 2 + 1], conics ? conics + i * 3 : NULL,
            opacities ? opacities + i : NULL, tile_size, tw, th, FN(emit_cb), &ctx
        );
    }
    return 0;
}

/* ---------------------------------------------------------------------- */
/* rasterize_to_pixels forward.  Reference: csrc/RasterizeToPixels3DGSSerialBatchFwd.cu:41-297,
 * per-pair math csrc/RasterizeToPixels3DGSDevice.cuh:37-97, constants include/Common.h:97-114.
 * margins (optional, [I,H,W]) receives, per pixel, the smallest relative distance of any
 * discrete decision (alpha threshold, transmittance stop, sigma sign, alpha clamp) from
 * flipping -- pixels with a tiny margin are legitimately implementation-dependent. */
int FN(gso_raster_fwd)(
    int64_t I, int64_t N, int64_t D, const REAL *means2d, const REAL *conics, const REAL *colors, const REAL *opacities,
    const REAL *backgrounds, const uint8_t *masks, uint32_t W, uint32_t H, uint32_t tile_size, uint32_t tw, uint32_t th,
    const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, REAL *render_colors, REAL *render_alphas,
    int32_t *last_ids, float *margins
)
{
    (void)N;
    const REAL ALPHA_TH = (REAL)(1.0f / 255.0f), MAX_A = (REAL)0.99f, T_TH = (REAL)1e-4f;
#pragma omp parallel for schedule(dynamic, 4)
    for(int64_t tile = 0; tile < I * (int64_t)tw * th; ++tile)
    {
        int64_t img = tile / ((int64_t)tw * th);
        int64_t tid = tile % ((int64_t)tw * th);
        uint32_t ty = (uint32_t)(tid / tw), tx = (uint32_t)(tid % tw);
        int32_t start = offsets[tile];
        int32_t end   = (tile == I * (int64_t)tw * th - 1) ? (int32_t)n_isects : offsets[tile + 1];
        const REAL *bg = backgrounds ? backgrounds + img * D : NULL;
        int masked     = masks && !masks[tile];
        for(uint32_t ly = 0; ly < tile_size; ++ly)
            for(uint32_t lx = 0; lx < tile_size; ++lx)
            {
                uint32_t i = ty * tile_size + ly, j = tx * tile_size + lx;
                if(i >= H || j >= W)
                    continue;
                int64_t pix = (img * H + i) * (int64_t)W + j;
                REAL *out   = render_colors + pix * D;
                if(masked)
                {
                    for(int64_t k = 0; k < D; ++k)
                        out[k] = bg ? bg[k] : (REAL)0;
                    render_alphas[pix] = 0;
                    last_ids[pix]      = 0;
                    if(margins)
                        margins[pix] = 1.0f;
                    continue;
                }
                REAL px = (REAL)j + (REAL)0.5, py = (REAL)i + (REAL)0.5;
                REAL T = 1;
                int32_t cur = 0;
                float margin = 1.0f;
                for(int64_t k = 0; k < D; ++k)
                    out[k] = 0;
                for(int32_t s = start; s < end; ++s)
                {
                    int32_t g = flatten_ids[s];
                    REAL dx = means2d[g * 2] - px, dy = means2d[g * 2 + 1] - py;
                    REAL a = conics[g * 3], b = conics[g * 3 + 1], c = conics[g * 3 + 2], op = opacities[g];
                    REAL sigma = (REAL)0.5 * (a * dx * dx + c * dy * dy) + b * dx * dy;
                    REAL vis = R_EXP(-sigma);
                    REAL ov    = op * vis;
                    REAL alpha = ov < MAX_A ? ov : MAX_A;
                    if(margins)
                    {
                        float m1 = (float)(fabs((double)(alpha - ALPHA_TH)) / (double)ALPHA_TH);
                        if(m1 < margin) margin = m1;
                        float m2 = (float)fabs((double)sigma); /* sigma sign */
                        if(sigma < (REAL)1e-3 && m2 < margin) margin = m2;
                    }
                    if(sigma < 0 || alpha < ALPHA_TH)
                        continue;
                    REAL next_T = T * ((REAL)1 - alpha);
                    if(margins)
                    {
                        float m3 = (float)(fabs((double)(next_T - T_TH)) / (double)T_TH);
                        if(m3 < margin) margin = m3;
                        float m4 = (float)(fabs((double)(ov - MAX_A)) / (double)MAX_A);
                        if(m4 < margin) margin = m4;
                    }
                    if(next_T <= T_TH)
                        break; /* exclusive */
                    REAL w = alpha * T;
                    const REAL *col = colors + (int64_t)g * D;
                    for(int64_t k = 0; k < D; ++k)
                        out[k] += col[k] * w;
                    cur = s;
                    T   = next_T;
                }
                render_alphas[pix] = (REAL)1 - T;
                if(bg)
                    for(int64_t k = 0; k < D; ++k)
                        out[k] = out[k] + T * bg[k];
                last_ids[pix] = cur;
                if(margins)
                    margins[pix] = margin;
            }
    }
    return 0;
}

/* rasterize_to_pixels backward.  Reference: csrc/RasterizeToPixels3DGSSerialBatchBwd.cu:41-320,
 * per-pair math csrc/RasterizeToPixels3DGSDevice.cuh:104-173.  Per-pair terms are evaluated in
 * REAL; the per-gaussian sums are accumulated in double.  abs_sums (optional, [I*N, 9+... ])
 * is not produced here; see gso_raster_bwd_abs for conditioning information.
 * Outputs (zero-initialised here): v_means2d [I*N,2], v_conics [I*N,3], v_colors [I*N,D],
 * v_opacities [I*N], optional v_means2d_abs [I*N,2], optional mag [I*N] = sum over pairs of the
 * absolute values of all terms (a conditioning scale for tolerance checks). */
int FN(gso_raster_bwd)(
    int64_t I, int64_t N, int64_t D, const REAL *means2d, const REAL *conics, const REAL *colors, const REAL *opacities,
    const REAL *backgrounds, const uint8_t *masks, uint32_t W, uint32_t H, uint32_t tile_size, uint32_t tw, uint32_t th,
    const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, const REAL *render_alphas,
    const int32_t *last_ids, const REAL *v_render_colors, const REAL *v_render_alphas, double *v_means2d, double *v_conics,
    double *v_colors, double *v_opacities, double *v_means2d_abs, double *mag
)
{
    const REAL ALPHA_TH = (REAL)(1.0f / 255.0f), MAX_A = (REAL)0.99f;
    memset(v_means2d, 0, sizeof(double) * (size_t)(I * N * 2));
    memset(v_conics, 0, sizeof(double) * (size_t)(I * N * 3));
    memset(v_colors, 0, sizeof(double) * (size_t)(I * N * D));
    memset(v_opacities, 0, sizeof(double) * (size_t)(I * N));
    if(v_means2d_abs)
        memset(v_means2d_abs, 0, sizeof(double) * (size_t)(I * N * 2));
    if(mag)
        memset(mag, 0, sizeof(double) * (size_t)(I * N * 4));
    if(D > 64)
        return -1;
#pragma omp parallel for schedule(dynamic, 4)
    for(int64_t tile = 0; tile < I * (int64_t)tw * th; ++tile)
    {
        if(masks && !masks[tile])
            continue;
        int64_t img = tile / ((int64_t)tw * th);
        int64_t tid = tile % ((int64_t)tw * th);
        uint32_t ty = (uint32_t)(tid / tw), tx = (uint32_t)(tid % tw);
        int32_t start = offsets[tile];
        int32_t end   = (tile == I * (int64_t)tw * th - 1) ? (int32_t)n_isects : offsets[tile + 1];
        if(end <= start)
            continue;
        const REAL *bg = backgrounds ? backgrounds + img * D : NULL;
        int32_t n      = end - start;
        /* tile-local accumulators: [n][ 2 xy, 3 conic, 1 opac, 2 abs, 4 mag, D rgb ] */
        const int stride = 12 + (int)D;
        double *acc = (double *)calloc((size_t)n * stride, sizeof(double));
        for(uint32_t ly = 0; ly < tile_size; ++ly)
            for(uint32_t lx = 0; lx < tile_size; ++lx)
            {
                uint32_t i = ty * tile_size + ly, j = tx * tile_size + lx;
                if(i >= H || j >= W)
                    continue;
                int64_t pix = (img * H + i) * (int64_t)W + j;
                REAL px = (REAL)j + (REAL)0.5, py = (REAL)i + (REAL)0.5;
                REAL T_final = (REAL)1 - render_alphas[pix];
                REAL T       = T_final;
                REAL buffer[64];
                for(int64_t k = 0; k < D; ++k)
                    buffer[k] = 0;
                const REAL *vrc = v_render_colors + pix * D;
                REAL vra        = v_render_alphas[pix];
                int32_t bin_final = last_ids[pix];
                for(int32_t s = end - 1; s >= start; --s)
                {
                    if(s > bin_final)
                        continue;
                    int32_t g = flatten_ids[s];
                    REAL dx = means2d[g * 2] - px, dy = means2d[g * 2 + 1] - py;
                    REAL a = conics[g * 3], b = conics[g * 3 + 1], c = conics[g * 3 + 2], op = opacities[g];
                    REAL sigma = (REAL)0.5 * (a * dx * dx + c * dy * dy) + b * dx * dy;
                    REAL vis = R_EXP(-sigma);
                    REAL ov    = op * vis;
                    REAL alpha = ov < MAX_A ? ov : MAX_A;
                    if(sigma < 0 || alpha < ALPHA_TH)
                        continue;
                    REAL oma = (REAL)1 - alpha;
                    REAL ra  = (REAL)1 / (oma > (REAL)1e-6f ? oma : (REAL)1e-6f);
                    T *= ra;
                    REAL fac = alpha * T;
                    double *A = acc + (size_t)(s - start) * stride;
                    const REAL *col = colors + (int64_t)g * D;
                    REAL v_alpha = 0;
                    double abs_va = 0; /* sum of |terms| inside v_alpha: its own conditioning */
                    for(int64_t k = 0; k < D; ++k)
                    {
                        A[12 + k] += (double)(fac * vrc[k]);
                        v_alpha += (col[k] * T - buffer[k] * ra) * vrc[k];
                        abs_va += (fabs((double)(col[k] * T)) + fabs((double)(buffer[k] * ra))) * fabs((double)vrc[k]);
                    }
                    v_alpha += T_final * ra * vra;
                    abs_va += fabs((double)(T_final * ra * vra));
                    if(bg)
                    {
                        REAL accum = 0;
                        for(int64_t k = 0; k < D; ++k)
                        {
                            accum += bg[k] * vrc[k];
                            abs_va += fabs((double)(T_final * ra * bg[k] * vrc[k]));
                        }
                        v_alpha += -T_final * ra * accum;
                    }
                    if(ov <= MAX_A)
                    {
                        REAL v_sigma = -ov * v_alpha;
                        REAL gx = v_sigma * (a * dx + b * dy), gy = v_sigma * (b * dx + c * dy);
                        double s_abs = fabs((double)ov) * abs_va;
                        A[0] += (double)gx;
                        A[1] += (double)gy;
                        A[2] += (double)((REAL)0.5 * v_sigma * dx * dx);
                        A[3] += (double)(v_sigma * dx * dy);
                        A[4] += (double)((REAL)0.5 * v_sigma * dy * dy);
                        A[5] += (double)(vis * v_alpha);
                        A[6] += fabs((double)gx);
                        A[7] += fabs((double)gy);
                        A[8] += s_abs * (fabs((double)(a * dx)) + fabs((double)(b * dy)) + fabs((double)(b * dx)) + fabs((double)(c * dy)));
                        A[9] += s_abs * (0.5 * (double)(dx * dx) + fabs((double)(dx * dy)) + 0.5 * (double)(dy * dy));
                        A[10] += fabs((double)vis) * abs_va;
                    }
                    for(int64_t k = 0; k < D; ++k)
                    {
                        A[11] += fabs((double)(fac * vrc[k]));
                        buffer[k] += col[k] * fac;
                    }
                }
            }
        for(int32_t s = 0; s < n; ++s)
        {
            int64_t g       = flatten_ids[start + s];
            const double *A = acc + (size_t)s * stride;
#define GSO_ATOMIC_ADD(dst, val)            \
    do                                      \
    {                                       \
        double v__ = (val);                 \
        if(v__ != 0.0)                      \
        {                                   \
            _Pragma("omp atomic")(dst) += v__; \
        }                                   \
    } while(0)
            GSO_ATOMIC_ADD(v_means2d[g * 2], A[0]);
            GSO_ATOMIC_ADD(v_means2d[g * 2 + 1], A[1]);
            GSO_ATOMIC_ADD(v_conics[g * 3], A[2]);
            GSO_ATOMIC_ADD(v_conics[g * 3 + 1], A[3]);
            GSO_ATOMIC_ADD(v_conics[g * 3 + 2], A[4]);
            GSO_ATOMIC_ADD(v_opacities[g], A[5]);
            if(v_means2d_abs)
            {
                GSO_ATOMIC_ADD(v_means2d_abs[g * 2], A[6]);
                GSO_ATOMIC_ADD(v_means2d_abs[g * 2 + 1], A[7]);
            }
            if(mag)
            {
                GSO_ATOMIC_ADD(mag[g * 4], A[8]);
                GSO_ATOMIC_ADD(mag[g * 4 + 1], A[9]);
                GSO_ATOMIC_ADD(mag[g * 4 + 2], A[10]);
                GSO_ATOMIC_ADD(mag[g * 4 + 3], A[11]);
            }
            for(int64_t k = 0; k < D; ++k)
                GSO_ATOMIC_ADD(v_colors[g * D + k], A[12 + k]);
#undef GSO_ATOMIC_ADD
        }
        free(acc);
    }
    return 0;
}

#undef FN
#undef CAT
#undef CAT_
