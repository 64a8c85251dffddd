/*
 * gsplat_b200.h -- C ABI of libgsplat_b200.so: the H100-native (sm_90a) replacement for the
 * CUDA operators behind gsplat.rasterization().
 *
 * This is the drop-in boundary.  Every entry point takes plain DEVICE pointers, sizes and a
 * cudaStream_t (passed as void*), allocates nothing that outlives the call (scratch comes from the
 * caller through *_workspace_bytes queries) and returns 0 on success or a negative GSB200_E_* code
 * (gsb200_error_string() gives the text).  The host side (gsplat_b200/*.py: torch.autograd.Function
 * wrappers with the reference's names and argument meaning) owns allocation, autograd and streams.
 *
 * Each function cites the reference operator schema it replaces
 * (/root/reference/gsplat/cuda/ext.cpp) and the Python wrapper that calls it
 * (/root/reference/gsplat/cuda/_wrapper.py).
 *
 * Layout conventions (the reference's): row-major contiguous fp32 unless noted; quaternions wxyz;
 * conics = (a, b, c) upper triangle of the inverse 2-D covariance; radii int32 [.., 2];
 * isect_ids int64 = image << (32 + tile_bits) | tile << 32 | float_bits(depth);
 * flatten_ids int32 index into [I * N].
 */
#ifndef GSPLAT_B200_H
#define GSPLAT_B200_H

#include <stddef.h>
#include <stdint.h>

/* FTheta camera parameters of the 3DGUT entry points (see gsb200_ut_projection_fwd). */
typedef struct
{
    int reference_poly;                /* 0: pixel distance -> angle is the reference polynomial, 1: angle -> pixel distance */
    float pixeldist_to_angle_poly[6];  /* backward polynomial, c0 .. c5 */
    float angle_to_pixeldist_poly[6];  /* forward polynomial, c0 .. c5 */
    float max_angle;                   /* radians from the optical axis */
    float linear_cde[3];               /* c, d, e of the linear map [[c, d], [e, 1]] */
} gsb200_ftheta_params;

#ifdef __cplusplus
extern "C"
{
#endif

#define GSB200_OK 0
#define GSB200_E_INVALID -1     /* bad argument (null pointer, negative size, ...)            */
#define GSB200_E_UNSUPPORTED -2 /* valid in the reference, not built here (camera model, channels, tile size) */
#define GSB200_E_CUDA -3        /* a CUDA runtime call / kernel launch failed (see gsb200_last_cuda_error) */
#define GSB200_E_WORKSPACE -4   /* workspace too small                                        */
#define GSB200_E_KEYBITS -5     /* (image, tile) id needs more than 32 key bits (csrc/Intersect.cpp:219-228) */

    const char *gsb200_version(void);
    /* sha256 (hex) over the CUDA sources and headers this binary was built from (gsplat_b200/build.py: source_hash()):
     * the built library is shipped next to its sources, this is how the two are matched. */
    const char *gsb200_source_hash(void);
    const char *gsb200_error_string(int code);
    /* cudaGetErrorString of the last CUDA failure seen by this library on the calling thread. */
    const char *gsb200_last_cuda_error(void);
    /* Bits needed to index `count` items (csrc/MathUtils.h:26-36 bits_for_count). Host-only. */
    uint32_t gsb200_bits_for_count(int64_t count);
    /* 1 when colour channel count D is compiled into the rasterizer (Config.h GSPLAT_NUM_CHANNELS analogue). */
    int gsb200_raster_supports_channels(int D);

    /* ---- quat_scale_to_covar_preci / _bwd : ext.cpp:984-991, _wrapper.py:657-716 ----
     * covars / precis: [N,3,3] or [N,6] when triu; either may be NULL (not requested). */
    int gsb200_quat_scale_to_covar_preci_fwd(
        int64_t N, const float *quats, const float *scales, int triu, float *covars, float *precis, void *stream
    );
    int gsb200_quat_scale_to_covar_preci_bwd(
        int64_t N, const float *quats, const float *scales, int triu, const float *v_covars, const float *v_precis,
        float *v_quats, float *v_scales, void *stream
    );

    /* ---- projection_ewa_3dgs_fused / _bwd : ext.cpp:1052-1063, _wrapper.py:819-963, 966-1063 ----
     * means [B,N,3]; covars [B,N,6] XOR (quats [B,N,4], scales [B,N,3]); opacities [B,N] or NULL;
     * viewmats [B,C,4,4]; Ks [B,C,3,3].  Outputs [B,C,N,*]; compensations NULL unless requested.
     * Culled gaussians get radii = 0 and ZEROED float outputs (the reference leaves them
     * uninitialised, csrc/Projection.cpp:395-404).  camera_model: 0 = pinhole (others: UNSUPPORTED). */
    int gsb200_projection_fwd(
        int64_t B, int64_t C, int64_t N, const float *means, const float *covars, const float *quats,
        const float *scales, const float *opacities, const float *viewmats, const float *Ks, uint32_t image_width,
        uint32_t image_height, float eps2d, float near_plane, float far_plane, float radius_clip, int camera_model,
        int32_t *radii, float *means2d, float *depths, float *conics, float *compensations, void *stream
    );
    /* v_* inputs are addressed as ptr[row * stride + k] with row = (b*C + c)*N + n, so that they may be
     * views into a packed gradient record (stride in floats; 2 / 1 / 3 / 1 for contiguous tensors).
     * Outputs are fully written (no pre-zeroing needed): v_means [B,N,3]; v_covars [B,N,6] or
     * (v_quats [B,N,4], v_scales [B,N,3]); v_viewmats [B,C,4,4] or NULL. Deterministic (no atomics
     * except for v_viewmats). */
    int gsb200_projection_bwd(
        int64_t B, int64_t C, int64_t N, const float *means, const float *covars, const float *quats,
        const float *scales, const float *viewmats, const float *Ks, uint32_t image_width, uint32_t image_height,
        float eps2d, int camera_model, const int32_t *radii, const float *conics, const float *compensations,
        const float *v_means2d, int64_t v_means2d_stride, const float *v_depths, int64_t v_depths_stride,
        const float *v_conics, int64_t v_conics_stride, const float *v_compensations, float *v_means,
        float *v_covars, float *v_quats, float *v_scales, float *v_viewmats, void *stream
    );

    /* ---- spherical_harmonics / _bwd : ext.cpp:994-1002, _wrapper.py:436-489 ----
     * Dense layout: means [B,N,3], viewmats [B,C,4,4], coeffs [N,K,D], masks [B,C,N] (bool bytes) or NULL
     * -> colors [B,C,N,D]; masked rows are written as 0.  degree in 0..4, (degree+1)^2 <= K. */
    int gsb200_sh_fwd(
        int64_t B, int64_t C, int64_t N, int64_t K, int64_t D, int degrees_to_use, const float *means,
        const float *viewmats, const float *coeffs, const uint8_t *masks, float *colors, void *stream
    );
    /* v_coeffs [N,K,D] fully written (zeros for unused bands / masked rows); v_means [B,N,3] or NULL;
     * v_dirsum [B,C,3] or NULL: per-image sum of the view-direction gradient, from which the caller forms
     * v_viewmats (dir = mean + R^T t; compute_v_viewmats of the reference schema). */
    int gsb200_sh_bwd(
        int64_t B, int64_t C, int64_t N, int64_t K, int64_t D, int degrees_to_use, const float *means,
        const float *viewmats, const float *coeffs, const uint8_t *masks, const float *v_colors, float *v_coeffs,
        float *v_means, float *v_dirsum, void *stream
    );

    /* ---- fused projection + conic + SH->RGB : the orchestrator's default training path
     * (csrc/Rendering.cpp:976-1117: projection_ewa_3dgs_fused then assemble_proj_features with
     * color_post = max(x + 0.5, 0)).  One pass over the gaussians, B = 1, D = 3, quats/scales input.
     * colors [C,N,3] = max(SH + 0.5, 0) for visible gaussians, 0 otherwise; a colour exactly on the kink
     * (SH + 0.5 == 0) is stored as -0.f, one clamped from below as +0.f, and gsb200_project_sh_bwd reads that zero's sign.
     * quats and sh_coeffs must be 16-byte aligned (128-bit loads), else GSB200_E_INVALID; the same holds for
     * gsb200_project_sh_fwd_rows, and for quats, sh_coeffs, v_quats and v_sh_coeffs of gsb200_project_sh_bwd. */
    int gsb200_project_sh_fwd(
        int64_t C, int64_t N, int64_t K, int degrees_to_use, const float *means, const float *quats,
        const float *scales, const float *opacities, const float *sh_coeffs, const float *viewmats, const float *Ks,
        uint32_t image_width, uint32_t image_height, float eps2d, float near_plane, float far_plane,
        float radius_clip, int calc_compensations, int32_t *radii, float *means2d, float *depths, float *conics,
        float *compensations, float *colors, void *stream
    );
    /* gsb200_project_sh_fwd (without compensations) whose epilogue also hands the two following stages what they would
     * otherwise recompute (round 2): tiles_per_gauss int32 [C,N] and totals int64 [3] exactly as
     * gsb200_isect_count_totals computes them from this call's means2d / radii / conics and the INPUT opacities
     * (AccuTile test, csrc/IntersectTile.cu:83-207), and row_records, 64 bytes per (camera, gaussian) row, 16-byte
     * aligned: {mean2d + axis-aligned half extents | ellipse axis + oriented half extents | pre-scaled conic + opacity |
     * r g b 0} -- the per-intersection record of the compositing kernels, so that gsb200_raster_fwd_rows only gathers.
     * Only rows with radii > 0 are written. */
    int gsb200_project_sh_fwd_rows(
        int64_t C, int64_t N, int64_t K, int degrees_to_use, const float *means, const float *quats,
        const float *scales, const float *opacities, const float *sh_coeffs, const float *viewmats, const float *Ks,
        uint32_t image_width, uint32_t image_height, float eps2d, float near_plane, float far_plane,
        float radius_clip, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, int32_t *radii,
        float *means2d, float *depths, float *conics, float *colors, void *row_records, int32_t *tiles_per_gauss,
        int64_t *totals, void *stream
    );
    /* Backward of the fused pass.  v_colors is the gradient w.r.t. the post-activation colours; it passes where the
     * stored colour is positive or -0.f (SH + 0.5 >= 0: at the kink the sub-gradient torch.clamp_min takes) and is
     * blocked at +0.f, so colours clamped by max(x, 0) elsewhere keep the mask colour > 0.  All outputs fully written;
     * deterministic.  seen_bits (optional,
     * ceil(N / 32) words): bit n%32 of word n/32 = gaussian n is visible in some camera of this call, i.e. its
     * gradient rows are not all zero -- the row bitmap gsb200_rows_allreduce_f32 consumes. */
    int gsb200_project_sh_bwd(
        int64_t C, int64_t N, int64_t K, int degrees_to_use, const float *means, const float *quats,
        const float *scales, const float *sh_coeffs, const float *viewmats, const float *Ks, uint32_t image_width,
        uint32_t image_height, float eps2d, const int32_t *radii, const float *conics, const float *compensations,
        const float *colors, const float *v_means2d, int64_t v_means2d_stride, const float *v_depths,
        int64_t v_depths_stride, const float *v_conics, int64_t v_conics_stride, const float *v_colors,
        int64_t v_colors_stride, const float *v_compensations, float *v_means, float *v_quats, float *v_scales,
        float *v_sh_coeffs, uint32_t *seen_bits, void *stream
    );

    /* ---- spherical harmonics on packed rows (reference: spherical_harmonics with batch_ids / camera_ids /
     * gaussian_ids, ext.cpp:994-1002, rendering.py:1001-1010).  Row i = (batch_ids[i], camera_ids[i],
     * gaussian_ids[i]); coeffs stay [N, K, D] and are indexed in the kernel.  colors / v_colors [nnz, D].
     * bwd: v_coeffs [N,K,D], v_means [B*N,3] (or NULL), v_dirsum [B*C,3] (or NULL) are zeroed here, then summed. */
    int gsb200_sh_rows_fwd(
        int64_t nnz, int64_t B, int64_t C, int64_t N, int64_t K, int64_t D, int degrees_to_use, const float *means,
        const float *viewmats, const float *coeffs, const int64_t *batch_ids, const int64_t *camera_ids,
        const int64_t *gaussian_ids, float *colors, void *stream
    );
    int gsb200_sh_rows_bwd(
        int64_t nnz, int64_t B, int64_t C, int64_t N, int64_t K, int64_t D, int degrees_to_use, const float *means,
        const float *viewmats, const float *coeffs, const int64_t *batch_ids, const int64_t *camera_ids,
        const int64_t *gaussian_ids, const float *v_colors, float *v_coeffs, float *v_means, float *v_dirsum,
        void *stream
    );

    /* ---- projection_ewa_3dgs_packed / _bwd : ext.cpp:1065-1077, _wrapper.py:1065-1191, host
     * csrc/Projection.cpp:858-1260, kernel csrc/ProjectionEWA3DGSPacked.cu ----
     * Two passes, nothing of size B*C*N is allocated.  Pass 1 leaves per-block counts and their scan in
     * `workspace` (gsb200_projection_packed_workspace_bytes) and the row total in *nnz_dev (device int32);
     * the caller reads it, allocates the [nnz, ...] outputs and runs pass 2 with the SAME workspace.
     * Rows are in ascending (batch, camera, gaussian) order; ids are int64 like the reference's; indptr
     * int32 [B*C + 1].  compensations NULL = not computed (and opacities are culled unscaled). */
    size_t gsb200_projection_packed_workspace_bytes(int64_t B, int64_t C, int64_t N);
    int gsb200_projection_packed_count(
        int64_t B, int64_t C, int64_t N, const float *means, const float *covars, const float *quats,
        const float *scales, const float *opacities, const float *viewmats, const float *Ks, uint32_t image_width,
        uint32_t image_height, float eps2d, float near_plane, float far_plane, float radius_clip,
        int calc_compensations, int camera_model, void *workspace, size_t workspace_bytes, int32_t *nnz_dev,
        void *stream
    );
    int gsb200_projection_packed_emit(
        int64_t B, int64_t C, int64_t N, const float *means, const float *covars, const float *quats,
        const float *scales, const float *opacities, const float *viewmats, const float *Ks, uint32_t image_width,
        uint32_t image_height, float eps2d, float near_plane, float far_plane, float radius_clip, int camera_model,
        const void *workspace, int32_t *indptr, int64_t *batch_ids, int64_t *camera_ids, int64_t *gaussian_ids,
        int32_t *radii, float *means2d, float *depths, float *conics, float *compensations, void *stream
    );
    /* sparse_grad != 0: one gradient row per packed row (v_means [nnz,3], v_covars [nnz,6] | v_quats [nnz,4] +
     * v_scales [nnz,3]; the caller wraps them as COO over gaussian_ids, Projection.cpp:1188-1206); otherwise
     * dense [B*N, *] outputs (zero-initialised here, summed over cameras with atomics). */
    int gsb200_projection_packed_bwd(
        int64_t B, int64_t C, int64_t N, int64_t nnz, const float *means, const float *covars, const float *quats,
        const float *scales, const float *viewmats, const float *Ks, uint32_t image_width, uint32_t image_height,
        float eps2d, int camera_model, const int64_t *batch_ids, const int64_t *camera_ids,
        const int64_t *gaussian_ids, const float *conics, const float *compensations, const float *v_means2d,
        int64_t v_means2d_stride, const float *v_depths, int64_t v_depths_stride, const float *v_conics,
        int64_t v_conics_stride, const float *v_compensations, int sparse_grad, float *v_means, float *v_covars,
        float *v_quats, float *v_scales, float *v_viewmats, void *stream
    );

    /* ---- intersect_tile : ext.cpp:1022-1026, _wrapper.py:1196-1266, host csrc/Intersect.cpp:170-329 ----
     * Unsorted output (the reference's sort=False), in row order.
     * Pass 1: tiles_per_gauss int32 [I*N] and their inclusive scan cum_tiles int64 [I*N].  conics + opacities
     * given -> AccuTile/SNUGBOX ellipse test, else AABB from radii.  The caller reads cum_tiles[I*N-1]
     * (= n_isects) to size the pass-2 outputs. */
    size_t gsb200_isect_scan_workspace_bytes(int64_t n_elements);
    int gsb200_isect_count(
        int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *conics,
        const float *opacities, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        int32_t *tiles_per_gauss, int64_t *cum_tiles, void *workspace, size_t workspace_bytes, void *stream
    );
    /* Pass 2: isect_ids int64 [n_isects], flatten_ids int32 [n_isects], emitted in row order.  Packed layout
     * (reference packed=True): pass image_ids int64 [N] (the image of each of the N rows); pass 1 is then
     * called with I = 1. */
    int gsb200_isect_emit(
        int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *depths, const float *conics,
        const float *opacities, const int64_t *cum_tiles, const int64_t *image_ids, uint32_t tile_size,
        uint32_t tile_width, uint32_t tile_height, int64_t *isect_ids, int32_t *flatten_ids, void *stream
    );
    /* Sorted output, first pass: the row-order count, and the totals the host reads -- totals[0] = n_isects,
     * totals[1] = rows that have tiles, totals[2] = largest tile count of a row (max_tiles_hint of gsb200_isect_sorted:
     * picks the one-thread-per-gaussian or the warp-cooperative emit kernel).  totals is int64 [3].  Rows as in
     * gsb200_isect_sorted: I*N, or N when image_ids int64 [N] is given.  tile_mask NULL, or uint8 [I, th, tw]: a row
     * then counts only the tiles whose byte is set, and a row whose image lies outside [0, I) counts none. */
    int gsb200_isect_count_totals(
        int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *conics, const float *opacities,
        const int64_t *image_ids, const uint8_t *tile_mask, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        int32_t *tiles_per_gauss, int64_t *totals, void *stream
    );
    /* Narrow keys (round 2): the rows are emitted in depth order, so the S-sized sort only needs the dense tile id
     * image * n_tiles + tile, as a key_bytes-wide (2 when I * n_tiles <= 65536, else 4) unsigned integer.
     * gsb200_isect_ids_from_tilekeys rebuilds the reference's sorted int64 isect_ids ((image << tile_bits | tile) << 32 |
     * depth bits; depths is indexed by flatten_ids) from the sorted tile ids of gsb200_isect_sorted, for callers that ask
     * for them. */
    int gsb200_isect_ids_from_tilekeys(
        int64_t n_isects, int key_bytes, const void *tile_keys, const int32_t *flatten_ids, const float *depths, int64_t I,
        uint32_t tile_width, uint32_t tile_height, int64_t *isect_ids, void *stream
    );
    /* The sorted intersection stage in ONE call, sized by capacities (round 2): rows-with-tiles compaction, depth
     * order, scan, emission of (dense tile id, row) pairs, stable sort on the tile id, offsets.  Inputs: the per-row tile
     * counts and `totals` (int64 [3], DEVICE memory) of gsb200_isect_count_totals / gsb200_project_sh_fwd_rows.
     * rows = I*N, or N when image_ids int64 [N] (packed layout, the image of each row) is given; I is always the number
     * of images (tile ids, offsets) and total_rows of the workspace size is that row count.  Every
     * launch is sized by cap_vis (<= rows) and cap_isects; the real counts are read on the device: entries past
     * totals[0] in tile_keys / flatten_ids ([cap_isects] each) are padding, nothing is written past a capacity, and
     * offsets int32 [I, th, tw] is exact whenever totals[1] <= cap_vis and totals[0] <= cap_isects.  A caller may
     * therefore launch with PREDICTED capacities before it has read the totals (the host read then overlaps this work
     * instead of idling the GPU: the sync being hidden is the reference's csrc/Intersect.cpp:258-259), use the first
     * totals[0] entries if both counts fit, and otherwise call again with capacities = totals.  key_bytes: 2 when
     * I * th * tw <= 65536, else 4.  tile_mask NULL, or the uint8 [I, th, tw] mask the counts were taken with: only the
     * tiles it sets are emitted. */
    size_t gsb200_isect_sorted_workspace_bytes(
        int64_t I, int64_t total_rows, int64_t cap_vis, int64_t cap_isects, int key_bytes, uint32_t tile_width,
        uint32_t tile_height
    );
    int gsb200_isect_sorted(
        int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *depths, const float *conics,
        const float *opacities, const int64_t *image_ids, const uint8_t *tile_mask, uint32_t tile_size, uint32_t tile_width,
        uint32_t tile_height, const int32_t *tiles_per_gauss, const int64_t *totals, int64_t cap_vis, int64_t cap_isects,
        int64_t max_tiles_hint, int key_bytes, void *tile_keys, int32_t *flatten_ids, int32_t *offsets, void *workspace,
        size_t workspace_bytes, void *stream
    );
    /* Publishes totals (int64 [3], device) into host_mapped (int64 [4], pinned / mapped host memory) with system-scope
     * stores from a one-warp kernel, then writes seq into host_mapped[3]: the host polls that word instead of waiting for
     * a copy (which takes a copy engine and queues behind PCIe uploads). */
    int gsb200_publish_totals(const int64_t *totals, int64_t *host_mapped, int64_t seq, void *stream);
    /* ---- intersect_offset : ext.cpp:1027, _wrapper.py:1328-1347 ---- offsets int32 [I, th, tw]. */
    int gsb200_isect_offsets(
        int64_t n_isects, const int64_t *isect_ids, int64_t I, uint32_t tile_width, uint32_t tile_height,
        int32_t *offsets, void *stream
    );

    /* Stage 1 of gsb200_raster_fwd on its own: gathers the depth-sorted per-intersection records into `records`
     * (gsb200_raster_records_bytes) and writes the longest-list-first tile order.  gsb200_raster_fwd does this itself; a
     * binding that does not keep `records` alive between forward and backward (INTEGRATION.md section B) calls this
     * in its backward, then gsb200_raster_bwd. */
    int gsb200_raster_pack(
        int64_t I, int D, const float *means2d, const float *conics, const float *colors, const float *opacities,
        uint32_t tile_width, uint32_t tile_height, const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects,
        void *records, void *stream
    );
    /* ---- rasterize_to_pixels_3dgs / _bwd : ext.cpp:1079-1089, _wrapper.py:1497-1562, 2010-2117 ----
     * Dense layout: means2d [I,N,2] conics [I,N,3] colors [I,N,D] opacities [I,N]
     * backgrounds [I,D] or NULL, masks [I,th,tw] bool bytes or NULL, offsets [I,th,tw], flatten_ids [n_isects].
     * tile_size must be 16.  `records` is caller scratch of gsb200_raster_records_bytes(n_isects, D, I*th*tw):
     * the forward packs the depth-sorted per-intersection records there (TMA-streamed by both passes)
     * plus a longest-list-first tile dispatch order; the caller keeps it alive for the backward.
     * Outputs: render_colors [I,H,W,D], render_alphas [I,H,W,1], last_ids int32 [I,H,W]. */
    size_t gsb200_raster_records_bytes(int64_t n_isects, int D, int64_t n_tiles);
    int gsb200_raster_fwd(
        int64_t I, int64_t N, int D, const float *means2d, const float *conics, const float *colors,
        const float *opacities, const float *backgrounds, const uint8_t *masks, uint32_t image_width,
        uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, const int32_t *offsets,
        const int32_t *flatten_ids, int64_t n_isects, void *records, float *render_colors, float *render_alphas,
        int32_t *last_ids, void *stream
    );
    /* gsb200_raster_fwd for D <= 4 from the row records of gsb200_project_sh_fwd_rows (the gaussians' means2d / conics /
     * colours / opacities are read from there); same outputs, same `records` for gsb200_raster_bwd. */
    int gsb200_raster_fwd_rows(
        int64_t I, int64_t N, int D, const void *row_records, const float *backgrounds, const uint8_t *masks,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, void *records, float *render_colors,
        float *render_alphas, int32_t *last_ids, void *stream
    );
    /* The gradients are ACCUMULATED into v_grad_records, one record per gaussian row g in [0, I*N): a row of
     * round_up4(6 + D + 2*absgrad) floats laid out
     *     [v_means2d 2 | v_conics 3 | v_opacities 1 | v_colors D | v_means2d_abs 2 if absgrad | zero pad].
     * The caller zero-fills the records; their base must be 16-byte aligned (GSB200_E_INVALID otherwise) and
     * rows * row width must stay below 2^32 (GSB200_E_UNSUPPORTED otherwise).
     * v_render_alphas may be NULL (no gradient flows into render_alphas). */
    int gsb200_raster_bwd(
        int64_t I, int64_t N, int D, const float *backgrounds, const uint8_t *masks, uint32_t image_width,
        uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, const int32_t *offsets,
        const int32_t *flatten_ids, int64_t n_isects, const void *records, const float *render_alphas,
        const int32_t *last_ids, const float *v_render_colors, const float *v_render_alphas, int absgrad,
        float *v_grad_records, void *stream
    );

    /* ---- sparse pixels: build_sparse_tile_layout, isect_tiles_sparse, rasterize_to_pixels_sparse
     * (_wrapper.py:1352-1665).  tile_size must be 16.
     * Layout: pixels int32 [P, 2] (row, col) inside the tile grid, image_ids int32 [P] in [0, n_images) (the caller
     * checks both).  gsb200_sparse_layout_sort sorts one key (dense tile id << 8 | in-tile position) per pixel and
     * writes the number of active tiles to n_active (device int64); the caller reads it, then
     * gsb200_sparse_layout_finish (same workspace) writes active_tiles int32 [AT] ascending, active_tile_mask bool
     * bytes [n_images, th, tw], tile_pixel_mask uint64 [AT, 4] (raster-order in-tile bits), tile_pixel_cumsum int64
     * [AT] (inclusive) and pixel_map int64 [P] (pixel index in (tile, in-tile) order). */
    size_t gsb200_sparse_layout_workspace_bytes(int64_t P, int64_t n_images, uint32_t tile_width, uint32_t tile_height);
    int gsb200_sparse_layout_sort(
        int64_t P, const int32_t *pixels, const int32_t *image_ids, int64_t n_images, uint32_t tile_size,
        uint32_t tile_width, uint32_t tile_height, void *workspace, size_t workspace_bytes, int64_t *n_active, void *stream
    );
    int gsb200_sparse_layout_finish(
        int64_t P, int64_t n_images, uint32_t tile_width, uint32_t tile_height, int64_t n_active, const void *workspace,
        size_t workspace_bytes, int32_t *active_tiles, uint8_t *active_tile_mask, uint64_t *tile_pixel_mask,
        int64_t *tile_pixel_cumsum, int64_t *pixel_map, void *stream
    );
    /* Tile intersection restricted to the tiles of active_tile_mask: gsb200_isect_count_totals and gsb200_isect_sorted
     * with that mask as tile_mask (dense rows [I, N], or packed rows [N] with int64 image_ids), then
     * gsb200_isect_active_offsets: tile_offsets int32 [n_active + 1] = the sorted stage's offsets [I, th, tw] at each
     * of active_tiles int32 [n_active], and n_isects.  An active tile id outside [0, I * th * tw) gets n_isects. */
    int gsb200_isect_active_offsets(
        int64_t n_active, const int32_t *active_tiles, int64_t I, uint32_t tile_width, uint32_t tile_height,
        const int32_t *offsets, int64_t n_isects, int32_t *tile_offsets, void *stream
    );
    /* Compositing of the requested pixels only: one CTA per active tile, tile_offsets [n_active + 1] of
     * gsb200_isect_active_offsets and flatten_ids of the masked gsb200_isect_sorted, the layout tensors from
     * gsb200_sparse_layout_finish.  Gaussian rows and backgrounds [n_images, D] / masks [n_images, th, tw] as in
     * gsb200_raster_fwd; `records` of gsb200_raster_records_bytes(n_isects, D, n_active).  Outputs in the original
     * pixel order: render_colors [P, D],
     * render_alphas [P], last_ids int32 [P].  The backward accumulates into the gradient records of gsb200_raster_bwd,
     * one per gaussian row g in [0, n_rows); v_render_colors [P, D], v_render_alphas [P] or NULL. */
    int gsb200_raster_sparse_fwd(
        int D, const float *means2d, const float *conics, const float *colors, const float *opacities,
        const float *backgrounds, const uint8_t *masks, uint32_t image_width, uint32_t image_height, uint32_t tile_size,
        uint32_t tile_width, uint32_t tile_height, int64_t n_active, const int32_t *active_tiles,
        const int32_t *tile_offsets, const int32_t *flatten_ids, int64_t n_isects, const uint64_t *tile_pixel_mask,
        const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, void *records, float *render_colors,
        float *render_alphas, int32_t *last_ids, void *stream
    );
    int gsb200_raster_sparse_bwd(
        int64_t n_rows, int D, const float *backgrounds, const uint8_t *masks, uint32_t image_width, uint32_t image_height,
        uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, int64_t n_active, const int32_t *active_tiles,
        const int32_t *tile_offsets, const int32_t *flatten_ids, int64_t n_isects, const uint64_t *tile_pixel_mask,
        const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, const void *records, const float *render_alphas,
        const int32_t *last_ids, const float *v_render_colors, const float *v_render_alphas, int absgrad,
        float *v_grad_records, void *stream
    );

    /* ---- 2DGS (surfel splatting), dense layout: projection_2dgs_fused / _bwd and rasterize_to_pixels_2dgs / _bwd
     * (ext.cpp, _wrapper.py:2633-2727, 2918-3150; kernels csrc/Projection2DGSFused.cu,
     * csrc/RasterizeToPixels2DGSSerialBatch{Fwd,Bwd}.cu).
     * Projection: means [B,N,3], quats [B,N,4], scales [B,N,3] (scales[..., 2] unused), viewmats [B,C,4,4], Ks [B,C,3,3].
     * Outputs [B,C,N,*]: radii int32 [.., 2], means2d [.., 2], depths, ray_transforms [.., 3, 3] (row-major
     * K * [R rot(q) diag(s0, s1, 1) columns 0, 1 | camera-space mean]), normals [.., 3] (camera space, facing the camera).
     * Culled rows (near / far, degenerate, radius_clip, off-screen) get radii = 0 and zero float outputs. */
    int gsb200_surfel_projection_fwd(
        int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales,
        const float *viewmats, const float *Ks, uint32_t image_width, uint32_t image_height, float near_plane,
        float far_plane, float radius_clip, int32_t *radii, float *means2d, float *depths, float *ray_transforms,
        float *normals, void *stream
    );
    /* All v_* inputs contiguous [B,C,N,*].  v_means [B,N,3], v_quats [B,N,4], v_scales [B,N,3] (v_scales[..., 2] = 0) are
     * fully written, summed over the cameras without atomics; v_viewmats [B,C,4,4] or NULL is zeroed here, then
     * accumulated. */
    int gsb200_surfel_projection_bwd(
        int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales,
        const float *viewmats, const float *Ks, const int32_t *radii, const float *ray_transforms, const float *v_means2d,
        const float *v_depths, const float *v_ray_transforms, const float *v_normals, float *v_means, float *v_quats,
        float *v_scales, float *v_viewmats, void *stream
    );
    /* Compositing, dense rows: means2d [I,N,2], ray_transforms [I,N,3,3], colors [I,N,D] (the last channel is the depth
     * that distortion and median depth use), opacities [I,N], normals [I,N,3], backgrounds [I,D] or NULL, masks
     * [I,th,tw] bool bytes or NULL, offsets [I,th,tw], flatten_ids [n_isects].  tile_size must be 16; D one of the
     * channel counts of gsb200_raster_supports_channels.  Outputs: render_colors [I,H,W,D], render_alphas, render_distort,
     * render_median [I,H,W,1], render_normals [I,H,W,3], last_ids and median_ids int32 [I,H,W] (indices into
     * flatten_ids). */
    int gsb200_surfel_raster_fwd(
        int64_t I, int64_t N, int D, const float *means2d, const float *ray_transforms, const float *colors,
        const float *opacities, const float *normals, const float *backgrounds, const uint8_t *masks,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, float *render_colors, float *render_alphas,
        float *render_normals, float *render_distort, float *render_median, int32_t *last_ids, int32_t *median_ids,
        void *stream
    );
    /* Gradient outputs are ACCUMULATED into contiguous rows (caller zero-initialises): v_means2d [I,N,2], v_ray_transforms
     * [I,N,3,3], v_colors [I,N,D], v_opacities [I,N], v_normals [I,N,3], v_densify [I,N,2] (v_ray_transforms[.., 0:2, 2]
     * * ray_transforms[.., 2, 2]), v_means2d_abs [I,N,2] or NULL.  v_render_alphas / _normals / _distort / _median may
     * be NULL (no gradient flows into that output). */
    int gsb200_surfel_raster_bwd(
        int64_t I, int64_t N, int D, const float *means2d, const float *ray_transforms, const float *colors,
        const float *opacities, const float *normals, const float *backgrounds, const uint8_t *masks,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, const float *render_colors,
        const float *render_alphas, const int32_t *last_ids, const int32_t *median_ids, const float *v_render_colors,
        const float *v_render_alphas, const float *v_render_normals, const float *v_render_distort,
        const float *v_render_median, float *v_means2d, float *v_ray_transforms, float *v_colors, float *v_opacities,
        float *v_normals, float *v_densify, float *v_means2d_abs, void *stream
    );
    /* Surfel compositing of the requested pixels only (rasterize_to_pixels_2dgs_sparse; no reference counterpart): one
     * CTA per active tile, the layout and lists of gsb200_raster_sparse_fwd.  The surfel rows, backgrounds [n_images, D]
     * and masks [n_images, th, tw] are those of gsb200_surfel_raster_fwd with n_rows rows in all (n_rows * 9 < 2^31).
     * Outputs in the original pixel order: render_colors [P, D], render_alphas, render_distort, render_median [P],
     * render_normals [P, 3], last_ids and median_ids int32 [P]; each the dense forward's value at that pixel.  The
     * backward ACCUMULATES into the gradient rows of gsb200_surfel_raster_bwd ([n_rows, *], caller zero-initialises);
     * v_render_* [P, *] with the same NULL rules. */
    int gsb200_surfel_raster_sparse_fwd(
        int64_t n_rows, int D, const float *means2d, const float *ray_transforms, const float *colors,
        const float *opacities, const float *normals, const float *backgrounds, const uint8_t *masks, uint32_t image_width,
        uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, int64_t n_active,
        const int32_t *active_tiles, const int32_t *tile_offsets, const int32_t *flatten_ids, int64_t n_isects,
        const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, float *render_colors,
        float *render_alphas, float *render_normals, float *render_distort, float *render_median, int32_t *last_ids,
        int32_t *median_ids, void *stream
    );
    int gsb200_surfel_raster_sparse_bwd(
        int64_t n_rows, int D, const float *means2d, const float *ray_transforms, const float *colors,
        const float *opacities, const float *normals, const float *backgrounds, const uint8_t *masks, uint32_t image_width,
        uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, int64_t n_active,
        const int32_t *active_tiles, const int32_t *tile_offsets, const int32_t *flatten_ids, int64_t n_isects,
        const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map,
        const float *render_colors, const float *render_alphas, const int32_t *last_ids, const int32_t *median_ids,
        const float *v_render_colors, const float *v_render_alphas, const float *v_render_normals,
        const float *v_render_distort, const float *v_render_median, float *v_means2d, float *v_ray_transforms,
        float *v_colors, float *v_opacities, float *v_normals, float *v_densify, float *v_means2d_abs, void *stream
    );

    /* ---- rasterize_to_indices_in_range / _2dgs (_wrapper.py:2486, :3154; kernels
     * csrc/RasterizeToIndices{3,2}DGSSerialBatch.cu, host csrc/Rasterization.cpp:954-1090) ----
     * The (pixel, gaussian) pairs the compositing forward (gsb200_raster_fwd / gsb200_surfel_raster_fwd) composites when
     * each pixel walks only the batches [range_start, range_end) of 256 records of its tile's list, starting from its
     * transmittance (float32 [I,H,W]).  A pair whose next transmittance is <= 1e-4 stops the pixel and is not a pair.
     * Dense rows: means2d [I,N,2], conics [I,N,3] / ray_transforms [I,N,3,3], opacities [I,N]; offsets [I,th,tw];
     * tile_size must be 16.  range_start / range_end >= 0; range_end past every list means "to the end".
     * Two calls with one workspace of gsb200_indices_workspace_bytes(I*H*W) bytes: emit = 0 counts every pixel's
     * pairs and writes their total to total (device int64 [1]); the caller reads it, then emit = 1 writes gaussian_ids
     * (flatten id % N), pixel_ids (row-major in the image) and image_ids, int64 [total], pixel-major over
     * (image, row, col) and front to back within a pixel. */
    size_t gsb200_indices_workspace_bytes(int64_t n_pixels);
    int gsb200_raster_indices(
        int64_t I, int64_t N, const float *means2d, const float *conics, const float *opacities,
        const float *transmittances, uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width,
        uint32_t tile_height, const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t range_start,
        int64_t range_end, int emit, void *workspace, size_t workspace_bytes, int64_t *total, int64_t *gaussian_ids,
        int64_t *pixel_ids, int64_t *image_ids, void *stream
    );
    int gsb200_surfel_indices(
        int64_t I, int64_t N, const float *means2d, const float *ray_transforms, const float *opacities,
        const float *transmittances, uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width,
        uint32_t tile_height, const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t range_start,
        int64_t range_end, int emit, void *workspace, size_t workspace_bytes, int64_t *total, int64_t *gaussian_ids,
        int64_t *pixel_ids, int64_t *image_ids, void *stream
    );

    /* ---- per-pixel contributor queries: rasterize_num_contributing_gaussians, rasterize_contributing_gaussian_ids,
     * rasterize_top_contributing_gaussian_ids and their _sparse forms (_wrapper.py:1668-2008, host
     * csrc/Rasterization.cpp:1380-1620).  Each pixel walks its tile's full list from T = 1 with the decisions of
     * gsb200_raster_indices (and so of gsb200_raster_fwd).  Rows: means2d [R,2], conics [R,3], opacities [R]; ids are
     * flatten id % N (dense rows [I,N,*]: the gaussian index; packed rows [nnz,*]: pass N = nnz, the row index).
     * Dense: offsets [I,th,tw], active_tiles = null, outputs row (image, y, x) of I*H*W.  Sparse (active_tiles non-null):
     * the layout of gsb200_sparse_layout_* and the per-active-tile offsets [n_active + 1] of gsb200_isect_active_offsets,
     * outputs row = the pixel's index in the caller's list [P].  tile_size must be 16.  Every pixel is written.
     *   count: counts int32 [rows] contributing pairs, alphas float32 [rows] (nullable) 1 - final T.
     *   ids:   ids int32 / weights float32 [rows, max_samples]: the first max_samples pairs front to back (later ones
     *          are dropped), weight alpha * T before the pair; -1 / 0 after a pixel's last pair.
     *   top:   ids / weights [rows, num_samples]: the num_samples heaviest pairs (a pair replaces the lightest slot,
     *          the first on ties, only when strictly heavier), front to back, -1 / 0 for empty slots.  num_samples must
     *          lie in [1, gsb200_contrib_max_samples()] (GSB200_E_UNSUPPORTED above it).
     * gsb200_contrib_max_samples: the largest num_samples the current device's opt-in shared memory per block holds, or
     * GSB200_E_CUDA without a device. */
    int gsb200_contrib_max_samples(void);
    int gsb200_contrib_count(
        int64_t I, int64_t N, const float *means2d, const float *conics, const float *opacities, uint32_t image_width,
        uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, const int32_t *offsets,
        const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
        const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int32_t *counts,
        float *alphas, void *stream
    );
    int gsb200_contrib_ids(
        int64_t I, int64_t N, const float *means2d, const float *conics, const float *opacities, uint32_t image_width,
        uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, const int32_t *offsets,
        const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
        const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int max_samples,
        int32_t *ids, float *weights, void *stream
    );
    int gsb200_contrib_top(
        int64_t I, int64_t N, const float *means2d, const float *conics, const float *opacities, uint32_t image_width,
        uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, const int32_t *offsets,
        const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
        const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int num_samples,
        int32_t *ids, float *weights, void *stream
    );

    /* ---- 2DGS per-pixel contributor queries: rasterize_num_contributing_gaussians_2dgs,
     * rasterize_contributing_gaussian_ids_2dgs, rasterize_top_contributing_gaussian_ids_2dgs and their _sparse forms (the
     * reference has no 2DGS contributor queries).  The arguments, outputs, checks and return codes of gsb200_contrib_*,
     * with ray_transforms [R,3,3] in place of conics; each pixel walks its tile's full list from T = 1 with the decisions
     * of gsb200_surfel_indices (and so of gsb200_surfel_raster_fwd: count's alphas are its render_alphas).  Dense
     * rows [I,N,*]; sparse lists from gsb200_isect_active_offsets on the surfel rows.
     * gsb200_surfel_contrib_max_samples: the num_samples bound of gsb200_surfel_contrib_top, taken from the surfel walk's
     * own staging arrays, or GSB200_E_CUDA without a device. */
    int gsb200_surfel_contrib_max_samples(void);
    int gsb200_surfel_contrib_count(
        int64_t I, int64_t N, const float *means2d, const float *ray_transforms, const float *opacities,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
        const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int32_t *counts,
        float *alphas, void *stream
    );
    int gsb200_surfel_contrib_ids(
        int64_t I, int64_t N, const float *means2d, const float *ray_transforms, const float *opacities,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
        const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int max_samples,
        int32_t *ids, float *weights, void *stream
    );
    int gsb200_surfel_contrib_top(
        int64_t I, int64_t N, const float *means2d, const float *ray_transforms, const float *opacities,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
        const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int num_samples,
        int32_t *ids, float *weights, void *stream
    );

    /* ---- 3DGUT (csrc/ut.cu): camera_model 0 pinhole (OpenCV: radial [B*C, 6], tangential [B*C, 2], thin prism
     * [B*C, 4], each optional; none at all is the perfect pinhole), 2 fisheye (OpenCV: radial [B*C, 4] optional, the
     * other two must be NULL) or 3 FTheta (ftheta non-NULL, the three coefficient arrays NULL); any other model is
     * GSB200_E_UNSUPPORTED.  ftheta is a host pointer, read when the call is made, and must be NULL for the other models.
     * FTheta: the parameters are shared by every camera; each camera's principal point is Ks (cx, cy) + 0.5 (FTheta's
     * image origin is the centre of the first pixel), fx and fy are unused.  reference_poly 0: the backward polynomial
     * (pixel distance -> angle) is the reference and the forward direction inverts it by 3 Newton steps; 1: the
     * forward polynomial (angle -> pixel distance) is, and the unprojection inverts it (a pixel whose last Newton step
     * stays above 1e-6 composites nothing).  Polynomial coefficients are c0 + c1 x + .. + c5 x^5; the image offset is
     * [[c, d], [e, 1]] times the radial offset.  Rays at max_angle or beyond are invalid.
     * global_z_order (projection): 1 culls on and returns the camera-frame z as the depth; 0 (FTheta only, else
     * GSB200_E_UNSUPPORTED) culls on and returns the distance |mean_c| from the camera centre.
     * Shutter: viewmats_rs NULL with rolling_shutter 4 is the global shutter (the pose of viewmats).  viewmats_rs
     * [B*C, 4, 4] (the end-of-frame pose) with rolling_shutter 0 top to bottom, 1 left to right, 2 bottom to top or 3
     * right to left exposes each image row or column at the pose interpolated between the two (translation lerp,
     * rotation slerp) at its relative frame time.  Any other pairing, or a rolling shutter over a single row / column,
     * is GSB200_E_INVALID.  The projection takes the mid-frame pose for the depths and the near / far cull.
     * UT projection: the rows of gsb200_projection_fwd (radii int32 [B,C,N,2], means2d, depths, conics, compensations or
     * NULL), culled rows radii 0 and zero floats; opacities [B,N] or NULL.  alpha^2 * (3 + kappa) must be > 0. */
    int gsb200_ut_projection_fwd(
        int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales, const float *opacities,
        const float *viewmats, const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
        const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
        int global_z_order, uint32_t image_width, uint32_t image_height, float eps2d, float near_plane, float far_plane,
        float radius_clip, float ut_alpha, float ut_beta, float ut_kappa, float ut_in_image_margin_factor,
        int ut_require_all_sigma_points_valid, int32_t *radii, float *means2d, float *depths, float *conics,
        float *compensations, void *stream
    );
    /* Compositing with each gaussian evaluated in 3-D along the pixel's world ray: means/quats/scales [B,N,*], colors
     * [B*C, N, D], opacities [B*C, N], backgrounds [B*C, D] or NULL, masks [B*C, th, tw] or NULL, the lists of
     * isect_offset_encode over the B*C images.  Outputs render_colors [B*C,H,W,D], render_alphas [B*C,H,W], last_ids
     * int32 [B*C,H,W] (-1: none).  The backward ACCUMULATES v_colors and v_opacities (caller zero-initialises) and
     * grad_records float [B*N, 12] (caller zero-initialises), then writes v_means, v_quats, v_scales [B,N,*]. */
    int gsb200_eval3d_fwd(
        int64_t B, int64_t C, int64_t N, int D, const float *means, const float *quats, const float *scales,
        const float *colors, const float *opacities, const float *backgrounds, const uint8_t *masks, const float *viewmats,
        const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
        const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, float *render_colors, float *render_alphas, int32_t *last_ids,
        void *stream
    );
    int gsb200_eval3d_bwd(
        int64_t B, int64_t C, int64_t N, int D, const float *means, const float *quats, const float *scales,
        const float *colors, const float *opacities, const float *backgrounds, const uint8_t *masks, const float *viewmats,
        const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
        const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, const float *render_alphas, const int32_t *last_ids,
        const float *v_render_colors, const float *v_render_alphas, float *grad_records, float *v_colors, float *v_opacities,
        float *v_means, float *v_quats, float *v_scales, void *stream
    );
    /* Eval3d compositing of the requested pixels only (rasterize_to_pixels_eval3d_sparse; no reference counterpart): one
     * CTA per active tile, the layout of gsb200_sparse_layout_* and the per-active-tile lists [n_active + 1] of
     * gsb200_isect_active_offsets on the UT rows.  The other arguments are those of gsb200_eval3d_fwd / _bwd, with
     * backgrounds [B*C, D] and masks [B*C, th, tw] indexed by the layout's image (the flattened (b, c)).  A requested
     * pixel inside the W x H image gets the dense forward's values there; one in the margin of a partial tile gets the
     * background (or 0), alpha 0 and last id -1, and passes no gradient.  Outputs in the original pixel order:
     * render_colors [P, D], render_alphas [P], last_ids int32 [P].  The backward reads render_alphas, last_ids,
     * v_render_colors [P, D] and v_render_alphas [P] (or NULL) per requested pixel and accumulates and writes the
     * gradients of gsb200_eval3d_bwd.  Every check runs before any launch; the return codes are those of the dense
     * entries and of gsb200_raster_sparse_fwd / _bwd. */
    int gsb200_eval3d_sparse_fwd(
        int64_t B, int64_t C, int64_t N, int D, const float *means, const float *quats, const float *scales,
        const float *colors, const float *opacities, const float *backgrounds, const uint8_t *masks, const float *viewmats,
        const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
        const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        int64_t n_active, const int32_t *active_tiles, const int32_t *tile_offsets, const int32_t *flatten_ids,
        int64_t n_isects, const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map,
        float *render_colors, float *render_alphas, int32_t *last_ids, void *stream
    );
    int gsb200_eval3d_sparse_bwd(
        int64_t B, int64_t C, int64_t N, int D, const float *means, const float *quats, const float *scales,
        const float *colors, const float *opacities, const float *backgrounds, const uint8_t *masks, const float *viewmats,
        const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
        const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        int64_t n_active, const int32_t *active_tiles, const int32_t *tile_offsets, const int32_t *flatten_ids,
        int64_t n_isects, const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map,
        const float *render_alphas, const int32_t *last_ids, const float *v_render_colors, const float *v_render_alphas,
        float *grad_records, float *v_colors, float *v_opacities, float *v_means, float *v_quats, float *v_scales,
        void *stream
    );

    /* ---- 3DGUT pair query and per-pixel contributor queries (rasterize_to_indices_in_range_eval3d,
     * rasterize_num_contributing_gaussians_eval3d, rasterize_contributing_gaussian_ids_eval3d,
     * rasterize_top_contributing_gaussian_ids_eval3d and their _sparse forms; the reference has no 3DGUT queries).  Each
     * pixel walks its tile's list with the decisions of gsb200_eval3d_fwd (its ray through the camera model and shutter,
     * the maximum response along it, the stop rule), so count's alphas are its render_alphas.  The geometry and camera
     * arguments are gsb200_eval3d_fwd's (images B*C, flatten ids over [B*C*N], ids = flatten id % N); the rest are those of
     * gsb200_raster_indices / gsb200_contrib_*, with their outputs, sparse layouts and return codes.  A pixel that does
     * not composite (outside the W x H image, or a ray that cannot be unprojected) has no pairs; with an output row it
     * gets count 0 and ids -1 / weights 0.  Checks, all before any launch: the sizes of gsb200_eval3d_fwd, the camera,
     * the sparse layout (active_tiles non-null), then the query's own.
     * gsb200_eval3d_contrib_max_samples: the num_samples bound of gsb200_eval3d_contrib_top for every camera and shutter,
     * or GSB200_E_CUDA without a device. */
    int gsb200_eval3d_indices(
        int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales, const float *opacities,
        const float *viewmats, const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
        const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
        const float *transmittances, uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width,
        uint32_t tile_height, const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t range_start,
        int64_t range_end, int emit, void *workspace, size_t workspace_bytes, int64_t *total, int64_t *gaussian_ids,
        int64_t *pixel_ids, int64_t *image_ids, void *stream
    );
    int gsb200_eval3d_contrib_max_samples(void);
    int gsb200_eval3d_contrib_count(
        int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales, const float *opacities,
        const float *viewmats, const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
        const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
        const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int32_t *counts,
        float *alphas, void *stream
    );
    int gsb200_eval3d_contrib_ids(
        int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales, const float *opacities,
        const float *viewmats, const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
        const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
        const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int max_samples,
        int32_t *ids, float *weights, void *stream
    );
    int gsb200_eval3d_contrib_top(
        int64_t B, int64_t C, int64_t N, const float *means, const float *quats, const float *scales, const float *opacities,
        const float *viewmats, const float *Ks, int camera_model, const float *radial_coeffs, const float *tangential_coeffs,
        const float *thin_prism_coeffs, const gsb200_ftheta_params *ftheta, const float *viewmats_rs, int rolling_shutter,
        uint32_t image_width, uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        const int32_t *offsets, const int32_t *flatten_ids, int64_t n_isects, int64_t n_active, const int32_t *active_tiles,
        const uint64_t *tile_pixel_mask, const int64_t *tile_pixel_cumsum, const int64_t *pixel_map, int num_samples,
        int32_t *ids, float *weights, void *stream
    );

    /* ---- MCMC strategy ops ("next" row): relocation (ext.cpp `relocation`, gsplat/relocation.py:64,
     * csrc/RelocationCUDA.cu:36-80) and in-place position perturbation (csrc/MCMCPerturbCUDA.cu:28-60,
     * gsplat/strategy/ops.py).  ratios int32 [N] already clamped to [1, n_max]; binoms [n_max, n_max]. */
    int gsb200_relocation(
        int64_t N, const float *opacities, const float *scales, const int32_t *ratios, const float *binoms, int n_max,
        float min_opacity, float *new_opacities, float *new_scales, void *stream
    );
    int gsb200_mcmc_perturb_positions(
        int64_t N, float *positions, const float *quats, const float *scales_log, const float *opacities_logit,
        const float *noise, float noise_scale, float t, float k, void *stream
    );

    /* ---- `adam` (ext.cpp, _wrapper.py:419-432, csrc/AdamCUDA.cu:34-70): selective Adam step in place on
     * param / exp_avg / exp_avg_sq [N, D]; rows with valid[n] == 0 (bool bytes, or NULL = all) are skipped. */
    int gsb200_adam(
        int64_t N, int64_t D, float *param, const float *param_grad, float *exp_avg, float *exp_avg_sq,
        const uint8_t *valid, float lr, float b1, float b2, float eps, void *stream
    );

    /* ---- fused photometric L1 of the train step (caller-side fusion; the reference trainer's
     * F.l1_loss(colors, pixels), examples/simple_trainer.py): loss[0] = mean |a - b| (device scalar, deterministic
     * two-level sum); bwd: v_a[i] = v_loss[0] / n * sign(a[i] - b[i]) with v_loss a device scalar. */
    size_t gsb200_l1_loss_workspace_bytes(void);
    int gsb200_l1_loss_fwd(int64_t n, const float *a, const float *b, float *loss, void *workspace, void *stream);
    int gsb200_l1_loss_bwd(int64_t n, const float *a, const float *b, const float *v_loss, float *v_a, void *stream);

    /* Fused SSIM loss of the train step (reference: gsplat/losses.py:110-201 torch_ssim_loss / ssim_loss, the
     * D-SSIM term at examples/simple_trainer.py:951-961; torch path: 11x11 Gaussian window sigma 1.5, zero padding,
     * per channel): loss[0] = 1 - mean SSIM(x, y) over B*C*H*W (device scalar, deterministic fixed-order sum).
     * Images are addressed as p[b*s[0] + c*s[1] + h*s[2] + w*s[3]] (element strides: NCHW views of NHWC renders are
     * read in place).  maps = 3*B*C*H*W floats kept for the backward (NULL: forward only); workspace:
     * gsb200_ssim_workspace_bytes.  Backward: v_x = v_loss[0] * d loss / d x, written through v_strides. */
    size_t gsb200_ssim_workspace_bytes(int64_t B, int64_t C, int64_t H, int64_t W);
    int gsb200_ssim_fwd(
        int64_t B, int64_t C, int64_t H, int64_t W, const float *x, const int64_t *x_strides, const float *y,
        const int64_t *y_strides, float *maps, void *workspace, float *loss, void *stream
    );
    int gsb200_ssim_bwd(
        int64_t B, int64_t C, int64_t H, int64_t W, const float *x, const int64_t *x_strides, const float *y,
        const int64_t *y_strides, const float *maps, const float *v_loss, float *v_x, const int64_t *v_strides, void *stream
    );

    /* ---- view-parallel gradient all-reduce (SURVEY.md section 8e; replaces the NCCL all-reduce of
     * gsplat_b200/distributed.py on NVSwitch systems) over NVLS multicast memory, in place.
     * Every rank calls this on its stream with the SAME n_floats (multiple of 4) and `blocks`:
     *   multicast_ptr   : multicast (all-GPU) address of the symmetric gradient buffer, 16-byte aligned
     *   signal_pads_dev : device array of `world` pointers, entry r = rank r's signal pad (zero-initialised,
     *                     peer-mapped; at least blocks * world * 4 bytes) -- used for the two rank barriers
     * On return (stream order) every rank's buffer holds the element-wise sum over the ranks. */
    int gsb200_nvls_allreduce_f32(
        void *multicast_ptr, int64_t n_floats, int rank, int world, void *const *signal_pads_dev,
        int64_t signal_pad_bytes, int blocks, void *stream
    );

    /* Same contract without the switch reduction (plain peer loads / stores over NVLink): buffers_dev = device
     * array of `world` pointers, entry r = rank r's symmetric buffer.  Moves less than the multicast scheme
     * only for world == 2. */
    int gsb200_p2p_allreduce_f32(
        void *const *buffers_dev, int64_t n_floats, int rank, int world, void *const *signal_pads_dev,
        int64_t signal_pad_bytes, int blocks, void *stream
    );

    /* Row-sparse all-reduce of a structure-of-arrays gradient buffer: n_segs segments of n_rows rows (segment k starts
     * seg_offsets_floats[k] floats into the buffer, seg_widths[k] floats per row); the buffer also holds, at
     * bitmap_offset_floats, every rank's "row touched" bitmap (ceil(n_rows / 32) words, written by
     * gsb200_project_sh_bwd).  A group of 32 rows is moved only if some rank touched it, inside it only the touched
     * rows.  multicast_ptr != NULL: in-switch reduction (multimem.ld_reduce / multimem.st); else peer loads / stores
     * through buffers_dev.  stats (optional device u64) += number of 16-byte vectors this rank reduced. */
    int gsb200_rows_allreduce_f32(
        void *multicast_ptr, void *const *buffers_dev, int n_segs, const int64_t *seg_offsets_floats,
        const int32_t *seg_widths, int64_t n_rows, int64_t bitmap_offset_floats, int rank, int world,
        void *const *signal_pads_dev, int64_t signal_pad_bytes, int blocks, void *stats, void *stream
    );

#ifdef __cplusplus
}
#endif
#endif /* GSPLAT_B200_H */
