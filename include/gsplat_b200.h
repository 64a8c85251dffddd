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
     * colors [C,N,3] = max(SH + 0.5, 0) for visible gaussians, 0 otherwise. */
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
    /* Backward of the fused pass.  v_colors is the gradient w.r.t. the post-activation colours
     * (the relu mask is re-derived).  All outputs fully written; deterministic.  seen_bits (optional,
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
     * Pass 0 (sorted output only): order int32 [rows] = the projected rows in ascending (image, depth bits,
     * row) order, culled rows (radii <= 0) last.  Emitting the intersections in this order leaves only the
     * (image, tile) key bits for the S-sized sort -- same final order as the reference's one stable sort on
     * (image, tile, depth).  rows = I*N, or N when image_ids (packed layout) is given. */
    size_t gsb200_isect_depth_order_workspace_bytes(int64_t I, int64_t total_rows);
    int gsb200_isect_depth_order(
        int64_t I, int64_t N, const int32_t *radii, const float *depths, const int64_t *image_ids, int32_t *order,
        void *workspace, size_t workspace_bytes, void *stream
    );
    /* Pass 1: tiles_per_gauss int32 [I*N] (row order) and the inclusive scan cum_tiles int64 [I*N] of the
     * counts taken in `order` (NULL = row order).  conics + opacities given -> AccuTile/SNUGBOX ellipse test,
     * else AABB from radii.  The caller reads cum_tiles[I*N-1] (= n_isects) to size the pass-2 outputs. */
    size_t gsb200_isect_scan_workspace_bytes(int64_t n_elements);
    int gsb200_isect_count(
        int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *conics,
        const float *opacities, const int32_t *order, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        int32_t *tiles_per_gauss, int64_t *cum_tiles, void *workspace, size_t workspace_bytes, void *stream
    );
    /* Pass 2: isect_ids int64 [n_isects], flatten_ids int32 [n_isects], emitted in `order` (NULL = row order,
     * the reference's unsorted output).  Packed layout (reference packed=True): pass image_ids int64 [N]
     * (the image of each of the N rows); pass 1 is then called with I = 1. */
    int gsb200_isect_emit(
        int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *depths, const float *conics,
        const float *opacities, const int64_t *cum_tiles, const int64_t *image_ids, const int32_t *order,
        uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, int64_t *isect_ids, int32_t *flatten_ids,
        void *stream
    );
    /* Faster pass 0 / 1 for the sorted dense layout (round 2): count first, in row order, and hand the host BOTH totals
     * -- totals[0] = n_isects, totals[1] = rows that have tiles, totals[2] = largest tile count of a row -- in one read; then order ONLY those rows:
     * gsb200_isect_order_visible compacts them (stable), sorts them by (image, depth) and scans their counts in that
     * order (order int32 [n_vis], cum_tiles int64 [n_vis]); gsb200_isect_emit_ordered emits from the n_vis ordered rows
     * (max_tiles_hint = totals[2], the largest tile count of a row, or 0: picks the one-thread-per-gaussian or the
     * warp-cooperative kernel).  totals is int64 [3].
     * Same intersections in the same final order as gsb200_isect_depth_order + gsb200_isect_count + gsb200_isect_emit. */
    int gsb200_isect_count_totals(
        int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *conics, const float *opacities,
        uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, int32_t *tiles_per_gauss, int64_t *totals,
        void *stream
    );
    size_t gsb200_isect_order_visible_workspace_bytes(int64_t I, int64_t total_rows, int64_t n_vis);
    int gsb200_isect_order_visible(
        int64_t I, int64_t N, int64_t n_vis, const int32_t *tiles_per_gauss, const float *depths,
        const int64_t *image_ids, int32_t *order, int64_t *cum_tiles, void *workspace, size_t workspace_bytes,
        void *stream
    );
    int gsb200_isect_emit_ordered(
        int64_t I, int64_t N, int64_t n_order, int64_t max_tiles_hint, const float *means2d, const int32_t *radii, const float *depths,
        const float *conics, const float *opacities, const int64_t *cum_tiles, const int64_t *image_ids,
        const int32_t *order, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, int64_t *isect_ids,
        int32_t *flatten_ids, void *stream
    );
    /* Narrow-key variant of the same pipeline (round 2): the rows are emitted in depth order, so the S-sized sort only
     * needs the dense tile id image * n_tiles + tile.  gsb200_isect_emit_tilekeys writes that id as a key_bytes-wide
     * (2 when I * n_tiles <= 65536, else 4) unsigned integer next to flatten_ids; gsb200_sort_tile_pairs sorts the pairs
     * (stable, key bits [0, end_bit)), gsb200_isect_offsets_tilekeys derives offsets int32 [I, th, tw] from the sorted
     * keys, and gsb200_isect_ids_from_tilekeys rebuilds the reference's sorted int64 isect_ids
     * ((image << tile_bits | tile) << 32 | depth bits; depths is indexed by flatten_ids) for callers that ask for them. */
    int gsb200_isect_emit_tilekeys(
        int64_t I, int64_t N, int64_t n_order, int64_t max_tiles_hint, const float *means2d, const int32_t *radii, const float *depths,
        const float *conics, const float *opacities, const int64_t *cum_tiles, const int64_t *image_ids,
        const int32_t *order, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, int key_bytes, void *tile_keys,
        int32_t *flatten_ids, void *stream
    );
    size_t gsb200_sort_tile_pairs_workspace_bytes(int64_t n_isects, int key_bytes, int end_bit);
    int gsb200_sort_tile_pairs(
        int64_t n_isects, int key_bytes, int end_bit, const void *keys_in, const int32_t *vals_in, void *keys_out,
        int32_t *vals_out, void *workspace, size_t workspace_bytes, void *stream
    );
    int gsb200_isect_offsets_tilekeys(
        int64_t n_isects, int key_bytes, const void *tile_keys, int64_t I, uint32_t tile_width, uint32_t tile_height,
        int32_t *offsets, void *stream
    );
    int gsb200_isect_ids_from_tilekeys(
        int64_t n_isects, int key_bytes, const void *tile_keys, const int32_t *flatten_ids, const float *depths, int64_t I,
        uint32_t tile_width, uint32_t tile_height, int64_t *isect_ids, void *stream
    );
    /* The sorted dense intersection stage in ONE call, sized by capacities (round 2): rows-with-tiles compaction, depth
     * order, scan, emission of (dense tile id, row) pairs, stable sort on the tile id, offsets.  Inputs: the per-row tile
     * counts and `totals` (int64 [3], DEVICE memory) of gsb200_isect_count_totals / gsb200_project_sh_fwd_rows.  Every
     * launch is sized by cap_vis (<= I * N) and cap_isects; the real counts are read on the device: entries past
     * totals[0] in tile_keys / flatten_ids ([cap_isects] each) are padding, nothing is written past a capacity, and
     * offsets int32 [I, th, tw] is exact whenever totals[1] <= cap_vis and totals[0] <= cap_isects.  A caller may
     * therefore launch with PREDICTED capacities before it has read the totals (the host read then overlaps this work
     * instead of idling the GPU: the sync being hidden is the reference's csrc/Intersect.cpp:258-259), use the first
     * totals[0] entries if both counts fit, and otherwise call again with capacities = totals.  key_bytes: 2 when
     * I * th * tw <= 65536, else 4. */
    size_t gsb200_isect_sorted_workspace_bytes(
        int64_t I, int64_t N, int64_t cap_vis, int64_t cap_isects, int key_bytes, uint32_t tile_width, uint32_t tile_height
    );
    int gsb200_isect_sorted(
        int64_t I, int64_t N, const float *means2d, const int32_t *radii, const float *depths, const float *conics,
        const float *opacities, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height,
        const int32_t *tiles_per_gauss, const int64_t *totals, int64_t cap_vis, int64_t cap_isects, int64_t max_tiles_hint,
        int key_bytes, void *tile_keys, int32_t *flatten_ids, int32_t *offsets, void *workspace, size_t workspace_bytes,
        void *stream
    );
    /* Publishes totals (int64 [3], device) into host_mapped (int64 [4], pinned / mapped host memory) with system-scope
     * stores from a one-warp kernel, then writes seq into host_mapped[3]: the host polls that word instead of waiting for
     * a copy (which takes a copy engine and queues behind PCIe uploads). */
    int gsb200_publish_totals(const int64_t *totals, int64_t *host_mapped, int64_t seq, void *stream);
    /* Stable radix sort of (isect_ids, flatten_ids) on key bits [begin_bit, end_bit)
     * (cub::DeviceRadixSort::SortPairs, csrc/IntersectTile.cu:1078-1121); begin_bit = 32 after pass 0. */
    size_t gsb200_sort_workspace_bytes(int64_t n_isects, int begin_bit, int end_bit);
    int gsb200_sort_pairs(
        int64_t n_isects, int begin_bit, int end_bit, const int64_t *keys_in, const int32_t *vals_in,
        int64_t *keys_out, int32_t *vals_out, void *workspace, size_t workspace_bytes, void *stream
    );
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
    /* Gradient outputs are ACCUMULATED into (caller zero-initialises): each is addressed as
     * ptr[g * stride + k], g in [0, I*N), so they may be views into one packed record per gaussian.
     * v_means2d_abs may be NULL (absgrad off); v_render_alphas may be NULL (no gradient flows into render_alphas). */
    int gsb200_raster_bwd(
        int64_t I, int64_t N, int D, const float *backgrounds, const uint8_t *masks, uint32_t image_width,
        uint32_t image_height, uint32_t tile_size, uint32_t tile_width, uint32_t tile_height, const int32_t *offsets,
        const int32_t *flatten_ids, int64_t n_isects, const void *records, const float *render_alphas,
        const int32_t *last_ids, const float *v_render_colors, const float *v_render_alphas, float *v_means2d,
        int64_t v_means2d_stride, float *v_conics, int64_t v_conics_stride, float *v_colors, int64_t v_colors_stride,
        float *v_opacities, int64_t v_opacities_stride, float *v_means2d_abs, int64_t v_means2d_abs_stride,
        void *stream
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
