/*
 * b200splat.h -- C ABI of libb200splat.so: the H100 (sm_90a) rasterizer hot path.
 *
 * This is the drop-in boundary below the gsplat Python operators.  Each entry point
 * replaces one function of the reference's pybind/libtorch module
 * (/root/reference/gsplat/gsplat/cuda/csrc/ext.cpp:4-18, declared in bindings.h:19-225);
 * the reference interface it replaces is cited per function.
 *
 * Conventions (all functions):
 *   - plain pointers + sizes, no torch types; every pointer is a DEVICE pointer unless
 *     marked "host"; outputs are caller-allocated and need NOT be zero-initialised
 *     (the kernels write every element, including the zeros the reference obtains
 *     from its torch::zeros allocations);
 *   - work is enqueued on `stream` (a cudaStream_t passed as void*; NULL = legacy
 *     default stream) of the CURRENT device and the call returns without synchronising;
 *   - return value 0 = success, negative = error (B200_ERR_*); b200_last_error()
 *     gives a thread-local message.  No exceptions cross the boundary; reentrant.
 *   - float = IEEE fp32, ids/offsets int32, sort keys int64 -- as in the reference.
 */
#ifndef B200SPLAT_H
#define B200SPLAT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define B200_API __attribute__((visibility("default")))
#else
#define B200_API
#endif

#define B200_ABI_VERSION 1
#define B200_MAX_BLUR_SAMPLES 10 /* helpers.cuh:222 */
#define B200_OK 0
#define B200_ERR_INVALID (-1) /* bad argument (the reference raises TORCH_CHECK / AT_ERROR) */
#define B200_ERR_CUDA (-2)    /* a CUDA runtime call or launch failed */

#define B200_SH_POLY 0 /* sh.cuh:268-340 */
#define B200_SH_FAST 1 /* sh.cuh:54-156  */

/* project_gaussians_backward flags */
#define B200_PROJ_EXACT 1u /* clamp-aware J and full dL/dviewmat: the gradients of the reference's
                              torch path (project_gaussians.py:81-112); 0 = reference CUDA path
                              (backward.cu:454-532 ignores the fov clamp; project_gaussians.py:272-307
                              approximates dL/dR) */

/* render-mode word of the fused *_mode entry points (Splatfacto's two render switches, splatfacto.py:842-858); 0 = the
 * entry points without _mode */
#define B200_OPACITY_CLASSIC 1u /* rasterize_mode "classic": opacity = sigmoid(logit), no compensation factor */
#define B200_COLOR_SIGMOID 2u   /* sh_degree 0: colour = sigmoid(sh_dc), no SH basis and no clamp; sh_rest unread */
#define B200_MODE_BITS (B200_OPACITY_CLASSIC | B200_COLOR_SIGMOID)

B200_API int b200_abi_version(void);
B200_API const char *b200_last_error(void);
/* Number of kernels this library has launched in this process (hand-written kernels 1 each, a cub
 * primitive counts its documented passes); bench.py reports the per-step delta as gpu_launches. */
B200_API long long b200_launch_count(void);

/* Size of one packed per-Gaussian blend record (bytes); scratch for the blend = N * this. */
B200_API size_t b200_packed_record_bytes(void);

/* ---- projection ------------------------------------------------------------------------
 * replaces project_gaussians_forward_tensor (bindings.h:43-72, bindings.cu:154-257; kernel
 * forward.cu:13-112).  lin_vel / ang_vel are DEVICE float[3] (NULL = zero) so the caller never
 * needs the .tolist() D2H sync of project_gaussians.py:178-179.  viewmat: >= 12 floats row-major.
 * Outputs: cov3d (N,6) xys (N,2) depths (N) pix_vels (N,2) radii (N) i32 conics (N,3)
 * compensation (N) num_tiles_hit (N) i32.  quat_norm_flag (optional DEVICE int32, caller-zeroed) is OR-ed with 1 if
 * any quaternion violates the reference's `quats.norm(dim=-1) - 1 < 1e-6` assert (project_gaussians.py:69), so the
 * caller can raise it at its next host sync instead of paying a separate reduction + sync. */
B200_API int b200_project_gaussians_forward(int num_points, const float *means3d, const float *scales, float glob_scale,
                                   const float *quats, const float *lin_vel, const float *ang_vel,
                                   float rolling_shutter_time, float exposure_time, const float *viewmat, float fx,
                                   float fy, float cx, float cy, unsigned img_height, unsigned img_width,
                                   unsigned block_width, float clip_thresh, float *cov3d, float *xys, float *depths,
                                   float *pix_vels, int32_t *radii, float *conics, float *compensation,
                                   int32_t *num_tiles_hit, int32_t *quat_norm_flag, void *stream);

/* replaces project_gaussians_backward_tensor (bindings.h:74-108, bindings.cu:259-358; kernel
 * backward.cu:371-451) AND the Python-side v_viewmat block (project_gaussians.py:272-307) AND adds
 * the camera-velocity gradients the reference only has through its torch path.
 * v_cov2d (N,3) / v_cov3d (N,6) are optional scratch outputs (NULL = not materialised).
 * v_mean3d (N,3) v_scale (N,3) v_quat (N,4) are written for every Gaussian (zeros where radii<=0).
 * v_lin_vel[3], v_ang_vel[3], v_viewmat[12] are optional; when non-NULL they are OVERWRITTEN with
 * the sums over Gaussians (block-reduced in the kernel, one atomic per block and component). */
B200_API int b200_project_gaussians_backward(int num_points, const float *means3d, const float *scales, float glob_scale,
                                    const float *quats, const float *lin_vel, const float *ang_vel,
                                    float rolling_shutter_time, float exposure_time, const float *viewmat, float fx,
                                    float fy, float cx, float cy, unsigned img_height, unsigned img_width,
                                    const float *cov3d, const int32_t *radii, const float *conics,
                                    const float *compensation, const float *v_xy, const float *v_depth,
                                    const float *v_pix_vel, const float *v_conic, const float *v_compensation,
                                    unsigned flags, float *v_cov2d, float *v_cov3d, float *v_mean3d, float *v_scale,
                                    float *v_quat, float *v_lin_vel, float *v_ang_vel, float *v_viewmat,
                                    void *stream);

/* replaces compute_cov2d_bounds_tensor (bindings.h:19-22, bindings.cu:19-60): conics (N,3), radii (N) f32 */
B200_API int b200_compute_cov2d_bounds(int num_pts, const float *cov2d, float *conics, float *radii, void *stream);

/* ---- spherical harmonics ----------------------------------------------------------------
 * replaces compute_sh_forward_tensor / compute_sh_backward_tensor (bindings.h:24-41,
 * bindings.cu:62-151; kernels sh.cuh:434-498).  coeffs (N,K,3), K = (degree+1)^2, 3 channels;
 * viewdirs (N,3) un-normalised; v_coeffs rows >= (degrees_to_use+1)^2 are written as zeros. */
B200_API int b200_compute_sh_forward(int method, int num_points, int degree, int degrees_to_use, const float *viewdirs,
                            const float *coeffs, float *colors, void *stream);
B200_API int b200_compute_sh_backward(int method, int num_points, int degree, int degrees_to_use, const float *viewdirs,
                             const float *v_colors, float *v_coeffs, void *stream);

/* ---- tile binning -----------------------------------------------------------------------
 * b200_cumulative_intersects replaces torch.cumsum in compute_cumulative_intersects
 * (gsplat/utils.py:106-125): inclusive int32 scan.  `total_host_pinned` (HOST, optional) receives
 * cum[N-1] by an async copy on `stream` (the caller synchronises before reading it); when `flag_dev` is given its
 * int32 is copied to total_host_pinned[1] in the same way (deferred quat-norm check, see above). */
B200_API size_t b200_scan_temp_bytes(int num_points);
B200_API int b200_cumulative_intersects(int num_points, const int32_t *num_tiles_hit, int32_t *cum_tiles_hit, void *temp,
                                        size_t temp_bytes, int32_t *total_host_pinned, const int32_t *flag_dev,
                                        void *stream);

/* replaces map_gaussian_to_intersects_tensor (bindings.h:199-209, bindings.cu:360-402; kernel
 * forward.cu:116-153).  Slots reserved by cum_tiles_hit but not emitted (the reference's "phantom"
 * entries, which keep their zeros init) are written as key 0 / id 0 here too. */
B200_API int b200_map_gaussian_to_intersects(int num_points, int num_intersects, const float *xys, const float *depths,
                                    const int32_t *radii, const int32_t *cum_tiles_hit, unsigned tiles_x,
                                    unsigned tiles_y, unsigned block_width, int64_t *isect_ids,
                                    int32_t *gaussian_ids, void *stream);

/* replaces torch.sort + torch.gather in bin_and_sort_gaussians (gsplat/utils.py:179-180): stable LSD
 * radix sort of (key, id) pairs on the bits that can be set (32 depth bits + ceil(log2(num_tiles))). */
B200_API size_t b200_sort_temp_bytes(int num_intersects);
B200_API int b200_sort_intersects(int num_intersects, int num_tiles, const int64_t *isect_ids, const int32_t *gaussian_ids,
                         int64_t *isect_ids_sorted, int32_t *gaussian_ids_sorted, void *temp, size_t temp_bytes,
                         void *stream);

/* replaces get_tile_bin_edges_tensor (bindings.h:211-215, bindings.cu:404-422; kernel forward.cu:158-180):
 * tile_bins (num_tiles,2) i32, (0,0) for empty tiles. */
B200_API int b200_get_tile_bin_edges(int num_intersects, int num_tiles, const int64_t *isect_ids_sorted, int32_t *tile_bins,
                            void *stream);

/* Fused fast path of bin_and_sort_gaussians for callers that only need what the blend consumes
 * (rasterize.py:146-163 discards the key arrays): gaussian_ids_sorted (I) and tile_bins (num_tiles,2), produced by a
 * two-level sort (Gaussians by depth, then pairs by tile id) that is order-identical to the stable sort of the
 * reference's 64-bit keys, phantom zero-key slots included.  `ws`: 256-byte aligned scratch of
 * b200_bin_tiles_ws_bytes(N, I) bytes.  num_intersects must equal sum(num_tiles_hit). */
B200_API size_t b200_bin_tiles_ws_bytes(int num_points, int num_intersects);
B200_API int b200_bin_tiles(int num_points, int num_intersects, const float *xys, const float *depths,
                            const int32_t *radii, const int32_t *num_tiles_hit, unsigned tiles_x, unsigned tiles_y,
                            unsigned block_width, void *ws, size_t ws_bytes, int32_t *gaussian_ids_sorted,
                            int32_t *tile_bins, void *stream);

/* Culled binning -- the path gsplat.rasterize_gaussians takes.  Same two-level sort, but a (tile, Gaussian) pair of
 * the reference's bbox (forward.cu:94-102: the square around a 3-sigma circle, inflated by the blur length) is kept only
 * if the Gaussian can reach alpha >= 1/255 inside that tile for some blur sample; dropped pairs cannot change any pixel,
 * survivors keep the reference's order, and the reference's phantom copies of Gaussian 0 survive iff it can touch
 * tile 0.  Two calls around ONE host sync:
 *   b200_bin_cull_count: per-Gaussian survivor counts (the 32-bit survival mask of every 32-tile chunk is kept for the
 *       emit pass), depth sort on a helper stream, offsets; totals_host_pinned[5] (HOST, pinned, async) =
 *       {sum(num_tiles_hit) i.e. the reference's num_intersects, phantom slots, Gaussian-0-touches-tile-0, culled
 *       entry count M, *flag_dev (0 if flag_dev is null: the deferred input-check word of
 *       b200_project_gaussians_forward rides along with the totals)};
 *   b200_bin_cull_emit: after the caller synchronised and allocated M ids -> gaussian_ids_sorted (M), tile_bins.
 * `packed` = records from b200_pack_records; ws_g (b200_bin_cull_ws_bytes(N) bytes) must stay alive and untouched
 * between the two calls; ws_e has b200_bin_cull_emit_ws_bytes(M) bytes; both 256-byte aligned. */
B200_API size_t b200_bin_cull_ws_bytes(int num_points);
B200_API size_t b200_bin_cull_emit_ws_bytes(int num_entries);
B200_API int b200_bin_cull_count(int num_points, const void *packed, const float *depths, const int32_t *radii,
                                 const int32_t *num_tiles_hit, unsigned img_height, unsigned img_width,
                                 unsigned block_width, unsigned n_blur_samples, float rolling_shutter_time,
                                 float exposure_time, void *ws_g, size_t ws_g_bytes, int32_t *totals_host_pinned,
                                 const int32_t *flag_dev, void *stream);
B200_API int b200_bin_cull_emit(int num_points, int num_entries, const void *packed, const int32_t *radii,
                                const int32_t *num_tiles_hit, unsigned img_height, unsigned img_width,
                                unsigned block_width, unsigned n_blur_samples, float rolling_shutter_time,
                                float exposure_time, const void *ws_g, void *ws_e, size_t ws_e_bytes,
                                int32_t *gaussian_ids_sorted, int32_t *tile_bins, void *stream);

/* Packed-record variants of the blend: b200_rasterize_forward/backward = b200_pack_records + these.  Lets a caller pack
 * once per render and share the records between culled binning, forward and backward.
 * out_alpha (H,W) may be null; when given it receives 1 - mean_s final_Ts, the alpha channel gsplat/rasterize.py:161-163
 * builds from final_Ts with two more passes.  v_output_alpha may be null (= a zero cotangent for that channel).
 * outputs_are_zero != 0: the six gradient arrays were already cleared by the caller (e.g. carved from one zero-filled
 * allocation), so the six memsets that otherwise precede the kernel are skipped. */
B200_API int b200_pack_records(int num_points, const float *xys, const float *pix_vels, const float *conics,
                               const float *colors, const float *opacities, void *packed, void *stream);
B200_API int b200_blend_forward_packed(unsigned img_height, unsigned img_width, unsigned block_width,
                                       unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                       const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                       float exposure_time, const float *background, float *out_img, float *final_Ts,
                                       int32_t *final_idx, float *out_alpha, void *stream);
B200_API int b200_blend_backward_packed(int num_points, unsigned img_height, unsigned img_width, unsigned block_width,
                                        unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                        const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                        float exposure_time, const float *background, const float *final_Ts,
                                        const int32_t *final_idx, const float *v_output, const float *v_output_alpha,
                                        float *v_xy, float *v_xy_abs, float *v_pix_vels, float *v_conic,
                                        float *v_colors, float *v_opacity, int outputs_are_zero, void *stream);

/* Launch order of the blend CTAs.  b200_blend_tile_order writes tile_order (int32[num_tiles], num_tiles = tiles_x *
 * tiles_y): a permutation of the tiles, longest tile_bins range first, so the costliest tiles start in the first wave
 * instead of trailing the launch.  The _ordered blend entry points run one CTA per tile in that order and otherwise
 * equal b200_blend_forward_packed_status (status may be null: no empty-render branch) and b200_blend_backward_packed:
 * the forward's outputs are bit-identical, the backward's differ only by the order of float atomics.  The entry points
 * without tile_order run the tiles in raster order. */
B200_API int b200_blend_tile_order(int num_tiles, const int32_t *tile_bins, int32_t *tile_order, void *stream);
B200_API int b200_blend_forward_packed_ordered(unsigned img_height, unsigned img_width, unsigned block_width,
                                               unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                               const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                               float exposure_time, const float *background, const int32_t *status,
                                               const int32_t *tile_order, float *out_img, float *final_Ts,
                                               int32_t *final_idx, float *out_alpha, void *stream);
B200_API int b200_blend_backward_packed_ordered(int num_points, unsigned img_height, unsigned img_width,
                                                unsigned block_width, unsigned n_blur_samples,
                                                const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                                                const void *packed, float rolling_shutter_time, float exposure_time,
                                                const float *background, const float *final_Ts, const int32_t *final_idx,
                                                const float *v_output, const float *v_output_alpha,
                                                const int32_t *tile_order, float *v_xy, float *v_xy_abs,
                                                float *v_pix_vels, float *v_conic, float *v_colors, float *v_opacity,
                                                int outputs_are_zero, void *stream);

/* ---- deterministic mode ----------------------------------------------------------------------------------------------
 * The backward entry points above add per-Gaussian (blend) and per-block (camera) partial sums with float atomics, so
 * their last bits depend on scheduling.  These variants compute the same gradients with every sum in a fixed order, so
 * repeated calls on the same inputs are bit-identical (gsplat uses them under torch.use_deterministic_algorithms).
 *
 * b200_blend_backward_packed_deterministic = b200_blend_backward_packed_ordered, except: each warp visit stores its 13
 * sums to the workspace at (list position, warp) instead of adding them; the list positions are grouped by Gaussian
 * (stable radix sort of (Gaussian id, position)); each Gaussian's sums are added in ascending position, then ascending
 * warp.  The six outputs are written for every Gaussian (zeros where it has no entry).  num_entries = length of
 * gaussian_ids_sorted; status (may be null) = the capacity-mode status of b200_bin_cull_emit_capacity: positions from
 * status[1] on are padding and join no Gaussian.  tile_order may be null (raster order); the result does not depend on
 * it.  ws: 256-byte aligned, b200_blend_backward_deterministic_ws_bytes(num_points, num_entries, block_width) bytes:
 * 52 bytes per (entry, warp) with 4 warps per entry at block_width 16 (8 otherwise), plus 16 bytes per entry, 8 per
 * Gaussian and the sort's temporary storage.
 *
 * b200_project_gaussians_backward_deterministic / b200_fused_preprocess_backward_deterministic = the entry points
 * without the suffix; each block stores its 18 camera partials to ws and one more small kernel sums them in block
 * order.  ws: 16-byte aligned, *_ws_bytes(num_points) bytes (18 floats per block of 256 / 128 Gaussians); unused when
 * no camera gradient is requested. */
B200_API size_t b200_blend_backward_deterministic_ws_bytes(int num_points, int num_entries, unsigned block_width);
B200_API int b200_blend_backward_packed_deterministic(int num_points, int num_entries, unsigned img_height,
                                                      unsigned img_width, unsigned block_width, unsigned n_blur_samples,
                                                      const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                                                      const void *packed, float rolling_shutter_time, float exposure_time,
                                                      const float *background, const float *final_Ts,
                                                      const int32_t *final_idx, const float *v_output,
                                                      const float *v_output_alpha, const int32_t *status,
                                                      const int32_t *tile_order, void *ws, size_t ws_bytes, float *v_xy,
                                                      float *v_xy_abs, float *v_pix_vels, float *v_conic,
                                                      float *v_colors, float *v_opacity, void *stream);
B200_API size_t b200_project_gaussians_backward_ws_bytes(int num_points);
B200_API int b200_project_gaussians_backward_deterministic(
    int num_points, const float *means3d, const float *scales, float glob_scale, const float *quats,
    const float *lin_vel, const float *ang_vel, float rolling_shutter_time, float exposure_time, const float *viewmat,
    float fx, float fy, float cx, float cy, unsigned img_height, unsigned img_width, const float *cov3d,
    const int32_t *radii, const float *conics, const float *compensation, const float *v_xy, const float *v_depth,
    const float *v_pix_vel, const float *v_conic, const float *v_compensation, unsigned flags, float *v_cov2d,
    float *v_cov3d, float *v_mean3d, float *v_scale, float *v_quat, float *v_lin_vel, float *v_ang_vel, float *v_viewmat,
    void *ws, size_t ws_bytes, void *stream);
B200_API size_t b200_fused_preprocess_backward_ws_bytes(int num_points);
B200_API int b200_fused_preprocess_backward_deterministic(
    int num_points, const float *means, const float *log_scales, const float *quats, const float *opacity_logit,
    const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use, const float *viewmat,
    const float *cam_pos, const float *lin_vel, const float *ang_vel, float rolling_shutter_time, float exposure_time,
    float fx, float fy, float cx, float cy, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, float *g_means, float *g_log_scales,
    float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel, float *g_ang_vel,
    float *g_viewmat, void *ws, size_t ws_bytes, void *stream);

/* ---- blend (blur + rolling shutter), 3 channels ------------------------------------------
 * replaces rasterize_forward_tensor (bindings.h:110-127, bindings.cu:424-503; kernel forward.cu:306-456).
 * packed_ws: scratch of num_points * b200_packed_record_bytes() bytes, 16-byte aligned (filled here).
 * out_img (H,W,3), final_Ts (H,W,S) f32, final_idx (H,W,S) i32.  background: DEVICE float[3]. */
B200_API int b200_rasterize_forward(int num_points, unsigned img_height, unsigned img_width, unsigned block_width,
                           unsigned n_blur_samples, const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                           const float *xys, const float *pix_vels, float rolling_shutter_time, float exposure_time,
                           const float *conics, const float *colors, const float *opacities, const float *background,
                           void *packed_ws, float *out_img, float *final_Ts, int32_t *final_idx, void *stream);

/* replaces rasterize_backward_tensor (bindings.h:168-197, bindings.cu:684-773; kernel backward.cu:143-369).
 * v_xy, v_xy_abs, v_pix_vels (N,2); v_conic, v_colors (N,3); v_opacity (N): overwritten (zeroed inside).
 * packed_ws as above (re-filled here, so forward and backward may use different scratch). */
B200_API int b200_rasterize_backward(int num_points, unsigned img_height, unsigned img_width, unsigned block_width,
                            unsigned n_blur_samples, const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                            const float *xys, const float *pix_vels, float rolling_shutter_time, float exposure_time,
                            const float *conics, const float *colors, const float *opacities, const float *background,
                            const float *final_Ts, const int32_t *final_idx, const float *v_output,
                            const float *v_output_alpha, void *packed_ws, float *v_xy, float *v_xy_abs,
                            float *v_pix_vels, float *v_conic, float *v_colors, float *v_opacity, void *stream);

/* ---- fused pre/post-processing on RAW Splatfacto parameters ("next" row f-1 of SURVEY.md section 8) -----------------
 * Folds the caller-side glue of nerfstudio/models/splatfacto.py:816-856 into one kernel each way:
 *   forward : exp(log_scales), quats/|quats|, projection (b200_project_gaussians_forward semantics), "fast" SH colour
 *             + clamp(rgb + 0.5, 0) for Gaussians that survive the bbox test, sigmoid(opacity_logit) * compensation,
 *             and the packed blend record  ->  packed (N * b200_packed_record_bytes()), depths, radii, num_tiles_hit
 *             (exactly the inputs of b200_bin_cull_count / b200_blend_*_packed).
 *   backward: blend gradients (v_xy, v_pix_vel (N,2); v_conic, v_colors (N,3); v_opacity (N)) -> gradients of the raw
 *             parameters, every row written (zeros for culled Gaussians), plus optional camera gradients
 *             (g_lin_vel[3], g_ang_vel[3], g_viewmat[12]; overwritten).  Projection gradients are the clamp-aware
 *             "exact" ones (B200_PROJ_EXACT).
 * Colour clamp: the forward stores a colour the clamp cut as -0.0f and an exact rgb + 0.5 == 0 as +0.0f, and the backward
 * passes the colour gradient where the record's colour has a clear sign bit (torch.clamp(min=0) is inclusive).  So the
 * backward expects `packed` as the fused forward kernels wrote it: records built by b200_pack_records, or recoloured by
 * b200_set_record_colors from clamped colours, hold +0 for cut colours and would pass their gradient.
 * sh_dc (N,3) and sh_rest (N,K-1,3) are the two Splatfacto tensors (no torch.cat needed); sh_bases = K. */
B200_API int b200_fused_preprocess_forward(int num_points, const float *means, const float *log_scales,
                                           const float *quats, const float *opacity_logit, const float *sh_dc,
                                           const float *sh_rest, int sh_bases, int degrees_to_use, const float *viewmat,
                                           const float *cam_pos, const float *lin_vel, const float *ang_vel,
                                           float rolling_shutter_time, float exposure_time, float fx, float fy, float cx,
                                           float cy, unsigned img_height, unsigned img_width, unsigned block_width,
                                           float clip_thresh, void *packed, float *depths, int32_t *radii,
                                           int32_t *num_tiles_hit, void *stream);
/* The forward in two halves, for a trainer that projects and bins image k+1 while the SH coefficients of step k are still
 * being exchanged / updated (gsplat.dp.PipelinedTrainer): b200_fused_geometry_forward reads the geometry parameters only
 * and leaves the records' colours 0; b200_fused_colors_forward fills clamp(SH colour + 0.5, 0) (a cut colour as -0, see
 * above) into the records of the
 * Gaussians with radii > 0 afterwards (the binning does not read colours).  Together they write what
 * b200_fused_preprocess_forward writes; b200_fused_preprocess_backward serves both. */
B200_API int b200_fused_geometry_forward(int num_points, const float *means, const float *log_scales, const float *quats,
                                         const float *opacity_logit, const float *viewmat, const float *lin_vel,
                                         const float *ang_vel, float rolling_shutter_time, float exposure_time, float fx,
                                         float fy, float cx, float cy, unsigned img_height, unsigned img_width,
                                         unsigned block_width, float clip_thresh, void *packed, float *depths,
                                         int32_t *radii, int32_t *num_tiles_hit, void *stream);
B200_API int b200_fused_colors_forward(int num_points, const float *means, const float *sh_dc, const float *sh_rest,
                                       int sh_bases, int degrees_to_use, const float *cam_pos, const int32_t *radii,
                                       void *packed, void *stream);
B200_API int b200_fused_preprocess_backward(int num_points, const float *means, const float *log_scales,
                                            const float *quats, const float *opacity_logit, const float *sh_dc,
                                            const float *sh_rest, int sh_bases, int degrees_to_use, const float *viewmat,
                                            const float *cam_pos, const float *lin_vel, const float *ang_vel,
                                            float rolling_shutter_time, float exposure_time, float fx, float fy, float cx,
                                            float cy, unsigned img_height, unsigned img_width, unsigned block_width,
                                            float clip_thresh, const void *packed, const int32_t *radii,
                                            const float *v_xy, const float *v_pix_vel, const float *v_conic,
                                            const float *v_colors, const float *v_opacity, float *g_means,
                                            float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc,
                                            float *g_sh_rest, float *g_lin_vel, float *g_ang_vel, float *g_viewmat,
                                            void *stream);

/* ---- view batches: B cameras of one scene in one call ----------------------------------------------------------------
 * The fused forward, culled binning and blend with a view dimension; camera v of the batch gives exactly the single-view
 * result (the single-view entry points run the same kernels with B = 1).  Layout, for B views of N Gaussians, T =
 * tiles_x * tiles_y tiles per view:
 *   records   Gaussian g of view v is record r = v * N + g: packed (B * N * 64 bytes, record id = r), depths, radii,
 *             num_tiles_hit (B * N), and the blend gradients (v_xy, v_xy_abs, v_pix_vels (B*N,2); v_conic, v_colors
 *             (B*N,3); v_opacity (B*N)).
 *   lists     tile t of view v is list key v * T + t: tile_bins (B * T, 2); the ids are record ids.  Each tile's list is
 *             that view's single-view list (stable sorts: depth order, ties by Gaussian id); every view's phantom entries
 *             (key v * T, id v * N, kept iff Gaussian 0 of the view can touch its tile 0) lead its tile 0.
 *   images    out_img (B,H,W,3), final_Ts / final_idx (B,H,W,S), out_alpha / v_output_alpha (B,H,W), v_output (B,H,W,3).
 *   cameras   viewmats (B,3,4) row major, cam_pos / lin_vel / ang_vel (B,3), intrinsics (B,4) = fx, fy, cx, cy per view
 *             (16-byte aligned); camera gradients g_lin_vel / g_ang_vel (B,3), g_viewmat (B,3,4), overwritten.
 * b200_fused_preprocess_forward_views: grid (ceil(N / 128), B).
 * b200_fused_preprocess_backward_views(_deterministic): one thread per Gaussian, the views in order; the raw-parameter
 *   gradients are the sums over the views, added in view order with separately rounded adds, so they equal the B
 *   single-view gradients added one after the other.  ws of the deterministic variant: 16-byte aligned,
 *   b200_fused_preprocess_backward_views_ws_bytes(B, N) bytes (18 floats per view and block of 128 Gaussians).
 * b200_bin_cull_count_views / b200_bin_cull_emit_views: b200_bin_cull_count / _emit over the B * N records, ONE host read
 *   for the batch.  ws_g: b200_bin_cull_views_ws_bytes(B, N) bytes (0: B * N exceeds int32); ws_e as for
 *   b200_bin_cull_emit (b200_bin_cull_emit_ws_bytes(M)).  totals_host_pinned[7] (HOST, pinned, may be null): the five
 *   words of b200_bin_cull_count summed over the views ([2]: view 0), then [5] phantom entries kept and [6] = 1 if the
 *   batch's reserved-slot total [0] does not fit in int32 (the lists cannot be built).  view_isect (DEVICE int32[B]):
 *   every view's reference num_intersects.
 * b200_blend_forward_views / b200_blend_backward_views(_deterministic): the blends over the batch lists, one CTA per
 *   (view, tile) in tile_order (b200_blend_tile_order over the B * T bins, required); a view whose view_isect is < 1 takes
 *   the empty-render branch (background, final_Ts = 0, alpha = 1).  The deterministic backward's ws is
 *   b200_blend_backward_deterministic_ws_bytes(B * N, M, block_width) bytes. */
B200_API int b200_fused_preprocess_forward_views(int num_views, int num_points, const float *means,
                                                 const float *log_scales, const float *quats, const float *opacity_logit,
                                                 const float *sh_dc, const float *sh_rest, int sh_bases,
                                                 int degrees_to_use, const float *viewmats, const float *cam_pos,
                                                 const float *lin_vel, const float *ang_vel, const float *intrinsics,
                                                 float rolling_shutter_time, float exposure_time, unsigned img_height,
                                                 unsigned img_width, unsigned block_width, float clip_thresh,
                                                 void *packed, float *depths, int32_t *radii, int32_t *num_tiles_hit,
                                                 void *stream);
B200_API int b200_fused_preprocess_backward_views(
    int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, float *g_means, float *g_log_scales,
    float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel, float *g_ang_vel,
    float *g_viewmat, void *stream);
B200_API size_t b200_fused_preprocess_backward_views_ws_bytes(int num_views, int num_points);
B200_API int b200_fused_preprocess_backward_views_deterministic(
    int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, float *g_means, float *g_log_scales,
    float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel, float *g_ang_vel,
    float *g_viewmat, void *ws, size_t ws_bytes, void *stream);
B200_API size_t b200_bin_cull_views_ws_bytes(int num_views, int num_points);
B200_API int b200_bin_cull_count_views(int num_views, int num_points, const void *packed, const float *depths,
                                       const int32_t *radii, const int32_t *num_tiles_hit, unsigned img_height,
                                       unsigned img_width, unsigned block_width, unsigned n_blur_samples,
                                       float rolling_shutter_time, float exposure_time, void *ws_g, size_t ws_g_bytes,
                                       int32_t *totals_host_pinned, int32_t *view_isect, const int32_t *flag_dev,
                                       void *stream);
B200_API int b200_bin_cull_emit_views(int num_views, int num_points, int num_entries, const void *packed,
                                      const int32_t *radii, const int32_t *num_tiles_hit, unsigned img_height,
                                      unsigned img_width, unsigned block_width, unsigned n_blur_samples,
                                      float rolling_shutter_time, float exposure_time, const void *ws_g, void *ws_e,
                                      size_t ws_e_bytes, int32_t *gaussian_ids_sorted, int32_t *tile_bins, void *stream);
B200_API int b200_blend_forward_views(int num_views, unsigned img_height, unsigned img_width, unsigned block_width,
                                      unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                      const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                      float exposure_time, const float *background, const int32_t *view_isect,
                                      const int32_t *tile_order, float *out_img, float *final_Ts, int32_t *final_idx,
                                      float *out_alpha, void *stream);
B200_API int b200_blend_backward_views(int num_views, int num_records, unsigned img_height, unsigned img_width,
                                       unsigned block_width, unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                       const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                       float exposure_time, const float *background, const float *final_Ts,
                                       const int32_t *final_idx, const float *v_output, const float *v_output_alpha,
                                       const int32_t *tile_order, float *v_xy, float *v_xy_abs, float *v_pix_vels,
                                       float *v_conic, float *v_colors, float *v_opacity, int outputs_are_zero,
                                       void *stream);
B200_API int b200_blend_backward_views_deterministic(int num_views, int num_records, int num_entries,
                                                     unsigned img_height, unsigned img_width, unsigned block_width,
                                                     unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                                     const int32_t *tile_bins, const void *packed,
                                                     float rolling_shutter_time, float exposure_time,
                                                     const float *background, const float *final_Ts,
                                                     const int32_t *final_idx, const float *v_output,
                                                     const float *v_output_alpha, const int32_t *tile_order, void *ws,
                                                     size_t ws_bytes, float *v_xy, float *v_xy_abs, float *v_pix_vels,
                                                     float *v_conic, float *v_colors, float *v_opacity, void *stream);

/* ---- visit records: a backward that replays what its forward blended ------------------------------------------------
 * b200_blend_records_visits(block_width): 1 when the three calls below run for that tile size (16x16 tiles, the paired
 *   two-pixel kernels), else 0; callers then take the entry points above.
 * b200_blend_forward_record = b200_blend_forward_views (num_views >= 1, one view = the single-image lists; view_isect
 *   may be null: no empty-render branch; tile_order required) with the same outputs bit for bit, and in addition:
 *   visit_mask, uint16[num_entries * 4] for the num_entries positions of gaussian_ids_sorted (the capacity in capacity
 *   mode): at (list position, warp of the tile's CTA) the blur samples at which some pixel of that warp blended the
 *   entry; tile_cost, int32[num_views * tiles]: per tile, the number of blended (warp, entry, sample) triples.
 * b200_blend_tile_order_cost: b200_blend_tile_order keyed on tile_cost instead of the list length (costliest first).
 * b200_blend_backward_replay(_deterministic) = b200_blend_backward_views(_deterministic) with the same results (the
 *   deterministic ones bit for bit), but each warp visits only the entries and samples visit_mask records; status as
 *   in b200_blend_backward_packed_deterministic (may be null); ws: b200_blend_backward_deterministic_ws_bytes.
 * Between the forward and the backward the caller keeps alive, unchanged: gaussian_ids_sorted, tile_bins, packed,
 *   final_Ts, final_idx and visit_mask (tile_cost only until b200_blend_tile_order_cost has run).  The backward reads a
 *   mask only at positions up to its warp's last contributor, all of which the forward wrote; a mask from other lists,
 *   records or outputs gives wrong gradients. */
B200_API int b200_blend_records_visits(unsigned block_width);
B200_API int b200_blend_forward_record(int num_views, unsigned img_height, unsigned img_width, unsigned block_width,
                                       unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                       const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                       float exposure_time, const float *background, const int32_t *view_isect,
                                       const int32_t *tile_order, float *out_img, float *final_Ts, int32_t *final_idx,
                                       float *out_alpha, void *visit_mask, int32_t *tile_cost, void *stream);
B200_API int b200_blend_tile_order_cost(int num_tiles, const int32_t *tile_cost, int32_t *tile_order, void *stream);
B200_API int b200_blend_backward_replay(int num_views, int num_records, unsigned img_height, unsigned img_width,
                                        unsigned block_width, unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                        const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                        float exposure_time, const float *background, const float *final_Ts,
                                        const int32_t *final_idx, const float *v_output, const float *v_output_alpha,
                                        const void *visit_mask, const int32_t *tile_order, float *v_xy, float *v_xy_abs,
                                        float *v_pix_vels, float *v_conic, float *v_colors, float *v_opacity,
                                        int outputs_are_zero, void *stream);
B200_API int b200_blend_backward_replay_deterministic(int num_views, int num_records, int num_entries,
                                                      unsigned img_height, unsigned img_width, unsigned block_width,
                                                      unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                                      const int32_t *tile_bins, const void *packed,
                                                      float rolling_shutter_time, float exposure_time,
                                                      const float *background, const float *final_Ts,
                                                      const int32_t *final_idx, const float *v_output,
                                                      const float *v_output_alpha, const int32_t *status,
                                                      const void *visit_mask, const int32_t *tile_order, void *ws,
                                                      size_t ws_bytes, float *v_xy, float *v_xy_abs, float *v_pix_vels,
                                                      float *v_conic, float *v_colors, float *v_opacity, void *stream);

/* ---- differentiable depth (splatfacto.py:881-897) ---------------------------------------------------------------------
 * D = the static blend (S = 1, no rolling shutter, zero background) of the records' view-space depths: the second
 * rasterize call Splatfacto makes with the depths as colours.  The records must come from the fused forward entry points
 * (b200_fused_preprocess_forward(_views), b200_fused_geometry_forward), which store the depth in the record's last
 * word; b200_pack_records stores 0 there.  Lists: the static lists of the same records (b200_bin_cull* with S = 1,
 * rs = exposure = 0), or lists that contain them (the colour pass's when rs == 0 and (exposure == 0 or S odd)).
 * Layouts are those of the view batches above, with B = num_views (1 for one camera): images (B,H,W), records B * N.
 * b200_blend_depth_forward: out_depth (B,H,W); final_T (B,H,W) float and final_idx (B,H,W) int32 for a backward, or
 *   both null.  view_isect (DEVICE int32[B]) may be null; a view whose entry is < 1 takes the empty-render branch
 *   (D = 0, final_T = 0, final_idx = 0).  tile_order: b200_blend_tile_order of tile_bins, or null for raster order.
 *   D is bit for bit channel 0 of b200_blend_forward_views / _packed at S = 1 on records whose colours are the depths.
 * b200_blend_depth_backward: with cotangent v_depth_img (B,H,W), ADDS the depth pass's gradients into v_xy (B*N,2),
 *   v_conic (B*N,3) and v_opacity (B*N) -- the colour backward's outputs -- and overwrites v_depth (B*N).
 * b200_blend_depth_backward_deterministic: the same sums in a fixed order (per Gaussian: ascending list position, then
 *   warp), every output OVERWRITTEN (add them to the colour pass's gradients yourself).  ws: 256-byte aligned,
 *   b200_blend_depth_backward_deterministic_ws_bytes(B * N, num_entries, block_width) bytes, num_entries = the list
 *   length.
 * b200_fused_preprocess_backward_views_depth(_deterministic): b200_fused_preprocess_backward_views(_deterministic) with
 *   v_depth (B*N) as the projection's depth cotangent; B = 1 with the camera's intrinsics gives the single-view result. */
B200_API int b200_blend_depth_forward(int num_views, unsigned img_height, unsigned img_width, unsigned block_width,
                                      const int32_t *gaussian_ids_sorted, const int32_t *tile_bins, const void *packed,
                                      const int32_t *view_isect, const int32_t *tile_order, float *out_depth,
                                      float *final_T, int32_t *final_idx, void *stream);
B200_API int b200_blend_depth_backward(int num_views, int num_records, unsigned img_height, unsigned img_width,
                                       unsigned block_width, const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                                       const void *packed, const float *final_T, const int32_t *final_idx,
                                       const float *v_depth_img, const int32_t *tile_order, float *v_xy, float *v_conic,
                                       float *v_opacity, float *v_depth, void *stream);
B200_API size_t b200_blend_depth_backward_deterministic_ws_bytes(int num_records, int num_entries, unsigned block_width);
B200_API int b200_blend_depth_backward_deterministic(int num_views, int num_records, int num_entries,
                                                     unsigned img_height, unsigned img_width, unsigned block_width,
                                                     const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                                                     const void *packed, const float *final_T, const int32_t *final_idx,
                                                     const float *v_depth_img, const int32_t *tile_order, void *ws,
                                                     size_t ws_bytes, float *v_xy, float *v_conic, float *v_opacity,
                                                     float *v_depth, void *stream);
B200_API int b200_fused_preprocess_backward_views_depth(
    int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, const float *v_depth, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, void *stream);
B200_API int b200_fused_preprocess_backward_views_depth_deterministic(
    int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, const float *v_depth, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, void *ws, size_t ws_bytes, void *stream);

/* ---- render modes: Splatfacto's "classic" opacities and degree-0 sigmoid colours ------------------------------------
 * Each *_mode entry point is the entry point named without _mode, with a leading mode word of B200_* flags:
 *   B200_OPACITY_CLASSIC  the record's opacity is sigmoid(opacity_logit) (rasterize_mode "classic", splatfacto.py:155,
 *                         :853-856); the backward drops the compensation VJP.
 *   B200_COLOR_SIGMOID    the record's colour is sigmoid(sh_dc) (sh_degree 0, splatfacto.py:847-848): no view direction,
 *                         no clamp; degrees_to_use is ignored, sh_bases may be any K >= 1, sh_rest and cam_pos are not
 *                         read, and the backward writes g_sh_rest ((N, K-1, 3)) as zeros.
 * mode 0 runs exactly the kernels of the entry point without _mode; a bit outside B200_MODE_BITS is B200_ERR_INVALID,
 * checked before any GPU work.  The geometry-only forward reads only the opacity bit and the colour fill only the colour
 * bit, so a trainer passes one word to all of them.  b200_fused_preprocess_backward_views_mode(_deterministic) take
 * v_depth after v_opacity like the _depth entry points, but nullable: null is the backward without depth. */
B200_API int b200_fused_preprocess_forward_views_mode(
    unsigned mode, int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, void *packed, float *depths, int32_t *radii, int32_t *num_tiles_hit, void *stream);
B200_API int b200_fused_preprocess_backward_views_mode(
    unsigned mode, int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, const float *v_depth, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, void *stream);
B200_API int b200_fused_preprocess_backward_views_mode_deterministic(
    unsigned mode, int num_views, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmats, const float *cam_pos, const float *lin_vel, const float *ang_vel, const float *intrinsics,
    float rolling_shutter_time, float exposure_time, unsigned img_height, unsigned img_width, unsigned block_width,
    float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy, const float *v_pix_vel,
    const float *v_conic, const float *v_colors, const float *v_opacity, const float *v_depth, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, void *ws, size_t ws_bytes, void *stream);
B200_API int b200_fused_geometry_forward_mode(unsigned mode, int num_points, const float *means, const float *log_scales,
                                              const float *quats, const float *opacity_logit, const float *viewmat,
                                              const float *lin_vel, const float *ang_vel, float rolling_shutter_time,
                                              float exposure_time, float fx, float fy, float cx, float cy,
                                              unsigned img_height, unsigned img_width, unsigned block_width,
                                              float clip_thresh, void *packed, float *depths, int32_t *radii,
                                              int32_t *num_tiles_hit, void *stream);
B200_API int b200_fused_colors_forward_mode(unsigned mode, int num_points, const float *means, const float *sh_dc,
                                            const float *sh_rest, int sh_bases, int degrees_to_use, const float *cam_pos,
                                            const int32_t *radii, void *packed, void *stream);
B200_API int b200_fused_preprocess_backward_mode(
    unsigned mode, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmat, const float *cam_pos, const float *lin_vel, const float *ang_vel, float rolling_shutter_time,
    float exposure_time, float fx, float fy, float cx, float cy, unsigned img_height, unsigned img_width,
    unsigned block_width, float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy,
    const float *v_pix_vel, const float *v_conic, const float *v_colors, const float *v_opacity, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, void *stream);
B200_API int b200_fused_preprocess_backward_mode_deterministic(
    unsigned mode, int num_points, const float *means, const float *log_scales, const float *quats,
    const float *opacity_logit, const float *sh_dc, const float *sh_rest, int sh_bases, int degrees_to_use,
    const float *viewmat, const float *cam_pos, const float *lin_vel, const float *ang_vel, float rolling_shutter_time,
    float exposure_time, float fx, float fy, float cx, float cy, unsigned img_height, unsigned img_width,
    unsigned block_width, float clip_thresh, const void *packed, const int32_t *radii, const float *v_xy,
    const float *v_pix_vel, const float *v_conic, const float *v_colors, const float *v_opacity, float *g_means,
    float *g_log_scales, float *g_quats, float *g_opacity_logit, float *g_sh_dc, float *g_sh_rest, float *g_lin_vel,
    float *g_ang_vel, float *g_viewmat, void *ws, size_t ws_bytes, void *stream);

/* ---- N-channel blend (no blur), fp16 accumulators like the reference ----------------------
 * replaces nd_rasterize_forward_tensor / nd_rasterize_backward_tensor (bindings.h:129-166,
 * bindings.cu:506-682; kernels forward.cu:185-304, backward.cu:22-141). */
B200_API int b200_nd_rasterize_forward(int num_points, unsigned img_height, unsigned img_width, unsigned block_width,
                              unsigned channels, const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                              const float *xys, const float *conics, const float *colors, const float *opacities,
                              const float *background, float *out_img, float *final_Ts, int32_t *final_idx,
                              void *stream);
B200_API int b200_nd_rasterize_backward(int num_points, unsigned img_height, unsigned img_width, unsigned block_width,
                               unsigned channels, const int32_t *gaussian_ids_sorted, const int32_t *tile_bins,
                               const float *xys, const float *conics, const float *colors, const float *opacities,
                               const float *background, const float *final_Ts, const int32_t *final_idx,
                               const float *v_output, const float *v_output_alpha, float *v_xy, float *v_xy_abs,
                               float *v_conic, float *v_colors, float *v_opacity, void *stream);

/* ---- photometric loss ("next" row f-3 of SURVEY section 8) -----------------------------------
 * Fused L1: loss[0] = mean |pred - target| over numel floats and, when grad is not null, grad = sign(pred - target) /
 * numel -- the cotangent rasterize_backward consumes -- in ONE pass; replaces the L1 term of the caller's loss
 * (nerfstudio/models/splatfacto.py:957, `torch.abs(gt_img - pred_img).mean()`) and its autograd chain.
 * ws: b200_l1_loss_ws_bytes() bytes of device scratch, 16-byte aligned, one per concurrent stream; pass
 * ws_is_zeroed = 1 if its first 4 bytes are zero (they are left zero on return), else they are cleared here.
 * Deterministic (block partial sums are added in block order). */
B200_API size_t b200_l1_loss_ws_bytes(void);
B200_API int b200_l1_loss(long long numel, const float *pred, const float *target, float *loss, float *grad, void *ws,
                          int ws_is_zeroed, void *stream);
/* The same with the caller's gamma step folded in (splatfacto.py:879-880 `clamp(rgb, max=1) ** (1 / gamma)` before the loss of
 * :957): pred_linear is the LINEAR render, loss[0] = mean |min(pred, 1)^(1/gamma) - target|, grad_linear = the cotangent w.r.t.
 * the linear image (torch's clamp / pow backward: (1/gamma) x^(1/gamma - 1) up to and including x = 1, 0 above, infinite at 0). */
B200_API int b200_l1_loss_gamma(long long numel, const float *pred_linear, const float *target, float gamma, float *loss,
                                float *grad_linear, void *ws, int ws_is_zeroed, void *stream);
/* The same against the dataset's uint8 image with the caller's ground-truth preparation folded in: uint8 -> float / 255
 * (splatfacto.py:900-910 get_gt_img), RGBA composited over `background` (3 DEVICE floats; :912-923 composite_with_background,
 * alpha * rgb + (1 - alpha) * background, unfused like torch), clamp(min = min_level) with min_level = min_rgb_level / 255
 * (:952-953; <= 0: off), optional mask (n_pixels floats: gt * mask, pred * mask, :957-964), L1 mean over 3 * n_pixels (:966).
 * channels = 3 or 4; gamma > 0 applies the gamma step to pred as in b200_l1_loss_gamma, <= 0: pred is used as it is;
 * target_out (3 * n_pixels floats or null) receives the prepared float target (what the SSIM term is taken against). */
B200_API int b200_l1_loss_u8(long long n_pixels, int channels, const float *pred, const unsigned char *target_u8,
                             const float *background, float min_level, float gamma, const float *mask, float *loss,
                             float *grad, float *target_out, void *ws, int ws_is_zeroed, void *stream);
/* b200_l1_loss_u8 for a render at 1/d of the target's resolution (Splatfacto's resolution schedule, splatfacto.py:660-667):
 * the target's area downscale (`resize_image`, :83-95: conv2d with a d x d box of weight 1/d^2 at stride d) rides in the
 * same pass, which reads the full-resolution image once.  target_u8 is (in_h, in_w, channels) bytes with rows of
 * in_w * channels bytes (no alignment asked); mask is in_h * in_w floats or null; pred, grad and target_out are
 * (in_h / d) * (in_w / d) * 3 floats (floored sizes; rows and columns past d * (in / d) are ignored, as by the strided conv2d).
 * d = 2, 4, 8 or 16.  Per output pixel, in the reference's order: every channel (alpha included) and the mask are pooled
 * from k / 255.0f, summed in float32 in one fixed order (rows top to bottom, pixels left to right) and scaled by 1/d^2
 * (exact); RGBA is composited over background with the POOLED alpha; clamp(min = min_level); both images times the pooled
 * mask; the gamma step on pred; L1 mean over 3 * (in_h / d) * (in_w / d).  grad is the cotangent w.r.t. the linear render.
 * Error bound (first order, u = 2^-24, one rounding per operation; torch's conv2d sums in an order of its own, so equality
 * with it bit for bit is not available; tests/downscale_f64.py restates this in float64 and evaluates it per element):
 *   pooled channel / alpha / mask p:  e_p = (d^2 - 1) u p   (d^2 non-negative terms; the mask bound uses its |values|)
 *   composite t = a c + (1 - a) bg:    e_t = (|c| + |bg|) e_a + |a| e_c + u (|a c| + 2 |(1 - a) bg| + |t|);  RGB: e_t = e_c
 *   clamp: e_t unchanged;  mask:       e_tm = |m| e_t + |t| e_m + u |t m|
 *   pred side y (gamma-corrected or not): e_y = |y| e_m + u |y m| with a mask, plus 4 u |y m| with gamma (powf, not
 *   correctly rounded);  loss: mean(e_tm + e_y) + the reduction's rounding, at most (depth) u L for its deepest chain.
 * Where |pred_img - target| exceeds e_tm + e_y the cotangent's sign is the reference's.  Deterministic. */
B200_API int b200_l1_loss_u8_area(int in_h, int in_w, int channels, int d, const float *pred, const unsigned char *target_u8,
                                  const float *background, float min_level, float gamma, const float *mask, float *loss,
                                  float *grad, float *target_out, void *ws, int ws_is_zeroed, void *stream);

/* SSIM term of the photometric loss, (1 - lambda) * L1 + lambda * (1 - SSIM) (nerfstudio/models/splatfacto.py:957-975;
 * SSIM = pytorch_msssim.SSIM(data_range=1, size_average=True, channel=C): 11-tap Gaussian window sigma 1.5, separable,
 * valid padding, K = (0.01, 0.03), mean over channels and the (H-10) x (W-10) valid positions).  Images are (H, W, C).
 *   b200_ssim_forward: ssim_out[0] = mean SSIM; if loss_out: loss_out[0] = (1 - lambda) * l1_loss[0] + lambda * (1 - SSIM)
 *       (l1_loss null = 0); if maps (b200_ssim_maps_bytes bytes): the three partial-derivative maps for the backward.
 *   b200_ssim_backward: grad = [v_scale[0] *] (add_scale * add_in + scale * dSSIM/dpred); add_in, v_scale optional.
 *       With add_in = the L1 cotangent, add_scale = 1 - lambda, scale = -lambda this is the photometric cotangent.
 * window11: optional HOST float[11], the normalised window taps (null = exp(-x^2 / 4.5) / sum evaluated in float here);
 *       SSIM of smooth images is sensitive to the last bits of the taps, so a binding that must reproduce
 *       pytorch_msssim passes the taps that library builds.
 * ws: b200_ssim_ws_bytes bytes, 16-byte aligned, ws_is_zeroed as for b200_l1_loss.  Deterministic. */
B200_API size_t b200_ssim_ws_bytes(unsigned img_height, unsigned img_width, unsigned channels);
B200_API size_t b200_ssim_maps_bytes(unsigned img_height, unsigned img_width, unsigned channels);
B200_API int b200_ssim_forward(unsigned img_height, unsigned img_width, unsigned channels, const float *pred,
                               const float *target, float *maps, float *ssim_out, float *loss_out, const float *l1_loss,
                               float ssim_lambda, const float *window11, void *ws, int ws_is_zeroed, void *stream);
B200_API int b200_ssim_backward(unsigned img_height, unsigned img_width, unsigned channels, const float *pred,
                                const float *target, const float *maps, float scale, const float *add_in,
                                float add_scale, const float *v_scale, const float *window11, float *grad,
                                void *stream);

/* ---- evaluation metrics of B views in one launch --------------------------------------------------------------------
 * What nerfstudio's ns-eval computes per image (Splatfacto's get_image_metrics_and_images, splatfacto.py:1006-1042),
 * LPIPS aside, for `views` images of one size:
 *   pred_linear (views, H, W, 3) float, the LINEAR render; y = min(pred, 1)^(1/gamma) (splatfacto.py:880), with the
 *       exponent (float)(1.0 / gamma); gamma == 1: y = min(pred, 1) exactly (no powf);
 *   target (views, H, W, channels), uint8 (target_is_u8 = 1) or float (0; the reference's float-image branch), channels
 *       3 or 4; prepared as b200_l1_loss_u8 prepares it with min_level 0 and no mask (its target_out, bit for bit):
 *       uint8 / 255, RGBA composited over `background` (3 DEVICE floats, needed for channels = 4);
 *   mse_out[v] = mean (y - t)^2 over 3 H W;  psnr_out[v] = 10 log10(1 / mse) (torchmetrics' PeakSignalNoiseRatio with
 *       data_range 1; +inf when mse == 0);  ssim_out[v] = the b200_ssim_forward value of (y, t) with the same window11.
 * One pass over each view's SSIM tiles; neither the prepared images nor the SSIM maps are written.  Every squared error
 * is summed once.  ws: b200_eval_metrics_ws_bytes(views, H, W) bytes, 16-byte aligned, one ticket per view in its first
 * 4 * views bytes (ws_is_zeroed as for b200_l1_loss: they are left zero on return).  Deterministic: each view's sums
 * run in one fixed order, so a view's metrics do not depend on the batch it is evaluated in and repeated calls agree bit
 * for bit.  views <= 21845 (three grid layers per view). */
B200_API size_t b200_eval_metrics_ws_bytes(unsigned views, unsigned img_height, unsigned img_width);
B200_API int b200_eval_metrics_views(unsigned views, unsigned img_height, unsigned img_width, unsigned channels,
                                     const float *pred_linear, const void *target, int target_is_u8,
                                     const float *background, float gamma, const float *window11, float *mse_out,
                                     float *psnr_out, float *ssim_out, void *ws, int ws_is_zeroed, void *stream);

/* ---- optimizer ("next" row f-2 of SURVEY section 8) ---------------------------------------------
 * One Adam update (no weight decay, no amsgrad: what nerfstudio/engine/optimizers.py:158-171 builds for every Splatfacto
 * group, eps = 1e-15) of `numel` consecutive floats of the flat {param, grad, exp_avg, exp_avg_sq} buffers:
 *   g' = grad_scale * grad;  m += (1 - beta1)(g' - m);  v = beta2 v + (1 - beta2) g'^2;
 *   param -= lr / (1 - beta1^step) * m / (sqrt(v) / sqrt(1 - beta2^step) + eps);   grad = 0 if zero_grad.
 * `step` counts from 1; the hyper-parameters are doubles so that 1 - beta, the bias corrections and lr / (1 - beta1^step)
 * are formed in double exactly like the Python optimizer forms them.  The four pointers may point anywhere into equally aligned buffers (same offset each), so a
 * trainer can update slice by slice as gradient exchanges complete. */
B200_API int b200_adam_step(long long numel, float *param, float *grad, float *exp_avg, float *exp_avg_sq, int step,
                            double lr, double beta1, double beta2, double eps, double grad_scale, int zero_grad,
                            void *stream);

/* Device-resident Adam: the step count, the bias corrections, per-group learning rates and a per-step VETO live on the
 * device, so a trainer that never synchronises with the host (CUDA-graph replays, capacity-mode binning below) can follow
 * Splatfacto's schedules and still skip the update of a step whose render turned out incomplete.  Splatfacto steps one
 * Adam per parameter group, each with its own rate and scheduler (nerfstudio/configs/method_configs.py, the splatfacto
 * optimizers); a single rate is one constant group.  Same arithmetic as b200_adam_step.
 *   state: DEVICE, b200_adam_state_bytes() bytes, zeroed by the caller before the first step; as int32 words: [2] optimizer
 *       steps applied, [3] the current step: 0 one count for every group, 1 vetoed, 2 per-group counts; [4] steps
 *       prepared, [5] steps vetoed, [6..15] indices (0-based, in `steps prepared` numbering) of the last 10 vetoed steps,
 *       slot = count % 10.
 *   group_table: DEVICE float[B200_ADAM_GROUP_TABLE_FLOATS], 16-byte aligned, zeroed by the caller before the first step:
 *       [g] lr_g(s) / (1 - beta1^t_g), [16 + g] 1 / sqrt(1 - beta2^t_g), [32 + g] t_g (int32: steps group g has taken),
 *       [48] the mask of the last prepared step (uint32, bit g = group g steps).  Without per-group counts only [g] is
 *       written, with t_g = the steps applied.
 *   b200_adam_prepare_step: once per step before the first update.  veto_flag: DEVICE int32 or null; non-zero = veto this
 *       step (a data-parallel caller reduces it with MAX across ranks first); it is cleared here, and a vetoed step leaves
 *       the group table as it was.  groups: HOST double[n_groups][B200_LR_GROUP_DOUBLES], read during the call and passed
 *       to the kernel by value (so it can be captured): {kind (0 constant, 1 exponential decay), lr_init, lr_final,
 *       lr_pre_warmup, warmup_steps, max_steps, ramp (0 cosine, 1 linear)}.  Kind 1 is nerfstudio's
 *       ExponentialDecayScheduler (engine/schedulers.py) under LambdaLR: lr_g(s) = lr_init * (func_lr(s) / lr_init), in
 *       double.  Kind 0 uses lr_init exactly.  The schedule position s is the index of the step being prepared, vetoed
 *       steps included: word [4] before the increment.  The state's own bias corrections count applied steps, and its
 *       lr / bc1 is group 0's.
 *       detached: DEVICE int32 or null.  Null: every group steps at the count of applied steps (word [3] = 0).  Otherwise
 *       each group keeps its own count t_g (word [3] = 2), for Splatfacto's detached eval cameras: nerfstudio steps an
 *       optimizer only when one of its parameters has a gradient (engine/optimizers.py:158-171), and torch's Adam keeps a
 *       step count per parameter.  *detached zero: every group steps.  Non-zero: only the groups of the bit mask
 *       detached_groups step, and group cond_group as well when s is a multiple of cond_every (cond_group < 0: none).  A
 *       group that steps advances t_g and gets new constants; the others keep both.
 *   b200_adam_update: the update of numel floats whose first one is GLOBAL flat index `offset`; the slice must start
 *       16-byte aligned.  A vetoed step moves nothing and clears the gradient slice.  zero_grad: 1 clears the gradient
 *       slice, 0 leaves it, B200_ADAM_CLEAR_ON_VETO clears it on a vetoed step only -- for a caller whose backward
 *       overwrites every gradient of the slice, which then needs no clear behind an applied step (and no masked group's
 *       clear: a detached image's rows are already zero).  n_segments == 0: every element uses
 *       the state's constants.  n_segments > 0: every element uses its own group's constants from group_table.
 *       segments: HOST long long[n_segments][B200_ADAM_SEGMENT_WORDS], sorted and disjoint, by value like `groups`:
 *       {begin, end, period, split, group_a, group_b}.  Global index i in [begin, end) belongs to group_a when
 *       period == 0 or (i - begin) % period < split, else to group_b.  An element in no segment, or in a group outside the
 *       step's mask, keeps its parameter and moments bit-unchanged; its gradient is cleared as zero_grad says.  The
 *       slice need not start or end on a segment boundary.  After a prepare with a `detached` word, pass the segment table: without one
 *       the update reads word [3] = 2 as a veto.  ctas_per_sm: 0 = many short CTAs; 1..32 = a background kernel for a
 *       caller that runs it on a second stream beside latency-bound work: at most ctas_per_sm resident CTAs of 256 threads
 *       per SM loop over the slice, so kernels launched beside it always find free thread slots instead of queueing
 *       behind a grid of thousands of short CTAs.  Same arithmetic, same result.
 * b200_detached_grad_rows: when *detached (DEVICE int32) is non-zero, grad[i] = 0 for i in each [begin, end) of ranges
 * (HOST long long[n_ranges][2], by value); otherwise nothing is touched.  The fused trainer clears the Gaussian and
 * background rows of a detached image's gradient with it, after the backward and before the scale regulariser. */
#define B200_ADAM_MAX_GROUPS 16
#define B200_ADAM_MAX_SEGMENTS 16
#define B200_LR_GROUP_DOUBLES 7
#define B200_ADAM_SEGMENT_WORDS 6
#define B200_ADAM_GROUP_TABLE_FLOATS 64
#define B200_DETACHED_MAX_RANGES 4
#define B200_ADAM_CLEAR_ON_VETO 2
B200_API size_t b200_adam_state_bytes(void);
B200_API int b200_adam_prepare_step(void *state, int32_t *veto_flag, const int32_t *detached, unsigned detached_groups,
                                    int cond_group, int cond_every, int n_groups, const double *groups, double beta1,
                                    double beta2, float *group_table, void *stream);
B200_API int b200_adam_update(long long numel, long long offset, float *param, float *grad, float *exp_avg,
                              float *exp_avg_sq, int n_segments, const long long *segments, const void *state,
                              const float *group_table, double beta1, double beta2, double eps, double grad_scale,
                              int zero_grad, int ctas_per_sm, void *stream);
B200_API int b200_detached_grad_rows(const int32_t *detached, int n_ranges, const long long *ranges, float *grad,
                                     void *stream);

/* ---- rasterization without a host sync ---------------------------------------------------------------------------
 * The reference reads the intersection count back to size its lists (gsplat/utils.py:123-124 `.item()`); the two-phase
 * culled binning above reads the culled count.  In CAPACITY mode the caller sizes the lists from a running high-water
 * mark instead: b200_bin_cull_count with totals_host_pinned = NULL, then b200_bin_cull_emit_capacity.  The id list has
 * `capacity` slots: the real entries in the reference's order, then padding that belongs to no tile.
 * status: DEVICE int32[4]: [0] |= 1 if this image's entries did not fit (lists incomplete: discard the render -- veto the
 * optimizer step with b200_adam_prepare_step, grow the capacity, repeat the image), [1] entries of this image, [2] running
 * maximum, [3] the reference's num_intersects of this image.  b200_blend_forward_packed_status = b200_blend_forward_packed
 * plus the reference's empty-render branch (rasterize.py:136-144: background image, final_Ts = 0, alpha = 1) taken on
 * the device when status[3] < 1.  b200_set_record_colors patches the colours of packed records (everything the binning
 * reads is colour-independent, so a caller may bin before it has shaded). */
B200_API int b200_bin_cull_emit_capacity(int num_points, int capacity, const void *packed, const int32_t *radii,
                                         const int32_t *num_tiles_hit, unsigned img_height, unsigned img_width,
                                         unsigned block_width, unsigned n_blur_samples, float rolling_shutter_time,
                                         float exposure_time, const void *ws_g, void *ws_e, size_t ws_e_bytes,
                                         int32_t *gaussian_ids_sorted, int32_t *tile_bins, int32_t *status, void *stream);
B200_API int b200_blend_forward_packed_status(unsigned img_height, unsigned img_width, unsigned block_width,
                                              unsigned n_blur_samples, const int32_t *gaussian_ids_sorted,
                                              const int32_t *tile_bins, const void *packed, float rolling_shutter_time,
                                              float exposure_time, const float *background, const int32_t *status,
                                              float *out_img, float *final_Ts, int32_t *final_idx, float *out_alpha,
                                              void *stream);
B200_API int b200_set_record_colors(int num_points, const float *colors, void *packed, void *stream);

/* ---- adaptive density control on the flat buffers ("next" row f-2 of SURVEY section 8) -----------------------------------
 * replaces the Python mask / torch.cat / optimizer-state surgery of nerfstudio/models/splatfacto.py:352-622:
 *   b200_densify_accumulate  after_train (:408-434): grad_norm += |absgrad|, vis_counts += 1, max_2d = max(., radius /
 *       max_dim), max_dim = max(H, W), for the Gaussians visible in this image (radii > 0); first != 0: the first image since the last
 *       refinement initialises all three for EVERY Gaussian (norm, 1, 0) like the reference does.
 *   b200_densify_plan        refinement_after + cull_gaussians (:443-566): every split / duplicate / cull decision and,
 *       by two prefix sums, the final row of every survivor in the reference's order (kept originals, the children of
 *       split sample 0, 1, ..., the duplicates).  Negative split_screen_size / cull_scale_thresh / cull_screen_size switch
 *       that criterion off (the reference's step schedule, :462, :545, :548); do_densify = 0 culls only.
 *       counts (DEVICE int32[4]): new row count, splits, duplicates, culled originals -- the caller reads it once to size
 *       the new buffers.  ws: b200_densify_ws_bytes(num_points, n_split_samples) bytes, 256-byte aligned, kept for the gathers.
 *   b200_densify_gather      writes one field of the new buffers: field 0 copy; 1 means (split children are placed at
 *       mean + R(q/|q|) (exp(log_scale) * z), z = row sample * n_splits + rank of `randn`, the caller's
 *       (n_split_samples * n_splits, 3) normal draw, :574-582); 2 log-scales (split children shrink by 1.6, :596);
 *       3 optimizer moment (children start at zero, :384-399).  src (N, width) -> dst (new count, width). */
B200_API int b200_densify_accumulate(int num_points, const float *absgrad, const int32_t *radii, float max_dim, int first,
                                     float *grad_norm, float *vis_counts, float *max_2d, void *stream);
B200_API size_t b200_densify_ws_bytes(int num_points, int n_split_samples);
B200_API int b200_densify_plan(int num_points, const float *log_scales, const float *opacity_logit, const float *grad_norm,
                               const float *vis_counts, const float *max_2d, float half_max_dim, float densify_grad_thresh,
                               float densify_size_thresh, float split_screen_size, int n_split_samples,
                               float cull_alpha_thresh, float cull_scale_thresh, float cull_screen_size, int do_densify,
                               void *ws, size_t ws_bytes, int32_t *counts, void *stream);
B200_API int b200_densify_gather(int num_points, int n_split_samples, int field, int width, const float *src, float *dst,
                                 const void *ws, const int32_t *counts, const float *log_scales, const float *quats,
                                 const float *randn, void *stream);

/* ---- camera pose optimisation (Splatfacto's SO3xR3 camera optimiser) ---------------------------------------------------
 * A camera row is 21 floats: viewmat (3x4 row major) 12 | lin_vel 3 | ang_vel 3 | cam_pos 3, as built from an OpenGL c2w by
 * gsplat.data.to_gsplat_camera (viewmat = [R^T | -R^T t] with R = c2w's rotation times diag(1,-1,-1), cam_pos = t).  A
 * pose row is 6 floats [trans 3 | rot 3], zero = no correction; pose is (num_cameras, 6), index DEVICE int64[num_views]
 * names each view's pose row.  Nothing is read from the host, so all three may be captured in a CUDA graph.
 *   b200_camera_pose_apply: out_rows[v] = row v with c2w' = c2w [exp_map_SO3xR3(pose[index[v]])] (cameras/lie_groups.py:
 *       24-59, camera_optimizers.py:175-187) turned into viewmat and cam_pos as above (splatfacto.py:734-745, :843); the
 *       velocities are copied.  A view whose index is outside [0, num_cameras) gets a row of NaNs.  out_rows must not alias rows.
 *   b200_camera_pose_backward: g_viewmat (num_views, 12), the gradient of the ADJUSTED viewmats, becomes the pose-row
 *       gradient, ADDED into g_pose (num_cameras, 6) at each view's index.  One CTA; views that share a pose row are added in
 *       view order with separately rounded adds, so the result is deterministic and equals num_views sequential calls.
 *       cam_pos carries no gradient (the reference detaches it).  Views with an out-of-range index add nothing.
 *   b200_camera_l2: the camera regulariser (camera_optimizers.py:189-195, :267-273) of an (num_rows, 6) block split 3 | 3:
 *       value[0] += w_a * mean_i |rows_i[0:3]| + w_b * mean_i |rows_i[3:6]|, and its gradient ADDED into g_rows (zero for
 *       a zero-norm half, as torch gives it).  One CTA, a fixed summation order, no atomics. */
B200_API int b200_camera_pose_apply(int num_views, int num_cameras, const float *rows, const float *pose,
                                    const int64_t *index, float *out_rows, void *stream);
B200_API int b200_camera_pose_backward(int num_views, int num_cameras, const float *rows, const float *pose,
                                       const int64_t *index, const float *g_viewmat, float *g_pose, void *stream);
B200_API int b200_camera_l2(int num_rows, const float *rows, float w_a, float w_b, float *g_rows, float *value,
                            void *stream);

/* ---- learnable background and scale regulariser (Splatfacto's background_color "auto", use_scale_regularization) -------
 * Nothing is read from the host, so all three may be captured in a CUDA graph.  b200_background_vjp and
 * b200_scale_regularizer reduce in a fixed order (per-thread, warp, block, then the block partials in block order by the
 * last block to finish) and are bit-reproducible from call to call, in deterministic mode or not.  ws: DEVICE,
 * b200_bg_scale_ws_bytes() bytes, 16-byte aligned; its first word is a ticket each call leaves at zero, so a caller that
 * zeroed the workspace once passes ws_is_zeroed = 1 (0 = cleared here first).  One workspace serves calls queued one after
 * another on one stream.
 *   b200_background_forward: background[c] = 1 / (1 + exp(-logit[c])) for c < 3 (splatfacto.py:706-707), the colour the
 *       blend kernels then read as `background`.
 *   b200_background_vjp: g_logit[c] = (v_b[c] * (1 - background[c])) * background[c] with v_b[c] = sum_px v_rgb[px][c] *
 *       (sum_s final_Ts[px][s]) * (1 / n_samples), the reference's v_background (gsplat/rasterize.py:266-270) through the
 *       sigmoid; v_rgb (num_pixels, 3), final_Ts (num_pixels, n_samples).  g_logit (3 floats) is OVERWRITTEN.
 *   b200_scale_regularizer: when word [4] of adam_state (the b200_adam_prepare_step state: steps prepared so far, the index of
 *       the step whose loss this is) is a multiple of `every`, value[0] += weight * mean_i(max(r_i, max_ratio) - max_ratio)
 *       with r_i = amax_j(exp(log_scales[i][j])) / amin_j(exp(log_scales[i][j])) (splatfacto.py:968-977), and its
 *       gradient, torch's (ties split evenly, half the gradient at r_i == max_ratio), ADDED into g_log_scales
 *       (num_points, 3); otherwise nothing is touched.  One thread per Gaussian row, no atomics. */
B200_API size_t b200_bg_scale_ws_bytes(void);
B200_API int b200_background_forward(const float *logit, float *background, void *stream);
B200_API int b200_background_vjp(long long num_pixels, int n_samples, const float *v_rgb, const float *final_Ts,
                                 const float *background, float *g_logit, void *ws, int ws_is_zeroed, void *stream);
B200_API int b200_scale_regularizer(int num_points, const float *log_scales, float max_ratio, float weight, int every,
                                    const void *adam_state, float *g_log_scales, float *value, void *ws, int ws_is_zeroed,
                                    void *stream);

#ifdef __cplusplus
}
#endif
#endif /* B200SPLAT_H */
