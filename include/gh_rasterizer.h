/*
 * gh_rasterizer.h -- C ABI of libgh_raster.so, the H100-native (sm_90a) strand-aligned
 * differentiable Gaussian rasterizer.
 *
 * Drop-in boundary.  These entry points are what the reference's native binding for this path
 * binds today:
 *
 *   reference (ext/diff_gaussian_rasterization_hair)                      replaced by
 *   --------------------------------------------------------------------  ------------------------------
 *   CudaRasterizer::Rasterizer::forward   (cuda_rasterizer/rasterizer.h:31-55,   gh_forward_preprocess()
 *                                          rasterizer_impl.cu:198-340)            + gh_forward_render()
 *   CudaRasterizer::Rasterizer::backward  (rasterizer.h:57-87,                    gh_backward()
 *                                          rasterizer_impl.cu:344-441)
 *   CudaRasterizer::Rasterizer::markVisible (rasterizer.h:24-29,                  gh_mark_visible()
 *                                          rasterizer_impl.cu:141-153)
 *   required<GeometryState/ImageState/BinningState>() (rasterizer_impl.h:65-72)   gh_*_workspace_size*()
 *   the three std::function<char*(size_t)> workspace callbacks                    two-phase protocol below
 *   (rasterize_points.cu:27-33,75-80)
 *
 * Conventions
 *   - every pointer is a DEVICE pointer to contiguous float32 / int32 data unless stated otherwise;
 *     NULL means "absent optional" (the reference's empty-tensor convention, __init__.py:210-222);
 *   - the library allocates no device memory and keeps no per-call state: the caller owns all buffers
 *     (outputs and the three opaque workspaces) and passes the CUDA stream explicitly (the reference
 *     uses the legacy default stream implicitly).  Entry points are re-entrant and may be called from
 *     several host threads (PyTorch calls gh_backward from its autograd thread) and for several
 *     devices.  The only process-wide state is diagnostic: an atomic kernel-launch counter, the
 *     optional stage timer (mutex-guarded sums, events created per stage on the caller's device) and
 *     the per-thread message behind gh_last_error();
 *   - matrices use the reference's row-vector (transposed) convention: viewmatrix[12..14] is the
 *     translation (auxiliary.h:58-66);
 *   - return value: 0 on success, a GH_E_* code otherwise; gh_last_error() gives the message for the
 *     calling thread;
 *   - `rotations` must be 16-byte aligned, `colors_precomp` 8-byte aligned (128-/64-bit loads).
 *
 * Two-phase forward (replaces the resize callbacks; the only host sync is the one the reference has
 * at rasterizer_impl.cu:285):
 *   1. gh_forward_workspace_sizes(P, W, H, &geom_bytes, &img_bytes); allocate both.
 *   2. gh_forward_preprocess(...): runs preprocess + per-tile histogram + scan, then copies the
 *      instance count R (= the reference's num_rendered) to the host and returns it.  Optionally it is
 *      handed a binning buffer sized from a guess of R; if R fits, it also runs the bucket scatter
 *      (*emitted = 1) and step 3 is skipped.
 *   3. gh_binning_workspace_size(R, &bytes); allocate.
 *   4. gh_forward_render(...): bucket scatter (unless emitted), per-tile sort, alpha compositing.
 * The three workspaces must be kept for gh_backward (the reference keeps its three byte tensors on
 * the autograd ctx, __init__.py:102).
 */
#ifndef GH_RASTERIZER_H_INCLUDED
#define GH_RASTERIZER_H_INCLUDED

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GH_NUM_CHANNELS_ABI 10   /* reference config.h:15 */

#define GH_OK 0
#define GH_E_INVALID_ARG 1      /* bad shape / alignment / missing mandatory input            */
#define GH_E_NO_COLORS 2        /* "For non-RGB, provide precomputed Gaussian colors!"         */
                                /* (rasterizer_impl.cu:244-247)                                */
#define GH_E_CUDA 3             /* a CUDA call or kernel failed                                */
#define GH_E_PREFILTERED 4      /* a point failed the near cull although prefiltered was set   */
                                /* (reference: device printf + __trap, auxiliary.h:156-160)    */

typedef void* gh_stream_t;      /* cudaStream_t */

/* ABI version; bumped on any signature change. */
int gh_abi_version(void);

/* Number of feature channels the library was built for (10). */
int gh_num_channels(void);

/* Number of CUDA kernels this library has launched since it was loaded (bench `gpu_launches`). */
unsigned long long gh_kernel_launch_count(void);

/*
 * Optional per-stage device timing for the roofline report: when enabled every stage is bracketed by
 * CUDA events on the caller's stream and synchronised (so it perturbs end-to-end time: keep it off in
 * timed regions).  Stage order: preprocess, tile_scan, emit, tile_sort, blend_forward, blend_backward,
 * preprocess_backward.  gh_stage_timing_read returns the number of stages.
 */
void gh_stage_timing_enable(int on);
int gh_stage_timing_read(double* ms_sum, unsigned long long* calls, int capacity);

/* Message of the last error on this thread ("" if none). */
const char* gh_last_error(void);

/* Sizes of the geometry (per-Gaussian) and image (per-pixel / per-tile) workspaces. */
int gh_forward_workspace_sizes(int P, int width, int height, size_t* geom_bytes, size_t* img_bytes);

/* Size of the binning (per-instance) workspace for R instances. */
int gh_binning_workspace_size(long long R, size_t* binning_bytes);

/*
 * Phase 1 of Rasterizer::forward.  Inputs as rasterizer.h:31-55 (D = active SH degree, M = SH
 * coefficients per Gaussian; `shs` is accepted for signature parity but, as in the reference build
 * with NUM_CHANNELS = 10, `colors_precomp` is mandatory).  Exactly one of (scales+rotations |
 * cov3D_precomp) is used when conic_precomp is NULL; when conic_precomp is given the conic is
 * taken from it.  means2D_precomp is never read (reference forward.cu:201-210).
 * Writes radii[P].  On return *num_rendered = R and *max_tile_len = longest per-tile list
 * (host values; the call synchronises `stream`).
 * Optional binning buffer: given binning_buffer of gh_binning_workspace_size(binning_capacity) bytes, the bucket
 * scatter (emit) is enqueued right behind the read-back of R, so it runs while the host waits and prepares phase 2.
 * *emitted = 1 if R <= binning_capacity: the buffer then holds the binned instances (pass it, with emitted = 1, to
 * gh_forward_render).  *emitted = 0 otherwise: nothing was written; size a buffer for R and call gh_forward_render
 * with emitted = 0.  binning_buffer = NULL, binning_capacity = 0 (emitted may then be NULL) runs no scatter here.
 * binning_capacity must lie in [0, 2^32); `emitted` is required with a buffer.
 */
int gh_forward_preprocess(
    int P, int D, int M,
    int width, int height,
    const float* means3D, const float* means2D_precomp, const float* shs,
    const float* colors_precomp, const float* opacities,
    const float* scales, float scale_modifier, const float* rotations,
    const float* cov3D_precomp, const float* conic_precomp,
    const float* viewmatrix, const float* projmatrix, const float* cam_pos,
    float tan_fovx, float tan_fovy, int prefiltered,
    int* radii,
    char* geom_buffer, char* img_buffer,
    char* binning_buffer, long long binning_capacity,
    int* num_rendered, int* max_tile_len, int* emitted,
    int debug, gh_stream_t stream);

/*
 * Phase 2 of Rasterizer::forward: binning + per-tile sort + front-to-back blend.
 * out_color is (C, H, W) channel-major, fully overwritten (background included).
 * emitted = 1 skips the bucket scatter that the first phase already ran into binning_buffer (gh_forward_preprocess /
 * gh_project_forward_binned reported *emitted = 1 for this buffer); emitted = 0 runs it here.
 */
int gh_forward_render(
    int P, int width, int height,
    const float* background, const float* colors_precomp,
    const int* radii,
    char* geom_buffer, char* binning_buffer, char* img_buffer,
    int num_rendered, int max_tile_len, int emitted,
    float* out_color,
    int debug, gh_stream_t stream);

/*
 * Rasterizer::backward (rasterizer.h:57-87).  Every element of every non-NULL gradient buffer is
 * written (zeros where nothing flows), so the caller need NOT zero-fill them (the reference's binding
 * does torch::zeros, rasterize_points.cu:160-168).  dL_dsh is never touched.  Shapes as there:
 * dL_dmean2D (P,3) [NDC units, z unused], dL_dconic (P,2,2) [.x .y .w used, .y = half the
 * off-diagonal derivative], dL_dopacity (P,1), dL_dcolor (P,C), dL_dmean3D (P,3), dL_dcov3D (P,6),
 * dL_dsh (P,M,3) [never written: SH path unreachable with C = 10], dL_dscale (P,3), dL_drot (P,4).
 * When conic_precomp is given (nothing flows through the geometry), dL_dmean2D, dL_dconic, dL_dopacity and
 * dL_dcolor may ALL be NULL: the blend backward's per-Gaussian accumulation records then stay in the geometry
 * workspace for gh_project_backward to consume directly (no unpack pass).
 *
 * det_buffer / det_bytes select the blend backward's summation order.  det_buffer == NULL (det_bytes 0): the
 * fast path, whose float sums depend on GPU scheduling (gradients agree run to run to ~1e-7, not bit for bit).
 * det_buffer != NULL: the deterministic path -- no atomics, every sum in a fixed order, so every gradient is a pure
 * function of the inputs (bit-identical across runs on the same GPU and build).  It needs det_bytes >=
 * gh_backward_det_workspace_size(P, R) bytes of device memory; a smaller buffer, or det_bytes != 0 without a
 * buffer, is rejected with GH_E_INVALID_ARG before anything is launched.
 */
int gh_backward_det_workspace_size(int P, long long R, size_t* bytes);

int gh_backward(
    int P, int D, int M, int R,
    int width, int height,
    const float* background,
    const float* means3D, const float* shs, const float* colors_precomp,
    const float* scales, float scale_modifier, const float* rotations,
    const float* cov3D_precomp, const float* conic_precomp,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    float tan_fovx, float tan_fovy,
    const int* radii,
    char* geom_buffer, char* binning_buffer, char* img_buffer,
    const float* dL_dpix,
    float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
    float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
    int debug, gh_stream_t stream,
    char* det_buffer, size_t det_bytes);

/* Rasterizer::markVisible: present[i] = (view-space z of point i > 0.2).  `present` is bool[P]. */
int gh_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                    unsigned char* present, gh_stream_t stream);

/*
 * Introspection of the opaque workspaces, for parity tests ("bit-exact tile keys and sort order").
 * Copies are device->device on `stream`; any output pointer may be NULL.
 *   keys_sorted[R]   = (tile_id << 32) | float_bits(depth)   in list order (reference point_list_keys)
 *   point_list[R]    = Gaussian index                        in list order (reference point_list)
 *   ranges[2*T]      = (start, end) per tile                 (reference imgState.ranges)
 *   final_T[W*H], n_contrib[W*H]                             (reference accum_alpha, n_contrib)
 *   depths[P], means2D[2*P], conic_opacity[4*P]              (reference geomState.*)
 */
int gh_debug_export(
    int P, int width, int height, long long R,
    const char* geom_buffer, const char* binning_buffer, const char* img_buffer,
    unsigned long long* keys_sorted, unsigned int* point_list, unsigned int* ranges,
    float* final_T, unsigned int* n_contrib,
    float* depths, float* means2D, float* conic_opacity,
    gh_stream_t stream);

/*
 * "Next" row (SURVEY.md 8f-2): fused multi-group Adam step with torch.optim.Adam's arithmetic
 * (reference: src/scene/gaussian_model.py:431-448, stepped at src/train_gaussians.py:174-181).
 * params/grads/exp_avg/exp_avg_sq are HOST arrays of n_groups (<= GH_ADAM_MAX_GROUPS) device pointers,
 * sizes[k] the element count and lrs[k] the learning rate of group k; `step` is 1-based and used when
 * step_state is NULL; otherwise step_state is a device int[2] {steps taken, scratch} owned by the caller
 * (zero-initialised) and the step count lives on the device (advanced only by steps that were not skipped).
 * nan_flag (device uint, may be NULL): when given, the step is skipped on the device if any gradient
 * holds a NaN and the flag is left non-zero (the reference's NaN guard without its host syncs).
 * skip_flag (device uint, may be NULL, read only): the step is also skipped when *skip_flag != 0 -- pass
 * the error word (local_sync + 2) or the nan_out word of gh_allreduce_p2p so that a failed or poisoned
 * gradient exchange never reaches the parameters.
 */
#define GH_ADAM_MAX_GROUPS 8
int gh_adam_step(int n_groups, float* const* params, const float* const* grads,
                 float* const* exp_avg, float* const* exp_avg_sq,
                 const unsigned long long* sizes, const float* lrs,
                 double beta1, double beta2, float eps, int step, int* step_state,
                 unsigned int* nan_flag, const unsigned int* skip_flag, gh_stream_t stream);

/*
 * "Next" row (SURVEY.md 8f-4): the image-space losses of the appearance stage, forward + backward in
 * one call, consuming the rasterizer's (10,H,W) output and producing dL/dout in the layout gh_backward
 * reads as dL_dpix.  Replaces, for this step of src/train_gaussians.py:
 *   l1_loss / ssim / or_loss            src/utils/loss_utils.py:19-48, 73-121
 *   the dir -> angle post-processing    src/gaussian_renderer/__init__.py:100-105
 *   the loss composition + NaN guard    src/train_gaussians.py:126-140
 * out_color (10,H,W): image 0..2, mask 3..4, dir 5..7, orientation confidence 8, depth 9.
 * gt_image (3,H,W), gt_mask (2,H,W), gt_orient_angle (1,H,W), gt_orient_conf (1,H,W): device float32.
 * workspace: gh_image_loss_workspace_size bytes, 8-byte aligned.
 * losses (device float[8]): total, Ll1, Lssim, Lmask, Lorient, sum of orientation weights,
 *   1 if Lorient was NaN (then it counts as 0 and has no gradient, like the reference), 0.
 * dL_dout (10,H,W): d total / d out_color, every element written.  No host synchronisation.
 * deterministic != 0: the five loss sums are formed without floating-point atomics, in a fixed order (per-CTA slots
 *   added in CTA order by the last CTA), so losses and dL_dout are bit-identical run to run; 0: one double atomicAdd
 *   per CTA and sum, the faster path.
 */
int gh_image_loss_workspace_size(int width, int height, size_t* bytes);
int gh_image_loss(int width, int height, const float* out_color, const float* gt_image,
                  const float* gt_mask, const float* gt_orient_angle, const float* gt_orient_conf,
                  float lambda_dl1, float lambda_dssim, float lambda_dmask, float lambda_dorient,
                  void* workspace, float* losses, float* dL_dout, gh_stream_t stream, int deterministic);

/*
 * The image loss of each training stage, in the same kernels as gh_image_loss (inputs, workspace and losses[8] as
 * there; gh_image_loss_workspace_size serves every stage):
 *   GH_LOSS_STAGE_APPEARANCE      src/train_gaussians.py:126-140, bit-identical to gh_image_loss
 *   GH_LOSS_STAGE_STRANDS         src/train_strands.py:128-147: Ll1 = l1_loss(image, gt_image) and
 *                                 Lssim = 1 - ssim(image, gt_image), both unmasked; Lmask and Lorient as appearance
 *   GH_LOSS_STAGE_LATENT_STRANDS  src/train_latent_strands.py:130-152: Ll1 unmasked, no SSIM term,
 *                                 LCE = l1_loss(mask[:1], gt_mask[:1]) (channel 3 only), LOR as Lorient
 * options (strand stages only):
 *   GH_LOSS_ORIENT_UNIT_WEIGHT    opt.use_gt_orient_conf == False: orientation weight 1, sum of weights W H;
 *                                 gt_orient_conf may then be NULL and is not read
 *   GH_LOSS_ORIENT_NO_CONF        opt.train_orient_conf == False: or_loss(..., confs=None), no conf factor and no
 *                                 log term; channel 8 of dL_dout is exactly 0
 * losses[8]: total, Ll1, Lssim, Lmask, Lorient, sum of orientation weights, Lorient-was-NaN, slot 7.  Stage 2: slot 2
 *   is 0, slot 3 holds LCE, slot 7 the terms replaced by 0 because they were NaN as a float bitmask (1 Ll1, 2 LCE);
 *   slot 7 is 0 in the other stages.  total is the reference's sum without its prior term (lambda_dsds Lsds or
 *   lambda_dsds LDF), in the reference's order, so a trainer that adds that term afterwards gets the reference's total.
 * dL_dout: every element written.  Channels 7 and 9 are 0; in stage 2 channel 4 is 0; a replaced term contributes
 *   exactly 0: Lorient / LOR channels 5, 6, 8, and in stage 2 Ll1 channels 0..2 and LCE channel 3.  Stage 1 replaces
 *   only Lorient, like the reference: a NaN Ll1 or Lssim stays NaN in the total.
 * deterministic: as gh_image_loss.
 * Refused with GH_E_INVALID_ARG before any CUDA call: a stage outside 0..2, option bits with stage 0, unknown option
 *   bits, lambda_dssim != 0 with stage 2, a NULL gt_orient_conf without GH_LOSS_ORIENT_UNIT_WEIGHT, and everything
 *   gh_image_loss refuses.
 */
#define GH_LOSS_STAGE_APPEARANCE     0
#define GH_LOSS_STAGE_STRANDS        1
#define GH_LOSS_STAGE_LATENT_STRANDS 2
#define GH_LOSS_ORIENT_UNIT_WEIGHT   1u
#define GH_LOSS_ORIENT_NO_CONF       2u
int gh_image_loss_stage(int width, int height, int stage, unsigned options,
                        const float* out_color, const float* gt_image, const float* gt_mask,
                        const float* gt_orient_angle, const float* gt_orient_conf,
                        float lambda_dl1, float lambda_dssim, float lambda_dmask, float lambda_dorient,
                        void* workspace, float* losses, float* dL_dout, gh_stream_t stream, int deterministic);

/*
 * Rendering without a backward: the maps src/render_gaussians.py:50-68 and src/render_strands.py:51-69 write for every
 * view, from the raw out_color (10,H,W) in one pass.  Every output is optional (NULL: not wanted):
 *   orient_angle        float (H,W)    the epilogue of src/gaussian_renderer/__init__.py:100-105, the same device code
 *                                      as the image losses
 *   orient_conf_masked  float (H,W)    orient_conf * hair_mask (what the scripts torch.save to orient_confs/)
 *   render_u8           uint8 (H,W,3)  save_image(render), interleaved RGB
 *   hair_mask_u8, head_mask_u8  uint8 (H,W)   save_image(mask[:1]), save_image(mask[1:])
 *   orient_u8           uint8 (H,W)    save_image(orient_angle * hair_mask)
 *   orient_vis_u8       uint8 (H,W,3)  save_image(vis_orient(orient_angle, hair_mask))  (src/utils/image_utils.py:22-37)
 *   orient_conf_vis_u8  uint8 (H,W,3)  save_image(vis_orient(orient_angle, 1 - 1 / (orient_conf * hair_mask + 1)))
 * save_image's bytes are x.mul(255).add_(0.5).clamp_(0, 255).to(uint8); every float operation here is rounded on its
 * own like the tensor code (no FMA contraction), so the bytes are those of that composition on the same raw image.
 * A NaN value becomes byte 0.  The byte maps must be 4-byte aligned.  One launch on `stream`, no allocation, no host
 * synchronisation; refuses (GH_E_INVALID_ARG, before any launch) bad sizes, a NULL out_color, more than 2^27 pixels.
 */
int gh_render_maps(int width, int height, const float* out_color, float* orient_angle, float* orient_conf_masked,
                   unsigned char* render_u8, unsigned char* hair_mask_u8, unsigned char* head_mask_u8,
                   unsigned char* orient_u8, unsigned char* orient_vis_u8, unsigned char* orient_conf_vis_u8,
                   gh_stream_t stream);

/*
 * One view's numbers of the trainers' training_report, from the raw out_color and the view's ground truth maps (as
 * gh_image_loss takes them), written to row (device float[8]) -- a caller evaluating N views hands in row i of an
 * (N,8) buffer and reads it back once.  stage: GH_LOSS_STAGE_*.
 *   APPEARANCE, STRANDS (src/train_gaussians.py:254-277, src/train_strands.py): render, mask, orient_angle and their
 *     ground truths clamped to [0,1]; l1 = mean |image - gt|; mask = mean |mask - gt_mask| over both channels;
 *     or = or_loss(angle, gt_angle, mask=gt_mask[:1], weight=gt_orient_conf); psnr = mean over the three channels of
 *     20 log10(1 / sqrt(mse_c)).
 *   LATENT_STRANDS (src/train_latent_strands.py:235-258): image and gt multiplied by gt_mask[:1] before l1 and psnr;
 *     ce_loss(mask[:1], gt_mask[:1]) in place of the mask term.
 * row: l1, mask or ce, or, psnr, ssim, mse_r, mse_g, mse_b.  The ssim slot is NaN: it is not computed.  A zero weight
 *   sum gives or = NaN (0 / 0) and mse_c = 0 gives psnr = inf, like the reference.
 * The sums are formed in a fixed order (per-CTA slots in the workspace, added in CTA order by the last CTA, in double):
 * the row is bit-identical run to run.  workspace: gh_eval_metrics_workspace_size bytes, 8-byte aligned.  Three stream
 * operations (memset + 2 launches), no allocation, no host synchronisation; refuses (GH_E_INVALID_ARG, before any CUDA
 * call) bad sizes, a NULL pointer, an unknown stage, a workspace that is misaligned or smaller than the size query's.
 */
int gh_eval_metrics_workspace_size(int width, int height, size_t* bytes);
int gh_eval_metrics(int width, int height, int stage, const float* out_color, const float* gt_image,
                    const float* gt_mask, const float* gt_orient_angle, const float* gt_orient_conf,
                    void* workspace, size_t workspace_bytes, float* row, gh_stream_t stream);

/*
 * SSIM and PSNR of B image pairs, forward only (src/metrics.py):
 *   ssim[i] = loss_utils.ssim(img1[i], img2[i]) with size_average: the 11x11 Gaussian window (sigma 1.5, float32 1-D
 *     taps as create_window builds them, applied separably), zero padding 5, C1 = 0.01^2, C2 = 0.03^2, the mean of
 *     ssim_map over 3 H W;
 *   psnr[i] = image_utils.psnr on a (1,3,H,W) image: 20 log10(1 / sqrt(mse)) with one mse over all 3 H W values
 *     (mse 0 gives +inf).
 * img1, img2: B pairs of planar (3,H,W) images (channel stride H W), pair i at element offset i * stride1 / stride2 --
 *   so a stack of raw (10,H,W) renders is read in place with stride 10 H W.  dtype GH_DTYPE_FLOAT32, or
 *   GH_DTYPE_UINT8 read as x / 255 rounded as torchvision's to_tensor rounds it: a uint8 pair and its float32
 *   conversion give the same bits.  flags: GH_SSIM_CLAMP_IMG1 / _IMG2 clamp that image to [0,1] after conversion (what
 *   training_report does to a render and its ground truth).  mask: NULL, or per pair a float32 (1,H,W) multiplier at
 *   offset i * mask_stride applied to both images (the latent strand stage's gt_mask[:1]), clamped to [0,1] with
 *   GH_SSIM_CLAMP_MASK.
 * ssim (device float, pair i at i * ssim_stride) is required, psnr (same layout) optional: NULL skips it.  Pointing
 *   them into slot 4 / 3 of an (N,8) gh_eval_metrics row buffer takes stride 8.
 * Sums are per-pixel terms in double, per CTA through a fixed-order block sum, the CTAs of a pair added in CTA order:
 *   the results are bit-identical run to run, and pair i's bits do not depend on B or on the other pairs.
 * workspace: gh_eval_ssim_workspace_size(B, W, H) bytes, 8-byte aligned.  debug != 0 synchronises after the launches
 * and reports a failure there.  Three stream operations (memset + 2 launches), no allocation, no host synchronisation
 * (unless debug).  Refused (GH_E_INVALID_ARG, before any CUDA call): B, W or H <= 0, B > 65535, B 3 H W or the strided
 * extent beyond 2^31 - 1 elements, overlapping pair strides, an unknown dtype code or flag bit, a NULL image, ssim or
 * workspace pointer, misaligned float arrays, a workspace that is misaligned or smaller than the size query's, and
 * debug != 0 while the stage timer is on.
 */
#define GH_DTYPE_FLOAT32 0
#define GH_DTYPE_UINT8   1
#define GH_SSIM_CLAMP_IMG1 1u
#define GH_SSIM_CLAMP_IMG2 2u
#define GH_SSIM_CLAMP_MASK 4u
int gh_eval_ssim_workspace_size(int B, int width, int height, size_t* bytes);
int gh_eval_ssim(int B, int width, int height, const void* img1, int dtype1, long long stride1,
                 const void* img2, int dtype2, long long stride2, const float* mask, long long mask_stride,
                 unsigned flags, float* ssim, long long ssim_stride, float* psnr, long long psnr_stride,
                 void* workspace, size_t workspace_bytes, int debug, gh_stream_t stream);

/*
 * Multi-GPU (SURVEY.md 8e): sum a float32 buffer that lives in SYMMETRIC memory (the same allocation on
 * every GPU of the node, each mapped into every process, e.g. torch.distributed._symmetric_memory) over
 * all ranks, in place, with one kernel per rank that reads and writes its peers' copies through NVLink.
 * Replaces the NCCL all-reduce of the gradient arena; every rank of the group must make the same call.
 * peer_bufs / peer_flags: HOST arrays of `world` device addresses (this process's mappings of every
 *   rank's buffer and of every rank's flag block; flag block = uint32[3 * world], zero-initialised once).
 * multicast_buf: NVLS multicast mapping of the buffer, or 0 (then plain peer loads/stores are used).
 * offset_floats, n_floats: the range to reduce (multiples of 4; buffers 16-byte aligned).
 * epoch: 1, 2, 3, ... strictly increasing per call on every rank.
 * local_sync: device uint32[8] of this rank, zero-initialised once; word 2 (sticky) becomes non-zero if a
 *   peer did not arrive within the wall-clock bound (GH_ALLREDUCE_TIMEOUT_MS, default 30000): the reduction
 *   of that call is then SKIPPED on this rank (no partial sums) and the buffer content is undefined.
 * nan_out (device uint, may be NULL): set to 1 if the SUM holds a NaN anywhere in the range (identical on
 *   every rank: the per-slice findings are exchanged with the exit barrier), else 0.
 * Tunables (environment, read per call): GH_ALLREDUCE_THREADS, GH_ALLREDUCE_CTAS_PER_SM,
 *   GH_ALLREDUCE_UNROLL (NVLS path: 16-byte requests in flight per thread).
 */
int gh_allreduce_p2p(const unsigned long long* peer_bufs, const unsigned long long* peer_flags,
                     unsigned long long multicast_buf, int rank, int world,
                     size_t offset_floats, size_t n_floats, unsigned int epoch,
                     unsigned int* local_sync, unsigned int* nan_out, gh_stream_t stream);

/*
 * "Next" row (SURVEY.md 8f-1): the caller-side projection preamble, fused.  One forward and one backward kernel
 * replace the PyTorch code that `render()` / `render_hair()` run before every rasterizer call:
 *   GaussianModel.get_conic / get_covariance_2d / get_covariance   src/scene/gaussian_model.py:230-315
 *   get_mean_2d :317-337, get_depths :339-342, get_direction_2d :344-393, filter_points :143-228
 *   the parameter activations :106-141, eval_sh (src/utils/sh_utils.py:57-112), the feature concatenation and the
 *   boolean-mask gathers (src/gaussian_renderer/__init__.py:29-83, :122-186; strand models:
 *   src/scene/gaussian_model_latent_strands.py:109-440).
 * Inputs are the RAW model parameters (device float32, contiguous): xyz (P,3), scaling (P,3), rotation (P,4, raw
 * quaternion, 16-byte aligned), dirs (P,3) or NULL, features_dc (P,1,3), features_rest (P,15,3) [NULL allowed for
 * sh_degree 0], opacity / label / orient_conf (P,1) or NULL when their activation is a constant; viewmatrix,
 * projmatrix (4,4, row-vector convention) and campos (3).
 * flags: bits 0-1 scale activation (0 identity, 1 exp), 2-3 opacity (0 identity, 1 sigmoid, 2 constant 1),
 *   4-5 label (0 identity, 1 sigmoid, 2 constant 1, 3 constant 0), 6-7 orientation confidence (0 identity, 1 exp,
 *   3 constant 0), 8-9 direction feature (0: s_max * R[argmax s], 1: normalize(dirs), 2: zero),
 *   10 strand mode: Gaussian i is segment i of a polyline (src/scene/gaussian_model_strands.py:435-454) and its
 *   geometry is derived from the segment vector d = dirs[i]: scales (|d|/2, scale, scale), rotation
 *   parallel_transport(e_x, d).  `scaling` then points to ONE device float, the strand thickness `scale` (no host
 *   read); `rotation`, `d_scaling` and `d_rotation` must be NULL; `dirs` and `d_dirs` are required; the scale
 *   activation must be 0 and the direction feature 1.  The backward folds the scale and rotation gradients into
 *   d_dirs (the direct term of each segment) and writes the gradient w.r.t. the segment midpoint to d_xyz: finish
 *   with gh_strand_backward.
 * det_eps: added to the 2-D determinant before inversion (1e-12 GaussianModel, 1e-7 strand models).
 * Forward outputs: means2D (P,3) NDC, colors (P,10), opacities (P,1), conic (P,3), cov3D (P,6) or NULL,
 *   visible (P) uint8 = the caller's prefilter.  Culled Gaussians are NOT compacted away: their conic is 0, which the
 *   rasterizer drops (zero determinant), so indices stay the model's own and `prefiltered` must be passed as 0.
 * Backward: the incoming gradients are either the four tensors gh_backward produces (dL_dmeans2D (P,3),
 *   dL_dconic (P,2,2) native layout, dL_dcolors (P,10), dL_dopacity (P,1)) or, when geom_buffer is given, the
 *   accumulation records that gh_backward leaves in the geometry workspace (see gh_backward: pass NULL for its four
 *   2-D gradient outputs).  Every row of every per-Gaussian gradient is written (zeros for culled Gaussians);
 *   any of d_dirs, d_opacity, d_label, d_orient_conf, d_means2D may be NULL.  d_camera (device float[37], or NULL):
 *   dL/dviewmatrix (16), dL/dprojmatrix (16), dL/dcampos (3), dL/dtan_fovx, dL/dtan_fovy -- summed per CTA and then
 *   in a fixed order by the last CTA (deterministic); needs `workspace` (gh_project_workspace_size bytes,
 *   16-byte aligned).  nan_flag (device uint, or NULL): OR-ed with 1 when any per-Gaussian gradient is NaN -- the
 *   optimizer's NaN guard without a second pass over the gradients (pass it to gh_adam_step as skip_flag; the caller
 *   zeroes it).
 */
int gh_project_workspace_size(int P, size_t* bytes);
int gh_project_forward(
    int P, int width, int height,
    const float* xyz, const float* scaling, const float* rotation, const float* dirs,
    const float* features_dc, const float* features_rest,
    const float* opacity, const float* label, const float* orient_conf,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    float tan_fovx, float tan_fovy, float scale_modifier, int sh_degree, unsigned int flags, float det_eps,
    float* means2D, float* colors, float* opacities, float* conic, float* cov3D, unsigned char* visible,
    gh_stream_t stream);
/* gh_project_forward + gh_forward_preprocess in ONE pass over the Gaussians (the fused render path): besides the
 * outputs of gh_project_forward it fills `radii` and the geometry / image workspaces exactly as gh_forward_preprocess
 * would when handed (xyz, conic, opacities) with prefiltered = 0 -- same device code, bit-identical radii, state
 * records and keys -- runs the tile scan and returns num_rendered / max_tile_len after the same 16-byte read-back.
 * binning_buffer, binning_capacity, emitted: the optional binning buffer of gh_forward_preprocess (same contract).
 * Continue with gh_forward_render.  Workspaces: gh_forward_workspace_sizes. */
int gh_project_forward_binned(
    int P, int width, int height,
    const float* xyz, const float* scaling, const float* rotation, const float* dirs,
    const float* features_dc, const float* features_rest,
    const float* opacity, const float* label, const float* orient_conf,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    float tan_fovx, float tan_fovy, float scale_modifier, int sh_degree, unsigned int flags, float det_eps,
    float* means2D, float* colors, float* opacities, float* conic, float* cov3D, unsigned char* visible,
    int* radii, char* geom_buffer, char* img_buffer, char* binning_buffer, long long binning_capacity,
    int* num_rendered, int* max_tile_len, int* emitted,
    gh_stream_t stream);
int gh_project_backward(
    int P, int width, int height,
    const float* xyz, const float* scaling, const float* rotation, const float* dirs,
    const float* features_dc, const float* features_rest,
    const float* opacity, const float* label, const float* orient_conf,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    float tan_fovx, float tan_fovy, float scale_modifier, int sh_degree, unsigned int flags, float det_eps,
    const unsigned char* visible,
    const char* geom_buffer,
    const float* dL_dmeans2D, const float* dL_dconic, const float* dL_dcolors, const float* dL_dopacity,
    float* d_xyz, float* d_scaling, float* d_rotation, float* d_dirs, float* d_features_dc, float* d_features_rest,
    float* d_opacity, float* d_label, float* d_orient_conf, float* d_means2D, float* d_camera,
    unsigned int* nan_flag, void* workspace, gh_stream_t stream);

/*
 * Capturable training iteration (CUDA graphs; DESIGN §16).  These entry points do the work of the calls they are named
 * after for the GaussianModel call shape (fused projection, conic supplied, records mode), but none of them
 * synchronises with the host, allocates, or takes a value that changes between iterations as a host argument, so a
 * stream capture of them can be replayed for every camera and every step:
 *   - tan(fov / 2) is read from `tan_fov`, a device float[2] (x, y);
 *   - R, the number of tile instances, and the longest tile list exist only on the device;
 *   - the binning buffer holds `capacity` records (gh_binning_workspace_size(capacity) bytes), the deterministic
 *     workspace gh_backward_det_workspace_size(P, capacity) bytes; capacity lies in [0, 2^32).
 * Overflow (R > capacity) is safe by construction: the first phase ORs GH_STATUS_BINNING_OVERFLOW into the caller's
 * device uint32 `status` and empties the frame -- every radius 0, every tile range (0, 0) -- so that no kernel reads
 * or writes a binning record at or beyond `capacity`, and every output is still written: the image is the background
 * (final_T = 1, n_contrib = 0), the accumulation records and all gradients are zero.  Pass `status` as the skip_flag
 * of gh_adam_step_capturable so that the iteration's update is skipped on the device, and zero it before each
 * iteration.  Each entry point rejects debug != 0, and any call while the stage timer is on, with GH_E_INVALID_ARG
 * before it launches anything.
 *
 * gh_project_forward_binned_capturable: gh_project_forward_binned (non-strand flags; no cov3D) with tan fov from the
 *   device, no read-back and no pinned memory; emit is always enqueued into `binning_buffer`.  num_rendered (device
 *   uint32, or NULL) receives R, also on overflow.  `status` is required.
 * gh_forward_render_capturable: per-tile sort and blend of gh_forward_render (emitted = 1) with R and the longest list
 *   taken on the device: the long-list split and segment sort are always launched, on grids bounded by T and
 *   `capacity`, and their CTAs leave at once when no list exceeds the in-kernel sort's 1792 records.  With the same
 *   inputs and R <= capacity the image, final_T, n_contrib and the sorted lists are bit-identical to gh_forward_render.
 * gh_backward_capturable: the records-mode blend backward of gh_backward (conic supplied, the four 2-D gradient
 *   outputs NULL): the accumulation records are left in the geometry workspace.  det_buffer selects the deterministic
 *   variant as in gh_backward (records bit-identical to it); NULL the fast one.  An empty or overflowed frame yields
 *   zero records (no host branch on R).
 * gh_project_backward_capturable: gh_project_backward with tan fov from the device.
 * gh_adam_step_capturable: gh_adam_step with `lrs` a DEVICE float[n_groups] and the device step count `step_state`
 *   mandatory; same arithmetic, so the same inputs give bit-identical parameters and moments.
 */
#define GH_STATUS_BINNING_OVERFLOW 1u
int gh_project_forward_binned_capturable(
    int P, int width, int height,
    const float* xyz, const float* scaling, const float* rotation, const float* dirs,
    const float* features_dc, const float* features_rest,
    const float* opacity, const float* label, const float* orient_conf,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree, unsigned int flags, float det_eps,
    float* means2D, float* colors, float* opacities, float* conic, unsigned char* visible,
    int* radii, char* geom_buffer, char* img_buffer, char* binning_buffer, long long capacity,
    unsigned int* status, unsigned int* num_rendered, int debug, gh_stream_t stream);
int gh_forward_render_capturable(
    int P, int width, int height, long long capacity,
    const float* background, const float* colors_precomp,
    char* geom_buffer, char* binning_buffer, char* img_buffer,
    float* out_color, int debug, gh_stream_t stream);
int gh_backward_capturable(
    int P, int width, int height, long long capacity,
    const float* background, const float* colors_precomp, const int* radii,
    char* geom_buffer, char* binning_buffer, char* img_buffer,
    const float* dL_dpix, int debug, gh_stream_t stream, char* det_buffer, size_t det_bytes);
int gh_project_backward_capturable(
    int P, int width, int height,
    const float* xyz, const float* scaling, const float* rotation, const float* dirs,
    const float* features_dc, const float* features_rest,
    const float* opacity, const float* label, const float* orient_conf,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree, unsigned int flags, float det_eps,
    const unsigned char* visible,
    const char* geom_buffer,
    const float* dL_dmeans2D, const float* dL_dconic, const float* dL_dcolors, const float* dL_dopacity,
    float* d_xyz, float* d_scaling, float* d_rotation, float* d_dirs, float* d_features_dc, float* d_features_rest,
    float* d_opacity, float* d_label, float* d_orient_conf, float* d_means2D, float* d_camera,
    unsigned int* nan_flag, void* workspace, int debug, gh_stream_t stream);
int gh_adam_step_capturable(int n_groups, float* const* params, const float* const* grads,
                            float* const* exp_avg, float* const* exp_avg_sq,
                            const unsigned long long* sizes, const float* lrs,
                            double beta1, double beta2, float eps, int* step_state,
                            unsigned int* nan_flag, const unsigned int* skip_flag, int debug, gh_stream_t stream);

/*
 * Capturable strand iteration (DESIGN §19): render_hair_strands -- the frozen head block of n_head Gaussians followed by
 * the S * L segments of a strand model (strand-major) -- under the contract of the capturable block above (tan fov
 * from the device float[2] `tan_fov`, R only on the device, a binning buffer of `capacity` records, the overflow
 * contract of GH_STATUS_BINNING_OVERFLOW; debug != 0 and the stage timer are refused before any launch).  The
 * P = n_head + S * L rows keep the order of the eager path (head rows first), so that with the same inputs radii, keys,
 * the sorted lists and the image are bit-identical to it.  Continue with gh_forward_render_capturable and
 * gh_backward_capturable over all P rows (colors, geom/img/binning buffers of this call).
 *
 * gh_hair_strands_forward_binned_capturable: gh_strand_midpoints into `midpoints` (S*L,3) (the strand rows' means),
 *   the head rows projected with `head_flags` (no strand bit; the head block has no dirs, label or orient_conf) and
 *   `head_det_eps`, the segment rows with `flags` (strand bit set; `scale` = one device float, the strand thickness)
 *   and `det_eps`, then one tile histogram, scan, capacity guard and emit over all P rows.  Outputs as in
 *   gh_project_forward_binned_capturable, with P rows.  n_head >= 0, S, L >= 0, 3 * S * L and n_head + S * L below 2^31,
 *   P > 0; with S * L == 0 only the head block is rendered.  `status` is required, num_rendered (device uint32) may be
 *   NULL.
 * gh_hair_strands_backward_capturable: the parameter backward of the segment rows alone, after gh_backward_capturable:
 *   the strand-mode projection backward reads the accumulation records of rows [n_head, P) in place from
 *   `geom_buffer` (the geometry workspace of the P-row forward; `visible` has P rows), writes dL/d midpoint to d_xyz
 *   (S*L,3, scratch) and the gradients of d_dirs, d_features_dc, d_features_rest, d_orient_conf (may be NULL), then
 *   gh_strand_backward completes d_dirs (S,L,3).  nan_flag (device uint32, may be NULL) as in gh_project_backward and
 *   gh_strand_backward.  No head-row and no camera gradients.  S, L > 0.
 */
int gh_hair_strands_forward_binned_capturable(
    int n_head, int S, int L, int width, int height,
    const float* head_xyz, const float* head_scaling, const float* head_rotation,
    const float* head_features_dc, const float* head_features_rest, const float* head_opacity,
    unsigned int head_flags, float head_det_eps,
    const float* origins, const float* dirs, const float* scale,
    const float* features_dc, const float* features_rest, const float* orient_conf,
    unsigned int flags, float det_eps,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree,
    float* midpoints,
    float* means2D, float* colors, float* opacities, float* conic, unsigned char* visible,
    int* radii, char* geom_buffer, char* img_buffer, char* binning_buffer, long long capacity,
    unsigned int* status, unsigned int* num_rendered, int debug, gh_stream_t stream);
int gh_hair_strands_backward_capturable(
    int n_head, int S, int L, int width, int height,
    const float* midpoints, const float* dirs, const float* scale,
    const float* features_dc, const float* features_rest, const float* orient_conf,
    unsigned int flags, float det_eps,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree,
    const unsigned char* visible, const char* geom_buffer,
    float* d_xyz, float* d_dirs, float* d_features_dc, float* d_features_rest, float* d_orient_conf,
    unsigned int* nan_flag, int debug, gh_stream_t stream);

/*
 * Capturable latent strand iteration (DESIGN §20): render_hair_segments -- the frozen head block of n_head Gaussians
 * followed by N given segment rows -- under the contract of the gh_hair_strands_*_capturable pair above.  The only
 * difference: the segment rows come as their midpoints `xyz` (N,3) and segment vectors `dirs` (N,3), the layout
 * GaussianModelHair.generate_strands leaves in _xyz and _dir (N = num_strands * (strand_length - 1), strand-major),
 * instead of as polylines.  So the forward runs no gh_strand_midpoints (xyz is read in place) and the backward no
 * gh_strand_backward (no cumulative sum to chain through).
 *
 * gh_hair_segments_forward_binned_capturable: the head rows projected with `head_flags` (no strand bit) and
 *   `head_det_eps`, the segment rows with `flags` (strand bit set; `scale` = one device float, the strand thickness)
 *   and `det_eps`, then one tile histogram, scan, capacity guard and emit over all P = n_head + N rows.  Outputs,
 *   status and num_rendered as in gh_hair_strands_forward_binned_capturable.  n_head >= 0, N >= 0, 3 * N and
 *   n_head + N below 2^31, P > 0; xyz and dirs are required even when N == 0.
 * gh_hair_segments_backward_capturable: after gh_backward_capturable, the strand-mode projection backward reads the
 *   accumulation records of rows [n_head, P) in place from `geom_buffer` and writes dL/dxyz to d_xyz (N,3), dL/ddirs to
 *   d_dirs (N,3), and d_features_dc, d_features_rest, d_orient_conf (may be NULL).  nan_flag (device uint32, may be
 *   NULL) as in gh_project_backward.  No head-row and no camera gradients.  N > 0.
 */
int gh_hair_segments_forward_binned_capturable(
    int n_head, int N, int width, int height,
    const float* head_xyz, const float* head_scaling, const float* head_rotation,
    const float* head_features_dc, const float* head_features_rest, const float* head_opacity,
    unsigned int head_flags, float head_det_eps,
    const float* xyz, const float* dirs, const float* scale,
    const float* features_dc, const float* features_rest, const float* orient_conf,
    unsigned int flags, float det_eps,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree,
    float* means2D, float* colors, float* opacities, float* conic, unsigned char* visible,
    int* radii, char* geom_buffer, char* img_buffer, char* binning_buffer, long long capacity,
    unsigned int* status, unsigned int* num_rendered, int debug, gh_stream_t stream);
int gh_hair_segments_backward_capturable(
    int n_head, int N, int width, int height,
    const float* xyz, const float* dirs, const float* scale,
    const float* features_dc, const float* features_rest, const float* orient_conf,
    unsigned int flags, float det_eps,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    const float* tan_fov, float scale_modifier, int sh_degree,
    const unsigned char* visible, const char* geom_buffer,
    float* d_xyz, float* d_dirs, float* d_features_dc, float* d_features_rest, float* d_orient_conf,
    unsigned int* nan_flag, int debug, gh_stream_t stream);

/*
 * Trainable cameras (DESIGN §17): the reference's BARF camera model (src/scene/cameras.py:95-152, use_barf = True) and
 * its camera Adam (src/train_gaussians.py:45-63, 183-196).  A rig of n cameras owns, on the device:
 *   base       float[n][18]  C = the float32 _colmap_transform (16, row-major), FoVx, FoVy (the camera's base state)
 *   residuals  float[n][8]   r = [w (3), u (3), f (2)] = _rotation_res, _translation_res, _fov_res (f = 0 without
 *                            trainable intrinsics)
 *   grad       float[n][8]   dL/dr, accumulated by gh_camera_backward
 *   touched    int[n]        1 for a row gh_camera_backward wrote since the last gh_camera_adam_step
 * with znear = 0.01, zfar = 100:
 *   viewmatrix = (C @ Res)^T, Res[:3] = lie.se3_to_SE3(cat(w, u)), Res[3] = (0, 0, 0, 1)
 *   projmatrix = viewmatrix @ getProjectionMatrix(znear, zfar, FoVx + f0, FoVy + f1)^T
 *   campos     = inverse(viewmatrix)[3, :3],   tan_fov = tan((FoV + f) / 2) per axis (x, y)
 * (arithmetic: gaussianhaircut_b200/csrc/gh_camera_math.h).  Every entry point reads the camera index from the device
 * int32 `index`, so a captured CUDA graph serves every view; an index outside [0, n) ORs GH_STATUS_CAMERA_INDEX into
 * the device uint32 `status` and the kernel touches nothing else.  None of them synchronises with the host.  Each
 * rejects n <= 0, a missing or misaligned (not 4-byte) pointer, debug != 0 and calls while the stage timer is on with
 * GH_E_INVALID_ARG before it launches anything.
 *
 * gh_camera_forward: the four outputs of camera `index` into viewmatrix (16), projmatrix (16), campos (3), tan_fov (2),
 *   row-major like the reference's tensors.
 * gh_camera_backward: d_camera (float[37], the layout of gh_project_backward's d_camera: dL/dviewmatrix, dL/dprojmatrix,
 *   dL/dcampos, dL/dtan_fov) -> dL/dr of row `index`, ADDED to grad[index]; touched[index] = 1.  `intrinsics` == 0:
 *   f is not trained and its two gradients are 0.  nan_flag (device uint32) is OR-ed with 1 when one is NaN.
 * gh_camera_adam_step: torch.optim.Adam (the arithmetic of gh_adam_step_capturable) on exactly the touched rows, each
 *   with its own step count steps[i]: columns 0-2, 3-5 and 6-7 (the last two only with `intrinsics`) use the device
 *   learning rates lrs[0] (rotation), lrs[1] (translation), lrs[2] (fov); exp_avg / exp_avg_sq are float[n][8].  The
 *   touched rows' gradients and marks are then cleared -- torch.optim.Adam after zero_grad(set_to_none=True): a camera
 *   that was not visited does not step.  When *nan_flag or *skip_flag (device uint32, may be NULL: e.g. the binning
 *   status word) is non-zero the update is skipped as a whole (moments and step counts unchanged), the gradients are
 *   still cleared.  *nan_flag is zeroed at the end.
 */
#define GH_STATUS_CAMERA_INDEX 2u
int gh_camera_forward(int n, const float* residuals, const float* base, const int* index,
                      float* viewmatrix, float* projmatrix, float* campos, float* tan_fov,
                      unsigned int* status, int debug, gh_stream_t stream);
int gh_camera_backward(int n, const float* residuals, const float* base, const int* index, int intrinsics,
                       const float* d_camera, float* grad, int* touched, unsigned int* nan_flag,
                       unsigned int* status, int debug, gh_stream_t stream);
int gh_camera_adam_step(int n, int intrinsics, float* residuals, float* grad, int* touched,
                        float* exp_avg, float* exp_avg_sq, int* steps, const float* lrs,
                        double beta1, double beta2, float eps, unsigned int* nan_flag,
                        const unsigned int* skip_flag, int debug, gh_stream_t stream);

/*
 * Strand geometry (src/scene/gaussian_model_strands.py:435-454) for the strand mode of the projection (flag bit 10).
 * S strands of L segments, strand-major rows; device float32, contiguous.
 * gh_strand_midpoints: origins (S,1,3), dirs (S,L,3) segment vectors -> xyz (S*L,3) segment midpoints
 *   0.5 (p_k + p_{k+1}), p_0 = origin, p_{k+1} = origin + sum_{j<=k} d_j (a warp scan per strand; any L >= 1).
 *   `xyz` may be a row block of a larger buffer.
 * gh_strand_backward: d_xyz (S*L,3) = dL/d midpoint, d_dirs (S*L,3) = the direct terms the projection backward wrote;
 *   d_dirs is overwritten IN PLACE with dL/dd_k = direct_k + 0.5 d_xyz_k + sum_{j>k} d_xyz_j.  nan_flag (device uint,
 *   or NULL): OR-ed with 1 when any total is NaN.
 */
int gh_strand_midpoints(int S, int L, const float* origins, const float* dirs, float* xyz, gh_stream_t stream);
int gh_strand_backward(int S, int L, const float* d_xyz, float* d_dirs, unsigned int* nan_flag, gh_stream_t stream);

/*
 * "Next" row (SURVEY.md 8f-3): adaptive density control -- the outcome of the reference's densify_and_prune
 * (src/scene/gaussian_model.py:723-737 = densify_and_clone :708-721 + densify_and_split :682-706 + prune_points
 * :613-630, each re-allocating every parameter and both Adam moments with mask gathers / torch.cat :595-654) in one
 * classification pass and one compaction pass.
 * gh_densify_classify: flags (P,4) int32, 16-byte aligned = [original survives (not split, not pruned), its clone
 *   survives, its two children survive, it is split (before the prune)].  grad_threshold / dense_extent
 *   (= percent_dense * scene extent) / min_opacity as in the reference; ws_limit = 0.1 * extent when the caller passes
 *   a max_screen_size, else 0 (test disabled).  The screen-size test itself never fires in the reference
 *   (max_radii2D is zeroed by densification_postfix before it is read, :674) and is therefore not an input.
 * gh_densify_scatter: src / exp_avg / exp_avg_sq / dst / dst_* are HOST arrays of n_tensors (<= 8) device pointers
 *   (row-major (P, row_floats[k]); exp_avg[k] NULL = tensor without optimizer state).  inclusive_prefix = inclusive
 *   prefix sums of flags over the Gaussians (P,4), n_keep / n_clone / n_split_kept = the totals of columns 0..2.
 *   samples (2 * n_split_all, 3): N(0, scale) draws, first-children block then second-children block
 *   (torch.normal(mean=0, std=get_scaling[mask].repeat(2, 1)), :690-692).  Destination rows follow the reference's
 *   order [surviving originals | surviving clones | first children | second children]; clones and children get zero
 *   moments; child xyz = R(q) sample + xyz, child log-scale = log(scale / 1.6).
 */
int gh_densify_classify(int P, const float* grad_accum, const float* denom, const float* log_scaling,
                        const float* opacity_logit, float grad_threshold, float dense_extent,
                        float min_opacity, float ws_limit, int* flags, gh_stream_t stream);
int gh_densify_scatter(int P, int n_tensors, const float* const* src, const float* const* exp_avg,
                       const float* const* exp_avg_sq, float* const* dst, float* const* dst_exp_avg,
                       float* const* dst_exp_avg_sq, const int* row_floats,
                       int xyz_index, int scaling_index, int rotation_index,
                       const int* flags, const int* inclusive_prefix, int n_keep, int n_clone, int n_split_kept,
                       const float* samples, int n_split_all, gh_stream_t stream);

/*
 * Exact 3-nearest-neighbour mean squared distance of a point cloud (the reference's `simple_knn._C.distCUDA2`,
 * called by GaussianModel.create_from_pcd, src/scene/gaussian_model.py:409, to size the initial Gaussians).
 * points (P,3) float32, 4-byte aligned; P in [0, 2^31).  For every point i with finite coordinates,
 *   out[i] = ((b0 + b1) + b2) / 3,  b0 <= b1 <= b2 the three smallest of s_j = (dx*dx + dy*dy) + dz*dz,
 *   dx = p_j.x - p_i.x, ..., over the finite points j != i (told apart by index: a duplicate is at distance 0), every
 *   operation rounded on its own; slots without a candidate are +inf (P <= 3 gives +inf).  A point with a NaN or
 *   infinite coordinate gets NaN and is nobody's neighbour.  The result depends only on the multiset of distances.
 * Two calls with the same workspace of gh_knn_workspace_size(P) bytes (any alignment; device memory), on one stream:
 *   gh_knn_morton: codes (P) int64, 8-byte aligned = 63-bit Morton codes of the finite points on their bounding box,
 *     INT64_MAX for the others;
 *   the caller sorts the codes: order (P) int64 = the permutation that sorts them (torch.sort(..., stable=True));
 *   gh_knn_mean_dist3: out (P) float32.  `order` must be a permutation of [0, P); an entry outside it is skipped.
 *     Any permutation gives the same result: the order only decides how fast the search prunes.
 * No host synchronisation; P = 0 launches nothing.
 */
int gh_knn_workspace_size(long long P, size_t* bytes);
int gh_knn_morton(long long P, const float* points, long long* codes, void* workspace, size_t bytes, gh_stream_t stream);
int gh_knn_mean_dist3(long long P, const float* points, const long long* order, float* out, void* workspace,
                      size_t bytes, gh_stream_t stream);

/*
 * Hair orientation maps (the reference's `calc_orients`, src/preprocessing/calc_orientation_maps.py:53-97, evaluated on
 * the whole image; DESIGN §15).  Image (H,W,C) uint8, C = 3 (RGB) or 4 (RGBA, alpha ignored), row-major.
 *   gray = 0.2989 r + 0.5870 g + 0.1140 b (float64);
 *   dog (H,W) float64 = G(gray, w_low) - G(gray, w_high), G = the separable Gaussian of scipy.ndimage.gaussian_filter
 *     (axis 0 first, mode 'nearest'), each axis with correlate1d's symmetric order: x[i] w[r], then
 *     + (x[i+jj] + x[i-jj]) w[r+jj] for jj = -r .. -1.  w_* (2r+1) float64 device arrays = the normalised weights
 *     exp(-0.5 / s^2 * x^2) / sum, r = int(4 s + 0.5) (the caller computes them, as scipy does, on the host);
 *   bank (N,K,K) float32 = the real Gabor filters in theta-major order c = j*G + g (j < num_filters, G = N/num_filters),
 *     each zero-padded to the centre of the odd K x K square; thetas (num_filters) float32;
 *   R_c(y,x) = sum_{ky,kx} bank[c][ky][kx] * float32(dog)[y+ky-K/2][x+kx-K/2] (cross-correlation, zero outside the
 *     image) in FP32 FMA; F_j = |R_{j*G+g}|; per group idx_g = argmax_j F_j (first on ties), var_g = the float32
 *     epilogue of gaussianhaircut_b200/csrc/gh_orient_math.h; orients (H,W) int64 = idx of the first group with the
 *     smallest var_g, var (H,W) float32 = that var_g.
 * One workspace of gh_orient_workspace_size(H, W, N, K, num_filters) bytes, 256-byte aligned device memory, serves both
 * calls in order on one stream: gh_orient_dog leaves float32(dog) in it for gh_orient_gabor.  Caps: odd K <=
 * GH_ORIENT_MAX_K, num_filters <= GH_ORIENT_MAX_FILTERS, N <= GH_ORIENT_MAX_N, radii <= GH_ORIENT_MAX_RADIUS; H, W > 0
 * with H*W < 2^31.  Bad arguments are rejected before any launch.  No host synchronisation, no atomics: the maps are
 * bit-reproducible.
 */
#define GH_ORIENT_MAX_K 17
#define GH_ORIENT_MAX_FILTERS 256
#define GH_ORIENT_MAX_N 4096
#define GH_ORIENT_MAX_RADIUS 4096
int gh_orient_workspace_size(int H, int W, int N, int K, int num_filters, size_t* bytes);
int gh_orient_dog(int H, int W, int C, const unsigned char* image, const double* w_low, int r_low,
                  const double* w_high, int r_high, double* dog, void* workspace, size_t bytes, gh_stream_t stream);
int gh_orient_gabor(int H, int W, const float* bank, int N, int K, int num_filters, const float* thetas,
                    long long* orients, float* var, void* workspace, size_t bytes, gh_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* GH_RASTERIZER_H_INCLUDED */
