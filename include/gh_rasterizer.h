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
 *      instance count R (= the reference's num_rendered) to the host and returns it.
 *   3. gh_binning_workspace_size(R, &bytes); allocate.
 *   4. gh_forward_render(...): bucket scatter, per-tile sort, alpha compositing.
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
    int* num_rendered, int* max_tile_len,
    int debug, gh_stream_t stream);

/*
 * Phase 2 of Rasterizer::forward: binning + per-tile sort + front-to-back blend.
 * out_color is (C, H, W) channel-major, fully overwritten (background included).
 */
int gh_forward_render(
    int P, int width, int height,
    const float* background, const float* colors_precomp,
    const int* radii,
    char* geom_buffer, char* binning_buffer, char* img_buffer,
    int num_rendered, int max_tile_len,
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
                 float beta1, float beta2, float eps, int step, int* step_state,
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
 * Continue with gh_binning_workspace_size + gh_forward_render.  Workspaces: gh_forward_workspace_sizes. */
int gh_project_forward_binned(
    int P, int width, int height,
    const float* xyz, const float* scaling, const float* rotation, const float* dirs,
    const float* features_dc, const float* features_rest,
    const float* opacity, const float* label, const float* orient_conf,
    const float* viewmatrix, const float* projmatrix, const float* campos,
    float tan_fovx, float tan_fovy, float scale_modifier, int sh_degree, unsigned int flags, float det_eps,
    float* means2D, float* colors, float* opacities, float* conic, float* cov3D, unsigned char* visible,
    int* radii, char* geom_buffer, char* img_buffer, int* num_rendered, int* max_tile_len,
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

#ifdef __cplusplus
}
#endif
#endif /* GH_RASTERIZER_H_INCLUDED */
