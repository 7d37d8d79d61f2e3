/*
 * psb200 — C-ABI of the H100-native (sm_90a) Gaussian-splatting hot path (libpsb200.so).
 *
 * Plain C, plain pointers and sizes, no torch / C++ types. Every pointer named *device* below is a
 * CUDA device pointer to contiguous float32 / int32 data on the current device; `stream` is a
 * cudaStream_t passed as void* (NULL = the legacy default stream the reference launches on).
 * All functions return >= 0 on success and a negative code on failure; psb_last_error() then returns a
 * human-readable reason (thread-local). CUDA launch errors ARE checked (the reference never checks,
 * SURVEY.md §2.2 quirk 13).
 *
 * Each entry point names the reference interface it replaces (paths relative to the Photo-SLAM tree).
 */
#ifndef PSB200_H_INCLUDED
#define PSB200_H_INCLUDED

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PSB_ERR_ARG   (-1)
#define PSB_ERR_CUDA  (-2)
#define PSB_ERR_SIZE  (-3)

/* Scratch allocator callback: must return a device pointer to at least `bytes` bytes that stays valid
 * until the matching backward call. Replaces the std::function<char*(size_t)> resize callbacks of
 * cuda_rasterizer/rasterizer.h:32-34 (created by src/rasterize_points.cu:28-34). */
typedef char* (*psb_alloc_fn)(size_t bytes, void* user);

int psb_version(void);
const char* psb_last_error(void);

/* Scratch sizes; pure functions of P / num_rendered / W*H like `required<State>(n)`,
 * cuda_rasterizer/rasterizer_impl.h:66-72. */
size_t psb_geometry_bytes(int P);
size_t psb_binning_bytes(int num_rendered);
size_t psb_image_bytes(int num_pixels);

/*
 * Forward rasterization. Replaces CudaRasterizer::Rasterizer::forward
 * (cuda_rasterizer/rasterizer.h:31-52, rasterizer_impl.cu:198-336); same argument meaning and order.
 * Optional inputs are NULL ("None" convention, src/gaussian_rasterizer.cpp:209-219): exactly one of
 * {shs, colors_precomp} and one of {scales+rotations, cov3D_precomp}.
 * viewmatrix / projmatrix: 4x4 column-major in memory (m[4*c + r]), device. out_color: [3,H,W] device.
 * radii: [P] int32 device or NULL. Returns num_rendered (number of (Gaussian, tile) instances).
 * Like the reference it blocks the host once (to size the binning scratch through the callback).
 */
int psb_rasterize_forward(psb_alloc_fn geometry_buffer, void* geometry_user,
                          psb_alloc_fn binning_buffer, void* binning_user,
                          psb_alloc_fn image_buffer, void* image_user,
                          int P, int D, int M,
                          const float* background, int width, int height,
                          const float* means3D, const float* shs, const float* colors_precomp,
                          const float* opacities, const float* scales, float scale_modifier,
                          const float* rotations, const float* cov3D_precomp,
                          const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                          float tan_fovx, float tan_fovy, int prefiltered,
                          float* out_color, int* radii, void* stream);

/*
 * Backward rasterization. Replaces CudaRasterizer::Rasterizer::backward
 * (cuda_rasterizer/rasterizer.h:54-82, rasterizer_impl.cu:340-432). R = value returned by forward;
 * the three scratch pointers are the chunks handed out by the forward callbacks. Gradient outputs are
 * caller-allocated, ZERO-INITIALISED device arrays with the reference's shapes
 * (src/rasterize_points.cu:148-157): dL_dmean2D [P,3] (x,y written), dL_dconic [P,2,2] (x,y,w written),
 * dL_dopacity [P], dL_dcolor [P,3], dL_dmean3D [P,3], dL_dcov3D [P,6], dL_dsh [P,M,3],
 * dL_dscale [P,3], dL_drot [P,4]. Rows of invisible Gaussians are left untouched.
 */
int psb_rasterize_backward(int P, int D, int M, int R,
                           const float* background, int width, int height,
                           const float* means3D, const float* shs, const float* colors_precomp,
                           const float* scales, float scale_modifier, const float* rotations,
                           const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                           const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                           char* geom_buffer, char* binning_buffer, char* image_buffer,
                           const float* dL_dpix,
                           float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                           float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                           void* stream);

/*
 * Depth on the operator path. D(p) = sum_i z_i alpha_i T_i as defined for the trainer below (un-normalised expected depth,
 * z = view-space depth, alpha and T those of the colour, no background term), rendered over the same full-rectangle
 * instance lists as psb_rasterize_forward.
 *
 * psb_rasterize_forward_depth: psb_rasterize_forward plus out_depth [H,W] (device). out_depth == NULL is psb_rasterize_forward.
 * Colour, radii, num_rendered and the scratch contents are bit-identical to psb_rasterize_forward's on the same inputs.
 *
 * psb_rasterize_backward_depth: psb_rasterize_backward plus dL_ddepth [H,W] (device, or NULL = psb_rasterize_backward) and
 * dL_dz [P] (caller-allocated, ZERO-INITIALISED, device), which receives dL/dz of every Gaussian. dL/dz is folded into dL_dmean3D,
 * and dL_dmean2D includes the depth term's screen-space part, so densification statistics taken from it include depth.
 * PSB_ERR_ARG for dL_ddepth without dL_dz, and for everything psb_rasterize_backward rejects.
 */
int psb_rasterize_forward_depth(psb_alloc_fn geometry_buffer, void* geometry_user,
                                psb_alloc_fn binning_buffer, void* binning_user,
                                psb_alloc_fn image_buffer, void* image_user,
                                int P, int D, int M,
                                const float* background, int width, int height,
                                const float* means3D, const float* shs, const float* colors_precomp,
                                const float* opacities, const float* scales, float scale_modifier,
                                const float* rotations, const float* cov3D_precomp,
                                const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                float tan_fovx, float tan_fovy, int prefiltered,
                                float* out_color, int* radii, float* out_depth, void* stream);
int psb_rasterize_backward_depth(int P, int D, int M, int R,
                                 const float* background, int width, int height,
                                 const float* means3D, const float* shs, const float* colors_precomp,
                                 const float* scales, float scale_modifier, const float* rotations,
                                 const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                                 const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                                 char* geom_buffer, char* binning_buffer, char* image_buffer,
                                 const float* dL_dpix,
                                 float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                                 float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                                 const float* dL_ddepth, float* dL_dz, void* stream);

/*
 * Deterministic backward on the operator path: for the same inputs and the same forward scratch, every output is bit-identical from
 * call to call. psb_rasterize_backward[_depth] add each (Gaussian, tile) sum into the gradient arrays with float atomics, so their
 * last bits depend on the order in which tiles finish; here each sum is stored in a slot of its own and one thread per Gaussian adds
 * its slots in a fixed order (the instances' emission order) and writes the result.
 *
 * psb_rasterize_backward_det_bytes: size of the scratch this needs, a pure function of (P, R): 48 B per instance and 4 B per Gaussian,
 * plus alignment (0 for a negative argument). It is separate from the three forward chunks, whose sizes and contents do not change.
 *
 * psb_rasterize_backward_deterministic: the argument list of psb_rasterize_backward_depth plus det_scratch (device, at least
 * psb_rasterize_backward_det_bytes(P, R) bytes, caller-allocated; its contents are irrelevant: the call zeroes what it reads) and
 * det_scratch_bytes, before the stream. dL_ddepth == NULL is colour only; with dL_ddepth, dL_dz is required. Outputs and their
 * meaning are those of psb_rasterize_backward[_depth] (caller-zeroed arrays; rows of invisible Gaussians left untouched).
 * PSB_ERR_ARG for a NULL or too small det_scratch, for dL_ddepth without dL_dz, and for everything psb_rasterize_backward rejects,
 * all checked before any CUDA call. P == 0 does nothing.
 */
size_t psb_rasterize_backward_det_bytes(int P, int R);
int psb_rasterize_backward_deterministic(int P, int D, int M, int R,
                                         const float* background, int width, int height,
                                         const float* means3D, const float* shs, const float* colors_precomp,
                                         const float* scales, float scale_modifier, const float* rotations,
                                         const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                                         const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                                         char* geom_buffer, char* binning_buffer, char* image_buffer,
                                         const float* dL_dpix,
                                         float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                                         float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                                         const float* dL_ddepth, float* dL_dz, void* det_scratch, size_t det_scratch_bytes,
                                         void* stream);

/*
 * Anti-aliasing on the operator path (the 2D Mip filter of Mip-Splatting, upstream diff-gaussian-rasterization's `antialiasing`).
 * With (a0, b, c0) the 2D covariance of a visible Gaussian before the 0.3 px^2 dilation, det0 = a0 c0 - b^2 and det1 the
 * determinant after it, h = sqrt(max(det0 / det1, 2.5e-5)) in [0.005, 1] and the splat blends with opacity o' = o h. A splat that
 * the dilation widens keeps the energy it had before, so small splats do not brighten at low resolution. Conic, radius, tile
 * rectangle, depth key, colour and clamp bits are unchanged, so radii, num_rendered, the sorted keys and values and the ranges are
 * bit-identical with antialiasing on and off; the exported conic_opacity[:, 3] (psb_debug_export) is o'.
 *
 * psb_rasterize_forward_aa: the argument list of psb_rasterize_forward_depth plus `antialiasing` (0 or 1) before the stream.
 * out_depth may be NULL. antialiasing = 0 is psb_rasterize_forward_depth bit for bit.
 *
 * psb_rasterize_backward_aa: the argument list of psb_rasterize_backward_deterministic plus `antialiasing` before the stream, for the
 * scratch of a psb_rasterize_forward_aa with the same flag. det_scratch == NULL selects the atomic backward (det_scratch_bytes is then
 * ignored), dL_ddepth == NULL means colour only. With antialiasing = 1, dL_dopacity receives dL/do (h dL/do'), and dL/dh joins the
 * covariance gradient (dL_dcov3D, dL_dscale, dL_drot, dL_dmean3D). antialiasing = 0 is psb_rasterize_backward_deterministic (or,
 * without det_scratch, psb_rasterize_backward_depth) bit for bit. No opacity argument is needed: o' is in the geometry scratch.
 *
 * Both return PSB_ERR_ARG, before any CUDA call, for an antialiasing value other than 0 or 1 and for everything the calls they extend
 * reject. The scratch sizes (psb_*_bytes, psb_rasterize_backward_det_bytes) do not change.
 */
int psb_rasterize_forward_aa(psb_alloc_fn geometry_buffer, void* geometry_user,
                             psb_alloc_fn binning_buffer, void* binning_user,
                             psb_alloc_fn image_buffer, void* image_user,
                             int P, int D, int M,
                             const float* background, int width, int height,
                             const float* means3D, const float* shs, const float* colors_precomp,
                             const float* opacities, const float* scales, float scale_modifier,
                             const float* rotations, const float* cov3D_precomp,
                             const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                             float tan_fovx, float tan_fovy, int prefiltered,
                             float* out_color, int* radii, float* out_depth, int antialiasing, void* stream);
int psb_rasterize_backward_aa(int P, int D, int M, int R,
                              const float* background, int width, int height,
                              const float* means3D, const float* shs, const float* colors_precomp,
                              const float* scales, float scale_modifier, const float* rotations,
                              const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                              const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                              char* geom_buffer, char* binning_buffer, char* image_buffer,
                              const float* dL_dpix,
                              float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                              float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                              const float* dL_ddepth, float* dL_dz, void* det_scratch, size_t det_scratch_bytes,
                              int antialiasing, void* stream);

/*
 * Opacity, normals and the second depth moment on the operator path: the planes the fused training step renders
 * (psb_trainer_forward, psb_trainer_forward_normal, psb_trainer_forward_moment), formed from the operator's inputs, culls, full-rectangle
 * instance lists and blend order. Per pixel p, over the Gaussians i that blend there with alpha_i and transmittance T_i:
 *   A(p)   = 1 - T_final(p)                the accumulated opacity; no background term (the colour keeps its own)
 *   N_c(p) = sum_i n_ic alpha_i T_i        [3,H,W], no background term
 *   M(p)   = sum_i z_i^2 alpha_i T_i       the second depth moment, with the z and alpha of D; no background term
 * n_i = +-V r_k: r_k is the column of R(q) belonging to the smallest of the three activated scales (ties: the lowest index), q the
 * rotation input as given (neither the operator's covariance nor the reference's computeCov3D normalises it; scale_modifier does not
 * change the arg-min), V the view rotation; the sign makes n_i . t_i <= 0, t_i the view-space mean. With antialiasing = 1 every plane
 * blends with o h, as the colour does. dL/dn reaches `rotations` only: the arg-min and the sign are piecewise constant. N needs scales
 * and rotations; A and M work for every input combination.
 *
 * psb_rasterize_planes_bytes: the plane_scratch that the normal plane needs, a pure function of (P, R): 16 B per Gaussian for n_i,
 * 12 B per Gaussian for dL/dn and, for the deterministic backward, 64 B per instance (pass R = 0 for the forward and the atomic
 * backward), plus alignment. Only calls that render N or take dL/dN read plane_scratch; its contents are irrelevant.
 *
 * psb_rasterize_forward_planes: the argument list of psb_rasterize_forward_aa with out_depth moved into `planes` (NULL record or NULL
 * field = not rendered), plus plane_scratch, plane_scratch_bytes (device, at least psb_rasterize_planes_bytes(P, 0) bytes with
 * out_normal). Without planes it is psb_rasterize_forward_aa bit for bit; with them, colour, radii, num_rendered, the scratch
 * contents and D are bit-identical to it.
 *
 * psb_rasterize_backward_planes: the argument list of psb_rasterize_backward_aa with dL_ddepth moved into `grads` (NULL record or NULL
 * field = no gradient), plus plane_scratch, plane_scratch_bytes (at least psb_rasterize_planes_bytes(P, deterministic ? R : 0) bytes
 * with dL_dnormal) and `deterministic` (0 or 1; 1 needs det_scratch as in psb_rasterize_backward_deterministic and is bit-identical
 * from call to call; 0 ignores det_scratch). dL_dz [P], caller-allocated and zeroed, is required with dL_ddepth or dL_ddepth2: dM/dz =
 * 2 z alpha T joins dL/dz, which is folded into dL_dmean3D. dL/dA and the alpha-part of dL/dM join every splat's dL/dalpha, so they
 * reach dL_dopacity, dL_dmean2D, dL_dconic and through them the covariance inputs. dL/dn is folded into dL_drot. Without gradients it is
 * psb_rasterize_backward_aa bit for bit (with det_scratch only when deterministic = 1).
 *
 * Both return PSB_ERR_ARG, before any CUDA call, for everything the calls they extend reject, an antialiasing or deterministic value
 * other than 0 or 1, N or dL/dN with cov3D_precomp, a missing or too small plane_scratch with N or dL/dN, dL_ddepth or dL_ddepth2
 * without dL_dz, and dL_dnormal without dL_drot. The scratch sizes psb_geometry_bytes, psb_binning_bytes, psb_image_bytes and
 * psb_rasterize_backward_det_bytes do not change.
 */
typedef struct psb_raster_planes {
	float* out_depth;   /* [H,W] D, as psb_rasterize_forward_depth */
	float* out_alpha;   /* [H,W] A */
	float* out_normal;  /* [3,H,W] N */
	float* out_depth2;  /* [H,W] M */
} psb_raster_planes;
typedef struct psb_raster_plane_grads {
	const float* dL_ddepth;   /* [H,W] */
	const float* dL_dalpha;   /* [H,W] */
	const float* dL_dnormal;  /* [3,H,W] */
	const float* dL_ddepth2;  /* [H,W] */
} psb_raster_plane_grads;
size_t psb_rasterize_planes_bytes(int P, int R);
int psb_rasterize_forward_planes(psb_alloc_fn geometry_buffer, void* geometry_user,
                                 psb_alloc_fn binning_buffer, void* binning_user,
                                 psb_alloc_fn image_buffer, void* image_user,
                                 int P, int D, int M,
                                 const float* background, int width, int height,
                                 const float* means3D, const float* shs, const float* colors_precomp,
                                 const float* opacities, const float* scales, float scale_modifier,
                                 const float* rotations, const float* cov3D_precomp,
                                 const float* viewmatrix, const float* projmatrix, const float* cam_pos,
                                 float tan_fovx, float tan_fovy, int prefiltered,
                                 float* out_color, int* radii, const psb_raster_planes* planes,
                                 void* plane_scratch, size_t plane_scratch_bytes, int antialiasing, void* stream);
int psb_rasterize_backward_planes(int P, int D, int M, int R,
                                  const float* background, int width, int height,
                                  const float* means3D, const float* shs, const float* colors_precomp,
                                  const float* scales, float scale_modifier, const float* rotations,
                                  const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                                  const float* campos, float tan_fovx, float tan_fovy, const int* radii,
                                  char* geom_buffer, char* binning_buffer, char* image_buffer,
                                  const float* dL_dpix,
                                  float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                                  float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot,
                                  const psb_raster_plane_grads* grads, float* dL_dz,
                                  void* det_scratch, size_t det_scratch_bytes,
                                  void* plane_scratch, size_t plane_scratch_bytes,
                                  int antialiasing, int deterministic, void* stream);

/* Near-plane visibility (view z > 0.2). Replaces CudaRasterizer::Rasterizer::markVisible
 * (cuda_rasterizer/rasterizer.h:24-29, rasterizer_impl.cu:141-153). present: [P] bytes (bool), device. */
int psb_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                     unsigned char* present, void* stream);

/*
 * Parity/debug export (tests only): expands this library's private scratch into the reference's
 * intermediate arrays so they can be compared element by element with the reference's GeometryState /
 * BinningState / ImageState (cuda_rasterizer/rasterizer_impl.h:30-64). Any output may be NULL.
 *   depths [P] f32, means2D [P,2] f32, conic_opacity [P,4] f32, rgb [P,3] f32, clamped [P,3] u8,
 *   tiles_touched [P] u32, keys_sorted [R] u64 = (tile << 32 | depth bits), values_sorted [R] u32,
 *   ranges [tiles,2] u32, n_contrib [W*H] u32, final_T [W*H] f32.
 * Entries of culled Gaussians (tiles_touched == 0) are written as zero.
 */
int psb_debug_export(int P, int R, int width, int height,
                     char* geom_buffer, char* binning_buffer, char* image_buffer,
                     float* depths, float* means2D, float* conic_opacity, float* rgb, unsigned char* clamped,
                     uint32_t* tiles_touched, uint64_t* keys_sorted, uint32_t* values_sorted,
                     uint32_t* ranges, uint32_t* n_contrib, float* final_T, void* stream);

/* Diagnostics: occupancy of the tile backward kernel on the current device. variant bit 0: depth, bit 1: deterministic, bit 2: opacity
 * gradient (dL/dA). Writes the resident blocks per SM (cudaOccupancyMaxActiveBlocksPerMultiprocessor at the dynamic shared memory the
 * launch uses), that dynamic shared memory in bytes, and the kernel's registers per thread. Any output may be NULL. */
int psb_debug_render_bwd_occupancy(int variant, int* blocks_per_sm, int* dyn_smem_bytes, int* regs_per_thread);

/* ------------------------------------------------------------------------------------------------
 * Trainer-level surface: one fused training iteration on the RAW model tensors.
 *
 * Replaces the body of GaussianMapper::trainForOneIteration (src/gaussian_mapper.cpp:677-772) /
 * GaussianTrainer::trainingOnce (src/gaussian_trainer.cpp:31-135) between "pick a keyframe" and
 * "densify": GaussianRenderer::render (src/gaussian_renderer.cpp:23-149) incl. the activations of
 * src/gaussian_model.cpp:48-71, loss_utils::l1_loss / ssim (include/loss_utils.h:28-124), loss.backward(),
 * max_radii2D / addDensificationStats (gaussian_mapper.cpp:714-719, gaussian_model.cpp:817-831) and
 * gaussians_->optimizer_->step() + zero_grad (torch::optim::Adam over the 6 groups of
 * gaussian_model.cpp:477-503). Tensor layouts are the reference's (include/gaussian_model.h):
 *   index 0 xyz [P,3] | 1 features_dc [P,1,3] | 2 features_rest [P,15,3] | 3 opacity [P,1] (logit) |
 *   4 scaling [P,3] (log) | 5 rotation [P,4] (w,x,y,z, unnormalised);   all device float32, contiguous.
 * ------------------------------------------------------------------------------------------------ */
#define PSB_ERR_RETRY (-4)

typedef struct psb_trainer psb_trainer; /* opaque: scratch arena of the iteration */

typedef struct psb_model {
	float* param[6];          /* parameters, updated in place by psb_trainer_step / psb_adam_update */
	float* exp_avg[6];        /* Adam first moments  (same shapes) */
	float* exp_avg_sq[6];     /* Adam second moments (same shapes) */
	float* max_radii2D;       /* [P]   or NULL */
	float* xyz_gradient_accum;/* [P,1] or NULL */
	float* denom;             /* [P,1] or NULL */
	int* exist_since_iter;    /* [P] int32 or NULL (GaussianModel::exist_since_iter_; only the densify / prune / insert entry points move it) */
	unsigned char* adam_live; /* [P] bytes or NULL: "the moments of this row may be non-zero". Contract: adam_live[i] == 0 implies that all
	                             118 moment floats of row i are exactly zero (a 1 may stand for zero moments too). psb_trainer_step then
	                             reads and updates nothing of a row whose byte is 0 and that no gradient reaches (Adam is an exact no-op on
	                             it), and sets the byte of every row it updates with a non-zero gradient. Anything else that writes moments
	                             must leave the contract intact or be followed by psb_adam_live_rebuild. NULL: the moments themselves are
	                             read to find such rows. psb_relocate clears the bytes of the rows whose moments it zeroes. Every other entry point ignores
	                             the field. */
} psb_model;

typedef struct psb_camera {
	const float* viewmatrix;  /* device, 16 floats, column-major (world_view_transform_ memory) */
	const float* projmatrix;  /* device, 16 floats (full_proj_transform_ memory) */
	const float* campos;      /* device, 3 floats */
	float tan_fovx, tan_fovy;
	int width, height;
} psb_camera;

typedef struct psb_step {
	float lr[6];              /* per-group learning rates, order as psb_model.param */
	float beta1, beta2, eps;  /* reference: 0.9, 0.999, 1e-15 (gaussian_model.cpp:483-485) */
	int step;                 /* 1-based Adam step count of THIS update */
	float lambda_dssim;       /* reference default 0.2 */
	int sh_degree;            /* active SH degree 0..3 */
	int update_densify_stats; /* != 0: fold max_radii2D / xyz_gradient_accum / denom updates in */
} psb_step;

int psb_trainer_create(psb_trainer** out);
int psb_trainer_destroy(psb_trainer* t);

/* Forward only, from raw parameters (GaussianMapper::renderFromPose, gaussian_mapper.cpp:1521-1569).
 * out_color [3,H,W] device; radii [P] int32 device or NULL. M must be 16. Asynchronous on `stream`. */
int psb_trainer_render(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                       const float* background, int sh_degree, float* out_color, int* radii, void* stream);

/* One fused iteration: render -> loss -> backward -> Adam (parameters and moments updated in place).
 * gt_image [3,H,W] device; mask [3,H,W] device or NULL (undistortion mask, gaussian_mapper.cpp:692);
 * out_color / radii optional outputs. Asynchronous: no host synchronisation happens inside. */
int psb_trainer_step(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                     const float* background, const float* gt_image, const float* mask, const psb_step* step,
                     float* out_color, int* radii, void* stream);
/* ------------------------------------------------------------------------------------------------
 * Depth. The rendered depth is the un-normalised expected depth D(p) = sum_i z_i alpha_i T_i (z_i = view-space depth of
 * Gaussian i; alpha, T exactly those of the colour; no background term). Rendering it leaves the colour image, the final
 * transmittance and the radii bit-identical. The depth loss (RGB-D keyframes) adds lambda_depth * depth_l1 to the loss:
 *   valid(p) = gt_depth(p) > 0 and, with a mask, mask[0,p] != 0;  depth_l1 = sum_valid |D - G| / max(N_valid, 1)
 * N_valid is counted on the device (no host synchronisation). The densification statistics include the depth term.
 * ------------------------------------------------------------------------------------------------ */
typedef struct psb_depth {
	const float* gt_depth;  /* [H,W] device, metres, <= 0 = no measurement; NULL = no depth loss */
	float lambda_depth;     /* finite, >= 0; > 0 exactly when gt_depth is given */
	float* out_depth;       /* [H,W] device or NULL */
} psb_depth;
/* psb_trainer_render plus D -> out_depth [H,W] (device; NULL = psb_trainer_render). */
int psb_trainer_render_depth(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                             const float* background, int sh_degree, float* out_color, int* radii, float* out_depth, void* stream);
/* ------------------------------------------------------------------------------------------------
 * Training against the caller's loss: the fused step split at the loss. psb_trainer_forward renders (colour, optional depth and
 * accumulated opacity) and returns the pass number; the caller evaluates any loss on those planes and its gradients w.r.t. them;
 * psb_trainer_backward_pixels runs the tile backward of that pass on the caller's planes, then the per-Gaussian stage of
 * psb_trainer_step (fused Adam) or of psb_trainer_backward (raw-parameter gradients). The built-in step runs the same kernels with
 * its own loss in between.
 * Accumulated opacity: A(p) = 1 - T_final(p) = sum_i alpha_i T_i, the weight of the splats in the pixel (D / A is the normalised
 * depth; 1 - A is the background's share of the colour). dA/dalpha_i = T_final / (1 - alpha_i).
 * ------------------------------------------------------------------------------------------------ */
/* psb_trainer_render_depth plus out_alpha [H,W] (device or NULL) = A. Colour, depth, radii and the pass's scratch are bit-identical to
 * psb_trainer_render_depth's. *pass (host, may be NULL) receives the pass number (the sequence number psb_trainer_overflow_info counts),
 * which psb_trainer_backward_pixels takes. Asynchronous on `stream`. */
int psb_trainer_forward(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                        const float* background, int sh_degree, float* out_color, int* radii, float* out_depth, float* out_alpha,
                        unsigned* pass, void* stream);
/* Per-pixel gradients of the caller's loss w.r.t. the outputs of one forward pass (device, contiguous float32). */
typedef struct psb_pixel_grads {
	const float* dL_dcolor;   /* [3,H,W], required */
	const float* dL_ddepth;   /* [H,W] or NULL: gradient w.r.t. the depth D */
	const float* dL_dalpha;   /* [H,W] or NULL: gradient w.r.t. the accumulated opacity A */
} psb_pixel_grads;
/* Backward of forward pass `pass` on the caller's gradients, then:
 *   grads == NULL: the fused Adam of psb_trainer_step (parameters, moments, model->adam_live and, with step->update_densify_stats,
 *                  the densification statistics are updated; step->step is the Adam step count of this update);
 *   grads != NULL: the raw-parameter gradients of psb_trainer_backward into grads[0..5] (and the statistics); parameters untouched.
 * A depth gradient takes dL/dz into the xyz gradient, as psb_trainer_step_depth does. In deterministic mode the result is bit-identical
 * from run to run for the same planes. step->lambda_dssim is not read.
 * Contract: `pass` is the context's latest forward pass, made by psb_trainer_forward (or psb_trainer_render / _render_depth), and
 * model, camera and background are those of that pass (the model's parameters must not change in between). PSB_ERR_ARG when `pass`
 * is not the latest pass, when the latest pass was a training call (step, backward, _begin: it has had its backward), when
 * psb_trainer_result regrew the arena since, when P, the image size or step->sh_degree differ from that pass, when the deterministic or the anti-aliasing mode was switched in between, for a
 * NULL dL_dcolor and for misaligned gradient segments. A pass that overflowed the binning arena makes this call a no-op on the model
 * and on grads' rows; psb_trainer_result reports PSB_ERR_RETRY for it. psb_trainer_result after this call reports the status and
 * the instance count only: out3 is left untouched. Stage timing: stage "loss" is the stream time between the two calls.
 * Asynchronous on `stream`. */
int psb_trainer_backward_pixels(psb_trainer* t, unsigned pass, int P, int M, const psb_model* model, const psb_camera* camera,
                                const float* background, const psb_pixel_grads* pixel_grads, const psb_step* step,
                                float* const* grads, void* stream);
/* psb_trainer_step / psb_trainer_backward with a depth term; depth == NULL is the plain call. PSB_ERR_ARG for a negative or
 * non-finite lambda_depth, or gt_depth without lambda_depth > 0 (or the reverse). */
int psb_trainer_step_depth(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                           const float* background, const float* gt_image, const float* mask, const psb_step* step,
                           float* out_color, int* radii, const psb_depth* depth, void* stream);
int psb_trainer_backward_depth(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                               const float* background, const float* gt_image, const float* mask, const psb_step* step,
                               float* out_color, int* radii, float* const* grads, const psb_depth* depth, void* stream);
/* ------------------------------------------------------------------------------------------------
 * Exposure compensation per keyframe: the built-in loss compares the target with the rendered image I [3,H,W] (background term
 * included) through the keyframe's 3x4 affine row E (row-major, element (r, j) = param[4 r + j]; identity = eye(3, 4), the layout of
 * graphdeco's exposure.json, where E[:3,:3] right-multiplies HWC pixels):
 *   I'(c,p) = sum_k E[k][c] I(k,p) + E[c][3];   X = mask * I';   L = (1 - lambda) mean|X - G| + lambda (1 - mean SSIM(X, G)) [+ depth]
 * The tile backward receives dL/dI(k,p) = sum_c E[k][c] g(c,p), g = dL/dI'. dL/dE[k][c] = sum_p g(c,p) I(k,p) (k < 3) and
 * dL/dE[c][3] = sum_p g(c,p) are added in a fixed order (no atomics): bit-identical from run to run in every mode. out_color stays the
 * raw render; psb_trainer_result reports the loss of X. Only the given row and its moments are read or written. The row's Adam step
 * uses step->beta1 / beta2 / eps, its own lr and its own step count, which the device advances (no host round trip). A pass that
 * overflows the binning arena leaves the row, its moments and its step count untouched (the repeated call then updates it once).
 * The data-parallel calls take a replicated table instead (psb_exposure_table); on the operator path a caller applies E in torch.
 * ------------------------------------------------------------------------------------------------ */
typedef struct psb_exposure {
	float* param;       /* [3,4] device, the row E_k (gradient mode: read only) */
	float* exp_avg;     /* [3,4] device (step only) */
	float* exp_avg_sq;  /* [3,4] device (step only) */
	int*   step;        /* [1] device int32: this row's Adam step count, advanced on the device (step only) */
	float  lr;          /* finite, >= 0 */
} psb_exposure;
/* psb_trainer_step_depth with an exposure row (NULL: exactly psb_trainer_step_depth). PSB_ERR_ARG, before any CUDA call, for everything
 * psb_trainer_step_depth rejects, a NULL param, exp_avg, exp_avg_sq or step, and a negative or non-finite lr. */
int psb_trainer_step_exposure(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                              const float* background, const float* gt_image, const float* mask, const psb_step* step,
                              float* out_color, int* radii, const psb_depth* depth, const psb_exposure* exposure, void* stream);
/* psb_trainer_backward_depth with an exposure row (NULL: exactly psb_trainer_backward_depth, exposure_grad ignored): the raw-parameter
 * gradients of the compensated loss, and dL/dE -> exposure_grad [12] device (zeros for a pass that overflowed the binning arena).
 * exposure->param is only read; lr must still be valid, the moments and step are ignored. PSB_ERR_ARG, before any CUDA call, for
 * everything psb_trainer_backward_depth rejects, a NULL param, a negative or non-finite lr and a NULL exposure_grad. */
int psb_trainer_backward_exposure(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                                  const float* background, const float* gt_image, const float* mask, const psb_step* step,
                                  float* out_color, int* radii, float* const* grads, const psb_depth* depth,
                                  const psb_exposure* exposure, float* exposure_grad, void* stream);
/* psb_trainer_result with out4 = {loss, l1, ssim, depth_l1} (depth_l1 = 0 when the last step had no depth term). */
int psb_trainer_result_depth(psb_trainer* t, float* out4, int* num_rendered, void* stream);
/* ------------------------------------------------------------------------------------------------
 * Rendered surface normals. Depth pins where a surface is, not which way it faces; the normal plane and its RGB-D term (DN-Splatter,
 * GS-SLAM) supervise the orientation of each Gaussian's flattest axis.
 * Per-Gaussian normal: q = the normalised (w, x, y, z) quaternion and R(q) the rotation the covariance is built from; k = argmin_c
 *   scaling[c] (the raw log-scale; ties go to the lowest index); r = column k of R(q), the world-space shortest axis; V = the upper-left
 *   3x3 of the view matrix, V[r][c] = viewmatrix[4 c + r]; m = V r and t = the view-space mean, formed as the forward forms it;
 *   n_i = m if m . t <= 0, else -m (the normal faces the camera). The 3D filter widens Sigma by f^2 I, which keeps its eigenvectors and so
 *   k; anti-aliasing changes only alpha: n_i is the same in every mode.
 * Normal plane: N_c(p) = sum_i n_ic alpha_i T_i, c = 0, 1, 2, with alpha and T exactly those of the colour (same blend order, culls and
 *   termination) and no background term. N is un-normalised, like D: N / |N| is the pixel's surface normal, in view space. Rendering it
 *   leaves colour, depth, A, radii and the pass's scratch bit-identical.
 * Backward: the three channels join the tile backward like z does for depth (alpha_i T_i dL/dN_c -> dL/dn_ic, and n_i . dL/dN joins
 *   dL/dalpha, so the term reaches opacity, conic, mean2D and the densification statistics); dL/dr = +-V^T dL/dn, with the sign of the
 *   flip, then through dR/dq and the quaternion normalisation into the rotation gradient. k and the flip are piecewise constant: no
 *   gradient to the scales or the mean.
 * Sensor normals (psb_depth_normals): fx = W / (2 tan_fovx), fy = H / (2 tan_fovy), X(u,v) = ((u + 0.5 - W/2) z / fx, (v + 0.5 - H/2) z / fy,
 *   z) with z = depth(u,v) (the seeding rule's back-projection); c = (X(u+1,v) - X(u-1,v)) x (X(u,v+1) - X(u,v-1)); n = c / |c|, flipped
 *   so that n . X(u,v) < 0. (0,0,0) on the image border, where any of the five depths is not finite or <= 0, where some neighbour has
 *   |z_nb - z| > max_rel_jump z (a depth edge) and where |c| = 0. Output: view-space normals [3,H,W], the frame N is rendered in. No
 *   atomics: bit-identical from run to run.
 * Normal term of the built-in loss: valid(p) = G_n(p) != (0,0,0) and, with a mask, mask[0,p] != 0 (the depth loss's convention);
 *   normal_l1 = sum_valid sum_c |N_c - G_c| / max(N_valid, 1); L += lambda_normal normal_l1; dL/dN_c = lambda_normal sign(N_c - G_c) /
 *   max(N_valid, 1) on valid pixels (sign(0) = 0). N_valid is counted on the device (no host synchronisation); in deterministic mode the
 *   sums are reduced in a fixed order. Comparing the un-normalised N with a unit G also pushes A towards 1 where normals are measured:
 *   deliberate, as the depth term does with D. Exposure compensation acts on colour only and does not touch this term.
 * The data-parallel calls take it through psb_dp_step_dist, psb_trainer_backward_begin_dist (+ _slab) and psb_trainer_backward_dist;
 * the rasterizer operator takes no normal term.
 * ------------------------------------------------------------------------------------------------ */
typedef struct psb_normal {
	const float* gt_normal;  /* [3,H,W] device, view-space unit normals, (0,0,0) = no measurement (psb_depth_normals); NULL = no normal term */
	float lambda_normal;     /* finite, >= 0; > 0 exactly when gt_normal is given */
	float* out_normal;       /* [3,H,W] device or NULL: the normal plane N */
} psb_normal;
/* psb_trainer_forward plus out_normal [3,H,W] (device) = N; NULL is exactly psb_trainer_forward. The other outputs are bit-identical to
 * psb_trainer_forward's. A pass with the plane may be followed by psb_trainer_backward_pixels_normal with a dL_dnormal. */
int psb_trainer_forward_normal(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                               const float* background, int sh_degree, float* out_color, int* radii, float* out_depth, float* out_alpha,
                               float* out_normal, unsigned* pass, void* stream);
/* psb_trainer_backward_pixels plus dL_dnormal [3,H,W] (device), the gradient w.r.t. N; NULL is exactly psb_trainer_backward_pixels.
 * PSB_ERR_ARG, before any CUDA call, for everything psb_trainer_backward_pixels rejects and for a dL_dnormal after a pass that rendered
 * no normal plane. */
int psb_trainer_backward_pixels_normal(psb_trainer* t, unsigned pass, int P, int M, const psb_model* model, const psb_camera* camera,
                                       const float* background, const psb_pixel_grads* pixel_grads, const float* dL_dnormal,
                                       const psb_step* step, float* const* grads, void* stream);
/* psb_trainer_step_exposure plus the normal term (normal == NULL: exactly psb_trainer_step_exposure). PSB_ERR_ARG, before any CUDA call,
 * for everything psb_trainer_step_exposure rejects, a negative or non-finite lambda_normal, and gt_normal without lambda_normal > 0 (or
 * the reverse). An out_normal alone renders the plane and trains as without it. A step that overflows the binning arena is a no-op:
 * repeating it applies the term once. */
int psb_trainer_step_normal(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                            const float* background, const float* gt_image, const float* mask, const psb_step* step,
                            float* out_color, int* radii, const psb_depth* depth, const psb_exposure* exposure, const psb_normal* normal,
                            void* stream);
/* psb_trainer_result with out5 = {loss, l1, ssim, depth_l1, normal_l1} (0 for a term the last step did not have). */
int psb_trainer_result_normal(psb_trainer* t, float* out5, int* num_rendered, void* stream);
/* Sensor normals of a depth image [H,W] (metres, <= 0 or not finite = no measurement) seen by `camera` (width, height, tan_fovx and
 * tan_fovy are read) -> out_normal [3,H,W] device. PSB_ERR_ARG, before any CUDA call, for a NULL camera, depth or output, a size that is
 * not positive, a tan_fov that is not finite and positive, and a max_rel_jump that is not finite and positive. Asynchronous. */
int psb_depth_normals(const psb_camera* camera, const float* depth, float max_rel_jump, float* out_normal, void* stream);
/* ------------------------------------------------------------------------------------------------
 * Depth-normal consistency (2DGS, PGSR): the normal of the map's own rendered depth should agree with its rendered normal plane. It
 * needs no sensor and is invariant to the depth scale, so it trains surface orientation on monocular and stereo keyframes too.
 * Inputs: D [H,W], A = 1 - T_final [H,W] and N [3,H,W] of one pass, seen by that pass's camera.
 * Normalised depth: Dbar(p) = D(p) / A(p) (an IEEE division) where A(p) >= alpha_min, else 0 (a hole to psb_depth_normals).
 * Depth normal: n_d = psb_depth_normals applied to Dbar with max_rel_jump (same back-projection, central differences, camera-facing
 *   flip, border, hole and depth-edge rules); n_d = (0,0,0) marks an invalid pixel.
 * Valid pixels: n_d(p) != 0 and, with a mask, mask[0,p] != 0 (the depth and normal terms' convention).
 * Loss: dn = sum_valid (1 - n_d(p) . N(p)) / max(N_valid, 1); L += lambda_dn dn. N stays un-normalised, as in the normal term: since
 *   |N| <= A <= 1 each summand is >= 0, and the term also pushes A towards 1 on valid pixels (deliberate, like the depth and normal terms).
 * Gradients: dL/dN(p) = -lambda_dn n_d(p) / max(N_valid, 1) on valid p. dL/dDbar(q) gathers from the valid p whose stencil reads q,
 *   through the normalisation (I - n n^T) / |c| and the cross product c = a x b, a = X(u+1) - X(u-1), b = X(v+1) - X(v-1),
 *   X(q) = Dbar(q) ray(q); the centre depth, the flip and validity are piecewise constant and carry no gradient. Then
 *   dL/dD = dL/dDbar / A and dL/dA = -dL/dDbar Dbar / A on pixels with A >= alpha_min. Both enter the tile backward with dL/dN, so the
 *   term reaches rotations (through N), positions, opacity and shape, and the densification statistics.
 * N_valid is counted on the device and the scale lambda_dn / max(N_valid, 1) read there; no float atomics on the planes, and in
 * deterministic mode the loss sums are reduced in a fixed order. With a depth and/or normal term in the same step, their gradients are
 * written first and this term adds into the same planes. Anti-aliasing, the 3D filter and exposure compose unchanged (exposure acts on
 * colour only). The data-parallel calls take it through psb_dp_step_dist, psb_trainer_backward_begin_dist (+ _slab) and
 * psb_trainer_backward_dist; the rasterizer operator takes no consistency term.
 * ------------------------------------------------------------------------------------------------ */
typedef struct psb_dn {
	float lambda_dn;          /* finite, > 0 */
	float alpha_min;          /* (0, 1] */
	float max_rel_jump;       /* finite, > 0: the depth-edge rule of psb_depth_normals */
	float* out_depth_normal;  /* [3,H,W] device or NULL: n_d, (0,0,0) where psb_depth_normals of Dbar gives it */
} psb_dn;
/* psb_trainer_step_normal plus the consistency term (dn == NULL: exactly psb_trainer_step_normal). The pass renders D, A and N (in the
 * context's own planes where the caller passes none). PSB_ERR_ARG, before any CUDA call and with the model untouched, for everything
 * psb_trainer_step_normal rejects, a lambda_dn that is not finite and > 0, an alpha_min outside (0, 1] and a max_rel_jump that is not
 * finite and > 0. A step that overflows the binning arena is a no-op: repeating it applies the term once. */
int psb_trainer_step_dn(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                        const float* background, const float* gt_image, const float* mask, const psb_step* step,
                        float* out_color, int* radii, const psb_depth* depth, const psb_exposure* exposure, const psb_normal* normal,
                        const psb_dn* dn, void* stream);
/* psb_trainer_result with out6 = {loss, l1, ssim, depth_l1, normal_l1, dn} (0 for a term the last step did not have). */
int psb_trainer_result_dn(psb_trainer* t, float* out6, int* num_rendered, void* stream);
/* The consistency term on a caller's planes (the two kernels of the built-in step): depth, alpha [H,W] and normal [3,H,W] device, mask
 * [H,W] device or NULL, seen by `camera` (width, height, tan_fovx and tan_fovy are read). dL_ddepth, dL_dalpha [H,W] and dL_dnormal [3,H,W]
 * are ADDED into; out2_host (or NULL) <- {dn, N_valid}. PSB_ERR_ARG, before any CUDA call, for a NULL camera, plane or dn, the camera
 * psb_depth_normals rejects and the dn values psb_trainer_step_dn rejects. Synchronises the stream; the same result every run. */
int psb_dn_loss(const psb_camera* camera, const float* depth, const float* alpha, const float* normal, const float* mask, const psb_dn* dn,
                float* dL_ddepth, float* dL_dalpha, float* dL_dnormal, float* out2_host, void* stream);
/* ------------------------------------------------------------------------------------------------
 * Depth distortion (2DGS): how many Gaussians along a ray share a pixel's weight. Colour alone can explain a view with a haze of
 * half-transparent Gaussians spread in depth; this term pulls each ray's weight onto one depth. It needs no sensor and no target.
 * Second depth moment: M(p) = sum_i z_i^2 alpha_i T_i, with z_i the view-space depth D uses and alpha_i, T_i exactly those of the colour
 *   (same blend order, culls and termination), no background term; un-normalised like D. Rendering it leaves colour, D, A, N, radii and
 *   the pass's scratch bit-identical. With A = 1 - T_final and D = sum_i z_i alpha_i T_i, sqrt(max(M / A - (D / A)^2, 0)) is the pixel's
 *   depth spread: a per-pixel uncertainty of the rendered depth.
 * Distortion of a pixel: dist_p = A M - D^2. With A = sum_i w_i (w_i = alpha_i T_i) this is (1/2) sum_i sum_j w_i w_j (z_i - z_j)^2, 2DGS's
 *   pairwise term in its squared form with a pair counted once. 2DGS measures z in NDC; this term uses view-space z (it reuses D and needs
 *   one accumulator, not two), so its units are depth^2 and its weight scales with the square of the scene's depth.
 *   dist_p is formed in double from the float planes (the products are exact; one rounding). The planes themselves carry float32
 *   rounding, and A M - D^2 cancels: relative to the spread sigma^2 = dist_p / A^2, the error is of order eps_float (Dbar / sigma)^2,
 *   Dbar = D / A: for Gaussians within 1e-3 Dbar of each other a pixel's distortion is known to about 6 %.
 * Loss: valid(p) = mask[0,p] != 0 with a mask, every pixel without one; dist = sum_valid dist_p / max(N_valid, 1); L += lambda_dist dist.
 * Gradients: k = lambda_dist / max(N_valid, 1) (a float32 IEEE division on the device; N_valid counted there); on valid pixels
 *   dL/dA += k M, dL/dD += (-2k) D and dL/dM = k A (0 elsewhere), each one float32 product and one sum, no contraction. The term adds after
 *   the depth, normal and consistency terms have written their gradients; planes no term wrote start at 0. In the tile backward M is one
 *   more channel with per-Gaussian value z_i^2: z_i^2 dL/dM joins dL/dalpha_i, and dL/dz_i gains sum_p alpha_i T_i 2 z_i dL/dM, so per
 *   Gaussian dL/dz_i = 2k sum_p w_i (A z_i - D) (2DGS's gradient). The term reaches positions, opacity and shape, and the densification
 *   statistics. No float atomics on the planes; in deterministic mode the loss sums are reduced in a fixed order. Anti-aliasing, the 3D
 *   filter and exposure compose unchanged (exposure acts on colour only). The data-parallel calls take it through psb_dp_step_dist,
 *   psb_trainer_backward_begin_dist (+ _slab) and psb_trainer_backward_dist; the rasterizer operator takes no distortion term.
 * ------------------------------------------------------------------------------------------------ */
typedef struct psb_dist {
	float lambda_dist;   /* finite, >= 0; 0 with out_depth2: the plane alone */
	float* out_depth2;   /* [H,W] device or NULL: the second depth moment M */
} psb_dist;
/* psb_trainer_forward_normal plus out_depth2 [H,W] (device) = M; NULL is exactly psb_trainer_forward_normal. The other outputs are
 * bit-identical to psb_trainer_forward_normal's; out_depth may be NULL. A pass with the plane may be followed by
 * psb_trainer_backward_pixels_moment with a dL_ddepth2. */
int psb_trainer_forward_moment(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                               const float* background, int sh_degree, float* out_color, int* radii, float* out_depth, float* out_alpha,
                               float* out_normal, float* out_depth2, unsigned* pass, void* stream);
/* psb_trainer_backward_pixels_normal plus dL_ddepth2 [H,W] (device), the gradient w.r.t. M; NULL is exactly
 * psb_trainer_backward_pixels_normal. pixel_grads->dL_ddepth may be NULL alongside it. PSB_ERR_ARG, before any CUDA call, for everything
 * psb_trainer_backward_pixels_normal rejects and for a dL_ddepth2 after a pass that rendered no second depth moment. */
int psb_trainer_backward_pixels_moment(psb_trainer* t, unsigned pass, int P, int M, const psb_model* model, const psb_camera* camera,
                                       const float* background, const psb_pixel_grads* pixel_grads, const float* dL_dnormal,
                                       const float* dL_ddepth2, const psb_step* step, float* const* grads, void* stream);
/* psb_trainer_step_dn plus the distortion term (dist == NULL: exactly psb_trainer_step_dn). With lambda_dist > 0 the pass renders D, A
 * and M (in the context's own planes where the caller passes none), and N too when a normal or consistency term is on. An out_depth2
 * alone (lambda_dist = 0) renders the plane and trains as without it. PSB_ERR_ARG, before any CUDA call and with the model untouched, for
 * everything psb_trainer_step_dn rejects and a lambda_dist that is negative or not finite. A step that overflows the binning arena is a
 * no-op: repeating it applies the term once. */
int psb_trainer_step_dist(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                          const float* background, const float* gt_image, const float* mask, const psb_step* step,
                          float* out_color, int* radii, const psb_depth* depth, const psb_exposure* exposure, const psb_normal* normal,
                          const psb_dn* dn, const psb_dist* dist, void* stream);
/* psb_trainer_result with out7 = {loss, l1, ssim, depth_l1, normal_l1, dn, dist} (0 for a term the last step did not have). After
 * psb_dp_step_dist, psb_trainer_backward_begin_dist and psb_trainer_backward_dist it reports this context's (this rank's) terms. */
int psb_trainer_result_dist(psb_trainer* t, float* out7, int* num_rendered, void* stream);
/* psb_trainer_backward_exposure plus the normal, consistency and distortion terms (all three NULL: exactly psb_trainer_backward_exposure):
 * the raw-parameter gradients of the loss psb_trainer_step_dist would train on, written to grads; the parameters do not move. The
 * rotation gradient takes dL/dn, and the distortion's dL/dz joins the xyz gradient. PSB_ERR_ARG, before any CUDA call, for everything
 * psb_trainer_backward_exposure rejects and the normal, dn and dist records psb_trainer_step_dist rejects. */
int psb_trainer_backward_dist(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                              const float* background, const float* gt_image, const float* mask, const psb_step* step,
                              float* out_color, int* radii, float* const* grads, const psb_depth* depth,
                              const psb_exposure* exposure, float* exposure_grad, const psb_normal* normal, const psb_dn* dn,
                              const psb_dist* dist, void* stream);

/* model->adam_live[i] = 1 if any of the 118 moments of row i is non-zero, else 0: one pass over the moments. Restores the
 * psb_model.adam_live contract after moments were written by anything but psb_trainer_step. Asynchronous on `stream`. */
int psb_adam_live_rebuild(int P, const psb_model* model, void* stream);

/* Data-parallel halves of the same iteration: psb_trainer_backward writes the gradients w.r.t. the RAW
 * parameters into grads[0..5] (shapes of psb_model.param; every row written, zeros for invisible Gaussians)
 * and updates the densification statistics but NOT the parameters; after the all-reduce of `grads`,
 * psb_adam_update applies torch::optim::Adam semantics with g = grads * grad_scale. */
int psb_trainer_backward(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                         const float* background, const float* gt_image, const float* mask, const psb_step* step,
                         float* out_color, int* radii, float* const* grads, void* stream);
int psb_adam_update(int P, int M, const psb_model* model, float* const* grads, const psb_step* step,
                    float grad_scale, void* stream);
/* Pipelined form of psb_trainer_backward: _begin runs render, loss and the tile backward (everything up to the 9
 * screen-space sums per Gaussian); _slab then produces the raw-parameter gradients of Gaussians [first, first+count)
 * (first a multiple of 128). grads[i] must point at the address where row 0 of tensor i WOULD be, i.e.
 * slab_buffer_i - first * floats_per_row_i: the kernel writes row g of tensor i at grads[i] + g * floats_per_row_i,
 * which lets the caller keep each slab's six gradient blocks contiguous and all-reduce slab k while slab k+1 is
 * still being computed. */
int psb_trainer_backward_begin(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                               const float* background, const float* gt_image, const float* mask, const psb_step* step,
                               float* out_color, int* radii, void* stream);
int psb_trainer_backward_slab(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                              const psb_step* step, int first, int count, float* const* grads, void* stream);
/* psb_trainer_backward_begin with a depth term (depth == NULL is the plain call; PSB_ERR_ARG as psb_trainer_step_depth). The
 * context remembers whether the last _begin or _begin_depth carried a depth target, and every _slab that follows takes the
 * depth term into its gradients; a plain _begin clears that again. _slab keeps its signature, and the caller runs every slab
 * of a depth _begin before the next _begin, exactly as without depth. */
int psb_trainer_backward_begin_depth(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                                     const float* background, const float* gt_image, const float* mask, const psb_step* step,
                                     float* out_color, int* radii, const psb_depth* depth, void* stream);
/* psb_trainer_backward_begin_depth plus the normal, consistency and distortion terms (all three NULL: exactly
 * psb_trainer_backward_begin_depth). The context records, before the pass and whether or not the call succeeds, which gradients the
 * pass leaves in its rows (dL/dz with a depth, consistency or distortion term; dL/dn with a normal or consistency term), and every _slab
 * that follows takes them into its gradients; a plain _begin or _begin_depth clears that again. A _slab after a _begin_dist that failed
 * before its pass returns PSB_ERR_ARG. PSB_ERR_ARG, before any CUDA call, for everything _begin_depth rejects and the normal, dn and dist
 * records psb_trainer_step_dist rejects. psb_trainer_result_dist reports this rank's terms. */
int psb_trainer_backward_begin_dist(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                                    const float* background, const float* gt_image, const float* mask, const psb_step* step,
                                    float* out_color, int* radii, const psb_depth* depth, const psb_normal* normal, const psb_dn* dn,
                                    const psb_dist* dist, void* stream);
/* Exposure on the slab and flat paths (the replicated table: see psb_exposure_table below). psb_trainer_backward_begin_table is
 * psb_trainer_backward_begin_dist and psb_trainer_backward_table is psb_trainer_backward_dist without its single-row exposure, each plus
 * the table (NULL: exactly the _dist call without exposure): this rank's view trains through row exposure->id, and its record (valid = 0
 * without a row or for an overflowing pass) goes to exposure->record; the table does not move. After gathering every rank's record,
 * psb_exposure_apply(world, records, table, step, 1/world) updates the table. PSB_ERR_ARG, before any CUDA call, for everything the
 * _dist call rejects, the table values psb_dp_step_table rejects and a NULL record. */
struct psb_exposure_table;
int psb_trainer_backward_begin_table(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                                     const float* background, const float* gt_image, const float* mask, const psb_step* step,
                                     float* out_color, int* radii, const psb_depth* depth, const psb_normal* normal, const psb_dn* dn,
                                     const psb_dist* dist, const struct psb_exposure_table* exposure, void* stream);
int psb_trainer_backward_table(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera,
                               const float* background, const float* gt_image, const float* mask, const psb_step* step,
                               float* out_color, int* radii, float* const* grads, const psb_depth* depth, const psb_normal* normal,
                               const psb_dn* dn, const psb_dist* dist, const struct psb_exposure_table* exposure, void* stream);
/* The table update of the data-parallel exposure rule from `world` records (device, rank-major [world][PSB_EXPOSURE_RECORD], as the
 * gradient modes write them), with step->beta1 / beta2 / eps: one kernel, the one psb_dp_step_table runs. A record whose K or id does
 * not fit the table is skipped. PSB_ERR_ARG, before any CUDA call, for a world outside 1..8, a NULL records, table or step, the table
 * values psb_dp_step_table rejects and a non-finite grad_scale. Asynchronous. */
int psb_exposure_apply(int world, const float* records, const struct psb_exposure_table* table, const psb_step* step, float grad_scale,
                       void* stream);
/* Same update on one flat range of n floats (any slice of a parameter tensor and the matching slices of its moments and
 * gradient) with an explicit learning rate: lets the caller pipeline chunked all-reduces with the optimizer. */
int psb_adam_flat(size_t n, float* param, float* exp_avg, float* exp_avg_sq, const float* grad, float lr,
                  const psb_step* step, float grad_scale, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Keyframe-sharded data parallelism over NVLink peer memory (SURVEY.md 8e): one process per GPU, replicated
 * Gaussians, rank r trains on its own view, K views per optimizer step (mean gradient). Replaces the
 * optimizer step of the reference iteration (src/gaussian_mapper.cpp:769-772) at world > 1 by a fused
 *   reduce-scatter (80-byte gradient records pushed by the per-Gaussian backward straight into the owner
 *   rank's inbox) -> Adam on the owned rows only (moments live on the owner) -> all-gather (the owner's Adam
 *   kernels store the updated rows into every rank's parameter tensors)
 * with no materialised reduced gradient and no collective call. Ownership: chunks of 128 Gaussians, chunk c
 * belongs to rank c % world. The six parameter tensors must live in this context's arena (psb_dp_params), which
 * is mapped into the peers with CUDA IPC: create on every rank -> exchange the psb_dp_ipc_handle blobs with any
 * host-side transport (torch.distributed, MPI, a socket) -> psb_dp_connect. Moments (psb_model.exp_avg*) stay
 * ordinary full-size tensors; only the rows this rank owns are read or written.
 * ------------------------------------------------------------------------------------------------ */
typedef struct psb_dp psb_dp;
int psb_dp_create(psb_dp** out, int rank, int world, int P);   /* world <= 8; every rank must pass the same P */
int psb_dp_handle_bytes(void);                                 /* size of one IPC handle blob (64) */
int psb_dp_ipc_handle(psb_dp* dp, void* out_handle);           /* this rank's blob */
int psb_dp_connect(psb_dp* dp, const void* handles);           /* world blobs, rank-major; no-op for world == 1 */
int psb_dp_params(psb_dp* dp, float** out6);                   /* device addresses of the six parameter tensors in the arena (order of psb_model.param) */
/* One data-parallel iteration: render -> loss -> tile backward -> per-Gaussian backward with records pushed to the
 * owners -> (device-side wait for every rank's records) -> Adam of the owned rows, updated rows stored to every rank.
 * Asynchronous: no host synchronisation, every cross-rank dependency is a device-side wait on an epoch flag. A view
 * whose binning arena overflows contributes a zero gradient to the step (psb_trainer_result still reports
 * PSB_ERR_RETRY and grows the arena): the replicas stay identical and no rank waits forever. Every rank must run with the same
 * psb_trainer_set_antialiasing mode: the records of an anti-aliased view differentiate o' = o h, and the owner adds them as they are. */
int psb_dp_step(psb_trainer* t, psb_dp* dp, int P, int M, const psb_model* model, const psb_camera* camera,
                const float* background, const float* gt_image, const float* mask, const psb_step* step,
                float* out_color, int* radii, void* stream);
/* psb_dp_step with this rank's depth term (depth == NULL is psb_dp_step; PSB_ERR_ARG as psb_trainer_step_depth). dL/dz joins
 * this rank's xyz gradient before its records are built, so the records and the owner-side Adam are those of psb_dp_step: the
 * ranks of one step may mix views with and without a depth target. psb_trainer_result_depth reports this rank's depth_l1; a
 * view that overflows the binning arena contributes a zero gradient, as in psb_dp_step. */
int psb_dp_step_depth(psb_trainer* t, psb_dp* dp, int P, int M, const psb_model* model, const psb_camera* camera,
                      const float* background, const float* gt_image, const float* mask, const psb_step* step,
                      float* out_color, int* radii, const psb_depth* depth, void* stream);
/* psb_dp_step_depth plus this rank's normal, consistency and distortion terms (all three NULL: exactly psb_dp_step_depth; the records as
 * in psb_trainer_step_dist). dL/dn joins this rank's rotation gradient and the distortion's dL/dz its xyz gradient before the records
 * are built, so the record format and the owner-side Adam are those of psb_dp_step: the ranks of one step may mix views with different
 * terms. A row that only the terms reach sends a record. psb_trainer_result_dist reports this rank's terms; a view that overflows the
 * binning arena contributes a zero gradient, as in psb_dp_step. PSB_ERR_ARG, before any CUDA call, for everything psb_dp_step_depth
 * rejects and the normal, dn and dist records psb_trainer_step_dist rejects. */
int psb_dp_step_dist(psb_trainer* t, psb_dp* dp, int P, int M, const psb_model* model, const psb_camera* camera,
                     const float* background, const float* gt_image, const float* mask, const psb_step* step,
                     float* out_color, int* radii, const psb_depth* depth, const psb_normal* normal, const psb_dn* dn,
                     const psb_dist* dist, void* stream);
/* ------------------------------------------------------------------------------------------------
 * Exposure compensation on the data-parallel steps: every rank holds the same exposure table (K rows E_k, the layout of
 * psb_exposure, their Adam moments and int32 step counts) and trains its view either without exposure (id = -1) or through row
 * id with learning rate lr. Rank r's loss is exactly the one psb_trainer_step_exposure builds with row E_id; its Gaussian gradients
 * travel as on the step without exposure. Then, for every id k that at least one rank with a valid record trained:
 *   g_k = grad_scale * sum, in rank order, of dL_r/dE_k over those ranks (grad_scale = 1/world: a dropped view still counts in it);
 *   row k takes one Adam step with step count step[k] + 1, step->beta1 / beta2 / eps and the lr of the lowest such rank; step[k]
 *   advances by one, however many ranks trained k.
 * Rows no valid record names keep their row, moments and step count bit for bit; a view that overflows its binning arena sends an
 * invalid record (its row is untouched unless another rank trained it). Every rank applies the same records in the same order with
 * the same kernel, so after the step every rank's table is bit-identical, in every mode. The table is never grown here: every rank
 * must hold the same K (a record whose K differs from the local K, or whose id is outside [0, K), is skipped on the device and, on
 * the NVLink step, sets psb_dp_status to 2).
 * Exposure record (PSB_EXPOSURE_RECORD floats, device): id | lr | K | valid | the 12 sums dL/dE in the layout of E. On the NVLink step
 *   it rides in each rank's meta row, beside the camera centre, with no extra flag or collective. The slab and flat paths write it to
 *   table->record; the caller gathers the world records (rank-major, world * 16 floats: one all-gather) and calls psb_exposure_apply.
 *   For the same per-rank gradients the three paths give bit-identical tables.
 * ------------------------------------------------------------------------------------------------ */
#define PSB_EXPOSURE_RECORD 16
typedef struct psb_exposure_table {
	float* param;       /* [K,3,4] device: row k = E_k */
	float* exp_avg;     /* [K,3,4] device */
	float* exp_avg_sq;  /* [K,3,4] device */
	int*   step;        /* [K] device int32 step counts */
	int    K;           /* >= 0, the same on every rank */
	int    id;          /* the row this rank trains this step, or -1 for none */
	float  lr;          /* this rank's learning rate: finite, >= 0 */
	float* record;      /* [PSB_EXPOSURE_RECORD] device: the gradient modes' output (slab and flat paths); unused by psb_dp_step_table */
} psb_exposure_table;
/* psb_dp_step_dist plus this rank's exposure (exposure == NULL: exactly psb_dp_step_dist, and the table is not read). The record of this
 * rank's view is published with its meta row; after the device-side wait for every rank's records, each rank updates its own table
 * (one kernel, before the owner-side Adam). P = 0 exchanges nothing and leaves the table untouched. PSB_ERR_ARG, before any CUDA call,
 * for everything psb_dp_step_dist rejects, an id outside [-1, K), K < 0, a NULL table array with K > 0, and a negative or non-finite lr. */
int psb_dp_step_table(psb_trainer* t, psb_dp* dp, int P, int M, const psb_model* model, const psb_camera* camera,
                      const float* background, const float* gt_image, const float* mask, const psb_step* step,
                      float* out_color, int* radii, const psb_depth* depth, const psb_normal* normal, const psb_dn* dn,
                      const psb_dist* dist, const psb_exposure_table* exposure, void* stream);
/* Enqueues a device-side wait until every rank's rows of the last psb_dp_step have landed in this rank's tensors. */
int psb_dp_sync(psb_dp* dp, void* stream);
/* 0 = healthy, 1 = a cross-rank wait timed out (PSB_DP_TIMEOUT_MS, default 20 s), 2 = an exposure record was refused (a K or id that
 * does not fit this rank's table). Synchronises the stream. */
int psb_dp_status(psb_dp* dp, void* stream);
int psb_dp_destroy(psb_dp* dp);

/* Returns the results of the last step / backward / render: out3 = {loss, l1, ssim} (host, may be NULL),
 * *num_rendered (may be NULL). Blocks only until those scalars have reached pinned host memory (an event recorded
 * right behind the loss kernel), NOT until the step has finished: the caller can read the loss of iteration i and
 * enqueue iteration i+1 while the backward half of i is still running. Use a stream/device synchronize to wait for
 * the step itself.
 * Returns PSB_ERR_RETRY when the binning arena was too small for a view SINCE THE LAST CALL of this function (the
 * record is sticky on the device: a queued step that overflowed is reported even if later steps fitted): that step
 * was a no-op on the model, the arena has been grown, call the step again. psb_trainer_overflow_info tells which
 * call it was: sequence numbers count the forward passes (render / step / backward) of this context from 1;
 * *first_seq = the first overflowing one, *count = how many overflowed, *current_seq = the latest pass enqueued. */
int psb_trainer_result(psb_trainer* t, float* out3, int* num_rendered, void* stream);
int psb_trainer_overflow_info(psb_trainer* t, unsigned* first_seq, unsigned* count, unsigned* current_seq);

/* Parity/debug export (tests only) of the last step / render of this context: per pixel the final transmittance
 * (final_T [H*W] f32, device, may be NULL) and the Gaussian index of the last blended splat (last_gauss [H*W] i32,
 * device, -1 = none, may be NULL) — the trainer-path counterpart of psb_debug_export's n_contrib / final_T, comparable
 * with the reference's point_list[ranges.x + n_contrib - 1] (cuda_rasterizer/forward.cu:352-365) even though the
 * tight instance lists number their entries differently. *num_rendered (host, may be NULL) = instance count. */
int psb_trainer_debug_state(psb_trainer* t, int width, int height, int* last_gauss, float* final_T, int* num_rendered, void* stream);

/* Optional per-stage timing with CUDA events recorded on the step's stream (bench.py uses it for the roofline numbers; off by
 * default). psb_trainer_stage_times fills ms[0..n) (n >= 7) and returns how many stages it filled:
 *   psb_trainer_step : 8 = preprocess, depth sort, binning (emit + tile sort + ranges), render forward, loss fwd+bwd, render
 *                      backward, per-Gaussian backward kernel, f_rest Adam kernel;
 *   psb_dp_step      : 10 = the first six, then push backward, wait for every rank's records, owner-side Adam, and ms[9] = the
 *                      wait at the start of the step for the previous step's rows. */
int psb_trainer_set_profiling(psb_trainer* t, int enable);
int psb_trainer_stage_times(psb_trainer* t, float* ms, int n);

/* Deterministic mode of a context (off by default; PSB_ERR_ARG for a NULL context). While it is on, every output of these calls
 * is bit-identical from run to run for the same inputs, the same build and the same GPU model: psb_trainer_step(_depth),
 * psb_trainer_backward(_depth), psb_trainer_backward_begin(_depth) + psb_trainer_backward_slab, psb_dp_step(_depth) at any
 * world size, and the scalars of psb_trainer_result(_depth). The tile backward then stores each (Gaussian, tile) sum in a slot
 * of its own and a gather adds every Gaussian's slots in a fixed order, instead of adding them into the Gaussian's row with
 * float atomics in whatever order the tiles finish; the loss sums are reduced in a fixed order too. It costs a slot buffer of
 * 48 B per instance of the binning capacity (grown with it) and the time of the gather, counted in the "render backward" stage.
 * The operator path has its own entry point, psb_rasterize_backward_deterministic. Not covered: the NCCL all-reduce that a caller runs between
 * psb_trainer_backward* and psb_adam_update: each rank's gradients are deterministic, the all-reduce's order is NCCL's. */
int psb_trainer_set_deterministic(psb_trainer* t, int enable);

/* Anti-aliasing mode of a context (off by default; PSB_ERR_ARG for a NULL context): while it is on, every pass of the context blends
 * each splat with o' = o h, the 2D Mip filter defined for psb_rasterize_forward_aa, and every backward behind such a pass
 * differentiates it (dL/do = h dL/do', dL/dh into the covariance gradient). It covers psb_trainer_render(_depth),
 * psb_trainer_forward, psb_trainer_step(_depth), psb_trainer_backward(_depth), psb_trainer_backward_begin(_depth) +
 * psb_trainer_backward_slab (the slabs follow the mode of their _begin), psb_trainer_backward_pixels and psb_dp_step(_depth), with no
 * new signatures, and combines with the deterministic mode. The mode is read when a pass starts; psb_trainer_backward_pixels refuses
 * a pass whose mode was switched after it. Every rank of a psb_dp_step must set the same mode (the owner-side Adam sums the ranks'
 * records as they are). With o' < o the tight instance lists can only get shorter. */
int psb_trainer_set_antialiasing(psb_trainer* t, int enable);

/* Stand-alone fused loss (tests / evaluation): L = (1-lambda) L1 + lambda (1 - SSIM), reference
 * include/loss_utils.h:28-124. image/gt/mask/dL_dimage device [3,H,W] (mask, dL_dimage may be NULL);
 * out3_host = {loss, l1, ssim}. Synchronises the stream. */
int psb_loss(int height, int width, const float* image, const float* gt_image, const float* mask,
             float lambda_dssim, float* dL_dimage, float* out3_host, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused densification. Replaces GaussianModel::densifyAndPrune and everything under it (src/gaussian_model.cpp:795-815,
 * densifyAndClone :763-793, densifyAndSplit :716-761, prunePoints :588-642, densificationPostfix :644-714): the reference
 * re-materialises all 59 parameters + 118 Adam moments per Gaussian four times (cat, cat, mask-index, mask-index) with a
 * blocking .item(); here every surviving row is read once and every output row written once.
 *   plan : evaluates the clone / split / prune predicates on the P source rows, scans them, returns counts_host[5] =
 *          {P_new, surviving originals, clones, surviving split children PER COPY, split-selected rows}. This is the one host
 *          round trip (the caller sizes the output tensors from P_new).
 *   apply: writes the P_new output rows of all six parameter tensors and their moments into `dst`, in the reference's row
 *          order [surviving originals | clones | split children copy 0 | copy 1]; new rows get zero moments; the three
 *          statistics arrays of `dst` are zeroed (reference :709-711). Split children: xyz = R(q)(z * exp(s)) + xyz,
 *          scaling = log(exp(s)/1.6); z = normal_samples [2 * n_split, 3] (row c * n_split + rank of the parent among the
 *          split-selected rows, the reference's repeat({N,1}) order) or, when NULL, Philox4x32-10 + Box-Muller keyed by
 *          (cfg.seed, cfg.offset, sample row): counter-based, identical on every data-parallel replica.
 * workspace: psb_densify_workspace_bytes(P) device bytes, the same buffer for plan and apply.
 * ------------------------------------------------------------------------------------------------ */
typedef struct psb_densify_cfg {
	float max_grad;          /* densify_grad_threshold */
	float min_opacity;       /* prune below (reference call sites: 0.005) */
	float extent;            /* scene extent (cameras_extent_) */
	float percent_dense;     /* GaussianModel::percentDense() */
	int max_screen_size;     /* != 0 enables the world-size prune (max exp(scaling) > 0.1 extent), like the reference */
	unsigned long long seed, offset;
} psb_densify_cfg;
size_t psb_densify_workspace_bytes(int P);
int psb_densify_plan(int P, const psb_model* src, const psb_densify_cfg* cfg, void* workspace, int* counts_host, void* stream);
int psb_densify_apply(int P, const psb_model* src, const psb_model* dst, int P_new, const psb_densify_cfg* cfg, const void* workspace,
                      const float* normal_samples, void* stream);
/* GaussianModel::prunePoints (src/gaussian_model.cpp:588-642) through the same machinery: plan from a byte mask (!= 0 = remove),
 * counts_host as above (only [0] and [1] non-zero), then psb_densify_apply with the same workspace compacts parameters, moments
 * and exist_since_iter; NOTE: like every densify apply it zeroes dst's statistics — pass keep_stats != 0 to compact them instead
 * (prunePoints keeps them, :637-641). */
int psb_prune_plan(int P, const unsigned char* mask, void* workspace, int* counts_host, void* stream);
int psb_prune_apply(int P, const psb_model* src, const psb_model* dst, int P_new, const void* workspace, int keep_stats, void* stream);
/* GaussianModel::increasePcd (src/gaussian_model.cpp:193-377, both overloads) minus the k-NN call: dst (P + n rows) = src rows
 * followed by n new Gaussians: xyz = points, features_dc = RGB2SH(colors) (include/sh_utils.h:138-141), features_rest = 0,
 * opacity = inverse_sigmoid(0.1), scaling = log(sqrt(max(dist2, 1e-7))) on all three axes (dist2 = psb_dist_cuda2 of the NEW
 * points), rotation = (1,0,0,0), zero moments, exist_since_iter = iteration; statistics of all rows reset to zero
 * (densificationPostfix :709-711). points/colors [n,3], dist2 [n]: device. */
int psb_insert_points(int P, const psb_model* src, const psb_model* dst, int n, const float* points, const float* colors,
                      const float* dist2, int iteration, void* stream);
/* GaussianModel::resetOpacity (src/gaussian_model.cpp:556-565, incl. its no-op clamp) + zeroed opacity moments, in place. */
int psb_reset_opacity(int P, float* opacity, float* exp_avg, float* exp_avg_sq, void* stream);
/* Every entry point above, from psb_densify_plan on, checks all of its arguments before its first CUDA call: a call that returns
 * PSB_ERR_ARG has enqueued nothing and written no device memory. */

/* ------------------------------------------------------------------------------------------------
 * Depth-guided seeding: new Gaussians on the pixels of an RGB-D keyframe that the map does not explain (the dense rule of SplaTAM,
 * Gaussian-SLAM and MonoGS: where the map's silhouette is weak, or where the sensor sees a surface in front of the map's). The reference
 * only adds rows at ORB keypoints, so a textureless wall, floor or ceiling never gets any.
 * Inputs: a camera (any pyramid level, W x H), A and D [H,W] = the accumulated opacity and the depth sum_i z_i alpha_i T_i the map renders
 * from it (psb_trainer_forward), G [H,W] = the keyframe's depth in metres (<= 0: no measurement), its image [3,H,W] and an optional mask
 * [3,H,W] of which only mask[0] is read (the depth loss's convention: mask[0,p] == 0 makes p unusable).
 *   grid      only pixels (u, v) with u % stride == 0 and v % stride == 0 are considered;
 *   valid     G finite, min_depth < G < max_depth, and not masked out;
 *   hole      A < alpha_min;
 *   in front  A >= alpha_min and __fmul_rn(G, A) < __fmul_rn(k, D), k = 1 - depth_rel formed in float32 on the host, each product rounded
 *             on its own (no FMA): the sensor sees a surface nearer than the map's normalised depth D / A by more than depth_rel
 *             (depth_rel = 1 turns the test off);
 *   selected  valid and (hole or in front).
 * Order and cap: the selected pixels are ranked in raster order (v W + u); with c selected and n <= c kept, the pixel of rank k is kept
 * iff floor((k + 1) n / c) > floor(k n / c) (64-bit integers): exactly n pixels, spread evenly over the image; n = c keeps all.
 * The row of a kept pixel (u, v), z = G(u, v): fx = W / (2 tan_fovx), fy = H / (2 tan_fovy);
 *   camera point (x, y, z) = ((u + 0.5 - W / 2) z / fx, (v + 0.5 - H / 2) z / fy, z): the exact inverse of the forward's projection
 *   (ndc_to_pix's half pixel included), so the centre projects onto the centre of pixel (u, v) at depth z;
 *   world point xyz = R^T (p - t), R[r][c] = viewmatrix[4 c + r], t[r] = viewmatrix[12 + r] (a rigid view matrix);
 *   colour = image(u, v); dist2 = (stride z / ((fx + fy) / 2))^2, i.e. an isotropic scale of one grid cell's footprint at depth z;
 *   everything else is psb_insert_points: features_dc = RGB2SH(colour), features_rest = 0, opacity = logit(0.1), rotation = (1,0,0,0),
 *   zero moments, exist_since_iter = iteration, the statistics of all rows zeroed. dst = the P rows of src (bit for bit) followed by the
 *   n new rows in the order of their rank.
 * No float atomics: the result is bit-identical from run to run and independent of the launch configuration.
 * psb_seed_plan selects and counts: counts_host[3] = {selected, holes, in front}; its read-back of the counts is the one host round trip.
 * psb_seed_apply writes dst (P + n rows) from src and the plan in `workspace`; asynchronous. The library remembers on the host, for the
 * last 16 workspaces planned, the camera size, the stride and the selected count of their plan; apply refuses a workspace without one.
 * workspace: psb_seed_workspace_bytes(W, H, stride) device bytes (0 for a bad size or stride), the same buffer for plan and apply.
 * Both return PSB_ERR_ARG, before any CUDA call, for a config outside the ranges below (NaN included), a missing camera, plane,
 * workspace or count array, and (apply) a view matrix missing, a tan_fov not finite and positive, n < 0, n > max_new, n above the plan's
 * selected count, and everything psb_insert_points rejects.
 * ------------------------------------------------------------------------------------------------ */
typedef struct psb_seed_cfg {
	float alpha_min;    /* (0, 1]: hole below this accumulated opacity */
	float depth_rel;    /* [0, 1]: in front when G < (1 - depth_rel) D / A */
	float min_depth;    /* >= 0 */
	float max_depth;    /* > min_depth */
	int stride;         /* >= 1 */
	int max_new;        /* >= 0: apply adds at most this many rows */
} psb_seed_cfg;
size_t psb_seed_workspace_bytes(int width, int height, int stride);
int psb_seed_plan(const psb_camera* camera, const float* alpha, const float* depth, const float* gt_depth, const float* mask,
                  const psb_seed_cfg* cfg, void* workspace, int* counts_host, void* stream);
int psb_seed_apply(int P, const psb_model* src, const psb_model* dst, int n, const psb_camera* camera, const float* gt_image,
                   const float* gt_depth, const psb_seed_cfg* cfg, const void* workspace, int iteration, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Bounded-budget densification: relocation of dead Gaussians and growth to a cap (3DGS-MCMC, Kheradmand et al., NeurIPS 2024; the
 * semantics of gsplat's MCMCStrategy relocate / sample_add). The reference has no counterpart. With o = sigmoid(opacity) and
 * s = exp(scaling), a row is DEAD when o <= min_opacity and ALIVE otherwise.
 *   Sampling     n draws with replacement from a candidate set with probability proportional to o: inclusive prefix sum of o over the
 *                candidates in row order, in double and in a fixed order; draw j takes u_j in [0, 1) and picks the first candidate
 *                whose cumulative sum exceeds (double)u_j * total (binary search). u_j = uniforms[j] when given, else the first word
 *                w of Philox4x32-10(counter = (j, sub, offset low, offset high), key = (seed low, seed high)) as
 *                min(((float)w + 0.5f) * 2^-32, 1 - 2^-24), sub = 1 in psb_relocate and 2 in psb_grow (the normals of the densify split
 *                and of the position noise use 0). Counter-based: every data-parallel replica draws the same rows.
 *   Multiplicity N_i = min(1 + number of draws that picked row i, 51).
 *   Correction   of a picked row (the paper's Eq. 9): o' = 1 - (1 - o)^(1/N), D = sum_{a=1..N} sum_{k=0..a-1} C(a-1,k) (-1)^k
 *                o'^(k+1) / sqrt(k+1), s' = s o / D on all three axes, o' clamped to [min_opacity, 1 - 1e-7]; stored as logit(o'),
 *                log(s') (a logit at the lower clamp is raised by a few ulps until sigmoid(logit) > min_opacity: a corrected row is
 *                alive). N copies of (o', s') have the alpha of the original at its centre. All 118 moments of a picked row are zeroed.
 * psb_relocate (in place, P unchanged): candidates = the alive rows, n = the number of dead rows. Dead row number j (in row order)
 *   becomes a copy of the corrected source of draw j (all 59 parameters) with zero moments, zero max_radii2D / xyz_gradient_accum /
 *   denom (those given) and exist_since_iter = cfg.iteration (if given). (gsplat leaves the overwritten rows' stale moments in place;
 *   here they are zeroed, which the adam_live contract wants anyway.) model->adam_live, when given, is cleared for the picked and the
 *   overwritten rows, so the contract holds afterwards. No dead row or no alive row: nothing is written. counts_host (host, may be
 *   NULL) receives {rows overwritten, dead rows}; only then does the call synchronise the stream — with NULL it is asynchronous.
 * psb_grow (out of place): dst = the P rows of src followed by n = P_new - P rows (0 <= n <= P; the caller picks
 *   P_new = min(cap, floor(factor P))). n draws over ALL rows; picked rows are corrected in dst; new row P + j is a copy of the
 *   corrected source of draw j with zero moments, zero statistics and exist_since_iter = cfg.iteration. The old rows keep their
 *   statistics, exist_since_iter and (unless picked) moments. n == 0 copies src. dst->adam_live is ignored. Asynchronous.
 * workspace: psb_relocate_workspace_bytes(P) device bytes, 8-byte aligned. uniforms: device [n] floats in [0, 1), or NULL.
 * PSB_ERR_ARG, before any CUDA call, for P < 0, P_new outside [P, 2 P], min_opacity outside [0, 1), and a missing model tensor or
 * workspace.
 * ------------------------------------------------------------------------------------------------ */
typedef struct psb_relocate_cfg {
	float min_opacity;       /* dead at or below (3DGS-MCMC: 0.005) */
	int iteration;           /* exist_since_iter of the rows written */
	unsigned long long seed, offset;
} psb_relocate_cfg;
size_t psb_relocate_workspace_bytes(int P);
int psb_relocate(int P, const psb_model* model, const psb_relocate_cfg* cfg, void* workspace, const float* uniforms, int* counts_host,
                 void* stream);
int psb_grow(int P, const psb_model* src, const psb_model* dst, int P_new, const psb_relocate_cfg* cfg, void* workspace,
             const float* uniforms, void* stream);

/* Position noise of 3DGS-MCMC behind an optimizer step (gsplat inject_noise_to_position), on the rows of the context's latest pass:
 *   xyz += Sigma xi * (lr_xyz * noise_lr) * g(o),  Sigma = R(q) diag(s^2) R(q)^T (q the normalised quaternion),
 *   g(o) = 1 / (1 + exp(-100 ((1 - o) - 0.995))):  ~1 for dead rows, < 1e-4 above o = 0.1, so only nearly dead Gaussians move.
 * xi ~ N(0, I_3): Box-Muller on the four words w0..w3 of Philox4x32-10(counter = (row, 0, step low, step high), key = seed) with
 * u_k = ((float)w_k + 0.5f) 2^-32: xi = (r0 cos(2 pi u1), r0 sin(2 pi u1), r1 cos(2 pi u3)), r0 = sqrt(-2 log min(u0, 1 - 2^-24)),
 * r1 likewise from u2 (the draw of the densify split). Counter-based and free of atomics: bit-identical from run to run.
 * It does nothing when the latest pass overflowed the binning arena (like every kernel of that step), so the repeated step adds the
 * noise exactly once. visible_only != 0 restricts it to the rows that pass saw (radius > 0): a region no recent keyframe sees gets no
 * gradient that could pull a row back, and noise there would be a random walk of the unobserved map; 0 is gsplat's behaviour.
 * PSB_ERR_ARG when the context has run no pass of P rows, for a missing tensor, and for a negative or non-finite lr_xyz / noise_lr.
 * Asynchronous on `stream`. */
int psb_trainer_inject_noise(psb_trainer* t, int P, const psb_model* model, float lr_xyz, float noise_lr, unsigned long long seed,
                             unsigned long long step, int visible_only, void* stream);

/* Opacity and scale regularisers of 3DGS-MCMC on the per-Gaussian stage: L += lambda_opacity mean sigmoid(opacity) + lambda_scale mean
 * exp(scaling) (means over the P rows; the scale term sums the three axes of a row, so gsplat's mean over all 3 P values is
 * lambda_scale / 3 here; the paper uses 0.01 for both). In raw-parameter terms
 * g_opacity += (lambda_opacity / P) o (1 - o) and g_scaling[c] += (lambda_scale / P) s_c, added where the kernel forms the raw
 * gradients, before Adam or the gradient store. They apply to THE ROWS THE PASS UPDATES (rows whose screen-space sums are non-zero),
 * not to all P rows as in gsplat: the fused step touches no other row, and decaying whatever this keyframe does not see would be wrong
 * for a SLAM map anyway (Adam turns a constant-sign gradient into a full step). Read when a pass starts, like anti-aliasing; both 0
 * (the default) runs exactly the kernels of a context that never called this. Covers psb_trainer_step*, psb_trainer_backward*
 * (the _begin / _slab pair included) and psb_trainer_backward_pixels; not psb_dp_step*, which ignore it. The loss scalars of
 * psb_trainer_result stay the image terms. PSB_ERR_ARG for a NULL context and a negative or non-finite lambda. */
int psb_trainer_set_regularizers(psb_trainer* t, float lambda_opacity, float lambda_scale);

/* ------------------------------------------------------------------------------------------------
 * 3D smoothing filter (Mip-Splatting, Yu et al., CVPR 2024: compute_3D_filter, get_scaling_with_3D_filter,
 * get_opacity_with_3D_filter). It bounds every Gaussian from below by the finest sampling interval at which any keyframe saw it, so a
 * Gaussian cannot shrink into a high-frequency artefact that shows when the map is viewed closer or at a higher resolution than it was
 * trained at. (The 2D filter of psb_trainer_set_antialiasing handles the opposite case, zooming out.)
 * Filter. Inputs: the rows' xyz [P,3] and K cameras, each with its view matrix (the layout of psb_camera.viewmatrix),
 *   focal_x = W / (2 tan_fovx), focal_y = H / (2 tan_fovy), W and H: the full-resolution keyframes. For row i and camera k,
 *   (x, y, z) = the view matrix applied to xyz_i exactly as the forward does, so the z test is the forward's near cull bit for bit.
 *   Camera k SEES row i when z > 0.2, u = x / z focal_x + W / 2 in [-0.15 W, 1.15 W] and v = y / z focal_y + H / 2 in [-0.15 H, 1.15 H].
 *   d_i = min z over the cameras that see row i; F = max focal_x over all K cameras; a row no camera sees takes d_i = max d over the rows
 *   that are seen; filter_i = d_i / F * sqrt(0.2). No row seen (K = 0 included): every filter_i = 0. Only minima and maxima are involved:
 *   the result is bit-identical from run to run.
 * Application. s = exp(scaling), o = sigmoid(opacity), f = filter_i:
 *   s'_c = sqrt(s_c^2 + f^2),  c = sqrt(prod_c s_c^2 / prod_c s'_c^2) (formed as the product of the three ratios),  o' = o c.
 *   R diag(s')^2 R^T = Sigma + f^2 I: the splat is the plain one with its 3D covariance widened isotropically, and c keeps its integral.
 *   With anti-aliasing the blend opacity is o c h, h from the 2D covariance of the widened splat. IEEE sqrt and division: f = 0 is the
 *   plain splat bit for bit (s' = s, c = 1).
 * Backward (the per-Gaussian stage), with dL/ds' from the covariance chain and g = dL/d(o c) (the opacity sum, times h with anti-aliasing):
 *   dL/ds_c = dL/ds'_c s_c / s'_c + o c g f^2 / (s_c s'_c^2),  dL/do = c g, then the exp and sigmoid chain to the raw parameters.
 * Not filtered: dL/dmean2D and the densification statistics, the densification size tests, the 3DGS-MCMC regularisers and position noise
 *   read the raw activations. max_radii2D takes the forward's radii, which are those of the filtered splat.
 * The caller decides when to recompute the filter (Mip-Splatting: after each densification and every 100 iterations); nothing here does.
 * ------------------------------------------------------------------------------------------------ */
/* filter [P] device float32 <- the filter of the P rows of xyz [P,3] (device) for the K cameras cams [K][20] (device: the view matrix's
 * 16 floats, then focal_x, focal_y, W, H; focal lengths and sizes positive). seen_host (host, may be NULL) receives the number of rows
 * seen by at least one camera; only then does the call synchronise the stream, otherwise it is asynchronous. PSB_ERR_ARG, before any CUDA
 * call, for P < 0, K < 0, a NULL xyz or filter with P > 0 and a NULL cams with K > 0. */
int psb_filter3d(int P, const float* xyz, int K, const float* cams, float* filter, int* seen_host, void* stream);
/* The 3D filter of a context: filter [P] device (as psb_filter3d leaves it) or NULL = off (the default; P is then ignored). While it is
 * set, every pass of the context applies it: psb_trainer_render(_depth), psb_trainer_forward, psb_trainer_step*, psb_trainer_backward*
 * and psb_trainer_backward_pixels, whose per-Gaussian stage differentiates it. The array is read by the passes (not copied): it must
 * stay valid and unchanged while they run. A pass whose P differs from the filter's returns PSB_ERR_ARG before any CUDA call. The
 * setting is recorded in the mode of every pass; psb_trainer_backward_pixels refuses a pass whose filter was switched (or replaced by
 * another array) after it. psb_dp_step*, psb_trainer_backward_begin* and psb_trainer_backward_slab return PSB_ERR_ARG while it is set.
 * Combines with the deterministic, anti-aliasing and regulariser modes. PSB_ERR_ARG for a NULL context and a filter with P < 0. */
int psb_trainer_set_filter3d(psb_trainer* t, const float* filter, int P);

/* ------------------------------------------------------------------------------------------------
 * Contribution scores: how much each Gaussian shows in a set of views, for pruning the ones no view shows.
 * For one pass (view) and one pixel p, Gaussian i blends with w_i(p) = alpha_i(p) T_i(p): exactly the factor the forward multiplies
 * its colour by (C = fma(T, c alpha, C)), T the transmittance before the splat, alpha that of the pass (anti-aliased opacity o h and
 * 3D-filtered opacity o c in those modes, the 0.99 clamp). Only (pixel, splat) pairs that blend count: not those with power > 0,
 * below pmin, with alpha < 1/255, nor the pair whose T test (T (1 - alpha) < 1e-4) ends the pixel. Over the passes of a sweep:
 *   max_weight[i] = max w_i(p) over all pixels and views, as the bits of a float32 (0 = never blended);
 *   sum_weight[i] = sum w_i(p) over all pixels and views, in units of 2^-PSB_CONTRIB_SUM_FRAC_BITS, each pixel's w truncated
 *                   (floor(w 2^26)) before it is added.
 * Both are integers accumulated with integer atomics (atomicMax on the bits: non-negative floats order like their bits; a u64 add), so
 * a sweep's result is bit-identical from run to run, in either deterministic mode and in any order of the views, and sums of
 * separate sweeps add exactly. A weight is at least 1e-4 / 255 (about 26 units), so every blended pair adds to the sum.
 * ------------------------------------------------------------------------------------------------ */
#define PSB_CONTRIB_SUM_FRAC_BITS 26
/* One pass of the sweep: psb_trainer_render of the view (in the context's anti-aliasing and 3D-filter modes; an ordinary forward pass of
 * the context, with the same colour, final T and last contributors) that also ADDS this view's scores into max_weight [P] (u32) and
 * sum_weight [P] (u64), device arrays the caller zeroes once per sweep. out_color [3,H,W] device, or NULL: the context's own image.
 * Asynchronous (no host synchronisation). A pass that overflows the binning arena adds nothing and is reported by psb_trainer_result
 * like a render: zero the arrays and repeat the sweep on the grown arena. PSB_ERR_ARG, before any CUDA call, for a NULL context,
 * camera, background, max_weight or sum_weight, P < 0, and a P that differs from the context's 3D filter's. */
int psb_trainer_contribution(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                             int sh_degree, uint32_t* max_weight, uint64_t* sum_weight, float* out_color, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Point-cloud helpers exported by the same shared objects in the reference.
 * ------------------------------------------------------------------------------------------------ */

/* Mean squared distance of every point to its 3 nearest neighbours. Replaces SimpleKNN::knn /
 * distCUDA2 (third_party/simple-knn/simple_knn.h:15-19, spatial.cu:15-26). points [P,3], mean_dists [P], device.
 * Asynchronous on `stream` (scratch from the stream-ordered allocator; no host round trips). */
int psb_dist_cuda2(int P, const float* points, float* mean_dists, void* stream);

/* p' = M p for a 4x4 column-major M (rows 0..2 used). Replaces the transform_points kernel behind
 * transformPoints (src/operate_points.cu:38-50, 73-93). Out-of-place: out_points [P,3]. */
int psb_transform_points(int P, const float* points, const float* transform, float* out_points, void* stream);

/* For rows with mask != 0: p' = M (scale * p), q' = quaternion(M3x3 * R(q)) (w,x,y,z). Replaces the
 * scale_and_transform_points kernel behind scaleAndTransformThenMarkVisiblePoints (src/operate_points.cu:52-71,
 * 95-143). Unmasked rows of the outputs are left untouched. fix_quaternion_write = 0 reproduces the reference's
 * insert_rot_to_rots exactly (cuda_rasterizer/operate_points.h:170-178 writes z into slot +2 and never writes
 * slot +3 — SURVEY.md §2.2 quirk 10); != 0 writes the intended (w,x,y,z). */
int psb_scale_transform_points(int P, float scale, const float* points, const float* rots, const float* transform,
                               const unsigned char* mask, float* out_points, float* out_rots,
                               int fix_quaternion_write, void* stream);

/* Depth image -> camera-space points for masked pixels (idx = v * width + u). Replaces the reproject_depths_pinhole
 * kernel behind reprojectDepthPinhole (src/stereo_vision.cu:39-61, 138-166). points [P,3] must be zero-initialised. */
int psb_reproject_depth_pinhole(int P, int width, float fx, float fy, float cx, float cy, const float* depths,
                                const unsigned char* mask, float* points, void* stream);

/* Keypoints with a 3-D point keep it; the others borrow the depth of the nearest keypoint (squared pixel distance
 * <= max_pixel_dist) that has one and are re-projected, or get z = -1. Replaces the kernel behind
 * monocularPinholeInactiveGeoDensifyBySearchingNeighborhoodKeypoints (src/stereo_vision.cu:63-136, 168-215), including
 * its colour indexing `colors[(int)(v * width + u) + c]`. Outputs [N,3], zero-initialised by the caller. */
int psb_neighbour_depth_pinhole(int N, int width, float fx, float fy, float cx, float cy, float max_pixel_dist,
                                const float* pixels, const unsigned char* has3D, const float* points_local,
                                const float* colors, float* out_points, float* out_colors, void* stream);

/* Standalone sort primitive (tests): stable LSD radix sort of (u32 key, u32 value) pairs on key bits
 * [0, nbits). keys/vals are device arrays of n elements, sorted in place. */
int psb_debug_sort_pairs(uint32_t* keys, uint32_t* vals, size_t n, int nbits, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PSB200_H_INCLUDED */
