// Internal interface of the trainer-step kernels (psb_train.cu, psb_loss.cu) — not installed.
#pragma once
#include "psb_kernels.h"

namespace psb {

// Raw trainer tensors in the reference's layout and order (include/gaussian_model.h; optimizer groups of
// src/gaussian_model.cpp:477-503): 0 xyz [P,3] | 1 features_dc [P,1,3] | 2 features_rest [P,15,3] |
// 3 opacity [P,1] | 4 scaling [P,3] | 5 rotation [P,4].  m / v = Adam exp_avg / exp_avg_sq of the same shapes.
struct TrainTensors {
	float* p[6];
	float* m[6];
	float* v[6];
};
struct GradSegments {
	float* g[6];
};
struct StepHyper {
	float lr[6];
	float beta1, beta2, eps;
	float inv_bc1;   // 1 / (1 - beta1^t)
	float bc2_sqrt;  // sqrt(1 - beta2^t)
	int D;           // active SH degree
};
struct DensifyStats {
	int enabled;
	float* max_radii2D;         // [P]
	float* xyz_gradient_accum;  // [P,1]
	float* denom;               // [P,1]
};
// The mode of one training-context pass, recorded when the pass runs; its tile backward and per-Gaussian stage run this variant.
struct PassMode {
	int D;       // SH degree of the pass; -1: no psb_trainer_backward_pixels may follow it
	bool det;    // deterministic mode
	bool aa;     // the forward was anti-aliased (launch_preprocess aa): slot 7 of the sink rows holds dL/do'
	bool depth;  // the sink rows carry dL/dz in slot 11 (render_bwd_kernel<F | BWD_DEPTH, GradSink>)
	float reg_opacity, reg_scale;  // psb_trainer_set_regularizers: lambda_opacity, lambda_scale (both 0: the variants without MODE_REG)
	const float* f3d;              // psb_trainer_set_filter3d: the 3D smoothing filter [P] the pass applies, or null (the variants without it)
	bool normals = false;          // the forward wrote n_i of its visible rows (launch_normals): a normal gradient may follow it
	bool normal = false;           // the sink rows are 16 floats and slots 12..14 hold dL/dn (render_bwd_kernel<F | BWD_NORMAL, GradSink>, MODE_NORMAL)
	bool moment = false;           // the forward wrote the second depth moment M (render_fwd_kernel<F | FWD_MOMENT>): a dL/dM may follow it
};
// lambda / P of the opacity and scale regularisers for the rows a per-Gaussian backward updates; both 0 = no regulariser
struct RegCoef {
	float opacity, scale;
};
inline RegCoef reg_coef(const PassMode& m, int P) { return {P > 0 ? m.reg_opacity / (float)P : 0.f, P > 0 ? m.reg_scale / (float)P : 0.f}; }

// ---- NVLink data-parallel step (psb_dp_*, include/psb200.h) -----------------------------------------------------------
// Ownership: Gaussians are cut into chunks of 128 (one block of the per-Gaussian backward); chunk c belongs to rank
// c % world and is that rank's local chunk c / world. Every rank holds a symmetric arena (same layout, peer-mapped through
// CUDA IPC): the six parameter tensors, an inbox [world][nlocal_max][128][20 floats], per-rank meta rows and epoch flags.
constexpr int DP_MAX_WORLD = 8;
constexpr int DP_REC = 20;   // floats per gradient record: g_xyz 3 | g_dc 3 | g_opacity 1 | g_scaling 3 | g_rotation 4 | masked dL/dRGB 3 | pad 2 | epoch
// The exposure record of one rank's step (psb_exposure_table): id | lr | K | valid | the 12 sums dL/dE (the layout of E). valid = 0: the
// rank trained no exposure row, or its pass overflowed the binning arena; the record then counts for nothing.
constexpr int EXP_REC = 16;
// One meta row per rank and step: camera centre 3 | SH degree | the exposure record [4, 20) | unused [20, 32)
constexpr int DP_META = 32;
constexpr int DP_META_EXP = 4;
struct DpPush {              // what the per-Gaussian backward needs to deliver its records
	float* inbox[DP_MAX_WORLD];        // inbox base of every rank (own included), peer-mapped
	float* meta[DP_MAX_WORLD];         // [world][DP_META] floats on every rank: row r = rank r's meta row of this step
	uint32_t* grad_flag[DP_MAX_WORLD]; // [world] epoch words on every rank: word r = "rank r's records of this epoch have landed"
	int world, rank, nlocal_max;
	uint32_t epoch;
};
struct DpShard {             // what the owner-side Adam kernels need
	float* param[DP_MAX_WORLD][6];     // the six parameter tensors on every rank (row of `rank` = local)
	uint32_t* param_flag[DP_MAX_WORLD];// [world] epoch words on every rank: word r = "rank r's updated rows have landed"
	const float* inbox;                // local inbox
	const float* meta;                 // local meta rows
	float* g_rest;                     // local scratch [nlocal_max*128][45]: summed f_rest gradient of the owned rows
	int world, rank, nlocal_max, nlocal, P;   // nlocal: owned chunks of this rank
	uint32_t epoch;
};
// exp_rec: this rank's exposure record of this step (local, EXP_REC floats), published in its meta row with the camera centre; null: the
// meta row says valid = 0
int launch_push_backward(int P, const TrainTensors& t, const Camera& cam, const GeomState& geom, float* sink, const StepHyper& h,
                         const DensifyStats& st, const uint32_t* counters, uint32_t capacity, const DpPush& dp, cudaStream_t stream,
                         const PassMode& mode, const float* exp_rec);
int launch_shard_adam(const DpShard& d, const TrainTensors& t, const StepHyper& h, float grad_scale, cudaStream_t stream, cudaEvent_t between = nullptr);
// spins (device side) until flags[0..world) >= epoch (world <= 32 words); after `timeout_ms` writes 1 to *status and gives up
int launch_wait_flags(const uint32_t* flags, int world, uint32_t epoch, uint32_t* status, cudaStream_t stream);

// Gaussians [first, P) (first must be a multiple of 128 so f_rest chunks stay 16-byte aligned)
// seeds: scratch [P][20] floats (per-Gaussian SH gradient seeds handed from the per-Gaussian kernel to the f_rest stream kernel; with
// adam_live, the momentum-only row list of frest_momentum_kernel and its length instead)
int launch_fused_backward(bool adam, int first, int P, const TrainTensors& t, const Camera& cam, const GeomState& geom, float* sink, float* seeds,
                          const StepHyper& h, const GradSegments& grads, const DensifyStats& st, const uint32_t* counters, uint32_t capacity,
                          cudaStream_t stream, cudaEvent_t between /* recorded between the two kernels (stage timing), or null */,
                          unsigned char* adam_live /* adam only: psb_model.adam_live, or null (the moments tell idle rows) */, const PassMode& mode,
                          const RegCoef& reg /* reg_coef(mode, the model's row count) */);
// 3DGS-MCMC position noise on xyz [P,3] (psb_trainer_inject_noise; kernel in psb_densify.cu, beside the Philox draw it shares with the
// split): lr = lr_xyz * noise_lr; tile_info != null: only rows the pass saw; no-op when counters[0] > capacity
int launch_position_noise(int P, float* xyz, const float* opacity, const float* scaling, const float* rotation, float lr, unsigned long long seed,
                          unsigned long long step, const uint4* tile_info, const uint32_t* counters, uint32_t capacity, cudaStream_t stream);
// adam_live[i] = any moment of row i non-zero (t.m / t.v: the 12 moment tensors)
int launch_adam_live_rebuild(int P, const TrainTensors& t, unsigned char* adam_live, cudaStream_t stream);
int launch_adam(size_t n, float* p, float* m, float* v, const float* g, float lr, const StepHyper& h, float grad_scale, cudaStream_t stream);
// partials != null (deterministic mode): scratch of loss_partials_doubles(H, W); the blocks store their sums there and one more
// launch adds them in a fixed order, so sums[] is the same every run (the default double atomics add in completion order)
// E != null: exposure compensation, the loss of mask * I' with I'(c) = sum_k E[k][c] I(k) + E[c][3] (E: device [3][4], row-major);
// dL_dimg then receives g = dL/dI' (mask factor applied) and launch_exposure must follow.
int launch_loss(int H, int W, const float* img, const float* gt, const float* mask, float lambda_dssim, float* dmap, double* sums,
                float* dL_dimg, cudaStream_t stream, double* partials, const float* E);
// The Adam state of one exposure row (psb_exposure): all device pointers, the step count advanced on the device.
struct ExposureUpdate {
	float* param;
	float* exp_avg;
	float* exp_avg_sq;
	int* step;
	float lr, beta1, beta2, eps;
};
// After launch_loss with E: dL_dpix (g) -> dL/dI in place, and the 12 sums dL/dE added in a fixed order (no atomics: the same every run).
// update != null: the Adam step of the row; else grad [12] device receives dL/dE. An overflowing pass (counters[0] > capacity) leaves
// the row, its moments and its step count untouched (grad: zeros). partials: exposure_blocks(H, W) * 12 doubles. Two launches.
// record != null (the data-parallel steps): the gradient mode writes the EXP_REC-float record instead of grad: id, lr and K as given,
// valid = 0 for an overflowing pass (sums zero), else 1 and the 12 sums.
struct ExposureRecordOut {
	float* rec;   // [EXP_REC] device
	int id, K;
	float lr;
};
int launch_exposure(int H, int W, const float* img, const float* E, float* dL_dpix, double* partials, const uint32_t* counters, uint32_t capacity,
                    const ExposureUpdate* update, float* grad, const ExposureRecordOut* record, cudaStream_t stream);
// A replicated exposure table [K][3][4] (+ moments, int32 step counts [K]) on one rank.
struct ExposureTable {
	float* param;
	float* exp_avg;
	float* exp_avg_sq;
	int* step;
	int K;
};
// One block: the world exposure records recs[r * stride .. + EXP_REC) (rank order) -> the table. For every id k of at least one valid
// record: g = grad_scale * the sum, in rank order, of the valid records' sums with that id; row k takes one Adam step (step count
// step[k] + 1, the lr of the lowest such rank, the betas and eps given), exactly the arithmetic of the single-GPU step's exposure update.
// Rows no valid record names are not touched. A valid record whose K differs from table.K or whose id is outside [0, K) is skipped and
// sets *status to 2 if it was 0 (status may be null).
int launch_exposure_apply(const float* recs, int stride, int world, const ExposureTable& table, float beta1, float beta2, float eps, float grad_scale,
                          uint32_t* status, cudaStream_t stream);
inline int exposure_blocks(int H, int W) { return min(cdiv(H * W, 256), kNumSMs * 8); }
constexpr size_t kExposurePartials = 12 * (size_t)kNumSMs * 8;   // doubles: enough for any image
// Depth L1 over the valid pixels (gt > 0 and, with a mask, mask[0, p] != 0): sums[0] = sum |D - G|, sums[1] = N_valid (zeroed here);
// dL_dD [H,W] = lambda * sign(D - G) / max(N_valid, 1) on valid pixels, 0 elsewhere. Two launches, no host synchronisation.
// partials: as launch_loss.
int launch_depth_loss(int H, int W, const float* depth, const float* gt_depth, const float* mask, float lambda_depth, double* sums, float* dL_dD,
                      cudaStream_t stream, double* partials);
inline int depth_loss_blocks(int H, int W) { return min(cdiv(H * W, 256), kNumSMs * 8); }
// Normal L1 (include/psb200.h, psb_normal) over the valid pixels (gt_normal != (0, 0, 0) and, with a mask, mask[0, p] != 0), normal and
// gt_normal [3,H,W]: sums[0] = sum_valid sum_c |N_c - G_c|, sums[1] = N_valid (zeroed here); dL_dN [3,H,W] = lambda sign(N - G) / max(N_valid, 1)
// on valid pixels, 0 elsewhere. The launch geometry of launch_depth_loss (same partials).
int launch_normal_loss(int H, int W, const float* normal, const float* gt_normal, const float* mask, float lambda_normal, double* sums, float* dL_dN,
                       cudaStream_t stream, double* partials);
// Depth-normal consistency (include/psb200.h, psb_dn) over the depth, opacity and normal planes of one pass whose camera is W x H pixels
// with tan_fovx / tan_fovy: sums[0] = sum_valid (1 - n_d . N), sums[1] = N_valid (zeroed here); out_dn [3,H,W] or null: n_d; dL_dD,
// dL_dA [H,W] and dL_dN [3,H,W] are ADDED into (no atomics). The loss pass has the launch geometry of launch_depth_loss (same partials);
// the gradient pass runs one thread per pixel. No host synchronisation.
int launch_dn_loss(int W, int H, float tan_fovx, float tan_fovy, const float* depth, const float* alpha, const float* normal, const float* mask,
                   float lambda, float alpha_min, float max_rel_jump, float* out_dn, double* sums, float* dL_dD, float* dL_dA, float* dL_dN,
                   cudaStream_t stream, double* partials);
// Depth distortion (include/psb200.h, psb_dist) over the depth D, opacity A and second-moment M planes [H,W] of one pass, mask [H,W] or
// null: sums[0] = sum_valid (A M - D^2) (each term formed in double), sums[1] = N_valid (zeroed here). With k = lambda / max(N_valid, 1)
// (a float division on the device): dL_dA += k M and dL_dD += -2k D on valid pixels (added into, no atomics), and dL_dM = k A there, 0
// elsewhere (written). The launch geometry of launch_depth_loss (same partials). No host synchronisation.
int launch_dist_loss(int H, int W, const float* depth, const float* alpha, const float* depth2, const float* mask, float lambda, double* sums,
                     float* dL_dD, float* dL_dA, float* dL_dM, cudaStream_t stream, double* partials);
// launch_loss runs one block per 16 x 16 tile and channel
inline size_t loss_partials_doubles(int H, int W)
{
	const int loss_blocks = 3 * cdiv(W, 16) * cdiv(H, 16);
	return 2 * (size_t)(loss_blocks > depth_loss_blocks(H, W) ? loss_blocks : depth_loss_blocks(H, W));
}

}  // namespace psb
