// Trainer-level C-ABI (declared in include/psb200.h): a context that owns the scratch arena of the fused
// training iteration, and the iteration itself:
//   preprocess(raw params) -> depth sort -> scan -> emit -> tile sort -> ranges -> render
//   -> fused L1+SSIM loss fwd/bwd -> tile backward -> fused per-Gaussian backward + Adam (+ densify stats)
// The same forward, tile backward and per-Gaussian stages also run around a caller's loss (psb_trainer_forward ->
// the caller's dL/dpixel planes -> psb_trainer_backward_pixels).
// No host synchronisation inside a step: the instance count stays on the device (the binning arena is sized
// from the previous iterations and grown on demand; an overflowing step degrades to a no-op and is reported
// by psb_trainer_result so the caller repeats it).
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <string>
#include "psb_train.h"
#include "../../include/psb200.h"

using namespace psb;

// The context's arena: every buffer has 256 bytes of slack past its elements. A chunk counts rows of the scratch state carved from it.
template <typename T>
using ArenaBuffer = CudaBuffer<T, 256>;
template <typename S>
using ArenaChunk = CudaBuffer<char, 256, false, StateBytes<S>>;

struct psb_trainer {
	ArenaChunk<GeomState> geom;  // P rows: reallocated whenever P changes
	ArenaChunk<ImgState> img;    // W*H pixels: reallocated whenever W*H changes
	ArenaChunk<BinState> bin;    // its count is the binning capacity (instances)
	ArenaBuffer<float> image, dL_dpix, dmap;  // [3][H*W], [3][H*W], [9][H*W]
	ArenaBuffer<float> sink, seeds;           // [P][12] ([P][16] once a normal pass has run; zeroed when allocated), [P][20]
	ArenaBuffer<float> depth_buf;  // depth loss: [2][H*W] = rendered depth (when the caller passes no out_depth) | dL/dD
	ArenaBuffer<float4> normals;   // normal passes: n_i of the visible rows [P], made by the first one
	ArenaBuffer<float> normal_buf; // normal loss: [6][H*W] = rendered normal plane (when the caller passes no out_normal) | dL/dN
	ArenaBuffer<float> alpha_buf;  // depth-normal consistency, depth distortion: [2][H*W] = rendered opacity A | dL/dA
	ArenaBuffer<float> moment_buf; // depth distortion: [2][H*W] = second depth moment M (when the caller passes no out_depth2) | dL/dM
	// device [10]: sum |I - G|, sum SSIM | depth loss: sum |D - G|, N_valid | normal loss: sum |N - G|, N_valid | consistency: sum (1 - n_d . N), N_valid
	//   | distortion: sum (A M - D^2), N_valid
	ArenaBuffer<double> sums;
	CudaBuffer<double, 0, true> h_sums;     // pinned [10]
	CudaBuffer<uint32_t, 0, true> h_count;  // pinned [4]: instance count of the last call | sticky overflow record {count, first seq, largest count}
	ArenaBuffer<uint32_t> ovf;     // device [4]: the sticky overflow record (tile_ranges_kernel), collected by psb_trainer_result
	// what the scratch was last carved for: set when ensure() succeeds, cleared (P = -1) when it fails or the binning chunk is lost
	struct Carved {
		int P = -1, W = 0, H = 0;
	} carved;
	uint32_t seq = 0;            // sequence number of the last forward pass (render / step / backward) of this context
	// the mode of pass `seq`: what psb_trainer_backward_pixels must match, and the variant every per-Gaussian stage behind it runs
	// (a psb_trainer_backward_begin* records it before its pass, so the _slab calls after it run that variant even if it failed)
	PassMode pass = {-1, false, false, false, 0.f, 0.f, nullptr};
	// anti-aliasing (psb_trainer_set_antialiasing): every forward pass blends with o' = o h (the 2D Mip filter), and every per-Gaussian
	// backward behind it runs the AA variant
	bool antialiasing = false;
	// opacity / scale regularisers (psb_trainer_set_regularizers): recorded in the mode of every pass that starts while they are set
	float reg_opacity = 0.f, reg_scale = 0.f;
	// 3D smoothing filter (psb_trainer_set_filter3d): the caller's [filter3d_P] device array, recorded in the mode of every pass that starts
	// while it is set; null = off
	const float* filter3d = nullptr;
	int filter3d_P = 0;
	uint32_t ovf_first = 0, ovf_count = 0;  // what the last PSB_ERR_RETRY was about (psb_trainer_overflow_info)
	// recorded once the instance count (and the loss sums) of the last call are in pinned memory; made last of the read-back set
	// (sums, h_sums, h_count, ovf), so it exists only when the whole set does
	cudaEvent_t readback = nullptr;
	float last_lambda = 0.2f;
	float last_lambda_depth = 0.f;
	float last_lambda_normal = 0.f;
	float last_lambda_dn = 0.f;
	float last_lambda_dist = 0.f;
	bool have_loss = false;
	bool have_depth_loss = false;  // the last step had a depth term (h_sums[2..3] belong to it)
	bool have_normal_loss = false; // the last step had a normal term (h_sums[4..5] belong to it)
	bool have_dn_loss = false;     // the last step had a depth-normal consistency term (h_sums[6..7] belong to it)
	bool have_dist_loss = false;   // the last step had a depth distortion term (h_sums[8..9] belong to it)
	// tight instance lists: only the tiles a splat can reach get an instance (see preprocess_fwd_kernel); PSB_TIGHT=0 keeps the
	// reference's full rectangles (A/B measurements only — images and gradients are the same either way)
	bool tight = !(getenv("PSB_TIGHT") && atoi(getenv("PSB_TIGHT")) == 0);
	// deterministic mode (psb_trainer_set_deterministic): its own scratch, made only while the mode is on and grown with the binning
	// capacity — the instance slots [capacity][12] floats (zeroed when allocated: every tag reads "not this pass"), the emission offsets
	// [P] and the loss partials (a normal pass's slots are [capacity][16] floats)
	bool deterministic = false;
	ArenaBuffer<float> det_slots;
	ArenaBuffer<uint32_t> det_base;
	ArenaBuffer<double> det_partials;
	// exposure compensation (psb_trainer_step_exposure / psb_trainer_backward_exposure): the block partials of the 12 exposure sums
	// [kExposurePartials] doubles, made by the first such call
	ArenaBuffer<double> exp_partials;
	// optional per-stage timing (CUDA events on the step's stream)
	bool profiling = false;
	// stage boundaries: 0 start | 1 preprocess | 2 depth sort | 3 binning | 4 render fwd | 5 loss | 6 render bwd |
	//   fused step:        7 per-Gaussian backward kernel | 8 f_rest Adam stream kernel
	//   data-parallel step: 7 push backward | 8 wait for every rank's records | 9 owner-side Adam (+ stores to every replica);
	//                       ev[NSTAGE] is recorded BEFORE the wait for the previous step's rows (stage "wait_params" = ev[NSTAGE] -> ev[0])
	static constexpr int NSTAGE = 11;   // (ev[10]: between the two owner-side Adam kernels of the data-parallel step)
	int last_stage = 0;  // index of the last boundary the last profiled call recorded
	cudaEvent_t ev[NSTAGE + 1] = {};
	bool ev_ready = false, ev_recorded = false;
	void mark(int i, cudaStream_t s) { if (profiling && ev_ready) cudaEventRecord(ev[i], s); }
	cudaEvent_t event(int i) const { return profiling && ev_ready ? ev[i] : nullptr; }
	// the last boundary of a profiled call: psb_trainer_stage_times reads the stages up to it
	void end_stages(int last, cudaStream_t s) { mark(last, s); last_stage = last; ev_recorded = profiling && ev_ready; }
	~psb_trainer()
	{
		if (ev_ready) for (cudaEvent_t e : ev) cudaEventDestroy(e);
		if (readback) cudaEventDestroy(readback);
	}
};

namespace {

// The context's own plane pairs a pass's loss terms use: depth_buf, normal_buf, alpha_buf, moment_buf ([2][H*W] each, [6][H*W] for the
// normal plane): the rendered plane, when the caller passes none, then its gradient.
struct OwnPlanes {
	bool depth, normal, alpha, moment;
};

// The scratch of a pass of P Gaussians over W x H pixels, each buffer's need stated once (CudaBuffer::grow drains the stream before it
// frees a buffer the last call's kernels may still use). Any failure leaves t->carved cleared: no call reads this scratch until an
// ensure() succeeds.
// mode.normals: a normal pass (n_i, 16-float sink rows and 64-byte deterministic slots); own: the context's plane pairs the pass's loss
// terms use.
int ensure(psb_trainer* t, int P, int W, int H, cudaStream_t stream, const PassMode& mode, const OwnPlanes& own)
{
	const bool normal = mode.normals;
	const size_t N = (size_t)W * H;
	// the binning arena grows to P * 6 + 64 Ki instances when it is empty, or when it is smaller and the last pass was over another P
	const size_t bin_need = t->bin.count() == 0 || t->carved.P != P ? (size_t)P * 6 + (1u << 16) : 0;
	t->carved = {};
	PSB_CUDA_OK(t->geom.grow((size_t)P, Fit::exact, false, stream));
	PSB_CUDA_OK(t->img.grow(N, Fit::exact, false, stream));
	PSB_CUDA_OK(t->image.grow(3 * N, Fit::at_least, false, stream));
	PSB_CUDA_OK(t->dL_dpix.grow(3 * N, Fit::at_least, false, stream));
	PSB_CUDA_OK(t->dmap.grow(9 * N, Fit::at_least, false, stream));
	if (own.depth) PSB_CUDA_OK(t->depth_buf.grow(2 * N, Fit::at_least, false, stream));
	if (normal) PSB_CUDA_OK(t->normals.grow((size_t)P, Fit::at_least, false, stream));
	if (own.normal) PSB_CUDA_OK(t->normal_buf.grow(6 * N, Fit::at_least, false, stream));
	if (own.alpha) PSB_CUDA_OK(t->alpha_buf.grow(2 * N, Fit::at_least, false, stream));
	if (own.moment) PSB_CUDA_OK(t->moment_buf.grow(2 * N, Fit::at_least, false, stream));
	PSB_CUDA_OK(t->sink.grow((size_t)P * (normal ? 16 : 12), Fit::at_least, true, stream));
	PSB_CUDA_OK(t->seeds.grow((size_t)P * 20, Fit::at_least, false, stream));
	if (!t->readback) {
		PSB_CUDA_OK(t->sums.grow(10, Fit::at_least, false, stream));
		PSB_CUDA_OK(t->h_sums.grow(10, Fit::at_least, false, stream));
		PSB_CUDA_OK(t->h_count.grow(4, Fit::at_least, true, stream));
		PSB_CUDA_OK(t->ovf.grow(4, Fit::at_least, false, stream));
		const uint32_t init[4] = {0u, 0xFFFFFFFFu, 0u, 0u};
		PSB_CUDA_OK(cudaMemcpy(t->ovf.get(), init, sizeof(init), cudaMemcpyHostToDevice));
		PSB_CUDA_OK(cudaEventCreateWithFlags(&t->readback, cudaEventDisableTiming));
	}
	PSB_CUDA_OK(t->bin.grow(bin_need, Fit::at_least, false, stream));
	if (t->deterministic) {
		PSB_CUDA_OK(t->det_slots.grow(t->bin.count() * (normal ? 16 : 12), Fit::at_least, true, stream));
		PSB_CUDA_OK(t->det_base.grow((size_t)P, Fit::at_least, false, stream));
		PSB_CUDA_OK(t->det_partials.grow(loss_partials_doubles(H, W), Fit::at_least, false, stream));
	}
	t->carved = {P, W, H};
	return 0;
}

Camera to_camera(const psb_camera* c)
{
	return make_camera(c->width, c->height, c->viewmatrix, c->projmatrix, c->campos, c->tan_fovx, c->tan_fovy);
}

// the scratch states of the last forward pass of P Gaussians over width x height pixels, carved from the context's arena
struct Scratch {
	GeomState geom;
	ImgState img;
	BinState bin;
};
Scratch carve_scratch(const psb_trainer* t, int P, int width, int height)
{
	char* gc = t->geom.get();
	char* ic = t->img.get();
	char* bc = t->bin.get();
	return {GeomState::from_chunk(gc, (size_t)P), ImgState::from_chunk(ic, (size_t)width * height), BinState::from_chunk(bc, t->bin.count())};
}

GaussIn raw_input(int P, int D, int M, const psb_model* m)
{
	GaussIn in;
	memset(&in, 0, sizeof(in));
	in.P = P; in.D = D; in.M = M;
	in.means3D = m->param[0]; in.sh_dc = m->param[1]; in.sh_rest = m->param[2];
	in.opacities = m->param[3]; in.scales = m->param[4]; in.rotations = m->param[5];
	in.scale_modifier = 1.0f;
	return in;
}

StepHyper to_hyper(const psb_step* s)
{
	StepHyper h;
	for (int i = 0; i < 6; i++) h.lr[i] = s->lr[i];
	h.beta1 = s->beta1; h.beta2 = s->beta2; h.eps = s->eps;
	h.inv_bc1 = (float)(1.0 / (1.0 - std::pow((double)s->beta1, s->step)));
	h.bc2_sqrt = (float)std::sqrt(1.0 - std::pow((double)s->beta2, s->step));
	h.D = s->sh_degree;
	return h;
}

TrainTensors train_tensors(const psb_model* m, bool moments)
{
	TrainTensors tt;
	for (int i = 0; i < 6; i++) {
		tt.p[i] = m->param[i];
		tt.m[i] = moments ? m->exp_avg[i] : nullptr;
		tt.v[i] = moments ? m->exp_avg_sq[i] : nullptr;
	}
	return tt;
}

DensifyStats densify_stats(const psb_model* m, const psb_step* s)
{
	DensifyStats st;
	st.enabled = (s->update_densify_stats && m->max_radii2D && m->xyz_gradient_accum && m->denom) ? 1 : 0;
	st.max_radii2D = m->max_radii2D; st.xyz_gradient_accum = m->xyz_gradient_accum; st.denom = m->denom;
	return st;
}

int check_model(int P, int M, const psb_model* m, bool need_moments)
{
	if (P < 0 || M != 16 || !m) { set_error_msg("psb_trainer: need P >= 0, M == 16 (SH degree 3 storage) and a model"); return PSB_ERR_ARG; }
	for (int i = 0; i < 6; i++) {
		if (P > 0 && (!m->param[i] || (need_moments && (!m->exp_avg[i] || !m->exp_avg_sq[i])))) { set_error_msg("psb_trainer: null model tensor"); return PSB_ERR_ARG; }
	}
	const uintptr_t a = reinterpret_cast<uintptr_t>(m->param[2]) | reinterpret_cast<uintptr_t>(m->param[5]) |
	                    (need_moments ? (reinterpret_cast<uintptr_t>(m->exp_avg[2]) | reinterpret_cast<uintptr_t>(m->exp_avg_sq[2]) |
	                                     reinterpret_cast<uintptr_t>(m->exp_avg[5]) | reinterpret_cast<uintptr_t>(m->exp_avg_sq[5])) : 0);
	if (a & 15) { set_error_msg("psb_trainer: features_rest / rotation tensors must be 16-byte aligned"); return PSB_ERR_ARG; }
	return 0;
}

// NULL: no depth. Otherwise lambda_depth finite and >= 0, and a target exactly when lambda_depth > 0.
int check_depth(const psb_depth* d, const char* fn)
{
	if (!d) return 0;
	if (!std::isfinite(d->lambda_depth) || d->lambda_depth < 0.f) {
		set_error_msg(std::string(fn).append(": lambda_depth must be finite and >= 0").c_str());
		return PSB_ERR_ARG;
	}
	if ((d->gt_depth != nullptr) != (d->lambda_depth > 0.f)) {
		set_error_msg(std::string(fn).append(": gt_depth and lambda_depth > 0 must be given together").c_str());
		return PSB_ERR_ARG;
	}
	return 0;
}

// NULL: no normal term. Otherwise lambda_normal finite and >= 0, and a target exactly when lambda_normal > 0.
int check_normal(const psb_normal* n, const char* fn)
{
	if (!n) return 0;
	if (!std::isfinite(n->lambda_normal) || n->lambda_normal < 0.f) {
		set_error_msg(std::string(fn).append(": lambda_normal must be finite and >= 0").c_str());
		return PSB_ERR_ARG;
	}
	if ((n->gt_normal != nullptr) != (n->lambda_normal > 0.f)) {
		set_error_msg(std::string(fn).append(": gt_normal and lambda_normal > 0 must be given together").c_str());
		return PSB_ERR_ARG;
	}
	return 0;
}

// NULL: no consistency term. Otherwise lambda_dn finite and > 0, alpha_min in (0, 1] and max_rel_jump finite and > 0.
int check_dn(const psb_dn* d, const char* fn)
{
	if (!d) return 0;
	if (!std::isfinite(d->lambda_dn) || !(d->lambda_dn > 0.f)) {
		set_error_msg(std::string(fn).append(": lambda_dn must be finite and > 0").c_str());
		return PSB_ERR_ARG;
	}
	if (!(d->alpha_min > 0.f && d->alpha_min <= 1.f)) {
		set_error_msg(std::string(fn).append(": alpha_min must lie in (0, 1]").c_str());
		return PSB_ERR_ARG;
	}
	if (!std::isfinite(d->max_rel_jump) || !(d->max_rel_jump > 0.f)) {
		set_error_msg(std::string(fn).append(": max_rel_jump must be finite and > 0").c_str());
		return PSB_ERR_ARG;
	}
	return 0;
}

// NULL: no distortion term. Otherwise lambda_dist finite and >= 0 (0: the plane alone, when out_depth2 is given).
int check_dist(const psb_dist* d, const char* fn)
{
	if (!d) return 0;
	if (!std::isfinite(d->lambda_dist) || d->lambda_dist < 0.f) {
		set_error_msg(std::string(fn).append(": lambda_dist must be finite and >= 0").c_str());
		return PSB_ERR_ARG;
	}
	return 0;
}

// NULL: no exposure. Otherwise a row (param), a finite lr >= 0 and, for a step (`adam`), the moments and the device step count; for the
// gradient mode a gradient output.
int check_exposure(const psb_exposure* e, bool adam, const float* grad, const char* fn)
{
	if (!e) return 0;
	if (!e->param || (adam && (!e->exp_avg || !e->exp_avg_sq || !e->step)) || (!adam && !grad)) {
		set_error_msg(std::string(fn).append(adam ? ": exposure needs param, exp_avg, exp_avg_sq and step" : ": exposure needs param and exposure_grad").c_str());
		return PSB_ERR_ARG;
	}
	if (!std::isfinite(e->lr) || e->lr < 0.f) {
		set_error_msg(std::string(fn).append(": exposure lr must be finite and >= 0").c_str());
		return PSB_ERR_ARG;
	}
	return 0;
}

// NULL: no table. Otherwise K >= 0, id in [-1, K), a finite lr >= 0, the row, moment and step arrays when K > 0 and, for the gradient
// modes (`record`), a record output.
int check_table(const psb_exposure_table* e, bool record, const char* fn)
{
	if (!e) return 0;
	if (e->K < 0 || e->id < -1 || e->id >= e->K) {
		set_error_msg(std::string(fn).append(": exposure id must be -1 or lie in [0, K), and K >= 0").c_str());
		return PSB_ERR_ARG;
	}
	if (e->K > 0 && (!e->param || !e->exp_avg || !e->exp_avg_sq || !e->step)) {
		set_error_msg(std::string(fn).append(": the exposure table needs param, exp_avg, exp_avg_sq and step").c_str());
		return PSB_ERR_ARG;
	}
	if (!std::isfinite(e->lr) || e->lr < 0.f) {
		set_error_msg(std::string(fn).append(": exposure lr must be finite and >= 0").c_str());
		return PSB_ERR_ARG;
	}
	if (record && !e->record) {
		set_error_msg(std::string(fn).append(": the exposure table needs a record output on this path").c_str());
		return PSB_ERR_ARG;
	}
	return 0;
}

// The row a table trains this step, as a gradient-mode psb_exposure (param only), and where its record goes.
struct TableRow {
	psb_exposure row;
	ExposureRecordOut rec;
	bool any;   // the rank trains a row (id >= 0)
};
TableRow table_row(const psb_exposure_table* e, float* rec)
{
	TableRow r{};
	if (!e || e->id < 0) return r;
	r.row.param = e->param + 12 * (size_t)e->id;
	r.row.lr = e->lr;
	r.rec = {rec, e->id, e->K, e->lr};
	r.any = true;
	return r;
}

ExposureTable exposure_table(const psb_exposure_table* e)
{
	return {e->param, e->exp_avg, e->exp_avg_sq, e->step, e->K};
}

// Gradient segments of P rows: six non-null pointers, features_rest and rotation 16-byte aligned (written with float4 stores).
int check_grads(float* const* grads, int P, const char* fn)
{
	if (!grads) { set_error_msg(std::string(fn).append(": grads required").c_str()); return PSB_ERR_ARG; }
	if (P <= 0) return 0;
	for (int i = 0; i < 6; i++)
		if (!grads[i]) { set_error_msg(std::string(fn).append(": null gradient segment").c_str()); return PSB_ERR_ARG; }
	if ((reinterpret_cast<uintptr_t>(grads[2]) | reinterpret_cast<uintptr_t>(grads[5])) & 15) {
		set_error_msg(std::string(fn).append(": the features_rest and rotation gradient segments must be 16-byte aligned").c_str());
		return PSB_ERR_ARG;
	}
	return 0;
}

// The mode of a pass that starts now, in the context's deterministic, anti-aliasing, regulariser and 3D-filter modes.
PassMode pass_mode(const psb_trainer* t, int D, bool depth)
{
	return {D, t->deterministic, t->antialiasing, depth, t->reg_opacity, t->reg_scale, t->filter3d};
}

// A pass over P rows while a 3D filter is set must be over the filter's rows.
int check_filter3d(const psb_trainer* t, int P, const char* fn)
{
	if (t->filter3d && P != t->filter3d_P) {
		set_error_msg(std::string(fn).append(": the 3D filter set with psb_trainer_set_filter3d has a different row count than P").c_str());
		return PSB_ERR_ARG;
	}
	return 0;
}

// The NVLink and slab-pipelined data-parallel calls take no 3D filter.
int refuse_filter3d(const psb_trainer* t, const char* fn)
{
	if (t && t->filter3d) {
		set_error_msg(std::string(fn).append(": the 3D filter is not wired into the data-parallel steps; psb_trainer_set_filter3d(t, NULL, 0) first").c_str());
		return PSB_ERR_ARG;
	}
	return 0;
}

// Stage 1 of every pass: forward of SH degree D from raw parameters into t->image (or out_color), with the planes of `planes`
// (launch_render_forward). Each plane in `own` is the caller's where `planes` gives one, else the first half of the context's own pair:
// `planes` returns the planes the pass rendered. mode.normals: n_i of the visible rows -> t->normals (planes.normals). The pass is
// recorded as `mode`, with D = -1 until it has been binned.
int forward_raw(psb_trainer* t, int P, int M, int D, const psb_model* model, const psb_camera* camera, const float* background,
                float* out_color, int* radii, Scratch& sc, Camera& cam, cudaStream_t stream, FwdPlanes& planes, const PassMode& mode,
                const OwnPlanes& own)
{
	int rc;
	t->pass = mode;
	t->pass.D = -1;
	if ((rc = ensure(t, P, camera->width, camera->height, stream, mode, own))) return rc;
	if (own.depth && !planes.out_depth) planes.out_depth = t->depth_buf.get();
	if (own.normal && !planes.out_normal) planes.out_normal = t->normal_buf.get();
	if (own.alpha && !planes.out_alpha) planes.out_alpha = t->alpha_buf.get();
	if (own.moment && !planes.out_depth2) planes.out_depth2 = t->moment_buf.get();
	planes.normals = mode.normals ? t->normals.get() : nullptr;
	cam = to_camera(camera);
	sc = carve_scratch(t, P, camera->width, camera->height);
	GeomState& geom = sc.geom;
	BinState& bin = sc.bin;
	ImgState& img = sc.img;
	const GaussIn in = raw_input(P, D, M, model);
	t->mark(0, stream);
	if ((rc = launch_preprocess(in, cam, radii, geom, /*raw=*/true, t->tight, stream, mode.aa, mode.f3d))) return rc;
	if (mode.normals && (rc = launch_normals(P, model->param[0], model->param[4], model->param[5], cam, geom.tile_info, t->normals.get(), stream))) return rc;
	t->mark(1, stream);
	if ((rc = launch_depth_sort_and_scan(P, geom, /*scan=*/false, stream))) return rc;
	t->mark(2, stream);
	if ((rc = launch_scan_binning(P, cam, geom, bin, img, t->bin.count(), t->tight, t->ovf.get(), ++t->seq, stream, mode.det ? t->det_base.get() : nullptr)))
		return rc;
	t->pass.D = mode.D;
	t->mark(3, stream);
	// the instance count travels to pinned memory as soon as it exists: psb_trainer_result waits on `readback`, not on the stream
	PSB_CUDA_OK(cudaMemcpyAsync(t->h_count.get(), geom.counters, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
	PSB_CUDA_OK(cudaMemcpyAsync(t->h_count.get() + 1, t->ovf.get(), 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
	PSB_CUDA_OK(cudaEventRecord(t->readback, stream));
	rc = launch_render_forward(cam, img.ranges, bin.inst[sorted_slot(cam.W, cam.H)], geom.rec, background, out_color ? out_color : t->image.get(), img.final_T,
	                           img.n_contrib, planes, stream);
	t->mark(4, stream);
	return rc;
}

// Stage 3 of every pass: the tile backward of the context's last forward pass (scratch sc, camera cam, mode t->pass) on per-pixel
// gradients -> the packed sink rows (planes.dL_ddepth: also dL/dz in slot 11; dL_dalpha: the opacity variant; dL_dnormal: the normal
// variant, 16-float rows with dL/dn in slots 12..14, after a pass with mode.normals; dL_ddepth2: the moment variant, its 2 z dL/dM in slot
// 11, after a pass with mode.moment). The deterministic slots and n_i are the context's. P > 0.
int tile_backward(psb_trainer* t, int P, const Scratch& sc, const Camera& cam, const float* background, const float* dL_dpix, BwdPlanes planes,
                  cudaStream_t stream)
{
	float* const rows = t->sink.get();
	GradSink sink;
	sink.mean2D = rows; sink.mean2D_stride = 12;
	sink.conic = rows + 3; sink.conic_stride = 12;
	sink.opacity = rows + 7; sink.opacity_stride = 12;
	sink.color = rows + 8; sink.color_stride = 12;
	sink.packed = 1;
	DetSlots det;
	det.slots = reinterpret_cast<float4*>(t->det_slots.get());
	det.base = t->det_base.get();
	det.tile_info = sc.geom.tile_info;
	det.counters = sc.geom.counters;
	det.capacity = (uint32_t)t->bin.count();
	det.seq = t->seq;
	det.P = P;
	det.tight = t->tight ? 1 : 0;
	planes.det = t->pass.det ? &det : nullptr;
	planes.normals = planes.dL_dnormal ? t->normals.get() : nullptr;
	// (the deterministic gather runs inside this call: stage "render bwd" covers it)
	int rc;
	if ((rc = launch_render_backward(cam, sc.img.ranges, sc.bin.inst[sorted_slot(cam.W, cam.H)], sc.geom.rec, background, sc.img.final_T, sc.img.n_contrib,
	                                 dL_dpix, sink, planes, stream)))
		return rc;
	t->mark(6, stream);
	return 0;
}

// What the first half of a training step leaves for its per-Gaussian stage, besides the sink rows (the view's screen-space sums; with a
// depth term also dL/dz in slot 11, which the per-Gaussian kernel that follows must consume: it runs the variant t->pass names).
struct TileBackward {
	GeomState geom;
	Camera cam;
};

// The built-in loss around the shared stages: forward -> loss (+ depth loss) -> pinned read-back of the loss sums -> (exposure) -> tile
// backward. `moments`: the caller's per-Gaussian stage updates the Adam moments of the model. exposure != NULL: the loss is that of the
// image through the row; exposure_grad == NULL: the row takes its Adam step (with step's betas and eps), else dL/dE -> exposure_grad;
// exposure_record != NULL: dL/dE goes to that data-parallel record instead (the row does not move).
int render_loss_backward(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                         const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, const psb_depth* depth,
                         bool moments, cudaStream_t stream, TileBackward& out, const psb_exposure* exposure, float* exposure_grad,
                         const psb_normal* normal, const psb_dn* dn, const psb_dist* dist, const ExposureRecordOut* exposure_record = nullptr)
{
	int rc;
	if (!t || !camera || !step || !background || !gt_image) { set_error_msg("psb_trainer_step: null argument"); return PSB_ERR_ARG; }
	if ((rc = check_model(P, M, model, moments))) return rc;
	if ((rc = check_filter3d(t, P, "psb_trainer_step"))) return rc;
	if (step->sh_degree < 0 || step->sh_degree > 3 || step->step < 1) { set_error_msg("psb_trainer_step: sh_degree in 0..3 and step >= 1 required"); return PSB_ERR_ARG; }
	const size_t npix = (size_t)camera->width * camera->height;
	// the depth-normal consistency term reads D, A and N of this pass and adds into dL/dD, dL/dA and dL/dN: it forces all three planes
	const bool dn_loss = dn != nullptr;
	// the distortion term reads D, A and M of this pass, adds into dL/dD and dL/dA and writes dL/dM: it forces those three planes
	const bool dist_loss = dist && dist->lambda_dist > 0.f;
	const bool depth_loss = depth && depth->gt_depth;
	const bool depth_pass = depth_loss || dn_loss || dist_loss;
	const bool normal_loss = normal && normal->gt_normal;
	const bool normal_grad = normal_loss || dn_loss;
	// each term's plane is the caller's or the context's own (forward_raw), and its gradient lives in the context. An out_normal or
	// out_depth2 alone renders the plane and leaves the backward that of the step without it.
	const OwnPlanes own{depth_pass, normal_grad, dn_loss || dist_loss, dist_loss};
	FwdPlanes planes{};
	planes.out_depth = depth ? depth->out_depth : nullptr;
	planes.out_normal = normal ? normal->out_normal : nullptr;
	planes.out_depth2 = dist ? dist->out_depth2 : nullptr;
	if (exposure) PSB_CUDA_OK(t->exp_partials.grow(kExposurePartials, Fit::at_least, false, stream));
	Scratch sc;
	Camera cam;
	PassMode mode = pass_mode(t, -1, depth_pass);
	mode.normals = planes.out_normal || own.normal;
	mode.normal = normal_grad;
	mode.moment = planes.out_depth2 || own.moment;
	// this pass gets its own tile backward below and its sink rows belong to this call's per-Gaussian stage (or to the _slab calls
	// that follow a _begin): psb_trainer_backward_pixels must not add a second backward of it (D = -1)
	if ((rc = forward_raw(t, P, M, step->sh_degree, model, camera, background, out_color, radii, sc, cam, stream, planes, mode, own))) return rc;
	float* const depth_plane = planes.out_depth;
	float* const normal_plane = planes.out_normal;
	float* const alpha_plane = planes.out_alpha;
	float* const depth2_plane = planes.out_depth2;
	float* const dL_ddepth = own.depth ? t->depth_buf.get() + npix : nullptr;
	float* const dL_dnormal = own.normal ? t->normal_buf.get() + 3 * npix : nullptr;
	float* const dL_dalpha = own.alpha ? t->alpha_buf.get() + npix : nullptr;
	float* const dL_ddepth2 = own.moment ? t->moment_buf.get() + npix : nullptr;
	const float* image = out_color ? out_color : t->image.get();
	double* partials = t->deterministic ? t->det_partials.get() : nullptr;
	if ((rc = launch_loss(cam.H, cam.W, image, gt_image, mask, step->lambda_dssim, t->dmap.get(), t->sums.get(), t->dL_dpix.get(), stream, partials,
	                      exposure ? exposure->param : nullptr)))
		return rc;
	if (depth_loss &&
	    (rc = launch_depth_loss(cam.H, cam.W, depth_plane, depth->gt_depth, mask, depth->lambda_depth, t->sums.get() + 2, dL_ddepth, stream, partials)))
		return rc;
	if (normal_loss &&
	    (rc = launch_normal_loss(cam.H, cam.W, normal_plane, normal->gt_normal, mask, normal->lambda_normal, t->sums.get() + 4, dL_dnormal, stream, partials)))
		return rc;
	// the consistency term adds into the gradient planes after the depth and normal terms wrote theirs; planes no term wrote start at 0
	if (dn_loss) {
		if (!depth_loss) PSB_CUDA_OK(cudaMemsetAsync(dL_ddepth, 0, npix * sizeof(float), stream));
		if (!normal_loss) PSB_CUDA_OK(cudaMemsetAsync(dL_dnormal, 0, 3 * npix * sizeof(float), stream));
		PSB_CUDA_OK(cudaMemsetAsync(dL_dalpha, 0, npix * sizeof(float), stream));
		if ((rc = launch_dn_loss(cam.W, cam.H, camera->tan_fovx, camera->tan_fovy, depth_plane, alpha_plane, normal_plane, mask, dn->lambda_dn, dn->alpha_min,
		                         dn->max_rel_jump, dn->out_depth_normal, t->sums.get() + 6, dL_ddepth, dL_dalpha, dL_dnormal, stream, partials)))
			return rc;
	}
	// the distortion term adds into dL/dD and dL/dA after the depth, normal and consistency terms wrote theirs (planes no term wrote start
	// at 0) and writes dL/dM
	if (dist_loss) {
		if (!depth_loss && !dn_loss) PSB_CUDA_OK(cudaMemsetAsync(dL_ddepth, 0, npix * sizeof(float), stream));
		if (!dn_loss) PSB_CUDA_OK(cudaMemsetAsync(dL_dalpha, 0, npix * sizeof(float), stream));
		if ((rc = launch_dist_loss(cam.H, cam.W, depth_plane, alpha_plane, depth2_plane, mask, dist->lambda_dist, t->sums.get() + 8, dL_ddepth, dL_dalpha,
		                           dL_ddepth2, stream, partials)))
			return rc;
	}
	// loss sums -> pinned memory right behind the loss kernel, so the host can read the loss of this iteration (and start
	// enqueueing the next one) while the backward half is still running
	PSB_CUDA_OK(cudaMemcpyAsync(t->h_sums.get(), t->sums.get(), (dist_loss ? 10 : dn_loss ? 8 : normal_loss ? 6 : depth_loss ? 4 : 2) * sizeof(double),
	                            cudaMemcpyDeviceToHost, stream));
	PSB_CUDA_OK(cudaEventRecord(t->readback, stream));
	t->last_lambda = step->lambda_dssim;
	t->last_lambda_depth = depth_loss ? depth->lambda_depth : 0.f;
	t->last_lambda_normal = normal_loss ? normal->lambda_normal : 0.f;
	t->last_lambda_dn = dn_loss ? dn->lambda_dn : 0.f;
	t->last_lambda_dist = dist_loss ? dist->lambda_dist : 0.f;
	t->have_loss = true;
	t->have_depth_loss = depth_loss;
	t->have_normal_loss = normal_loss;
	t->have_dn_loss = dn_loss;
	t->have_dist_loss = dist_loss;
	if (exposure) {
		// dL/dI for the tile backward and the row's update (or gradient), inside stage "loss"; the row moves only after every read of it
		ExposureUpdate u{exposure->param, exposure->exp_avg, exposure->exp_avg_sq, exposure->step, exposure->lr, step->beta1, step->beta2, step->eps};
		if ((rc = launch_exposure(cam.H, cam.W, image, exposure->param, t->dL_dpix.get(), t->exp_partials.get(), P > 0 ? sc.geom.counters : nullptr,
		                          (uint32_t)t->bin.count(), exposure_grad || exposure_record ? nullptr : &u, exposure_grad, exposure_record, stream)))
			return rc;
	}
	t->mark(5, stream);
	if (P == 0) return 0;
	if ((rc = tile_backward(t, P, sc, cam, background, t->dL_dpix.get(), BwdPlanes{dL_ddepth, nullptr, dL_dalpha, nullptr, dL_dnormal, dL_ddepth2, nullptr},
	                        stream)))
		return rc;
	out.geom = sc.geom;
	out.cam = cam;
	return 0;
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------------------
// NVLink data-parallel context (psb_dp_*): the symmetric arena of one rank and its peer mappings.
// ------------------------------------------------------------------------------------------------------------------------
struct psb_dp {
	int rank = 0, world = 1, P = 0;
	int nchunks = 0, nlocal_max = 0, nlocal = 0;
	CudaBuffer<char> base;                      // local arena (cudaMalloc: exportable through CUDA IPC)
	char* peer[DP_MAX_WORLD] = {};              // arena of every rank in this process' address space (peer[rank] == base)
	size_t off_param[6] = {}, off_inbox = 0, off_meta = 0, off_gflag = 0, off_pflag = 0, bytes = 0;
	CudaBuffer<float> g_rest;                   // local scratch
	CudaBuffer<uint32_t> status;                // local word: 1 = a cross-rank wait timed out, 2 = an exposure record was refused
	CudaBuffer<float> exp_rec;                  // local [EXP_REC]: this rank's exposure record of the step, published in its meta row
	uint32_t epoch = 0;
	bool connected = false;
	cudaIpcMemHandle_t handle;
};

namespace {
void dp_layout(psb_dp* d)
{
	size_t o = 0;
	for (int i = 0; i < 6; i++) { d->off_param[i] = o; o = align_up(o + (size_t)d->P * row_floats(i) * sizeof(float), 256); }
	d->off_inbox = o; o = align_up(o + (size_t)d->world * d->nlocal_max * 128 * DP_REC * sizeof(float), 256);
	d->off_meta = o; o += DP_MAX_WORLD * DP_META * sizeof(float);
	d->off_gflag = o; o += 256;
	d->off_pflag = o; o += 256;
	d->bytes = o;
}
}  // namespace

extern "C" {

int psb_dp_create(psb_dp** out, int rank, int world, int P)
{
	if (!out || world < 1 || world > DP_MAX_WORLD || rank < 0 || rank >= world || P < 0) { set_error_msg("psb_dp_create: need 0 <= rank < world <= 8, P >= 0"); return PSB_ERR_ARG; }
	psb_dp* d = new psb_dp();
	d->rank = rank; d->world = world; d->P = P;
	d->nchunks = (P + 127) / 128;
	d->nlocal_max = (d->nchunks + world - 1) / world;
	d->nlocal = d->nchunks > rank ? (d->nchunks - rank + world - 1) / world : 0;
	dp_layout(d);
	// (zeroed on the legacy default stream, as cudaMemset does)
	cudaError_t e = d->base.grow(d->bytes, Fit::exact, true, nullptr);
	if (e == cudaSuccess) e = d->g_rest.grow((size_t)d->nlocal_max * 128 * kRestFloats + 64, Fit::exact, false, nullptr);
	if (e == cudaSuccess) e = d->status.grow(1, Fit::exact, true, nullptr);
	if (e == cudaSuccess) e = d->exp_rec.grow(EXP_REC, Fit::exact, true, nullptr);
	if (e == cudaSuccess && world > 1) e = cudaIpcGetMemHandle(&d->handle, d->base.get());
	if (e != cudaSuccess) {
		set_error("psb_dp_create", e, __FILE__, __LINE__);
		delete d;
		return PSB_ERR_CUDA;
	}
	d->peer[rank] = d->base.get();
	d->connected = world == 1;
	*out = d;
	return 0;
}

int psb_dp_handle_bytes(void) { return (int)sizeof(cudaIpcMemHandle_t); }

int psb_dp_ipc_handle(psb_dp* d, void* out_handle)
{
	if (!d || !out_handle) { set_error_msg("psb_dp_ipc_handle: null"); return PSB_ERR_ARG; }
	memcpy(out_handle, &d->handle, sizeof(cudaIpcMemHandle_t));
	return 0;
}

int psb_dp_connect(psb_dp* d, const void* handles)
{
	if (!d || (d->world > 1 && !handles)) { set_error_msg("psb_dp_connect: null"); return PSB_ERR_ARG; }
	for (int j = 0; j < d->world; j++) {
		if (j == d->rank || d->peer[j]) continue;
		cudaIpcMemHandle_t h;
		memcpy(&h, static_cast<const char*>(handles) + (size_t)j * sizeof(h), sizeof(h));
		void* p = nullptr;
		PSB_CUDA_OK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
		d->peer[j] = static_cast<char*>(p);
	}
	d->connected = true;
	return 0;
}

int psb_dp_params(psb_dp* d, float** out6)
{
	if (!d || !out6) { set_error_msg("psb_dp_params: null"); return PSB_ERR_ARG; }
	for (int i = 0; i < 6; i++) out6[i] = reinterpret_cast<float*>(d->base.get() + d->off_param[i]);
	return 0;
}

int psb_dp_destroy(psb_dp* d)
{
	if (!d) return 0;
	cudaDeviceSynchronize();
	for (int j = 0; j < d->world; j++)
		if (j != d->rank && d->peer[j]) cudaIpcCloseMemHandle(d->peer[j]);
	delete d;
	return 0;
}

// Enqueues a wait (device side) until every rank's parameter rows of the last psb_dp_step have landed in THIS rank's
// tensors: after it, the local replica is complete and may be read by anything that follows on `stream`.
int psb_dp_sync(psb_dp* d, void* stream_)
{
	if (!d) { set_error_msg("psb_dp_sync: null"); return PSB_ERR_ARG; }
	if (d->epoch == 0 || d->P == 0 || d->world == 1) return 0;   // (one rank: everything is on the caller's stream)
	return launch_wait_flags(reinterpret_cast<const uint32_t*>(d->base.get() + d->off_pflag), d->world, d->epoch, d->status.get(), (cudaStream_t)stream_);
}

// 0 = healthy, 1 = a cross-rank wait timed out (a peer never arrived); synchronises the stream
int psb_dp_status(psb_dp* d, void* stream_)
{
	if (!d) { set_error_msg("psb_dp_status: null"); return PSB_ERR_ARG; }
	uint32_t st = 0;
	PSB_CUDA_OK(cudaMemcpyAsync(&st, d->status.get(), sizeof(st), cudaMemcpyDeviceToHost, (cudaStream_t)stream_));
	PSB_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream_));
	return (int)st;
}

int psb_dp_step_depth(psb_trainer* t, psb_dp* d, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                      const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, const psb_depth* depth,
                      void* stream_)
{
	return psb_dp_step_dist(t, d, P, M, model, camera, background, gt_image, mask, step, out_color, radii, depth, nullptr, nullptr, nullptr, stream_);
}

int psb_dp_step_dist(psb_trainer* t, psb_dp* d, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                     const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, const psb_depth* depth,
                     const psb_normal* normal, const psb_dn* dn, const psb_dist* dist, void* stream_)
{
	return psb_dp_step_table(t, d, P, M, model, camera, background, gt_image, mask, step, out_color, radii, depth, normal, dn, dist, nullptr, stream_);
}

int psb_dp_step_table(psb_trainer* t, psb_dp* d, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                      const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, const psb_depth* depth,
                      const psb_normal* normal, const psb_dn* dn, const psb_dist* dist, const psb_exposure_table* exposure, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	int rc;
	const char* fn = exposure ? "psb_dp_step_table" : normal || dn || dist ? "psb_dp_step_dist" : "psb_dp_step_depth";
	if ((rc = check_depth(depth, fn))) return rc;
	if ((rc = check_normal(normal, fn))) return rc;
	if ((rc = check_dn(dn, fn))) return rc;
	if ((rc = check_dist(dist, fn))) return rc;
	if ((rc = check_table(exposure, false, fn))) return rc;
	if ((rc = refuse_filter3d(t, fn))) return rc;
	if (!d || !d->connected || P != d->P || !model) { set_error_msg("psb_dp_step: context not connected or built for a different P"); return PSB_ERR_ARG; }
	if ((rc = check_model(P, M, model, true))) return rc;
	for (int i = 0; i < 6; i++)
		if (P > 0 && model->param[i] != reinterpret_cast<float*>(d->base.get() + d->off_param[i])) {
			set_error_msg("psb_dp_step: the model's parameter tensors must be the arena tensors returned by psb_dp_params");
			return PSB_ERR_ARG;
		}
	const uint32_t epoch = ++d->epoch;
	t->mark(psb_trainer::NSTAGE, stream);
	// every rank's updated rows of the previous step must have landed here before this step reads the parameters
	if (epoch > 1 && P > 0 && d->world > 1)
		if ((rc = launch_wait_flags(reinterpret_cast<const uint32_t*>(d->base.get() + d->off_pflag), d->world, epoch - 1, d->status.get(), stream))) return rc;
	// render, loss, tile backward (the 9 screen-space sums per Gaussian; with a depth, consistency or distortion term also dL/dz in slot 11,
	// with a normal or consistency term 16-float rows with dL/dn in slots 12..14: the push backward below runs the variant t->pass names and
	// consumes them, where a plain one would leave them in the sink for the next step)
	// with a row: its 12 sums dL/dE and the valid flag go to the local record, which the signal behind the push backward publishes in this
	// rank's meta row (every rank's row updates only after every rank's records have landed, in exposure_apply_kernel below)
	const TableRow tr = table_row(exposure, d->exp_rec.get());
	TileBackward tb;
	if ((rc = render_loss_backward(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, depth, false, stream, tb,
	                               tr.any ? &tr.row : nullptr, nullptr, normal, dn, dist, tr.any ? &tr.rec : nullptr)) ||
	    P == 0)
		return rc;
	const TrainTensors tt = train_tensors(model, true);
	const StepHyper h = to_hyper(step);
	DpPush push;
	memset(&push, 0, sizeof(push));
	DpShard sh;
	memset(&sh, 0, sizeof(sh));
	for (int j = 0; j < d->world; j++) {
		push.inbox[j] = reinterpret_cast<float*>(d->peer[j] + d->off_inbox);
		push.meta[j] = reinterpret_cast<float*>(d->peer[j] + d->off_meta);
		push.grad_flag[j] = reinterpret_cast<uint32_t*>(d->peer[j] + d->off_gflag);
		sh.param_flag[j] = reinterpret_cast<uint32_t*>(d->peer[j] + d->off_pflag);
		for (int i = 0; i < 6; i++) sh.param[j][i] = reinterpret_cast<float*>(d->peer[j] + d->off_param[i]);
	}
	push.world = d->world; push.rank = d->rank; push.nlocal_max = d->nlocal_max; push.epoch = epoch;
	sh.inbox = reinterpret_cast<const float*>(d->base.get() + d->off_inbox);
	sh.meta = reinterpret_cast<const float*>(d->base.get() + d->off_meta);
	sh.g_rest = d->g_rest.get();
	sh.world = d->world; sh.rank = d->rank; sh.nlocal_max = d->nlocal_max; sh.nlocal = d->nlocal; sh.P = P; sh.epoch = epoch;
	// push backward (records go straight into the owners' inboxes) + signal; wait until every rank's records have landed -> Adam of
	// the owned rows, updated rows stored to every replica + signal
	if ((rc = launch_push_backward(P, tt, tb.cam, tb.geom, t->sink.get(), h, densify_stats(model, step), tb.geom.counters, (uint32_t)t->bin.count(), push, stream,
	                               t->pass, tr.any ? d->exp_rec.get() : nullptr)))
		return rc;
	t->mark(7, stream);
	t->mark(8, stream);
	if ((rc = launch_wait_flags(reinterpret_cast<const uint32_t*>(d->base.get() + d->off_gflag), d->world, epoch, d->status.get(), stream))) return rc;
	// every rank's meta row of this step has landed: each rank applies the same exposure records to its own copy of the table. It runs
	// before the shard Adam's "rows landed" signal, and a peer writes its next step's meta row only after it has seen that signal (the
	// wait at the top of its next step), so no meta row is overwritten while this kernel reads it.
	if (exposure &&
	    (rc = launch_exposure_apply(reinterpret_cast<const float*>(d->base.get() + d->off_meta) + DP_META_EXP, DP_META, d->world, exposure_table(exposure),
	                                step->beta1, step->beta2, step->eps, 1.0f / (float)d->world, d->status.get(), stream)))
		return rc;
	if ((rc = launch_shard_adam(sh, tt, h, 1.0f / (float)d->world, stream, t->event(10)))) return rc;
	t->end_stages(9, stream);
	return 0;
}

int psb_dp_step(psb_trainer* t, psb_dp* d, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, void* stream_)
{
	return psb_dp_step_depth(t, d, P, M, model, camera, background, gt_image, mask, step, out_color, radii, nullptr, stream_);
}

int psb_trainer_create(psb_trainer** out)
{
	if (!out) { set_error_msg("psb_trainer_create: null"); return PSB_ERR_ARG; }
	*out = new psb_trainer();
	return 0;
}

int psb_trainer_destroy(psb_trainer* t)
{
	delete t;
	return 0;
}

static int forward_impl(const char* fn, psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                        int sh_degree, float* out_color, int* radii, FwdPlanes planes, unsigned* pass, cudaStream_t stream)
{
	int rc;
	if (!t || !camera || !background || !out_color) { set_error_msg(std::string(fn).append(": null argument").c_str()); return PSB_ERR_ARG; }
	if ((rc = check_model(P, M, model, false))) return rc;
	if ((rc = check_filter3d(t, P, fn))) return rc;
	Scratch sc;
	Camera cam;
	t->have_loss = false;
	PassMode mode = pass_mode(t, sh_degree, false);
	mode.normals = planes.out_normal != nullptr;
	mode.moment = planes.out_depth2 != nullptr;
	if ((rc = forward_raw(t, P, M, sh_degree, model, camera, background, out_color, radii, sc, cam, stream, planes, mode, OwnPlanes{}))) return rc;
	if (pass) *pass = t->seq;
	return 0;
}

int psb_trainer_forward_normal(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background, int sh_degree,
                               float* out_color, int* radii, float* out_depth, float* out_alpha, float* out_normal, unsigned* pass, void* stream_)
{
	return forward_impl(out_normal ? "psb_trainer_forward_normal" : "psb_trainer_forward", t, P, M, model, camera, background, sh_degree, out_color, radii,
	                    FwdPlanes{out_depth, out_alpha, nullptr, out_normal, nullptr}, pass, (cudaStream_t)stream_);
}

int psb_trainer_forward_moment(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background, int sh_degree,
                               float* out_color, int* radii, float* out_depth, float* out_alpha, float* out_normal, float* out_depth2, unsigned* pass,
                               void* stream_)
{
	const char* fn = out_depth2 ? "psb_trainer_forward_moment" : out_normal ? "psb_trainer_forward_normal" : "psb_trainer_forward";
	return forward_impl(fn, t, P, M, model, camera, background, sh_degree, out_color, radii, FwdPlanes{out_depth, out_alpha, nullptr, out_normal, out_depth2},
	                    pass, (cudaStream_t)stream_);
}

int psb_trainer_forward(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background, int sh_degree,
                        float* out_color, int* radii, float* out_depth, float* out_alpha, unsigned* pass, void* stream_)
{
	return forward_impl("psb_trainer_forward", t, P, M, model, camera, background, sh_degree, out_color, radii,
	                    FwdPlanes{out_depth, out_alpha, nullptr, nullptr, nullptr}, pass, (cudaStream_t)stream_);
}

int psb_trainer_render(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background, int sh_degree,
                       float* out_color, int* radii, void* stream_)
{
	return forward_impl("psb_trainer_render", t, P, M, model, camera, background, sh_degree, out_color, radii, FwdPlanes{}, nullptr, (cudaStream_t)stream_);
}

int psb_trainer_render_depth(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background, int sh_degree,
                             float* out_color, int* radii, float* out_depth, void* stream_)
{
	return forward_impl("psb_trainer_render_depth", t, P, M, model, camera, background, sh_degree, out_color, radii,
	                    FwdPlanes{out_depth, nullptr, nullptr, nullptr, nullptr}, nullptr, (cudaStream_t)stream_);
}

static_assert(EXP_REC == PSB_EXPOSURE_RECORD, "the exposure record of the kernels is the header's");
static_assert(kScoreFracBits == PSB_CONTRIB_SUM_FRAC_BITS, "the score kernel's fixed-point unit is the header's");

int psb_trainer_contribution(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background, int sh_degree,
                             uint32_t* max_weight, uint64_t* sum_weight, float* out_color, void* stream_)
{
	const char* fn = "psb_trainer_contribution";
	int rc;
	if (!t || !camera || !background || !max_weight || !sum_weight) { set_error_msg("psb_trainer_contribution: null argument"); return PSB_ERR_ARG; }
	if (P < 0) { set_error_msg("psb_trainer_contribution: need P >= 0"); return PSB_ERR_ARG; }
	if ((rc = check_model(P, M, model, false))) return rc;
	if ((rc = check_filter3d(t, P, fn))) return rc;
	Scratch sc;
	Camera cam;
	t->have_loss = false;
	FwdPlanes planes{};
	planes.score = {max_weight, reinterpret_cast<unsigned long long*>(sum_weight)};
	return forward_raw(t, P, M, sh_degree, model, camera, background, out_color, nullptr, sc, cam, (cudaStream_t)stream_, planes,
	                   pass_mode(t, sh_degree, false), OwnPlanes{});
}

int psb_trainer_backward_pixels(psb_trainer* t, unsigned pass, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                                const psb_pixel_grads* pixel_grads, const psb_step* step, float* const* grads, void* stream_)
{
	return psb_trainer_backward_pixels_normal(t, pass, P, M, model, camera, background, pixel_grads, nullptr, step, grads, stream_);
}

int psb_trainer_backward_pixels_normal(psb_trainer* t, unsigned pass, int P, int M, const psb_model* model, const psb_camera* camera,
                                       const float* background, const psb_pixel_grads* pixel_grads, const float* dL_dnormal, const psb_step* step,
                                       float* const* grads, void* stream_)
{
	return psb_trainer_backward_pixels_moment(t, pass, P, M, model, camera, background, pixel_grads, dL_dnormal, nullptr, step, grads, stream_);
}

int psb_trainer_backward_pixels_moment(psb_trainer* t, unsigned pass, int P, int M, const psb_model* model, const psb_camera* camera,
                                       const float* background, const psb_pixel_grads* pixel_grads, const float* dL_dnormal, const float* dL_ddepth2,
                                       const psb_step* step, float* const* grads, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	int rc;
	const bool adam = grads == nullptr;
	if (!t || !camera || !background || !pixel_grads || !step) { set_error_msg("psb_trainer_backward_pixels: null argument"); return PSB_ERR_ARG; }
	if (!pixel_grads->dL_dcolor) { set_error_msg("psb_trainer_backward_pixels: dL_dcolor is required"); return PSB_ERR_ARG; }
	if (pass == 0 || pass != t->seq || t->pass.D < 0) {
		set_error_msg("psb_trainer_backward_pixels: `pass` is not the context's latest forward pass (or the arena was regrown since)");
		return PSB_ERR_ARG;
	}
	if (P != t->carved.P || camera->width != t->carved.W || camera->height != t->carved.H || step->sh_degree != t->pass.D) {
		set_error_msg("psb_trainer_backward_pixels: P, the image size and step->sh_degree must be those of the forward pass");
		return PSB_ERR_ARG;
	}
	if (t->pass.det != t->deterministic) {
		set_error_msg("psb_trainer_backward_pixels: the deterministic mode changed since the forward pass");
		return PSB_ERR_ARG;
	}
	if (t->pass.aa != t->antialiasing) {
		set_error_msg("psb_trainer_backward_pixels: the anti-aliasing mode changed since the forward pass");
		return PSB_ERR_ARG;
	}
	if (t->pass.f3d != t->filter3d) {
		set_error_msg("psb_trainer_backward_pixels: the 3D filter changed since the forward pass");
		return PSB_ERR_ARG;
	}
	if (dL_dnormal && !t->pass.normals) {
		set_error_msg("psb_trainer_backward_pixels_normal: dL_dnormal needs a pass that rendered the normal plane (psb_trainer_forward_normal)");
		return PSB_ERR_ARG;
	}
	if (dL_ddepth2 && !t->pass.moment) {
		set_error_msg("psb_trainer_backward_pixels_moment: dL_ddepth2 needs a pass that rendered the second depth moment (psb_trainer_forward_moment)");
		return PSB_ERR_ARG;
	}
	if (step->step < 1) { set_error_msg("psb_trainer_backward_pixels: step >= 1 required"); return PSB_ERR_ARG; }
	if ((rc = check_model(P, M, model, adam))) return rc;
	if (!adam && (rc = check_grads(grads, P, "psb_trainer_backward_pixels"))) return rc;
	t->have_loss = false;
	t->mark(5, stream);   // stage "loss": the caller's, between the two calls
	if (P == 0) return 0;
	const Scratch sc = carve_scratch(t, P, camera->width, camera->height);
	const Camera cam = to_camera(camera);
	// (a moment gradient leaves 2 z dL/dM in slot 11: the per-Gaussian stage consumes dL/dz)
	t->pass.depth = pixel_grads->dL_ddepth != nullptr || dL_ddepth2 != nullptr;
	t->pass.normal = dL_dnormal != nullptr;
	if ((rc = tile_backward(t, P, sc, cam, background, pixel_grads->dL_dcolor,
	                        BwdPlanes{pixel_grads->dL_ddepth, nullptr, pixel_grads->dL_dalpha, nullptr, dL_dnormal, dL_ddepth2, nullptr}, stream)))
		return rc;
	GradSegments gs{};
	if (!adam)
		for (int i = 0; i < 6; i++) gs.g[i] = grads[i];
	rc = launch_fused_backward(adam, 0, P, train_tensors(model, adam), cam, sc.geom, t->sink.get(), t->seeds.get(), to_hyper(step), gs, densify_stats(model, step),
	                           sc.geom.counters, (uint32_t)t->bin.count(), stream, t->event(7), adam ? model->adam_live : nullptr, t->pass, reg_coef(t->pass, P));
	t->end_stages(8, stream);
	return rc;
}

int psb_trainer_step(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                     const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, void* stream_)
{
	return psb_trainer_step_depth(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, nullptr, stream_);
}

int psb_trainer_step_depth(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                           const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, const psb_depth* depth,
                           void* stream_)
{
	return psb_trainer_step_exposure(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, depth, nullptr, stream_);
}

int psb_trainer_step_exposure(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                              const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, const psb_depth* depth,
                              const psb_exposure* exposure, void* stream_)
{
	return psb_trainer_step_normal(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, depth, exposure, nullptr, stream_);
}

int psb_trainer_step_normal(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                            const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, const psb_depth* depth,
                            const psb_exposure* exposure, const psb_normal* normal, void* stream_)
{
	return psb_trainer_step_dn(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, depth, exposure, normal, nullptr, stream_);
}

int psb_trainer_step_dn(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                        const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, const psb_depth* depth,
                        const psb_exposure* exposure, const psb_normal* normal, const psb_dn* dn, void* stream_)
{
	return psb_trainer_step_dist(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, depth, exposure, normal, dn, nullptr,
	                             stream_);
}

int psb_trainer_step_dist(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                          const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, const psb_depth* depth,
                          const psb_exposure* exposure, const psb_normal* normal, const psb_dn* dn, const psb_dist* dist, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	int rc;
	const char* fn = dist ? "psb_trainer_step_dist"
	                 : dn ? "psb_trainer_step_dn" : normal ? "psb_trainer_step_normal" : exposure ? "psb_trainer_step_exposure" : "psb_trainer_step_depth";
	if ((rc = check_depth(depth, fn))) return rc;
	if ((rc = check_exposure(exposure, true, nullptr, fn))) return rc;
	if ((rc = check_normal(normal, fn))) return rc;
	if ((rc = check_dn(dn, fn))) return rc;
	if ((rc = check_dist(dist, fn))) return rc;
	TileBackward tb;
	if ((rc = render_loss_backward(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, depth, true, stream, tb, exposure,
	                               nullptr, normal, dn, dist)) ||
	    P == 0)
		return rc;
	rc = launch_fused_backward(true, 0, P, train_tensors(model, true), tb.cam, tb.geom, t->sink.get(), t->seeds.get(), to_hyper(step), GradSegments{},
	                           densify_stats(model, step), tb.geom.counters, (uint32_t)t->bin.count(), stream, t->event(7), model->adam_live, t->pass, reg_coef(t->pass, P));
	t->end_stages(8, stream);
	return rc;
}

int psb_adam_live_rebuild(int P, const psb_model* model, void* stream_)
{
	int rc;
	if ((rc = check_model(P, 16, model, true))) return rc;
	if (P > 0 && !model->adam_live) { set_error_msg("psb_adam_live_rebuild: model->adam_live is NULL"); return PSB_ERR_ARG; }
	return launch_adam_live_rebuild(P, train_tensors(model, true), model->adam_live, (cudaStream_t)stream_);
}

// The gradient-mode built-in step behind psb_trainer_backward_dist and psb_trainer_backward_table, its arguments checked: the raw-parameter
// gradients -> grads, dL/dE -> exposure_grad or the record.
static int backward_flat(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background, const float* gt_image,
                         const float* mask, const psb_step* step, float* out_color, int* radii, float* const* grads, const psb_depth* depth,
                         const psb_exposure* exposure, float* exposure_grad, const psb_normal* normal, const psb_dn* dn, const psb_dist* dist,
                         const ExposureRecordOut* record, cudaStream_t stream)
{
	int rc;
	TileBackward tb;
	if ((rc = render_loss_backward(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, depth, false, stream, tb, exposure,
	                               exposure_grad, normal, dn, dist, record)) ||
	    P == 0)
		return rc;
	GradSegments gs;
	for (int i = 0; i < 6; i++) gs.g[i] = grads[i];
	rc = launch_fused_backward(false, 0, P, train_tensors(model, false), tb.cam, tb.geom, t->sink.get(), t->seeds.get(), to_hyper(step), gs, densify_stats(model, step),
	                           tb.geom.counters, (uint32_t)t->bin.count(), stream, t->event(7), nullptr, t->pass, reg_coef(t->pass, P));
	t->end_stages(8, stream);
	return rc;
}

// A table whose rank trains no row this step still writes its record, with valid = 0 (all zeros), for the hosts' gather.
static int clear_record(const psb_exposure_table* e, const TableRow& tr, cudaStream_t stream)
{
	if (e && !tr.any) PSB_CUDA_OK(cudaMemsetAsync(e->record, 0, EXP_REC * sizeof(float), stream));
	return 0;
}

int psb_trainer_backward_depth(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                               const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, float* const* grads,
                               const psb_depth* depth, void* stream_)
{
	return psb_trainer_backward_exposure(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, grads, depth, nullptr, nullptr,
	                                     stream_);
}

int psb_trainer_backward_exposure(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                                  const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, float* const* grads,
                                  const psb_depth* depth, const psb_exposure* exposure, float* exposure_grad, void* stream_)
{
	return psb_trainer_backward_dist(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, grads, depth, exposure, exposure_grad,
	                                 nullptr, nullptr, nullptr, stream_);
}

int psb_trainer_backward_dist(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                              const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, float* const* grads,
                              const psb_depth* depth, const psb_exposure* exposure, float* exposure_grad, const psb_normal* normal, const psb_dn* dn,
                              const psb_dist* dist, void* stream_)
{
	int rc;
	const bool terms = normal || dn || dist;
	if ((rc = check_depth(depth, terms ? "psb_trainer_backward_dist" : exposure ? "psb_trainer_backward_exposure" : "psb_trainer_backward_depth"))) return rc;
	if ((rc = check_exposure(exposure, false, exposure_grad, terms ? "psb_trainer_backward_dist" : "psb_trainer_backward_exposure"))) return rc;
	if ((rc = check_normal(normal, "psb_trainer_backward_dist"))) return rc;
	if ((rc = check_dn(dn, "psb_trainer_backward_dist"))) return rc;
	if ((rc = check_dist(dist, "psb_trainer_backward_dist"))) return rc;
	if ((rc = check_grads(grads, P, terms ? "psb_trainer_backward_dist" : "psb_trainer_backward"))) return rc;
	return backward_flat(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, grads, depth, exposure, exposure ? exposure_grad : nullptr,
	                     normal, dn, dist, nullptr, (cudaStream_t)stream_);
}

int psb_trainer_backward_table(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                               const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, float* const* grads,
                               const psb_depth* depth, const psb_normal* normal, const psb_dn* dn, const psb_dist* dist,
                               const psb_exposure_table* exposure, void* stream_)
{
	int rc;
	const char* fn = "psb_trainer_backward_table";
	if ((rc = check_depth(depth, fn))) return rc;
	if ((rc = check_normal(normal, fn))) return rc;
	if ((rc = check_dn(dn, fn))) return rc;
	if ((rc = check_dist(dist, fn))) return rc;
	if ((rc = check_table(exposure, true, fn))) return rc;
	if ((rc = check_grads(grads, P, fn))) return rc;
	const TableRow tr = table_row(exposure, exposure ? exposure->record : nullptr);
	if ((rc = backward_flat(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, grads, depth, tr.any ? &tr.row : nullptr, nullptr,
	                        normal, dn, dist, tr.any ? &tr.rec : nullptr, (cudaStream_t)stream_)))
		return rc;
	return clear_record(exposure, tr, (cudaStream_t)stream_);
}

int psb_trainer_backward(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                         const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, float* const* grads,
                         void* stream_)
{
	return psb_trainer_backward_depth(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, grads, nullptr, stream_);
}

int psb_trainer_backward_begin_depth(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                                     const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii,
                                     const psb_depth* depth, void* stream_)
{
	return psb_trainer_backward_begin_dist(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, depth, nullptr, nullptr, nullptr,
	                                       stream_);
}

int psb_trainer_backward_begin_dist(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                                    const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii,
                                    const psb_depth* depth, const psb_normal* normal, const psb_dn* dn, const psb_dist* dist, void* stream_)
{
	return psb_trainer_backward_begin_table(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, depth, normal, dn, dist, nullptr,
	                                        stream_);
}

int psb_trainer_backward_begin_table(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                                     const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii,
                                     const psb_depth* depth, const psb_normal* normal, const psb_dn* dn, const psb_dist* dist,
                                     const psb_exposure_table* exposure, void* stream_)
{
	int rc;
	const char* fn = exposure ? "psb_trainer_backward_begin_table" : normal || dn || dist ? "psb_trainer_backward_begin_dist" : "psb_trainer_backward_begin_depth";
	if ((rc = check_depth(depth, fn))) return rc;
	if ((rc = check_normal(normal, fn))) return rc;
	if ((rc = check_dn(dn, fn))) return rc;
	if ((rc = check_dist(dist, fn))) return rc;
	if ((rc = check_table(exposure, true, fn))) return rc;
	if ((rc = refuse_filter3d(t, fn))) return rc;
	// recorded whether or not the call below succeeds (render_loss_backward records the same rows again): dL/dz in slot 11 with a depth,
	// consistency or distortion term, 16-float rows with dL/dn with a normal or consistency term. The variants that read them give the
	// plain result on rows without those gradients.
	if (t) {
		t->pass = pass_mode(t, -1, (depth && depth->gt_depth) || dn || (dist && dist->lambda_dist > 0.f));
		t->pass.normal = (normal && normal->gt_normal) || dn;
	}
	const TableRow tr = table_row(exposure, exposure ? exposure->record : nullptr);
	TileBackward tb;
	if ((rc = render_loss_backward(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, depth, false, (cudaStream_t)stream_, tb,
	                               tr.any ? &tr.row : nullptr, nullptr, normal, dn, dist, tr.any ? &tr.rec : nullptr)))
		return rc;
	return clear_record(exposure, tr, (cudaStream_t)stream_);
}

int psb_exposure_apply(int world, const float* records, const psb_exposure_table* table, const psb_step* step, float grad_scale, void* stream_)
{
	int rc;
	if (world < 1 || world > DP_MAX_WORLD || !records || !table || !step) {
		set_error_msg("psb_exposure_apply: need 1 <= world <= 8, records, a table and a step");
		return PSB_ERR_ARG;
	}
	if ((rc = check_table(table, false, "psb_exposure_apply"))) return rc;
	if (!std::isfinite(grad_scale)) { set_error_msg("psb_exposure_apply: grad_scale must be finite"); return PSB_ERR_ARG; }
	return launch_exposure_apply(records, EXP_REC, world, exposure_table(table), step->beta1, step->beta2, step->eps, grad_scale, nullptr,
	                             (cudaStream_t)stream_);
}

int psb_trainer_backward_begin(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const float* background,
                               const float* gt_image, const float* mask, const psb_step* step, float* out_color, int* radii, void* stream_)
{
	return psb_trainer_backward_begin_depth(t, P, M, model, camera, background, gt_image, mask, step, out_color, radii, nullptr, stream_);
}

int psb_trainer_backward_slab(psb_trainer* t, int P, int M, const psb_model* model, const psb_camera* camera, const psb_step* step, int first,
                              int count, float* const* grads, void* stream_)
{
	int rc;
	if (!t || !camera || !step || !grads || t->carved.P != P) { set_error_msg("psb_trainer_backward_slab: bad argument / no matching backward_begin"); return PSB_ERR_ARG; }
	if ((rc = check_model(P, M, model, false))) return rc;
	if ((rc = refuse_filter3d(t, "psb_trainer_backward_slab"))) return rc;
	if (first < 0 || count < 0 || first + count > P || (first % 128) != 0) { set_error_msg("psb_trainer_backward_slab: slab must start at a multiple of 128"); return PSB_ERR_ARG; }
	if (count == 0) return 0;
	if ((rc = check_grads(grads, count, "psb_trainer_backward_slab"))) return rc;
	// a _begin_dist that failed before its pass made the 16-float rows it recorded: there is nothing of that pass to read
	if (t->pass.normal && t->sink.count() < (size_t)P * 16) { set_error_msg("psb_trainer_backward_slab: no matching backward_begin"); return PSB_ERR_ARG; }
	const GeomState geom = carve_scratch(t, P, t->carved.W, t->carved.H).geom;
	GradSegments gs;
	for (int i = 0; i < 6; i++) gs.g[i] = grads[i];
	return launch_fused_backward(false, first, first + count, train_tensors(model, false), to_camera(camera), geom, t->sink.get(), t->seeds.get(), to_hyper(step), gs,
	                             densify_stats(model, step), geom.counters, (uint32_t)t->bin.count(), (cudaStream_t)stream_, nullptr, nullptr, t->pass, reg_coef(t->pass, P));
}

int psb_adam_update(int P, int M, const psb_model* model, float* const* grads, const psb_step* step, float grad_scale, void* stream_)
{
	int rc;
	if ((rc = check_model(P, M, model, true))) return rc;
	if (!grads || !step || step->step < 1) { set_error_msg("psb_adam_update: bad argument"); return PSB_ERR_ARG; }
	const StepHyper h = to_hyper(step);
	for (int i = 0; i < 6; i++)
		if ((rc = launch_adam((size_t)P * row_floats(i), model->param[i], model->exp_avg[i], model->exp_avg_sq[i], grads[i], step->lr[i], h, grad_scale,
		                      (cudaStream_t)stream_)))
			return rc;
	return 0;
}

int psb_adam_flat(size_t n, float* param, float* exp_avg, float* exp_avg_sq, const float* grad, float lr, const psb_step* step,
                  float grad_scale, void* stream_)
{
	if (!step || step->step < 1 || (n > 0 && (!param || !exp_avg || !exp_avg_sq || !grad))) { set_error_msg("psb_adam_flat: bad argument"); return PSB_ERR_ARG; }
	const StepHyper h = to_hyper(step);
	return launch_adam(n, param, exp_avg, exp_avg_sq, grad, lr, h, grad_scale, (cudaStream_t)stream_);
}

static int result_impl(psb_trainer* t, float* out, int n_out, int* num_rendered, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	if (!t || t->carved.P < 0) { set_error_msg("psb_trainer_result: no step has run"); return PSB_ERR_ARG; }
	PSB_CUDA_OK(cudaEventSynchronize(t->readback));
	uint32_t* const h_count = t->h_count.get();
	const uint32_t n = t->carved.P > 0 ? h_count[0] : 0;
	if (num_rendered) *num_rendered = (int)n;
	const uint32_t n_ovf = t->carved.P > 0 ? h_count[1] : 0;
	if (n_ovf > 0) {
		// One or more views since the last collection needed more instances than the binning arena holds: those calls were
		// no-ops on the model (fused step) / contributed zero gradients (data-parallel modes). The record is sticky on the device,
		// so a queued overflow is reported here even when later steps fitted. Grow the arena (the remaining kernels may still be
		// in flight: drain first), clear the record, tell the caller which call it was.
		PSB_CUDA_OK(cudaStreamSynchronize(stream));
		PSB_CUDA_OK(cudaDeviceSynchronize());
		uint32_t rec[3];
		PSB_CUDA_OK(cudaMemcpy(rec, t->ovf.get(), sizeof(rec), cudaMemcpyDeviceToHost));
		t->ovf_count = rec[0]; t->ovf_first = rec[1];
		const uint32_t init[4] = {0u, 0xFFFFFFFFu, 0u, 0u};
		PSB_CUDA_OK(cudaMemcpy(t->ovf.get(), init, sizeof(init), cudaMemcpyHostToDevice));
		h_count[1] = 0;
		t->pass.D = -1;   // the scratch of the last pass is gone: no psb_trainer_backward_pixels for it
		const cudaError_t e = t->bin.grow((size_t)(rec[2] * 1.25) + (1u << 16), Fit::exact, false, stream);
		if (e != cudaSuccess) {
			t->carved = {};   // no binning chunk: nothing may read the last pass's scratch
			set_error("psb_trainer_result: growing the binning arena", e, __FILE__, __LINE__);
			return PSB_ERR_CUDA;
		}
		set_error_msg("psb_trainer: binning arena was too small for a view; it has been grown, repeat the call (psb_trainer_overflow_info says which)");
		return PSB_ERR_RETRY;
	}
	if (out && t->have_loss) {
		const double* h_sums = t->h_sums.get();
		const double inv_n = 1.0 / (3.0 * (double)t->carved.W * (double)t->carved.H);
		const float l1 = (float)(h_sums[0] * inv_n), ss = (float)(h_sums[1] * inv_n);
		const float dl1 = t->have_depth_loss ? (float)(h_sums[2] / (h_sums[3] > 1.0 ? h_sums[3] : 1.0)) : 0.f;
		const float nl1 = t->have_normal_loss ? (float)(h_sums[4] / (h_sums[5] > 1.0 ? h_sums[5] : 1.0)) : 0.f;
		const float dn = t->have_dn_loss ? (float)(h_sums[6] / (h_sums[7] > 1.0 ? h_sums[7] : 1.0)) : 0.f;
		const float dist = t->have_dist_loss ? (float)(h_sums[8] / (h_sums[9] > 1.0 ? h_sums[9] : 1.0)) : 0.f;
		out[0] = (1.0f - t->last_lambda) * l1 + t->last_lambda * (1.0f - ss);
		if (t->have_depth_loss) out[0] += t->last_lambda_depth * dl1;
		if (t->have_normal_loss) out[0] += t->last_lambda_normal * nl1;
		if (t->have_dn_loss) out[0] += t->last_lambda_dn * dn;
		if (t->have_dist_loss) out[0] += t->last_lambda_dist * dist;
		out[1] = l1;
		out[2] = ss;
		if (n_out > 3) out[3] = dl1;
		if (n_out > 4) out[4] = nl1;
		if (n_out > 5) out[5] = dn;
		if (n_out > 6) out[6] = dist;
	}
	return 0;
}

int psb_trainer_result(psb_trainer* t, float* out3, int* num_rendered, void* stream_)
{
	return result_impl(t, out3, 3, num_rendered, stream_);
}

int psb_trainer_result_depth(psb_trainer* t, float* out4, int* num_rendered, void* stream_)
{
	return result_impl(t, out4, 4, num_rendered, stream_);
}

int psb_trainer_result_normal(psb_trainer* t, float* out5, int* num_rendered, void* stream_)
{
	return result_impl(t, out5, 5, num_rendered, stream_);
}

int psb_trainer_result_dn(psb_trainer* t, float* out6, int* num_rendered, void* stream_)
{
	return result_impl(t, out6, 6, num_rendered, stream_);
}

int psb_trainer_result_dist(psb_trainer* t, float* out7, int* num_rendered, void* stream_)
{
	return result_impl(t, out7, 7, num_rendered, stream_);
}

// Parity/debug export (tests only): per pixel, the final transmittance and the Gaussian index of the last blended splat
// (-1: none) of the last step / render. List positions (n_contrib) are private — tight lists number the instances
// differently from the reference — but the splat they name is comparable with the reference's
// point_list[ranges[tile].x + n_contrib - 1] (cuda_rasterizer/forward.cu:352-365).
__global__ void export_last_splat_kernel(int W, int H, int grid_x, const uint2* __restrict__ ranges, const uint32_t* __restrict__ point_list,
                                         const uint32_t* __restrict__ n_contrib, const float* __restrict__ final_T, int* __restrict__ last_gauss,
                                         float* __restrict__ T_out)
{
	const int pix = blockIdx.x * blockDim.x + threadIdx.x;
	if (pix >= W * H) return;
	const int x = pix % W, y = pix / W;
	const uint2 r = ranges[(y / PSB_TILE_Y) * grid_x + x / PSB_TILE_X];
	const uint32_t n = n_contrib[pix];
	if (last_gauss) last_gauss[pix] = n ? (int)point_list[r.x + n - 1] : -1;
	if (T_out) T_out[pix] = final_T[pix];
}

int psb_trainer_debug_state(psb_trainer* t, int width, int height, int* last_gauss, float* final_T, int* num_rendered, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	if (!t || t->carved.P < 0 || t->carved.W != width || t->carved.H != height) { set_error_msg("psb_trainer_debug_state: no step of that size has run"); return PSB_ERR_ARG; }
	const Scratch sc = carve_scratch(t, t->carved.P, width, height);
	export_last_splat_kernel<<<(width * height + 255) / 256, 256, 0, stream>>>(width, height, tile_grid(width, height).x, sc.img.ranges,
	                                                                        sc.bin.inst[sorted_slot(width, height)], sc.img.n_contrib, sc.img.final_T,
	                                                                        last_gauss, final_T);
	PSB_LAUNCH_OK();
	if (num_rendered) {
		PSB_CUDA_OK(cudaMemcpyAsync(num_rendered, sc.geom.counters, sizeof(int), cudaMemcpyDeviceToHost, stream));
		PSB_CUDA_OK(cudaStreamSynchronize(stream));
	}
	return 0;
}

int psb_trainer_overflow_info(psb_trainer* t, unsigned* first_seq, unsigned* count, unsigned* current_seq)
{
	if (!t) { set_error_msg("psb_trainer_overflow_info: null"); return PSB_ERR_ARG; }
	if (first_seq) *first_seq = t->ovf_first;
	if (count) *count = t->ovf_count;
	if (current_seq) *current_seq = t->seq;
	return 0;
}

int psb_trainer_set_profiling(psb_trainer* t, int enable)
{
	if (!t) return PSB_ERR_ARG;
	if (enable && !t->ev_ready) {
		for (int i = 0; i <= psb_trainer::NSTAGE; i++) {
			const cudaError_t e = cudaEventCreate(&t->ev[i]);
			if (e != cudaSuccess) {   // all of them or none
				while (i-- > 0) cudaEventDestroy(t->ev[i]);
				set_error("cudaEventCreate(&t->ev[i])", e, __FILE__, __LINE__);
				return PSB_ERR_CUDA;
			}
		}
		t->ev_ready = true;
	}
	t->profiling = enable != 0;
	t->ev_recorded = false;
	return 0;
}

int psb_trainer_set_deterministic(psb_trainer* t, int enable)
{
	if (!t) { set_error_msg("psb_trainer_set_deterministic: null context"); return PSB_ERR_ARG; }
	t->deterministic = enable != 0;   // (its scratch is made by the next call that runs a pass)
	return 0;
}

int psb_trainer_set_antialiasing(psb_trainer* t, int enable)
{
	if (!t) { set_error_msg("psb_trainer_set_antialiasing: null context"); return PSB_ERR_ARG; }
	t->antialiasing = enable != 0;   // (takes effect at the next pass; the scratch does not change)
	return 0;
}

int psb_trainer_set_regularizers(psb_trainer* t, float lambda_opacity, float lambda_scale)
{
	if (!t || !std::isfinite(lambda_opacity) || !std::isfinite(lambda_scale) || lambda_opacity < 0.f || lambda_scale < 0.f) {
		set_error_msg("psb_trainer_set_regularizers: a context and finite lambdas >= 0 required");
		return PSB_ERR_ARG;
	}
	t->reg_opacity = lambda_opacity; t->reg_scale = lambda_scale;   // (take effect at the next pass)
	return 0;
}

int psb_trainer_set_filter3d(psb_trainer* t, const float* filter, int P)
{
	if (!t || (filter && P < 0)) { set_error_msg("psb_trainer_set_filter3d: a context, and P >= 0 with a filter"); return PSB_ERR_ARG; }
	t->filter3d = filter;   // (takes effect at the next pass)
	t->filter3d_P = filter ? P : 0;
	return 0;
}

int psb_trainer_inject_noise(psb_trainer* t, int P, const psb_model* model, float lr_xyz, float noise_lr, unsigned long long seed,
                             unsigned long long step, int visible_only, void* stream_)
{
	if (!t || !model || P < 0 || !std::isfinite(lr_xyz) || !std::isfinite(noise_lr) || lr_xyz < 0.f || noise_lr < 0.f) {
		set_error_msg("psb_trainer_inject_noise: a context, a model, P >= 0 and finite lr_xyz, noise_lr >= 0 required");
		return PSB_ERR_ARG;
	}
	if (t->carved.P != P) { set_error_msg("psb_trainer_inject_noise: the context's latest pass was not over P rows"); return PSB_ERR_ARG; }
	if (P == 0) return 0;
	if (!model->param[0] || !model->param[3] || !model->param[4] || !model->param[5] || (reinterpret_cast<uintptr_t>(model->param[5]) & 15)) {
		set_error_msg("psb_trainer_inject_noise: xyz, opacity, scaling and a 16-byte aligned rotation tensor required");
		return PSB_ERR_ARG;
	}
	const GeomState geom = carve_scratch(t, P, t->carved.W, t->carved.H).geom;
	return launch_position_noise(P, model->param[0], model->param[3], model->param[4], model->param[5], lr_xyz * noise_lr, seed, step,
	                             visible_only ? geom.tile_info : nullptr, geom.counters, (uint32_t)t->bin.count(), (cudaStream_t)stream_);
}

// ms[i] = time between stage boundaries i and i+1 of the last profiled step (see psb_trainer::ev), i < n; entries beyond the last
// recorded boundary are 0. Fused step: 8 stages (preprocess, depth sort, binning, render fwd, loss, render bwd, per-Gaussian
// backward kernel, f_rest Adam kernel). Data-parallel step: 9 stages (..., render bwd, push backward, wait for the ranks' records,
// owner-side Adam) and ms[9] = the wait for the previous step's rows at the start of the step. Synchronises. Returns the number of
// stages filled.
int psb_trainer_stage_times(psb_trainer* t, float* ms, int n)
{
	if (!t || !ms || n < 7 || !t->ev_recorded) { set_error_msg("psb_trainer_stage_times: no profiled step"); return PSB_ERR_ARG; }
	PSB_CUDA_OK(cudaEventSynchronize(t->ev[t->last_stage]));
	for (int i = 0; i < n; i++) ms[i] = 0.f;
	int filled = 0;
	for (int i = 0; i < t->last_stage && i < n; i++, filled++) PSB_CUDA_OK(cudaEventElapsedTime(&ms[i], t->ev[i], t->ev[i + 1]));
	if (t->last_stage == 9 && n > 9) { PSB_CUDA_OK(cudaEventElapsedTime(&ms[9], t->ev[psb_trainer::NSTAGE], t->ev[0])); filled = 10; }
	if (t->last_stage == 9 && n > 10) { PSB_CUDA_OK(cudaEventElapsedTime(&ms[10], t->ev[10], t->ev[9])); filled = 11; }   // the f_rest kernel + signal alone
	return filled;
}

int psb_loss(int height, int width, const float* image, const float* gt_image, const float* mask, float lambda_dssim, float* dL_dimage,
             float* out3_host, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	if (height <= 0 || width <= 0 || !image || !gt_image) { set_error_msg("psb_loss: bad argument"); return PSB_ERR_ARG; }
	const size_t N = (size_t)height * width;
	// stream-ordered scratch: no device-wide synchronisation
	StreamScratch<float> dmap(stream);
	StreamScratch<double> sums(stream);
	PSB_CUDA_OK(dmap.alloc(9 * N));
	if (sums.alloc(2) != cudaSuccess) { set_error_msg("psb_loss: out of device memory"); return PSB_ERR_CUDA; }
	int rc;
	if ((rc = launch_loss(height, width, image, gt_image, mask, lambda_dssim, dmap.get(), sums.get(), dL_dimage, stream, nullptr, nullptr))) return rc;
	double h[2] = {0, 0};
	cudaMemcpyAsync(h, sums.get(), sizeof(h), cudaMemcpyDeviceToHost, stream);
	if (cudaStreamSynchronize(stream) != cudaSuccess) return PSB_ERR_CUDA;
	if (out3_host) {
		const double inv_n = 1.0 / (3.0 * (double)N);
		const float l1 = (float)(h[0] * inv_n), ss = (float)(h[1] * inv_n);
		out3_host[0] = (1.0f - lambda_dssim) * l1 + lambda_dssim * (1.0f - ss);
		out3_host[1] = l1;
		out3_host[2] = ss;
	}
	return 0;
}

}  // extern "C"
