// Trainer step kernels: the per-Gaussian backward fused with the activations' backward, the Adam update of
// all 59 parameters of the Gaussian and the densification statistics — one read and one write of every
// parameter / moment, no gradient tensor in memory. Two launches per iteration:
//
//   gaussian_backward_kernel  one thread per Gaussian: screen-space sums -> gradients of the 14 small parameters
//                             + their Adam update + densification statistics + the 18-float SH gradient "seed"
//                             (latency-bound: every global load is issued at the top of the kernel, the f_rest
//                             parameter rows it has to read arrive by one TMA bulk copy per block);
//   frest_stream_kernel       Adam over the [P,15,3] SH rows (76 % of the parameter bytes), one float4 per thread,
//                             gradient = seed products; runs at the HBM copy rate.
// With the caller's live byte (MODE_ADAM_LIVE) the per-Gaussian kernel applies the f_rest Adam to the rows it staged, and
//   frest_momentum_kernel     applies it (g = 0) to the live rows it did not stage, from a list that kernel leaves.
//
// Replaces, per iteration of reference GaussianMapper::trainForOneIteration (src/gaussian_mapper.cpp:614-774):
//   computeCov2DCUDA + preprocessCUDA backward (cuda_rasterizer/backward.cu:144-396),
//   autograd through sigmoid / exp / normalize / cat (src/gaussian_model.cpp:48-71),
//   9 torch::zeros gradient tensors incl. [P,16,3] (src/rasterize_points.cu:148-157),
//   max_radii2D / addDensificationStats (gaussian_mapper.cpp:714-719, gaussian_model.cpp:817-831),
//   torch::optim::Adam::step over 6 parameter groups + zero_grad (gaussian_mapper.cpp:769-772).
#include "psb_backward.cuh"
#include "psb_train.h"
#include <cstdlib>
#include <cstdint>
#include <cstring>

namespace psb {

namespace {

constexpr int TB = 128;        // Gaussians per block
constexpr int A_MINBLOCKS = 5; // __launch_bounds__ minimum blocks per SM of gaussian_backward_kernel
constexpr int REST = kRestFloats;  // floats per f_rest row (15 coefficients x 3 channels)
constexpr int SEED = 20;       // floats per seed row: w_1..w_15 at [0..14], masked dL/dRGB at [16..18]

struct AdamCoef {
	float beta1, beta2, eps, inv_bc1, inv_bc2_sqrt;
	__host__ __device__ explicit AdamCoef(const StepHyper& h)
		: beta1(h.beta1), beta2(h.beta2), eps(h.eps), inv_bc1(h.inv_bc1), inv_bc2_sqrt(1.0f / h.bc2_sqrt) {}
};

// gaussian_backward_kernel modes
constexpr int MODE_GRADS = 0;  // dense gradients of the raw parameters -> `grads` (NCCL data-parallel path / tests)
constexpr int MODE_ADAM = 1;   // fused single-GPU step: parameters and moments updated in place
constexpr int MODE_PUSH = 2;   // NVLink data-parallel step: 80-byte gradient records pushed into the owner rank's inbox
constexpr int MODE_ADAM_LIVE = 3;  // MODE_ADAM with the caller's per-row live byte (psb_model.adam_live): rows that are neither live nor
                                   // reached by a gradient are not read beyond that byte and the visibility word
constexpr int MODE_DEPTH = 8;      // OR'd into MODE_GRADS / MODE_ADAM / MODE_ADAM_LIVE / MODE_PUSH: slot 11 of the sink row holds dL/dz (view-space depth,
                                   // render_bwd_kernel<F | BWD_DEPTH, Sink>) and joins dL/dxyz through the view matrix's z row
constexpr int MODE_AA = 16;        // OR'd into any of the above: the forward was anti-aliased (o' = o h, preprocess_fwd_kernel<true, true>), slot 7
                                   // holds dL/do'; dL/dh joins the covariance gradient and the opacity gradient is h dL/do' sigma'
constexpr int MODE_REG = 32;       // OR'd into MODE_GRADS / MODE_ADAM / MODE_ADAM_LIVE (each optionally | MODE_DEPTH | MODE_AA), not MODE_PUSH: the opacity
                                   // and scale regularisers of 3DGS-MCMC (psb_trainer_set_regularizers) join the raw gradients of the rows the
                                   // pass reached: g_opacity += reg.opacity o (1 - o), g_scaling[c] += reg.scale s_c (reg = lambda / P)
constexpr int MODE_F3D = 64;       // OR'd into MODE_GRADS / MODE_ADAM / MODE_ADAM_LIVE (each optionally | MODE_DEPTH | MODE_AA | MODE_REG), not MODE_PUSH:
                                   // the forward applied the 3D smoothing filter f3d[idx] (preprocess_fwd_kernel<true, AA, true>): the covariance is
                                   // rebuilt from s' = sqrt(s^2 + f^2), and the filter's opacity factor c joins the scale and opacity gradients
constexpr int MODE_NORMAL = 128;   // OR'd into MODE_GRADS / MODE_ADAM / MODE_ADAM_LIVE (each optionally | MODE_DEPTH | MODE_AA | MODE_REG | MODE_F3D)
                                   // and into MODE_PUSH (optionally | MODE_DEPTH | MODE_AA): the sink rows are 16 floats (render_bwd_kernel<F | BWD_NORMAL, Sink>) and
                                   // slots 12..14 hold dL/dn; the rotation gradient takes dL/dq of n = sign V r_k(q) (normal_axis_backward)

// torch::optim::Adam single-tensor update (LibTorch adam.cpp): exp_avg.mul_(b1).add_(g, 1-b1);
// exp_avg_sq.mul_(b2).addcmul_(g, g, 1-b2); denom = exp_avg_sq.sqrt()/sqrt(bc2) + eps; p.addcdiv_(exp_avg, denom, -lr/bc1).
// sqrt and the division go through the MUFU unit (rsqrt / rcp, ~1-2 ulp): 59 IEEE sqrt+div sequences per
// Gaussian would otherwise make this HBM-streaming kernel issue-bound.
__device__ __forceinline__ void adam1(float& p, float& m, float& v, float g, float lr_eff, const AdamCoef& c)
{
	m = m * c.beta1 + (1.f - c.beta1) * g;
	v = v * c.beta2 + (1.f - c.beta2) * g * g;
	const float sq = v > 0.f ? v * rsqrtf(v) : 0.f;
	const float denom = sq * c.inv_bc2_sqrt + c.eps;
	p = p - lr_eff * __fdividef(m, denom);
}

__device__ __forceinline__ void adam4(float4& p, float4& m, float4& v, const float4 g, float lr_eff, const AdamCoef& c)
{
	adam1(p.x, m.x, v.x, g.x, lr_eff, c);
	adam1(p.y, m.y, v.y, g.y, lr_eff, c);
	adam1(p.z, m.z, v.z, g.z, lr_eff, c);
	adam1(p.w, m.w, v.w, g.w, lr_eff, c);
}

// Adam over the 4 elements at p, m, v (16-byte aligned) with gradient g. A zero gradient on zero moments is an exact no-op of Adam
// (m' = v' = 0, p' = p - lr * 0 / (0 + eps) = p): such elements (Gaussians no view has reached since their moments were created) are
// neither read beyond their moments nor rewritten, and false is returned. Otherwise the moments are stored back and the new
// parameters are returned in `pp` for the caller to store.
__device__ __forceinline__ bool adam_noop(float g, float m, float v) { return g == 0.f && m == 0.f && v == 0.f; }

__device__ __forceinline__ bool adam4_unless_noop(const float* p, float* m, float* v, const float4 g, float lr_eff, const AdamCoef& c, float4& pp)
{
	float4 mm = __ldcs(reinterpret_cast<const float4*>(m)), vv = __ldcs(reinterpret_cast<const float4*>(v));
	if (adam_noop(g.x, mm.x, vv.x) && adam_noop(g.y, mm.y, vv.y) && adam_noop(g.z, mm.z, vv.z) && adam_noop(g.w, mm.w, vv.w)) return false;
	pp = __ldcs(reinterpret_cast<const float4*>(p));
	adam4(pp, mm, vv, g, lr_eff, c);
	__stcs(reinterpret_cast<float4*>(m), mm); __stcs(reinterpret_cast<float4*>(v), vv);
	return true;
}

// The 14 small parameters of one Gaussian (or their moments, or their gradients), by tensor: xyz 3 (tensor 0) | f_dc 3 (1) |
// scaling 3 (4) | opacity 1 (3) | rotation 4 (5).
struct SmallRow {
	float xyz[3], dc[3], sc[3], op;
	float4 rot;
};

__device__ __forceinline__ void load_small(SmallRow& r, float* const* ts, int idx)
{
#pragma unroll
	for (int c = 0; c < 3; c++) { r.xyz[c] = ts[0][3 * idx + c]; r.dc[c] = ts[1][3 * idx + c]; r.sc[c] = ts[4][3 * idx + c]; }
	r.op = ts[3][idx];
	r.rot = reinterpret_cast<const float4*>(ts[5])[idx];
}

__device__ __forceinline__ void store_small(float* const* ts, int idx, const SmallRow& r)
{
#pragma unroll
	for (int c = 0; c < 3; c++) { ts[0][3 * idx + c] = r.xyz[c]; ts[1][3 * idx + c] = r.dc[c]; ts[4][3 * idx + c] = r.sc[c]; }
	ts[3][idx] = r.op;
	reinterpret_cast<float4*>(ts[5])[idx] = r.rot;
}

// MODE_ADAM_LIVE: rows that are live after the step but had no f_rest row staged (hidden, out of view, or reached through dL/dz /
// dL/dn only). Their f_rest gradient is zero, but their moments still move the parameters: frest_momentum_kernel updates them.
// rows[0 .. *count) in no particular order (every row's update is independent of the others); *count is zeroed before the step.
struct MomentumList {
	uint32_t* rows;   // [P]
	uint32_t* count;
};

// any of the 14 values is non-zero
__device__ __forceinline__ bool any_nonzero(const SmallRow& r)
{
	bool nz = false;
#pragma unroll
	for (int c = 0; c < 3; c++) nz = nz || r.xyz[c] != 0.f || r.dc[c] != 0.f || r.sc[c] != 0.f;
	return nz || r.op != 0.f || r.rot.x != 0.f || r.rot.y != 0.f || r.rot.z != 0.f || r.rot.w != 0.f;
}

// any of the 28 moments is non-zero. (The order of the tests is the one that keeps the spill reloads of the fused Adam modes of
// gaussian_backward_kernel, which hold the moments across the backward, lowest.)
__device__ __forceinline__ bool any_nonzero(const SmallRow& m, const SmallRow& v)
{
	bool nz = m.op != 0.f || v.op != 0.f || m.rot.x != 0.f || m.rot.y != 0.f || m.rot.z != 0.f || m.rot.w != 0.f || v.rot.x != 0.f || v.rot.y != 0.f ||
	          v.rot.z != 0.f || v.rot.w != 0.f;
	const float* m3[3] = {m.xyz, m.dc, m.sc};
	const float* v3[3] = {v.xyz, v.dc, v.sc};
#pragma unroll
	for (int a = 0; a < 3; a++)
#pragma unroll
		for (int c = 0; c < 3; c++) nz = nz || m3[a][c] != 0.f || v3[a][c] != 0.f;
	return nz;
}

// Adam over the 14 small parameters with the gradient g * gs, each tensor at its own learning rate h.lr[i] / (1 - beta1^t)
__device__ __forceinline__ void adam_small(SmallRow& p, SmallRow& m, SmallRow& v, const SmallRow& g, float gs, const StepHyper& h, const AdamCoef& ac)
{
#pragma unroll
	for (int c = 0; c < 3; c++) {
		adam1(p.xyz[c], m.xyz[c], v.xyz[c], g.xyz[c] * gs, h.lr[0] * ac.inv_bc1, ac);
		adam1(p.dc[c], m.dc[c], v.dc[c], g.dc[c] * gs, h.lr[1] * ac.inv_bc1, ac);
		adam1(p.sc[c], m.sc[c], v.sc[c], g.sc[c] * gs, h.lr[4] * ac.inv_bc1, ac);
	}
	adam1(p.op, m.op, v.op, g.op * gs, h.lr[3] * ac.inv_bc1, ac);
	const float4 gr = make_float4(g.rot.x * gs, g.rot.y * gs, g.rot.z * gs, g.rot.w * gs);
	adam4(p.rot, m.rot, v.rot, gr, h.lr[5] * ac.inv_bc1, ac);
}

// ADAM = true : fused update (parameters and moments of the 14 small parameters updated in place).
// ADAM = false: gradients w.r.t. the RAW parameters are written to `grads` (reference tensor shapes) for the
//               data-parallel path (all-reduce between this kernel and adam_kernel).
//
// Block = 128 Gaussians, one thread each. The SH gradient of coefficient k, channel ch is w_k(dir) * dL/dRGB[ch]
// (clamp-masked): the thread leaves the 15 weights and the 3 masked colour gradients in `seeds` ([P][SEED] floats) and
// frest_stream_kernel expands them. The f_rest parameter rows the SH backward has to READ (view-direction term of
// dL/dxyz) arrive by one TMA bulk copy per block; each thread walks its own row in shared memory (row stride 45 words:
// bank-conflict free).
//
// MODE_ADAM_LIVE (contract of psb_model.adam_live: byte 0 => all 118 moments of the row are zero) reads per row first the live
// byte and the visibility word, then only what the row needs: visible rows their screen-space sums, render meta word and
// densification statistics; live rows (and rows whose sums are non-zero) their 14 small parameters and, for live rows, their 28
// moments (a row reached for the first time starts from the zero moments the contract guarantees). The f_rest rows are staged
// only for rows with non-zero sums — the only rows whose view-direction term of dL/dxyz can be non-zero — each warp copying its
// own rows with 4-byte async copies into a compacted region of s_p (one coalesced 180-byte run per row; the whole-block TMA copy
// would move every row, since nearly every block holds some live row). No seed row is written: a last phase applies the f_rest
// Adam to the staged rows (phase 2 below), and the rows that are live after this step without a staged row go to `mom` for
// frest_momentum_kernel. The live byte is set for every row that received a gradient.
//
// MODE_DEPTH: dL/dxyz += dL/dz (V[2], V[6], V[10]). A row whose only non-zero sum is slot 11 has a gradient (its parameters are loaded and
// updated, its live byte set) but no SH gradient: the view-direction term depends on dL/dRGB only, so its f_rest row is not staged.
//
// MODE_NORMAL: a row whose only non-zero sums are slots 12..14 has a gradient (the rotation's) but no SH gradient, as with MODE_DEPTH. Under
// MODE_PUSH such a row sends a record: its g_rot is non-zero.
//
// MODE_REG: `reg` is read by these instantiations only. The regularisers touch exactly the rows that have a gradient anyway (`reached`), so
// the dirty / live decisions and the memory traffic are those of the variant without it.
//
// MODE_F3D: `f3d` is read by these instantiations only, for the rows whose backward runs. With dL/ds' from the covariance chain and
// g = dL/d(o c) (slot 7, times h under AA): dL/ds_c = dL/ds'_c s_c / s'_c + o c g f^2 / (s_c s'_c^2) and dL/do = c g. The regularisers, the
// densification statistics and dL/dmean2D keep the unfiltered activations.
template <int MODE>
__global__ void __launch_bounds__(TB, A_MINBLOCKS) gaussian_backward_kernel(int first, int P, TrainTensors t, Camera cam, GeomState geom, float4* __restrict__ sink,
                                                            StepHyper h, GradSegments grads, DensifyStats st,
                                                            const uint32_t* __restrict__ counters, uint32_t capacity, float4* __restrict__ seeds,
                                                            DpPush dp, unsigned char* __restrict__ adam_live, RegCoef reg,
                                                            const float* __restrict__ f3d, MomentumList mom)
{
	constexpr bool DEPTH = (MODE & MODE_DEPTH) != 0;
	constexpr bool AA = (MODE & MODE_AA) != 0;
	constexpr bool REG = (MODE & MODE_REG) != 0;
	constexpr bool F3D = (MODE & MODE_F3D) != 0;
	constexpr bool NORMAL = (MODE & MODE_NORMAL) != 0;
	constexpr int BASE = MODE & ~(MODE_DEPTH | MODE_AA | MODE_REG | MODE_F3D | MODE_NORMAL);
	constexpr int SR = NORMAL ? 4 : 3;  // float4 lanes per sink row
	static_assert(!F3D || BASE != MODE_PUSH, "no 3D filter on the NVLink step");
	constexpr bool LIVE = BASE == MODE_ADAM_LIVE;
	constexpr bool ADAM = BASE == MODE_ADAM || LIVE;
	__shared__ __align__(128) float s_p[TB * REST];  // f_rest parameter rows of this block (TMA destination; LIVE: compacted per warp)
	__shared__ __align__(16) float s_w[TB][SEED];    // seed rows of this block (copied out 128-bit coalesced at the end; LIVE: read by
	                                                 // the f_rest Adam phase instead)
	__shared__ __align__(8) uint64_t s_bar;

	// A binning arena that turned out too small leaves the tile lists incomplete. Fused step: no-op (the host sees the
	// same counter, grows the arena and repeats the step). Data-parallel modes: this view contributes a ZERO gradient to
	// the step (every rank still takes part in the exchange, so the replicas stay identical and nobody waits forever).
	const bool overflow = counters[0] > capacity;
	if (ADAM && overflow) return;

	const int tid = threadIdx.x;
	const int base = first + blockIdx.x * TB;  // this launch covers Gaussians [first, P)
	const int rows = min(TB, P - base);
	const uint32_t row_bytes = (uint32_t)rows * REST * sizeof(float);
	const uint32_t bulk_bytes = row_bytes & ~15u;
	const int rem_floats = (int)(row_bytes & 15u) / 4;
	const size_t goff = (size_t)base * REST;

	if (!LIVE && tid == 0) {
		mbar_init(&s_bar, 1);
		mbar_fence_init();
		mbar_arrive_expect_tx(&s_bar, bulk_bytes);
		bulk_g2s(s_p, t.p[2] + goff, bulk_bytes, &s_bar);
		for (int i = 0; i < rem_floats; i++) s_p[bulk_bytes / 4 + i] = t.p[2][goff + bulk_bytes / 4 + i];  // < 16 trailing bytes (last block)
	}
	if (!LIVE) __syncthreads();  // the mbarrier must be initialised before any other thread waits on it

	const int idx = base + tid;
	const bool valid = idx < P;
	const AdamCoef ac(h);

	// ---- phase 1a: everything that does not need the staged rows
	bool visible = false;
	float3 g_xyz = make_float3(0, 0, 0), g_scale = make_float3(0, 0, 0);
	float4 g_rot = make_float4(0, 0, 0, 0);
	float g_opac = 0.f;
	float3 mean = make_float3(0, 0, 1), dc = make_float3(0, 0, 0);
	float3 dL_dcolor = make_float3(0, 0, 0);
	uint32_t clamp_bits = 0;
	// the 14 small parameters (every Gaussian needs them for its Adam update): issued up front, with the
	// screen-space sums, as one batch of independent loads — a single memory round trip instead of a chain
	SmallRow p = {{0, 0, 1}, {0, 0, 0}, {0, 0, 0}, 0.f, make_float4(1, 0, 0, 0)};
	// ... and their moments (consumed last): loaded here as well so their latency hides behind the whole backward
	SmallRow m, v;
	if (LIVE) m = v = SmallRow{};  // (a row reached for the first time starts from zero moments)
	float st_rad = 0.f, st_acc = 0.f, st_den = 0.f;
	bool was_live = false;  // LIVE: live byte before this step
	bool staged = false;    // non-zero screen-space sums (LIVE: the f_rest row is staged)
	bool reached = false;   // staged, or (DEPTH) a non-zero dL/dz: the sink row was added to and has a gradient
	int rest_slot = tid;    // this row's f_rest row in s_p
	float4 s0 = make_float4(0, 0, 0, 0), s1 = s0, s2 = s0, s3 = s0;
	uint32_t meta = 0;
	auto load_moments = [&]() { load_small(m, t.m, idx); load_small(v, t.v, idx); };
	// rows nothing was added to (culled or hidden Gaussians) are zero since the last step: only the others are re-zeroed for the next one
	auto take_sink = [&]() {
		staged = s0.x != 0.f || s0.y != 0.f || s0.w != 0.f || s1.x != 0.f || s1.z != 0.f || s1.w != 0.f || s2.x != 0.f || s2.y != 0.f || s2.z != 0.f;
		reached = staged || (DEPTH && s2.w != 0.f);
		if constexpr (NORMAL) reached = reached || s3.x != 0.f || s3.y != 0.f || s3.z != 0.f;
		if (reached) { const float4 z = make_float4(0, 0, 0, 0); sink[SR * idx] = z; sink[SR * idx + 1] = z; sink[SR * idx + 2] = z; }
		if constexpr (NORMAL) if (reached) sink[SR * idx + 3] = make_float4(0, 0, 0, 0);
	};
	if (LIVE) {
		if (valid) {
			was_live = adam_live[idx] != 0;
			visible = geom.tile_info[idx].z != 0;  // (an overflowing step has returned above)
			if (was_live) load_small(p, t.p, idx);  // (the moments are loaded after the backward: fewer registers held across it)
			if (visible) {
				if (st.enabled) { st_rad = st.max_radii2D[idx]; st_acc = st.xyz_gradient_accum[idx]; st_den = st.denom[idx]; }
				s0 = sink[SR * idx]; s1 = sink[SR * idx + 1]; s2 = sink[SR * idx + 2];
				if constexpr (NORMAL) s3 = sink[SR * idx + 3];
				meta = __float_as_uint(geom.rec[idx].q2.w);
				take_sink();  // (only visible rows were added to)
				if (reached && !was_live) load_small(p, t.p, idx);  // first gradient of this row: its moments are zero by contract, not read
				if (st.enabled) {  // (here: fewer registers held across the backward)
					st.max_radii2D[idx] = fmaxf(st_rad, (float)rec_radius(meta));
					st.xyz_gradient_accum[idx] = st_acc + sqrtf(s0.x * s0.x + s0.y * s0.y);
					st.denom[idx] = st_den + 1.0f;
				}
			}
		}
		// f_rest rows of the rows with non-zero sums -> this warp's 32-row region of s_p, compacted; the copies land while the
		// geometry backward below runs. Their f_rest moments, which phase 2 reads, are prefetched into L2 at the same time (lanes 0-2:
		// m, 3-5: v; floats 0, 32 and 44 of a 180-byte row touch each 128-byte line it spans), so that phase 2 waits on L2, not HBM.
		const int lane = tid & 31, wbase = tid & ~31;
		const uint32_t ball = __ballot_sync(0xffffffffu, staged);
		uint32_t b = ball;
		for (int r = wbase; b != 0u; r++, b &= b - 1u) {
			const size_t e = (size_t)(base + wbase + __ffs(b) - 1) * REST;
			const float* src = t.p[2] + e;
			float* dst = s_p + r * REST;
			cp_async4(dst + lane, src + lane);
			if (lane < REST - 32) cp_async4(dst + 32 + lane, src + 32 + lane);
			if (lane < 6) prefetch_l2_evict_last((lane < 3 ? t.m[2] : t.v[2]) + e + (lane % 3 == 0 ? 0 : lane % 3 == 1 ? 32 : REST - 1));
		}
		rest_slot = wbase + __popc(ball & ((1u << lane) - 1u));
	}
	if (valid) {
		uint32_t tt = 0;
		if (!LIVE) {
			if (ADAM) load_moments();
			if (st.enabled) { st_rad = st.max_radii2D[idx]; st_acc = st.xyz_gradient_accum[idx]; st_den = st.denom[idx]; }
			tt = geom.tile_info[idx].z;
			s0 = sink[SR * idx]; s1 = sink[SR * idx + 1]; s2 = sink[SR * idx + 2];
			if constexpr (NORMAL) s3 = sink[SR * idx + 3];
			meta = __float_as_uint(geom.rec[idx].q2.w);
			load_small(p, t.p, idx);
			visible = tt != 0 && !overflow;
			take_sink();
		}
		// LIVE: a visible row with zero sums has zero gradients (and may not have its parameters loaded): statistics only
		if (visible && (!LIVE || reached)) {
			// sink row: [0,1] mean2D.xy | [3,4,6] conic.xyw | [7] opacity | [8,9,10] rgb
			const float2 dL_dmean2D = make_float2(s0.x, s0.y);
			const float3 dL_dconic = make_float3(s0.w, s1.x, s1.z);
			const float dL_dopacity = s1.w;
			dL_dcolor = make_float3(s2.x, s2.y, s2.z);
			mean = make_float3(p.xyz[0], p.xyz[1], p.xyz[2]);
			dc = make_float3(p.dc[0], p.dc[1], p.dc[2]);
			const float3 sraw = make_float3(p.sc[0], p.sc[1], p.sc[2]);
			const float4 qraw = p.rot;
			const float oraw = p.op;
			clamp_bits = rec_clamp_bits(meta);
			// activations exactly as in the forward (preprocess_fwd_kernel<RAW>)
			const float3 s = make_float3(expf(sraw.x), expf(sraw.y), expf(sraw.z));
			const float qn = fmaxf(sqrtf(qraw.x * qraw.x + qraw.y * qraw.y + qraw.z * qraw.z + qraw.w * qraw.w), 1e-12f);
			const float4 q = make_float4(qraw.x / qn, qraw.y / qn, qraw.z / qn, qraw.w / qn);
			const float sig = 1.0f / (1.0f + expf(-oraw));
			float3 sf = s;  // F3D: s', the scale the forward drew
			float f2 = 0.f, f3d_c = 1.f;
			if (F3D) {
				const float f = f3d[idx];
				f2 = f * f;
				f3d_c = filter3d_widen(sf, f);
			}
			float cov3D[6], dL_dcov[6];
			cov3d_from_scale_rot(sf, 1.0f, q, cov3D);
			float aa_h = 1.f;  // AA: dL/dh = o c dL/do'
			gaussian_backward_geom<AA>(cam, mean, cov3D, dL_dmean2D, dL_dconic, g_xyz, dL_dcov, F3D ? sig * f3d_c : sig, dL_dopacity, false, &aa_h);
			float3 dL_dscale;
			float4 dL_drot;
			cov3d_backward(sf, 1.0f, q, dL_dcov, dL_dscale, dL_drot);
			if constexpr (NORMAL) {  // n_i as the forward formed it (normals_kernel): same q, raw scales and view-space mean
				const NormalAxis ax = normal_axis(q, sraw, xform4x3(mean, cam.view), cam.view);
				const float4 dq = normal_axis_backward(q, ax, make_float3(s3.x, s3.y, s3.z), cam.view);
				dL_drot.x += dq.x; dL_drot.y += dq.y; dL_drot.z += dq.z; dL_drot.w += dq.w;
			}
			if (F3D && f2 > 0.f) {  // (f = 0: s' = s and c = 1, nothing to add)
				const float k = sig * f3d_c * (AA ? aa_h * dL_dopacity : dL_dopacity) * f2;   // o c dL/d(o c) f^2
				dL_dscale.x = dL_dscale.x * (s.x / sf.x) + (k != 0.f ? k / (s.x * sf.x * sf.x) : 0.f);
				dL_dscale.y = dL_dscale.y * (s.y / sf.y) + (k != 0.f ? k / (s.y * sf.y * sf.y) : 0.f);
				dL_dscale.z = dL_dscale.z * (s.z / sf.z) + (k != 0.f ? k / (s.z * sf.z * sf.z) : 0.f);
			}
			// autograd of the activations (src/gaussian_model.cpp:48-71): exp, normalize, sigmoid
			g_scale = make_float3(dL_dscale.x * s.x, dL_dscale.y * s.y, dL_dscale.z * s.z);
			const float qd = q.x * dL_drot.x + q.y * dL_drot.y + q.z * dL_drot.z + q.w * dL_drot.w;
			g_rot = make_float4((dL_drot.x - q.x * qd) / qn, (dL_drot.y - q.y * qd) / qn, (dL_drot.z - q.z * qd) / qn, (dL_drot.w - q.w * qd) / qn);
			// dL/do = c dL/d(o c); c sits at the leaf so that f = 0 (c = 1) rounds and contracts exactly like the variant without F3D
			g_opac = (AA ? aa_h * dL_dopacity : dL_dopacity) * (F3D ? f3d_c : 1.0f) * sig * (1.0f - sig);
			if (DEPTH) {  // z = V[2] x + V[6] y + V[10] z + V[14] (column-major view matrix)
				const float dz = s2.w;
				g_xyz.x += dz * cam.view[2]; g_xyz.y += dz * cam.view[6]; g_xyz.z += dz * cam.view[10];
			}
			if (REG && reached) {
				g_opac += reg.opacity * sig * (1.0f - sig);
				g_scale.x += reg.scale * s.x; g_scale.y += reg.scale * s.y; g_scale.z += reg.scale * s.z;
			}
		}
		// every visible row counts, hidden ones included (the reference's denom counts them too)
		if (!LIVE && visible && st.enabled) {
			st.max_radii2D[idx] = fmaxf(st_rad, (float)rec_radius(meta));
			st.xyz_gradient_accum[idx] = st_acc + sqrtf(s0.x * s0.x + s0.y * s0.y);
			st.denom[idx] = st_den + 1.0f;
		}
	}

	if (LIVE) {
		cp_async_wait_all();  // this thread's copies have landed ...
		__syncwarp();         // ... and every lane's: each warp reads only its own region of s_p
	} else {
		mbar_wait(&s_bar, 0);  // f_rest rows have landed
		__syncthreads();       // (also publishes thread 0's trailing plain stores)
	}

	// ---- phase 1b: SH backward seeds; the view-direction term completes dL/dxyz
	float3 g_dc = make_float3(0, 0, 0);
	float gm[3] = {0.f, 0.f, 0.f};  // clamp-masked dL/dRGB: the f_rest gradient is w_k * gm
	{
		const float* rp = s_p + rest_slot * REST;
		float w[16];
#pragma unroll
		for (int k = 0; k < 16; k++) w[k] = 0.f;
		if (LIVE ? staged : visible) {
			const float3 campos = make_float3(cam.campos[0], cam.campos[1], cam.campos[2]);
			const float3 sh_dmean = sh_backward_t(
				h.D, mean, campos, clamp_bits, dL_dcolor,
				[&](int k, int ch) { return k == 0 ? (ch == 0 ? dc.x : (ch == 1 ? dc.y : dc.z)) : rp[3 * (k - 1) + ch]; },
				[&](int k, int ch, float g) { if (k == 0) { if (ch == 0) g_dc.x = g; else if (ch == 1) g_dc.y = g; else g_dc.z = g; } },
				w);
			g_xyz.x += sh_dmean.x; g_xyz.y += sh_dmean.y; g_xyz.z += sh_dmean.z;
			gm[0] = ((clamp_bits >> 0) & 1u) ? 0.f : dL_dcolor.x;
			gm[1] = ((clamp_bits >> 1) & 1u) ? 0.f : dL_dcolor.y;
			gm[2] = ((clamp_bits >> 2) & 1u) ? 0.f : dL_dcolor.z;
		}
		if (BASE != MODE_PUSH) {
			const int ncoef = (h.D + 1) * (h.D + 1);
#pragma unroll
			for (int k = 1; k < 16; k++) s_w[tid][k - 1] = (k < ncoef) ? w[k] : 0.f;
			s_w[tid][15] = 0.f; s_w[tid][16] = gm[0]; s_w[tid][17] = gm[1]; s_w[tid][18] = gm[2]; s_w[tid][19] = 0.f;
		}
	}
	const SmallRow g = {{g_xyz.x, g_xyz.y, g_xyz.z}, {g_dc.x, g_dc.y, g_dc.z}, {g_scale.x, g_scale.y, g_scale.z}, g_opac, g_rot};
	// the row has a gradient: one of its 14 small-parameter gradients, or one of gm (its f_rest gradient), is non-zero
	const bool gnz = any_nonzero(g) || gm[0] != 0.f || gm[1] != 0.f || gm[2] != 0.f;
	if (BASE == MODE_PUSH) {
		// gradient record of this Gaussian for its owner rank (see DpPush): the SH weights are NOT sent, the owner
		// re-evaluates w_k(dir) from its bit-identical copy of xyz and this rank's camera centre
		s_w[tid][0] = g_xyz.x; s_w[tid][1] = g_xyz.y; s_w[tid][2] = g_xyz.z;
		s_w[tid][3] = g_dc.x; s_w[tid][4] = g_dc.y; s_w[tid][5] = g_dc.z;
		s_w[tid][6] = g_opac;
		s_w[tid][7] = g_scale.x; s_w[tid][8] = g_scale.y; s_w[tid][9] = g_scale.z;
		s_w[tid][10] = g_rot.x; s_w[tid][11] = g_rot.y; s_w[tid][12] = g_rot.z; s_w[tid][13] = g_rot.w;
		s_w[tid][14] = gm[0]; s_w[tid][15] = gm[1]; s_w[tid][16] = gm[2];
		s_w[tid][17] = 0.f; s_w[tid][18] = 0.f;
		// a visible Gaussian hidden behind nearer splats receives no gradient: like an invisible one it sends nothing
		s_w[tid][19] = __uint_as_float(visible && gnz ? dp.epoch : 0u);
	}

	// ---- the 14 small parameters of this Gaussian
	bool momentum_only = false;  // LIVE: live after this step, no f_rest row staged
	if (valid) {
		// a zero gradient on zero moments is an exact no-op of Adam (see adam4_unless_noop): hidden / never-reached Gaussians are not rewritten
		bool idle = false;
		if (LIVE) {
			if (gnz && !was_live) adam_live[idx] = 1;
			idle = !(gnz || was_live);
			momentum_only = !idle && !staged;
			if (was_live) load_moments();
		} else if (ADAM) {
			idle = !(any_nonzero(g) || any_nonzero(m, v));
		}
		if (ADAM && !idle) {
			adam_small(p, m, v, g, 1.f, h, ac);
			store_small(t.p, idx, p); store_small(t.m, idx, m); store_small(t.v, idx, v);
		} else if (BASE == MODE_GRADS) {
			store_small(grads.g, idx, g);
		}
	}

	if (LIVE) {
		const int lane = tid & 31, wbase = tid & ~31;
		// momentum-only rows -> the list, one atomic per warp
		const uint32_t mball = __ballot_sync(0xffffffffu, momentum_only);
		if (mball != 0u) {
			uint32_t at = 0;
			if (lane == 0) at = atomicAdd(mom.count, (uint32_t)__popc(mball));
			at = __shfl_sync(0xffffffffu, at, 0);
			if (momentum_only) mom.rows[at + __popc(mball & ((1u << lane) - 1u))] = (uint32_t)idx;
		}
		// ---- phase 2 (LIVE): Adam over this warp's staged f_rest rows, walked as one flat array of n x 45 elements so that no lane
		// idles on a row's 13-element tail. Parameters from s_p, gradient w_k * gm[ch] from s_w, moments from global memory; a
		// per-element no-op skip gives the bits of frest_stream_kernel's per-float4 one (g = m = v = 0 leaves p unchanged). The r-th
		// staged row of the warp is that of lane __fns(sball, 0, r + 1): its seeds are that thread's s_w row, its parameters s_p's row
		// wbase + r.
		__syncwarp();  // this warp's s_w rows are written
		const uint32_t sball = __ballot_sync(0xffffffffu, staged);
		const int n = __popc(sball) * REST;
		const float lr_eff = h.lr[2] * ac.inv_bc1;
		constexpr int U = 2;  // elements per lane in flight (more raise the spills of the variants)
		for (int f0 = lane; f0 < n; f0 += 32 * U) {
			uint32_t ge[U], rl[U];  // element index in the f_rest tensors | the row's lane
			float mm[U], vv[U];
#pragma unroll
			for (int u = 0; u < U; u++) {
				const int f = f0 + 32 * u;
				if (f < n) {
					const int r = f / REST;
					rl[u] = __fns(sball, 0, r + 1);
					ge[u] = (uint32_t)(base + wbase + rl[u]) * REST + (uint32_t)(f - r * REST);
					mm[u] = __ldcs(t.m[2] + ge[u]); vv[u] = __ldcs(t.v[2] + ge[u]);
				}
			}
#pragma unroll
			for (int u = 0; u < U; u++) {
				const int f = f0 + 32 * u;
				if (f < n) {
					const int r = f / REST, e = f - r * REST, k = e / 3;
					const float* sw = s_w[wbase + rl[u]];
					const float g = sw[k] * sw[16 + (e - 3 * k)];
					if (!adam_noop(g, mm[u], vv[u])) {
						float pp = s_p[(wbase + r) * REST + e];
						adam1(pp, mm[u], vv[u], g, lr_eff, ac);
						__stcs(t.p[2] + ge[u], pp); __stcs(t.m[2] + ge[u], mm[u]); __stcs(t.v[2] + ge[u], vv[u]);
					}
				}
			}
		}
		return;
	}
	__syncthreads();

	if (BASE != MODE_PUSH) {
		// seed rows of this block -> global, 128-bit coalesced
		const float4* src = reinterpret_cast<const float4*>(&s_w[0][0]);
		float4* dst = seeds + (size_t)base * (SEED / 4);
		for (int i = tid; i < rows * (SEED / 4); i += TB) dst[i] = src[i];
		return;
	}
	// MODE_PUSH: the block's records go straight into the inbox of the rank that owns this 128-Gaussian chunk (remote
	// stores over NVLink: fire and forget, they overlap the arithmetic of the blocks still running). Rows this view does
	// not see are not sent: their stale epoch word tells the owner to count them as zero.
	{
		const int chunk = base / TB;
		const int owner = chunk % dp.world, lc = chunk / dp.world;
		float4* dst = reinterpret_cast<float4*>(dp.inbox[owner]) + ((size_t)dp.rank * dp.nlocal_max + lc) * (TB * (SEED / 4));
		const float4* src = reinterpret_cast<const float4*>(&s_w[0][0]);
		for (int i = tid; i < rows * (SEED / 4); i += TB) {
			if (__float_as_uint(s_w[i / (SEED / 4)][19]) == dp.epoch) dst[i] = src[i];
		}
		// "all my records of this step have landed": dp_signal_kernel, queued right behind this kernel, publishes the camera centre
		// and raises the flags after ONE system-scope fence (the kernel boundary orders it after every store of this grid).
	}
}

// Adam over the f_rest rows of Gaussians [first, P) (ADAM) or their gradient written out
// (!ADAM), one float4 per thread. The gradient of element (row, k, ch) is seed[row][k-1] * seed[row][16+ch].
// (MODE_ADAM_LIVE updates the f_rest rows in gaussian_backward_kernel and frest_momentum_kernel instead.)
template <bool ADAM>
__global__ void __launch_bounds__(256) frest_stream_kernel(uint32_t e_first, uint32_t e_end, float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                                                           float* __restrict__ gout, const float* __restrict__ seeds, float lr_eff, AdamCoef ac,
                                                           const uint32_t* __restrict__ counters, uint32_t capacity)
{
	if (ADAM && counters[0] > capacity) return;  // overflowing fused step: no-op (see gaussian_backward_kernel; !ADAM: the seeds are zero)
	const uint32_t e = e_first + 4u * (blockIdx.x * 256u + threadIdx.x);
	if (e >= e_end) return;
	uint32_t row = e / REST;
	int c = (int)(e - row * REST);
	const float* sd = seeds + (size_t)row * SEED;
	float g[4];
#pragma unroll
	for (int j = 0; j < 4; j++) {
		const int k = c / 3, ch = c - 3 * k;
		g[j] = sd[k] * sd[16 + ch];
		if (++c == REST) { c = 0; sd += SEED; }
	}
	if (e + 4 <= e_end) {
		if (ADAM) {
			float4 pp;
			if (adam4_unless_noop(p + e, m + e, v + e, make_float4(g[0], g[1], g[2], g[3]), lr_eff, ac, pp)) __stcs(reinterpret_cast<float4*>(p + e), pp);
		} else {
			__stcs(reinterpret_cast<float4*>(gout + e), make_float4(g[0], g[1], g[2], g[3]));
		}
	} else {  // < 4 trailing elements (P not a multiple of 4)
		for (uint32_t j = 0; e + j < e_end; j++) {
			if (ADAM) adam1(p[e + j], m[e + j], v[e + j], g[j], lr_eff, ac);
			else gout[e + j] = g[j];
		}
	}
}

// MODE_ADAM_LIVE: Adam with a zero gradient over the f_rest rows of the momentum-only rows gaussian_backward_kernel listed (see
// MomentumList), one warp per row over a fixed grid; lanes take elements lane and lane + 32 of the 45. An overflowing step is a no-op.
constexpr int MOM_THREADS = 256;
__global__ void __launch_bounds__(MOM_THREADS) frest_momentum_kernel(MomentumList mom, float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                                                                     float lr_eff, AdamCoef ac, const uint32_t* __restrict__ counters, uint32_t capacity)
{
	if (counters[0] > capacity) return;
	const uint32_t n = *mom.count;
	const int lane = threadIdx.x & 31;
	const uint32_t nwarps = gridDim.x * (MOM_THREADS / 32);
	for (uint32_t i = blockIdx.x * (MOM_THREADS / 32) + threadIdx.x / 32; i < n; i += nwarps) {
		const uint32_t e0 = mom.rows[i] * REST + lane, e1 = e0 + 32;
		const bool two = lane < REST - 32;
		float p0 = __ldcs(p + e0), m0 = __ldcs(m + e0), v0 = __ldcs(v + e0), p1 = 0.f, m1 = 0.f, v1 = 0.f;
		if (two) { p1 = __ldcs(p + e1); m1 = __ldcs(m + e1); v1 = __ldcs(v + e1); }
		if (!adam_noop(0.f, m0, v0)) {
			adam1(p0, m0, v0, 0.f, lr_eff, ac);
			__stcs(p + e0, p0); __stcs(m + e0, m0); __stcs(v + e0, v0);
		}
		if (two && !adam_noop(0.f, m1, v1)) {
			adam1(p1, m1, v1, 0.f, lr_eff, ac);
			__stcs(p + e1, p1); __stcs(m + e1, m1); __stcs(v + e1, v1);
		}
	}
}

// live[i] = any of the 118 moments of row i is non-zero (psb_adam_live_rebuild: repairs psb_model.adam_live after the moments were
// written by anything other than the fused step). One thread per row; not on the per-iteration path.
__global__ void __launch_bounds__(256) adam_live_rebuild_kernel(int P, TrainTensors t, unsigned char* __restrict__ live)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const int width[6] = {row_floats(0), row_floats(1), row_floats(2), row_floats(3), row_floats(4), row_floats(5)};
	bool nz = false;
#pragma unroll
	for (int q = 0; q < 6; q++) {
		const float* m = t.m[q] + (size_t)i * width[q];
		const float* v = t.v[q] + (size_t)i * width[q];
		for (int k = 0; k < width[q]; k++) nz = nz || m[k] != 0.f || v[k] != 0.f;
	}
	live[i] = nz ? 1 : 0;
}

// Plain Adam over one flat tensor (data-parallel path, after the gradient all-reduce). 128-bit accesses.
__global__ void __launch_bounds__(256) adam_kernel(size_t n4, float4* __restrict__ p, float4* __restrict__ m, float4* __restrict__ v,
                                                   const float4* __restrict__ g, float lr, AdamCoef c, float grad_scale)
{
	const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n4) return;
	float4 pp = p[i], mm = m[i], vv = v[i];
	const float4 gg = g[i];
	adam4(pp, mm, vv, make_float4(gg.x * grad_scale, gg.y * grad_scale, gg.z * grad_scale, gg.w * grad_scale), lr * c.inv_bc1, c);
	p[i] = pp; m[i] = mm; v[i] = vv;
}
__global__ void adam_tail_kernel(size_t start, size_t n, float* p, float* m, float* v, const float* g, float lr, AdamCoef c, float grad_scale)
{
	const size_t i = start + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) adam1(p[i], m[i], v[i], g[i] * grad_scale, lr * c.inv_bc1, c);
}


// ------------------------------------------------------------------------------------------------------------------------
// NVLink data-parallel step, owner side. After every rank's records of this epoch have landed (launch_wait_flags), the
// owner of a chunk sums the <= world records of each of its rows, applies Adam to its rows only (moments exist only on the
// owner) and writes the updated parameters into EVERY rank's parameter tensors (remote stores over NVLink): reduce-scatter,
// sharded optimizer and all-gather without a materialised reduced gradient and without a collective call.
// ------------------------------------------------------------------------------------------------------------------------

// One block per owned chunk, one thread per Gaussian: the 14 small parameters (Adam + all-gather) and the summed f_rest gradient row.
// The updated small parameters leave through shared memory: each of the five tensors' 128-row chunk is contiguous in every replica, so
// it is sent to each rank as fully coalesced 16-byte stores (a thread storing its own 3-float rows would emit 4-byte stores at a
// 12-byte stride: a third of every NVLink write packet used — measured 0.55 ms of the 1.04 ms owner stage at N = 8).
__global__ void __launch_bounds__(TB) shard_adam_small_kernel(DpShard d, TrainTensors t, StepHyper h, float grad_scale)
{
	__shared__ __align__(16) float s_g[TB * REST];
	__shared__ __align__(16) float s_out[TB * 14];   // [xyz 384 | f_dc 384 | scaling 384 | opacity 128 | rotation 512] in tensor-chunk layout
	const int tid = threadIdx.x, lc = blockIdx.x;
	const int chunk = lc * d.world + d.rank;
	const int idx = chunk * TB + tid;
	const bool valid = idx < d.P;

	SmallRow acc = {};  // summed records
	float G[REST];
#pragma unroll
	for (int i = 0; i < REST; i++) G[i] = 0.f;
	SmallRow p = {{0, 0, 1}, {0, 0, 0}, {0, 0, 0}, 0.f, make_float4(1, 0, 0, 0)};
	SmallRow m = {}, v = {};
	bool live = false;
	if (valid) {
		// every rank's epoch word of this row first (independent loads: one round trip instead of one per source)
		float4 tail[DP_MAX_WORLD];
#pragma unroll
		for (int s = 0; s < DP_MAX_WORLD; s++) {
			tail[s] = make_float4(0.f, 0.f, 0.f, 0.f);
			if (s < d.world) tail[s] = (reinterpret_cast<const float4*>(d.inbox) + (((size_t)s * d.nlocal_max + lc) * TB + tid) * (DP_REC / 4))[4];
		}
		load_small(m, t.m, idx);
		load_small(v, t.v, idx);
		load_small(p, t.p, idx);
		const float3 pos = make_float3(p.xyz[0], p.xyz[1], p.xyz[2]);
#pragma unroll
		for (int s = 0; s < DP_MAX_WORLD; s++) {
			if (s >= d.world || __float_as_uint(tail[s].w) != d.epoch) continue;  // rank s sent nothing for this Gaussian in this step
			const float4* r = reinterpret_cast<const float4*>(d.inbox) + (((size_t)s * d.nlocal_max + lc) * TB + tid) * (DP_REC / 4);
			const float4 r0 = r[0], r1 = r[1], r2 = r[2], r3 = r[3];
			acc.xyz[0] += r0.x; acc.xyz[1] += r0.y; acc.xyz[2] += r0.z; acc.dc[0] += r0.w;
			acc.dc[1] += r1.x; acc.dc[2] += r1.y; acc.op += r1.z; acc.sc[0] += r1.w;
			acc.sc[1] += r2.x; acc.sc[2] += r2.y; acc.rot.x += r2.z; acc.rot.y += r2.w;
			acc.rot.z += r3.x; acc.rot.w += r3.y;
			const float gm[3] = {r3.z, r3.w, tail[s].x};
			const float* mt = d.meta + DP_META * s;
			const int deg = (int)mt[3], ncoef = (deg + 1) * (deg + 1);
			float w[16];
			sh_basis(sh_dir(make_float3(pos.x - mt[0], pos.y - mt[1], pos.z - mt[2])), w);
#pragma unroll
			for (int k = 1; k < 16; k++)
#pragma unroll
				for (int ch = 0; ch < 3; ch++) G[3 * (k - 1) + ch] += (k < ncoef ? w[k] : 0.f) * gm[ch];
		}
		// zero gradient on zero moments = an exact no-op of Adam: nothing to update (hidden / never-reached Gaussians)
		live = any_nonzero(m, v) || any_nonzero(acc);
		if (live) {
			adam_small(p, m, v, acc, grad_scale, h, AdamCoef(h));
			store_small(t.m, idx, m); store_small(t.v, idx, v);
		}
	}
	// the block's (updated or unchanged) small parameters in tensor-chunk layout
#pragma unroll
	for (int c = 0; c < 3; c++) { s_out[3 * tid + c] = p.xyz[c]; s_out[384 + 3 * tid + c] = p.dc[c]; s_out[768 + 3 * tid + c] = p.sc[c]; }
	s_out[1152 + tid] = p.op;
	reinterpret_cast<float4*>(s_out + 1280)[tid] = p.rot;
	// summed f_rest gradient row -> local scratch (coalesced through shared memory; row stride 45 words is conflict-free)
#pragma unroll
	for (int i = 0; i < REST; i++) s_g[tid * REST + i] = G[i] * grad_scale;
	const bool any_live = __syncthreads_or(live);
	float4* dst = reinterpret_cast<float4*>(d.g_rest + (size_t)lc * (TB * REST));
	const float4* src = reinterpret_cast<const float4*>(s_g);
	for (int i = tid; i < TB * REST / 4; i += TB) dst[i] = src[i];
	// all-gather by remote stores: every replica (this one included) receives the chunk of each tensor as coalesced 16-byte stores.
	// Destinations are visited starting at rank + 1, so ranks running in step aim at different receivers. A chunk in which no row moved
	// (all hidden / never reached) is not sent at all.
	if (any_live) {
		const int rows = min(TB, d.P - chunk * TB);
		const int tsel[5] = {0, 1, 4, 3, 5}, width[5] = {3, 3, 3, 1, 4}, soff[5] = {0, 384, 768, 1152, 1280};
		for (int jj = 0; jj < d.world; jj++) {
			const int j = (d.rank + 1 + jj) % d.world;
#pragma unroll
			for (int q = 0; q < 5; q++) {
				const int n = rows * width[q];   // floats of this tensor's chunk; the chunk starts 16-byte aligned (128 rows x width x 4 B)
				float* gdst = d.param[j][tsel[q]] + (size_t)chunk * TB * width[q];
				const float* ssrc = s_out + soff[q];
				for (int i = tid; i < n / 4; i += TB) reinterpret_cast<float4*>(gdst)[i] = reinterpret_cast<const float4*>(ssrc)[i];
				if (tid < (n & 3)) gdst[(n & ~3) + tid] = ssrc[(n & ~3) + tid];
			}
		}
	}
}

// Adam over the f_rest rows of the owned chunks, one block per chunk (5760 floats), 128-bit accesses; the updated values go
// to every rank. Rows nobody has ever seen (g = m = v = 0) are left alone: their Adam update is exactly zero.
__global__ void __launch_bounds__(256) shard_adam_frest_kernel(DpShard d, TrainTensors t, float lr_eff, AdamCoef ac)
{
	const int lc = blockIdx.x;
	const int chunk = lc * d.world + d.rank;
	const size_t e0 = (size_t)chunk * (TB * REST);
	const size_t e_end = (size_t)d.P * REST;
	float* p = t.p[2];
	float* m = t.m[2];
	float* v = t.v[2];
	const float* g = d.g_rest + (size_t)lc * (TB * REST);
	for (int i = threadIdx.x; i < TB * REST / 4; i += 256) {
		const size_t e = e0 + 4 * (size_t)i;
		if (e >= e_end) break;
		if (e + 4 <= e_end) {
			float4 pp;
			if (!adam4_unless_noop(p + e, m + e, v + e, __ldcs(reinterpret_cast<const float4*>(g + 4 * i)), lr_eff, ac, pp)) continue;
			for (int jj = 0; jj < d.world; jj++) {
				const int j = (d.rank + 1 + jj) % d.world;
				*reinterpret_cast<float4*>(d.param[j][2] + e) = pp;
			}
		} else {  // < 4 trailing elements (P * 45 not a multiple of 4)
			for (size_t k = e; k < e_end; k++) {
				float pp = p[k], mm = m[k], vv = v[k];
				adam1(pp, mm, vv, g[k - e0], lr_eff, ac);
				m[k] = mm; v[k] = vv;
				for (int j = 0; j < d.world; j++) d.param[j][2][k] = pp;
			}
		}
	}
	// "my updated rows have landed everywhere": dp_signal_kernel behind this kernel
}

// One warp, queued right behind a data kernel of the data-parallel step: lane j publishes (optionally) this rank's meta row and then
// raises this rank's epoch word on rank j. Stream order puts it after every store of the data kernel; the single system-scope fence
// orders those stores (cumulativity) before the flag for an observer on another GPU. It replaces a fence in every block of the data
// kernel because a system-scope fence per block costs microseconds while NVLink stores are in flight.
// The meta row carries this rank's exposure record (written earlier on this stream by the exposure update), or valid = 0 without one.
struct DpSignal {
	uint32_t* flag[DP_MAX_WORLD];
	float* meta[DP_MAX_WORLD];   // null: no meta row
	const float* campos;
	const float* exp_rec;        // [EXP_REC] local, or null
	int world, rank, degree;
	uint32_t epoch;
};
__global__ void dp_signal_kernel(DpSignal s)
{
	const int j = threadIdx.x;
	if (j < s.world && s.meta[j]) {
		float* mt = s.meta[j] + DP_META * s.rank;
		mt[0] = s.campos[0]; mt[1] = s.campos[1]; mt[2] = s.campos[2]; mt[3] = (float)s.degree;
		float* er = mt + DP_META_EXP;
		if (s.exp_rec) {
#pragma unroll
			for (int q = 0; q < EXP_REC; q++) er[q] = s.exp_rec[q];
		} else {
			er[0] = -1.f; er[3] = 0.f;   // id -1, not valid
		}
	}
	__threadfence_system();
	__syncwarp();
	if (j < s.world) *reinterpret_cast<volatile uint32_t*>(s.flag[j] + s.rank) = s.epoch;
}

__device__ __forceinline__ unsigned long long global_timer_ns()
{
	unsigned long long t;
	asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
	return t;
}

// One warp: lane r waits for flags[r] >= epoch (written by rank r over NVLink). Bounded: a peer that never arrives (crashed
// process) must not hang this GPU — after timeout_ns the kernel records the failure and returns.
__global__ void wait_flags_kernel(const uint32_t* flags, int world, uint32_t epoch, uint32_t* status, unsigned long long timeout_ns)
{
	const int lane = threadIdx.x;
	if (lane >= world) return;
	const volatile uint32_t* f = flags + lane;
	const unsigned long long t0 = global_timer_ns();
	while ((int32_t)(*f - epoch) < 0) {
		__nanosleep(200);
		if (global_timer_ns() - t0 > timeout_ns) { atomicExch(status, 1u); break; }
	}
	__threadfence_system();
}

// The only launch of gaussian_backward_kernel: MODE picked at run time by launch_gaussian_backward.
template <int MODE, typename... Args>
void run_gaussian_backward(int first, int P, cudaStream_t stream, Args... args)
{
	gaussian_backward_kernel<MODE><<<cdiv(P - first, TB), TB, 0, stream>>>(first, P, args...);
}

// Gaussians [first, P) in mode `mode` (MODE_GRADS, MODE_ADAM, MODE_ADAM_LIVE or MODE_PUSH, each optionally | MODE_DEPTH, | MODE_AA and
// | MODE_NORMAL; all but MODE_PUSH optionally | MODE_REG and | MODE_F3D)
int launch_gaussian_backward(int mode, int first, int P, const TrainTensors& t, const Camera& cam, const GeomState& geom, float* sink,
                             const StepHyper& h, const GradSegments& grads, const DensifyStats& st, const uint32_t* counters, uint32_t capacity,
                             float* seeds, const DpPush& dp, unsigned char* adam_live, cudaStream_t stream, const RegCoef& reg, const float* f3d,
                             const MomentumList& mom)
{
	if (P - first <= 0) return 0;
	float4* sink4 = reinterpret_cast<float4*>(sink);
	float4* seeds4 = reinterpret_cast<float4*>(seeds);
#define PSB_BACKWARD_CASE(M) \
	case M: run_gaussian_backward<M>(first, P, stream, t, cam, geom, sink4, h, grads, st, counters, capacity, seeds4, dp, adam_live, reg, f3d, mom); break
#define PSB_BACKWARD_CASE_F3D(M) PSB_BACKWARD_CASE(M); PSB_BACKWARD_CASE(M | MODE_F3D)
#define PSB_BACKWARD_CASE_REG(M) PSB_BACKWARD_CASE_F3D(M); PSB_BACKWARD_CASE_F3D(M | MODE_REG)
#define PSB_BACKWARD_CASE_NRM(M) PSB_BACKWARD_CASE_REG(M | MODE_NORMAL); PSB_BACKWARD_CASE_REG(M | MODE_NORMAL | MODE_DEPTH); \
	PSB_BACKWARD_CASE_REG(M | MODE_NORMAL | MODE_AA); PSB_BACKWARD_CASE_REG(M | MODE_NORMAL | MODE_DEPTH | MODE_AA)
	switch (mode) {
		PSB_BACKWARD_CASE_NRM(MODE_GRADS);
		PSB_BACKWARD_CASE_NRM(MODE_ADAM);
		PSB_BACKWARD_CASE_NRM(MODE_ADAM_LIVE);
		PSB_BACKWARD_CASE_REG(MODE_GRADS);
		PSB_BACKWARD_CASE_REG(MODE_ADAM);
		PSB_BACKWARD_CASE_REG(MODE_ADAM_LIVE);
		PSB_BACKWARD_CASE(MODE_PUSH);
		PSB_BACKWARD_CASE_REG(MODE_GRADS | MODE_DEPTH);
		PSB_BACKWARD_CASE_REG(MODE_ADAM | MODE_DEPTH);
		PSB_BACKWARD_CASE_REG(MODE_ADAM_LIVE | MODE_DEPTH);
		PSB_BACKWARD_CASE(MODE_PUSH | MODE_DEPTH);
		PSB_BACKWARD_CASE_REG(MODE_GRADS | MODE_AA);
		PSB_BACKWARD_CASE_REG(MODE_ADAM | MODE_AA);
		PSB_BACKWARD_CASE_REG(MODE_ADAM_LIVE | MODE_AA);
		PSB_BACKWARD_CASE(MODE_PUSH | MODE_AA);
		PSB_BACKWARD_CASE_REG(MODE_GRADS | MODE_DEPTH | MODE_AA);
		PSB_BACKWARD_CASE_REG(MODE_ADAM | MODE_DEPTH | MODE_AA);
		PSB_BACKWARD_CASE_REG(MODE_ADAM_LIVE | MODE_DEPTH | MODE_AA);
		PSB_BACKWARD_CASE(MODE_PUSH | MODE_DEPTH | MODE_AA);
		PSB_BACKWARD_CASE(MODE_PUSH | MODE_NORMAL);
		PSB_BACKWARD_CASE(MODE_PUSH | MODE_NORMAL | MODE_DEPTH);
		PSB_BACKWARD_CASE(MODE_PUSH | MODE_NORMAL | MODE_AA);
		PSB_BACKWARD_CASE(MODE_PUSH | MODE_NORMAL | MODE_DEPTH | MODE_AA);
		default: set_error_msg("launch_gaussian_backward: unknown mode"); return -1;
	}
#undef PSB_BACKWARD_CASE_NRM
#undef PSB_BACKWARD_CASE_REG
#undef PSB_BACKWARD_CASE_F3D
#undef PSB_BACKWARD_CASE
	PSB_LAUNCH_OK();
	return 0;
}

// dp_signal_kernel for `world` ranks: raises this rank's word in flag[j] of every rank j; with meta, first publishes campos, degree and
// the exposure record exp_rec (null: none)
int launch_signal(uint32_t* const* flag, float* const* meta, const float* campos, int degree, int world, int rank, uint32_t epoch,
                  cudaStream_t stream, const float* exp_rec = nullptr)
{
	DpSignal s;
	memset(&s, 0, sizeof(s));
	for (int j = 0; j < world; j++) { s.flag[j] = flag[j]; s.meta[j] = meta ? meta[j] : nullptr; }
	s.campos = campos; s.exp_rec = exp_rec; s.degree = degree; s.world = world; s.rank = rank; s.epoch = epoch;
	dp_signal_kernel<<<1, 32, 0, stream>>>(s);
	PSB_LAUNCH_OK();
	return 0;
}

}  // namespace

int launch_fused_backward(bool adam, int first, int P, const TrainTensors& t, const Camera& cam, const GeomState& geom, float* sink, float* seeds,
                          const StepHyper& h, const GradSegments& grads, const DensifyStats& st, const uint32_t* counters, uint32_t capacity,
                          cudaStream_t stream, cudaEvent_t between, unsigned char* adam_live, const PassMode& mode, const RegCoef& reg)
{
	if (P - first <= 0) return 0;
	if (!seeds) { set_error_msg("launch_fused_backward: seed scratch missing"); return -1; }
	if ((size_t)P * REST >= (size_t)UINT32_MAX - 8) { set_error_msg("psb_trainer: too many Gaussians for 32-bit element indices"); return -1; }
	DpPush nodp;
	memset(&nodp, 0, sizeof(nodp));
	unsigned char* live = adam ? adam_live : nullptr;
	const int variant = (live ? MODE_ADAM_LIVE : adam ? MODE_ADAM : MODE_GRADS) | (mode.depth ? MODE_DEPTH : 0) | (mode.aa ? MODE_AA : 0) |
	                    (reg.opacity != 0.f || reg.scale != 0.f ? MODE_REG : 0) | (mode.f3d ? MODE_F3D : 0) | (mode.normal ? MODE_NORMAL : 0);
	// LIVE writes no seed rows: the seed scratch ([P][20] floats) holds the momentum-only list instead
	const MomentumList mom = {reinterpret_cast<uint32_t*>(seeds), reinterpret_cast<uint32_t*>(seeds) + P};
	if (live) PSB_CUDA_OK(cudaMemsetAsync(mom.count, 0, sizeof(uint32_t), stream));
	int rc;
	if ((rc = launch_gaussian_backward(variant, first, P, t, cam, geom, sink, h, grads, st, counters, capacity, seeds, nodp, live, stream, reg, mode.f3d,
	                                   mom)))
		return rc;
	if (between) cudaEventRecord(between, stream);
	const AdamCoef ac(h);
	if (live) {
		int dev = 0, sms = 0;  // grid: a full SM's worth of threads on every SM (the list length is known on the device only)
		PSB_CUDA_OK(cudaGetDevice(&dev));
		PSB_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
		frest_momentum_kernel<<<sms * (2048 / MOM_THREADS), MOM_THREADS, 0, stream>>>(mom, t.p[2], t.m[2], t.v[2], h.lr[2] * ac.inv_bc1, ac, counters, capacity);
		PSB_LAUNCH_OK();
		return 0;
	}
	const uint32_t e0 = (uint32_t)first * REST, e1 = (uint32_t)P * REST;
	const unsigned gridB = (unsigned)(((size_t)(e1 - e0) + 1023) / 1024);
	if (adam) frest_stream_kernel<true><<<gridB, 256, 0, stream>>>(e0, e1, t.p[2], t.m[2], t.v[2], nullptr, seeds, h.lr[2] * ac.inv_bc1, ac, counters, capacity);
	else frest_stream_kernel<false><<<gridB, 256, 0, stream>>>(e0, e1, nullptr, nullptr, nullptr, grads.g[2], seeds, 0.f, ac, counters, capacity);
	PSB_LAUNCH_OK();
	return 0;
}

int launch_adam_live_rebuild(int P, const TrainTensors& t, unsigned char* live, cudaStream_t stream)
{
	if (P <= 0) return 0;
	adam_live_rebuild_kernel<<<cdiv(P, 256), 256, 0, stream>>>(P, t, live);
	PSB_LAUNCH_OK();
	return 0;
}

int launch_push_backward(int P, const TrainTensors& t, const Camera& cam, const GeomState& geom, float* sink, const StepHyper& h,
                         const DensifyStats& st, const uint32_t* counters, uint32_t capacity, const DpPush& dp, cudaStream_t stream,
                         const PassMode& mode, const float* exp_rec)
{
	const GradSegments nog = {};
	int rc;
	if (mode.f3d) { set_error_msg("launch_push_backward: the 3D filter is not wired into the NVLink step"); return -1; }
	if ((rc = launch_gaussian_backward(MODE_PUSH | (mode.depth ? MODE_DEPTH : 0) | (mode.aa ? MODE_AA : 0) | (mode.normal ? MODE_NORMAL : 0), 0, P, t, cam, geom, sink, h, nog, st, counters, capacity, nullptr, dp,
	                                   nullptr, stream, RegCoef{0.f, 0.f}, nullptr, MomentumList{})))
		return rc;
	return launch_signal(dp.grad_flag, dp.meta, cam.campos, h.D, dp.world, dp.rank, dp.epoch, stream, exp_rec);
}

int launch_shard_adam(const DpShard& d, const TrainTensors& t, const StepHyper& h, float grad_scale, cudaStream_t stream, cudaEvent_t between)
{
	if (d.nlocal > 0) {
		const AdamCoef ac(h);
		shard_adam_small_kernel<<<d.nlocal, TB, 0, stream>>>(d, t, h, grad_scale);
		PSB_LAUNCH_OK();
		if (between) cudaEventRecord(between, stream);
		shard_adam_frest_kernel<<<d.nlocal, 256, 0, stream>>>(d, t, h.lr[2] * ac.inv_bc1, ac);
		PSB_LAUNCH_OK();
	}
	return launch_signal(d.param_flag, nullptr, nullptr, 0, d.world, d.rank, d.epoch, stream);
}

int launch_wait_flags(const uint32_t* flags, int world, uint32_t epoch, uint32_t* status, cudaStream_t stream)
{
	static const unsigned long long timeout_ns = (unsigned long long)(getenv("PSB_DP_TIMEOUT_MS") ? atoll(getenv("PSB_DP_TIMEOUT_MS")) : 20000) * 1000000ull;
	wait_flags_kernel<<<1, 32, 0, stream>>>(flags, world, epoch, status, timeout_ns);
	PSB_LAUNCH_OK();
	return 0;
}

int launch_adam(size_t n, float* p, float* m, float* v, const float* g, float lr, const StepHyper& h, float grad_scale, cudaStream_t stream)
{
	if (n == 0) return 0;
	const AdamCoef c(h);
	const bool aligned = ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(g)) & 15) == 0;
	const size_t n4 = aligned ? n / 4 : 0;
	if (n4) {
		adam_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, stream>>>(n4, reinterpret_cast<float4*>(p), reinterpret_cast<float4*>(m), reinterpret_cast<float4*>(v),
		                                                             reinterpret_cast<const float4*>(g), lr, c, grad_scale);
		PSB_LAUNCH_OK();
	}
	if (n4 * 4 < n) {  // unaligned tensors / < 4 trailing elements: ONE scalar launch over the remainder
		adam_tail_kernel<<<(unsigned)((n - n4 * 4 + 255) / 256), 256, 0, stream>>>(n4 * 4, n, p, m, v, g, lr, c, grad_scale);
		PSB_LAUNCH_OK();
	}
	return 0;
}

}  // namespace psb
