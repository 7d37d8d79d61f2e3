// Fused densify / clone / split / prune (declared in include/psb200.h).
//
// Replaces reference GaussianModel::densifyAndPrune and everything under it (src/gaussian_model.cpp:795-815 driver,
// :763-793 clone, :716-761 split, :588-642 prunePoints, :644-714 densificationPostfix) — in the reference dozens of
// LibTorch launches, three re-materialisations of all 59 parameters + 118 Adam moments per Gaussian (cat, cat, mask-index,
// mask-index) and a blocking `.item()` — by three launches that read every surviving row ONCE and write every output row ONCE:
//
//   densify_mask_kernel     per Gaussian: the reference's three predicates evaluated on the ORIGINAL rows
//                             clone   |grad| >= tau  &&  max exp(scaling) <= percent_dense * extent              (:769-774)
//                             split   grad  >= tau  &&  max exp(scaling) >  percent_dense * extent              (:726-731)
//                             prune   sigmoid(opacity) < min_opacity || (max_screen_size && max exp(s) > 0.1 extent)  (:806-811)
//                           (the max_radii2D > max_screen_size term of :808 can never fire in the reference: densificationPostfix
//                            has just reset max_radii2D_ to zeros, :711 — reproduced by not evaluating it), composed into what
//                           survives of each row's up to four output rows {itself, its clone, split child 0, split child 1};
//                           per-block counts.
//   densify_scan_kernel     one block: exclusive scan of the block counts -> block offsets + totals (the only value the host
//                           needs: the new row count, to size the output tensors).
//   densify_scatter_kernel  per block of 128 source rows: destination rows from the scan, then every parameter / moment tensor
//                           is streamed through once (coalesced reads, run-coalesced writes). Output order = the reference's:
//                           [surviving originals | clones | split children copy 0 | split children copy 1], each in source
//                           order (cat order of :666-681 after the two prunePoints calls). New rows get zero moments (:675-676);
//                           split children get xyz = R(q) (z * exp(s)) + xyz and scaling = log(exp(s) / 1.6) (:733-738), with z
//                           either injected (tests: same numbers as the oracle) or drawn from Philox4x32-10 + Box-Muller keyed by
//                           (seed, offset, child row) — counter-based, so every data-parallel replica draws identical samples.
#include <climits>
#include <cmath>
#include <mutex>
#include <string>
#include "psb_common.cuh"
#include "../../include/psb200.h"

namespace psb {

namespace {

constexpr int DN_TB = 128;
constexpr uint32_t F_ORIG = 1u, F_CLONE = 2u, F_CHILD = 4u, F_SPLIT = 8u;

struct DensifyCfg {
	float tau, min_opacity, size_thr, ws_thr;
	int ws_prune;
};

__device__ __forceinline__ float sigmoidf(float x) { return 1.0f / (1.0f + expf(-x)); }

__global__ void __launch_bounds__(DN_TB) densify_mask_kernel(int P, const float* __restrict__ scaling, const float* __restrict__ opacity,
                                                           const float* __restrict__ accum, const float* __restrict__ denom, DensifyCfg cfg,
                                                           uint8_t* __restrict__ flags, uint32_t* __restrict__ block_counts)
{
	__shared__ uint32_t s_cnt[DN_TB / 32][4];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int i = blockIdx.x * DN_TB + tid;
	uint32_t f = 0;
	if (i < P) {
		float g = accum[i] / denom[i];
		if (isnan(g)) g = 0.0f;
		const float s0 = expf(scaling[3 * i]), s1 = expf(scaling[3 * i + 1]), s2 = expf(scaling[3 * i + 2]);
		const float smax = fmaxf(s0, fmaxf(s1, s2));
		const float act = sigmoidf(opacity[i]);
		const bool sel_c = sqrtf(__fmul_rn(g, g)) >= cfg.tau && smax <= cfg.size_thr;
		const bool sel_s = g >= cfg.tau && smax > cfg.size_thr;
		const bool prune_self = act < cfg.min_opacity || (cfg.ws_prune && smax > cfg.ws_thr);
		// children carry scaling = log(exp(s) * (1/1.6)) (ATen divides by a CPU scalar through its reciprocal); the prune test sees exp() of that
		const float inv = 1.0f / 1.6f;
		const float c0 = expf(logf(__fmul_rn(s0, inv))), c1 = expf(logf(__fmul_rn(s1, inv))), c2 = expf(logf(__fmul_rn(s2, inv)));
		const bool prune_child = act < cfg.min_opacity || (cfg.ws_prune && fmaxf(c0, fmaxf(c1, c2)) > cfg.ws_thr);
		if (!sel_s && !prune_self) f |= F_ORIG;
		if (sel_c && !prune_self) f |= F_CLONE;
		if (sel_s) f |= F_SPLIT;
		if (sel_s && !prune_child) f |= F_CHILD;
		flags[i] = (uint8_t)f;
	}
#pragma unroll
	for (int k = 0; k < 4; k++) {
		const uint32_t b = __ballot_sync(0xffffffffu, (f >> k) & 1u);
		if (lane == 0) s_cnt[warp][k] = __popc(b);
	}
	__syncthreads();
	if (tid < 4) {
		uint32_t t = 0;
#pragma unroll
		for (int w = 0; w < DN_TB / 32; w++) t += s_cnt[w][tid];
		block_counts[4 * blockIdx.x + tid] = t;
	}
}

// exclusive scan of [nblocks][4] counts by ONE block; totals[0..3] = sums
__global__ void __launch_bounds__(1024) densify_scan_kernel(int nblocks, const uint32_t* __restrict__ counts, uint32_t* __restrict__ offsets,
                                                          uint32_t* __restrict__ totals)
{
	__shared__ uint32_t s_w[32][4];
	__shared__ uint32_t s_run[4];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (tid < 4) s_run[tid] = 0;
	__syncthreads();
	for (int b0 = 0; b0 < nblocks; b0 += 1024) {
		const int b = b0 + tid;
		uint32_t v[4], inc[4];
#pragma unroll
		for (int k = 0; k < 4; k++) {
			v[k] = b < nblocks ? counts[4 * b + k] : 0u;
			inc[k] = v[k];
#pragma unroll
			for (int o = 1; o < 32; o <<= 1) {
				const uint32_t u = __shfl_up_sync(0xffffffffu, inc[k], o);
				if (lane >= o) inc[k] += u;
			}
			if (lane == 31) s_w[warp][k] = inc[k];
		}
		__syncthreads();
		uint32_t base[4];
#pragma unroll
		for (int k = 0; k < 4; k++) {
			uint32_t wb = 0;
			for (int w = 0; w < warp; w++) wb += s_w[w][k];
			base[k] = s_run[k] + wb + inc[k] - v[k];
			if (b < nblocks) offsets[4 * b + k] = base[k];
		}
		__syncthreads();
		if (tid == 1023) {
#pragma unroll
			for (int k = 0; k < 4; k++) s_run[k] = base[k] + v[k];
		}
		__syncthreads();
	}
	if (tid < 4) totals[tid] = s_run[tid];
}

// ---- Philox4x32-10 (Salmon et al. 2011), the counter-based generator cuRAND / ATen use; written out: no cuRAND dependency
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key)
{
	constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
	for (int r = 0; r < 10; r++) {
		const uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
		const uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
		ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
		key.x += W0; key.y += W1;
	}
	return ctr;
}
// three standard normals for child row j: Box-Muller on the four 32-bit words of Philox(counter = (j, 0, offset), key = seed)
__device__ __forceinline__ float3 normal3(unsigned long long seed, unsigned long long offset, uint32_t j)
{
	const uint4 r = philox4x32_10(make_uint4(j, 0u, (uint32_t)offset, (uint32_t)(offset >> 32)), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
	const float k = 2.3283064365386963e-10f;  // 2^-32
	const float u0 = ((float)r.x + 0.5f) * k, u1 = ((float)r.y + 0.5f) * k, u2 = ((float)r.z + 0.5f) * k, u3 = ((float)r.w + 0.5f) * k;
	const float ra = sqrtf(-2.0f * logf(fminf(u0, 0.99999994f))), rb = sqrtf(-2.0f * logf(fminf(u2, 0.99999994f)));
	float sa, ca, sb, cb;
	sincosf(6.283185307179586f * u1, &sa, &ca);
	sincosf(6.283185307179586f * u3, &sb, &cb);
	(void)sb;
	return make_float3(ra * ca, ra * sa, rb * cb);
}

struct DensifyTensors {
	const float* p[6]; const float* m[6]; const float* v[6];   // source [P]
	float* dp[6]; float* dm[6]; float* dv[6];                   // destination [P_new]
	const int* exist; int* dexist;                              // exist_since_iter (optional): children / clones inherit the parent's (:741, :781)
	const float* stat[3]; float* dstat[3];                      // statistics, compacted only by prunePoints (null otherwise)
};

__global__ void __launch_bounds__(DN_TB) densify_scatter_kernel(int P, DensifyTensors t, const uint8_t* __restrict__ flags,
                                                              const uint32_t* __restrict__ block_offsets, const uint32_t* __restrict__ totals,
                                                              const float* __restrict__ samples, unsigned long long seed, unsigned long long offset)
{
	__shared__ int s_dst[4][DN_TB];
	__shared__ float s_cxyz[2][DN_TB][3];
	__shared__ uint32_t s_wcnt[DN_TB / 32][4];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int base = blockIdx.x * DN_TB;
	const int rows = min(DN_TB, P - base);
	const int i = base + tid;
	const uint32_t f = i < P ? flags[i] : 0u;
	uint32_t pre[4];
#pragma unroll
	for (int k = 0; k < 4; k++) {
		const uint32_t b = __ballot_sync(0xffffffffu, (f >> k) & 1u);
		pre[k] = __popc(b & ((1u << lane) - 1u));
		if (lane == 0) s_wcnt[warp][k] = __popc(b);
	}
	__syncthreads();
	const uint32_t K0 = totals[0], K1 = totals[1], K2 = totals[2], NS = totals[3];
#pragma unroll
	for (int k = 0; k < 4; k++) {
		for (int w = 0; w < warp; w++) pre[k] += s_wcnt[w][k];
		pre[k] += block_offsets[4 * blockIdx.x + k];
	}
	s_dst[0][tid] = (f & F_ORIG) ? (int)pre[0] : -1;
	s_dst[1][tid] = (f & F_CLONE) ? (int)(K0 + pre[1]) : -1;
	s_dst[2][tid] = (f & F_CHILD) ? (int)(K0 + K1 + pre[2]) : -1;
	s_dst[3][tid] = (f & F_CHILD) ? (int)(K0 + K1 + K2 + pre[2]) : -1;
	if (f & F_CHILD) {
		// reference :733-736: samples = normal(0, exp(scaling)); new_xyz = build_rotation(rotation) @ samples + xyz
		const float4 qr = reinterpret_cast<const float4*>(t.p[5])[i];
		const float n = sqrtf(qr.x * qr.x + qr.y * qr.y + qr.z * qr.z + qr.w * qr.w);
		const float r = qr.x / n, x = qr.y / n, y = qr.z / n, z = qr.w / n;
		const float R00 = 1.f - 2.f * (y * y + z * z), R01 = 2.f * (x * y - r * z), R02 = 2.f * (x * z + r * y);
		const float R10 = 2.f * (x * y + r * z), R11 = 1.f - 2.f * (x * x + z * z), R12 = 2.f * (y * z - r * x);
		const float R20 = 2.f * (x * z - r * y), R21 = 2.f * (y * z + r * x), R22 = 1.f - 2.f * (x * x + y * y);
		const float s0 = expf(t.p[4][3 * i]), s1 = expf(t.p[4][3 * i + 1]), s2 = expf(t.p[4][3 * i + 2]);
		const float px = t.p[0][3 * i], py = t.p[0][3 * i + 1], pz = t.p[0][3 * i + 2];
#pragma unroll
		for (int c = 0; c < 2; c++) {
			const uint32_t j = (uint32_t)c * NS + pre[3];  // row of the [2 * n_split, 3] sample block (repeat({N,1}) order)
			float3 zz;
			if (samples) zz = make_float3(samples[3 * (size_t)j], samples[3 * (size_t)j + 1], samples[3 * (size_t)j + 2]);
			else zz = normal3(seed, offset, j);
			const float a = zz.x * s0, b = zz.y * s1, d = zz.z * s2;
			s_cxyz[c][tid][0] = R00 * a + R01 * b + R02 * d + px;
			s_cxyz[c][tid][1] = R10 * a + R11 * b + R12 * d + py;
			s_cxyz[c][tid][2] = R20 * a + R21 * b + R22 * d + pz;
		}
	}
	__syncthreads();

	if (i < P) {
		if (t.exist) {
			const int ex = t.exist[i];
#pragma unroll
			for (int o = 0; o < 4; o++) if (s_dst[o][tid] >= 0) t.dexist[s_dst[o][tid]] = ex;
		}
		if (t.stat[0] && s_dst[0][tid] >= 0) {
#pragma unroll
			for (int q = 0; q < 3; q++) t.dstat[q][s_dst[0][tid]] = t.stat[q][i];
		}
	}

	const float inv = 1.0f / 1.6f;
#pragma unroll
	for (int ti = 0; ti < 6; ti++) {
		const int k = row_floats(ti);
		const float* __restrict__ sp = t.p[ti] + (size_t)base * k;
		const float* __restrict__ sm = t.m[ti] + (size_t)base * k;
		const float* __restrict__ sv = t.v[ti] + (size_t)base * k;
		for (int e = tid; e < rows * k; e += DN_TB) {
			const int r = e / k, c = e - r * k;
			const int d0 = s_dst[0][r], d1 = s_dst[1][r], d2 = s_dst[2][r], d3 = s_dst[3][r];
			if (d0 < 0 && d1 < 0 && d2 < 0) continue;  // row vanishes (pruned, or a split parent whose children are pruned)
			const float pv = sp[e];
			if (d0 >= 0) {
				const size_t o = (size_t)d0 * k + c;
				t.dp[ti][o] = pv; t.dm[ti][o] = sm[e]; t.dv[ti][o] = sv[e];
			}
			if (d1 >= 0) {
				const size_t o = (size_t)d1 * k + c;
				t.dp[ti][o] = pv; t.dm[ti][o] = 0.f; t.dv[ti][o] = 0.f;
			}
			if (d2 >= 0) {
				float v0 = pv, v1 = pv;
				if (ti == 0) { v0 = s_cxyz[0][r][c]; v1 = s_cxyz[1][r][c]; }
				else if (ti == 4) { v0 = v1 = logf(__fmul_rn(expf(pv), inv)); }
				const size_t o0 = (size_t)d2 * k + c, o1 = (size_t)d3 * k + c;
				t.dp[ti][o0] = v0; t.dm[ti][o0] = 0.f; t.dv[ti][o0] = 0.f;
				t.dp[ti][o1] = v1; t.dm[ti][o1] = 0.f; t.dv[ti][o1] = 0.f;
			}
		}
	}
}

// reference GaussianModel::resetOpacity (src/gaussian_model.cpp:556-565): inverse_sigmoid(min(sigmoid(o), ones_like(...))) — the
// misplaced parenthesis makes the clamp a no-op (SURVEY §2.2 quirk 9) — and fresh (zero) Adam moments for the opacity group (:576-578)
__global__ void reset_opacity_kernel(int P, float* __restrict__ opacity, float* __restrict__ m, float* __restrict__ v)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const float a = fminf(sigmoidf(opacity[i]), 1.0f);
	opacity[i] = logf(a / (1.0f - a));
	m[i] = 0.f; v[i] = 0.f;
}

// prunePoints: flags from a byte mask
__global__ void __launch_bounds__(DN_TB) prune_mask_kernel(int P, const uint8_t* __restrict__ mask, uint8_t* __restrict__ flags, uint32_t* __restrict__ block_counts)
{
	__shared__ uint32_t s_cnt[DN_TB / 32];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int i = blockIdx.x * DN_TB + tid;
	const uint32_t f = (i < P && !mask[i]) ? F_ORIG : 0u;
	if (i < P) flags[i] = (uint8_t)f;
	const uint32_t b = __ballot_sync(0xffffffffu, f & 1u);
	if (lane == 0) s_cnt[warp] = __popc(b);
	__syncthreads();
	if (tid < 4) {
		uint32_t t = 0;
		if (tid == 0) for (int w = 0; w < DN_TB / 32; w++) t += s_cnt[w];
		block_counts[4 * blockIdx.x + tid] = t;
	}
}

// increasePcd: the n appended rows (reference src/gaussian_model.cpp:222-262)
__global__ void insert_fill_kernel(int P, int n, const float* __restrict__ points, const float* __restrict__ colors, const float* __restrict__ dist2,
                                   int iteration, DensifyTensors t)
{
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= n) return;
	const size_t d = (size_t)P + j;
	const float sc = logf(sqrtf(fmaxf(dist2[j], 0.0000001f)));
	const float a = 0.1f * 1.0f;
	const float op = logf(a / (1.0f - a));
#pragma unroll
	for (int c = 0; c < 3; c++) {
		t.dp[0][3 * d + c] = points[3 * (size_t)j + c];
		t.dp[1][3 * d + c] = (colors[3 * (size_t)j + c] - 0.5f) / kSH_C0;   // RGB2SH
		t.dp[4][3 * d + c] = sc;
	}
	for (int c = 0; c < kRestFloats; c++) t.dp[2][kRestFloats * d + c] = 0.f;
	t.dp[3][d] = op;
	reinterpret_cast<float4*>(t.dp[5])[d] = make_float4(1.f, 0.f, 0.f, 0.f);
	if (t.dexist) t.dexist[d] = iteration;
}

// ------------------------------------------------------------------------------------------------------------------------
// Depth-guided seeding (include/psb200.h, psb_seed_*): the pixels of an RGB-D keyframe that the map does not explain become new rows
// through the insert body above. Both kernels walk the stride grid, g = gv * gw + gu for the pixel (gu * stride, gv * stride); g grows
// with the raster index v * W + u, so the rank of a pixel among the selected ones is its rank in g. Counts per block of 128 grid pixels
// are [selected, holes, in front, 0], the [nblocks][4] shape densify_scan_kernel scans. No atomics: the result does not depend on the
// launch configuration.
// ------------------------------------------------------------------------------------------------------------------------
constexpr uint8_t SEED_HOLE = 1, SEED_FRONT = 2;

struct SeedGrid {
	int W, H, stride, gw, ng;   // image size, stride, grid width, grid pixels
};

struct SeedTest {
	float alpha_min, k, min_depth, max_depth;   // k = 1 - depth_rel, formed in float32 on the host
};

__global__ void __launch_bounds__(DN_TB) seed_mask_kernel(SeedGrid g, SeedTest s, const float* __restrict__ alpha, const float* __restrict__ depth,
                                                        const float* __restrict__ gt_depth, const float* __restrict__ mask,
                                                        uint8_t* __restrict__ flags, uint32_t* __restrict__ block_counts)
{
	__shared__ uint32_t s_cnt[DN_TB / 32][3];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int i = blockIdx.x * DN_TB + tid;
	uint32_t f = 0;
	if (i < g.ng) {
		const int gv = i / g.gw, gu = i - gv * g.gw;
		const size_t idx = (size_t)gv * g.stride * g.W + (size_t)gu * g.stride;
		const float G = gt_depth[idx];
		const bool valid = isfinite(G) && G > s.min_depth && G < s.max_depth && (!mask || mask[idx] != 0.f);
		const float A = alpha[idx];
		const bool hole = A < s.alpha_min;
		const bool front = A >= s.alpha_min && __fmul_rn(G, A) < __fmul_rn(s.k, depth[idx]);
		f = valid ? (hole ? SEED_HOLE : (front ? SEED_FRONT : 0u)) : 0u;
		flags[i] = (uint8_t)f;
	}
	const uint32_t b_sel = __ballot_sync(0xffffffffu, f != 0u), b_hole = __ballot_sync(0xffffffffu, f == SEED_HOLE);
	const uint32_t b_front = __ballot_sync(0xffffffffu, f == SEED_FRONT);
	if (lane == 0) { s_cnt[warp][0] = __popc(b_sel); s_cnt[warp][1] = __popc(b_hole); s_cnt[warp][2] = __popc(b_front); }
	__syncthreads();
	if (tid < 4) {
		uint32_t t = 0;
		if (tid < 3)
			for (int w = 0; w < DN_TB / 32; w++) t += s_cnt[w][tid];
		block_counts[4 * blockIdx.x + tid] = t;
	}
}

struct SeedCam {
	const float* view;       // device, column-major: R[r][c] = view[4 c + r], t[r] = view[12 + r]
	float fx, fy, half_w, half_h, scale;   // scale = stride / ((fx + fy) / 2)
};

// Rank of each selected pixel (block offset from the scan + the block's ballots), the cap test against the n of the caller, and the
// kept pixel's point, colour and dist2 at its output slot floor(k n / c). n <= c = totals[0], n > 0.
__global__ void __launch_bounds__(DN_TB) seed_emit_kernel(SeedGrid g, SeedCam cam, int n, const uint8_t* __restrict__ flags,
                                                        const uint32_t* __restrict__ block_offsets, const uint32_t* __restrict__ totals,
                                                        const float* __restrict__ gt_image, const float* __restrict__ gt_depth,
                                                        float* __restrict__ points, float* __restrict__ colors, float* __restrict__ dist2)
{
	__shared__ uint32_t s_wcnt[DN_TB / 32];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int i = blockIdx.x * DN_TB + tid;
	const bool sel = i < g.ng && flags[i] != 0;
	const uint32_t b = __ballot_sync(0xffffffffu, sel);
	if (lane == 0) s_wcnt[warp] = __popc(b);
	__syncthreads();
	if (!sel) return;
	uint64_t k = block_offsets[4 * blockIdx.x] + __popc(b & ((1u << lane) - 1u));
	for (int w = 0; w < warp; w++) k += s_wcnt[w];
	const uint64_t c = totals[0], nn = (uint64_t)n;
	const uint64_t j = k * nn / c;
	if ((k + 1) * nn / c == j) return;   // not kept
	const int gv = i / g.gw, gu = i - gv * g.gw;
	const int u = gu * g.stride, v = gv * g.stride;
	const size_t idx = (size_t)v * g.W + u, plane = (size_t)g.W * g.H;
	const float z = gt_depth[idx];
	// the inverse of the forward's projection (ndc_to_pix: pix = x / z f + W / 2 - 1 / 2): the point lands on the centre of pixel (u, v)
	const float px = ((float)u + 0.5f - cam.half_w) * z / cam.fx;
	const float py = ((float)v + 0.5f - cam.half_h) * z / cam.fy;
	const float* m = cam.view;
	const float d0 = px - m[12], d1 = py - m[13], d2 = z - m[14];
#pragma unroll
	for (int r = 0; r < 3; r++) {
		points[3 * j + r] = m[4 * r] * d0 + m[4 * r + 1] * d1 + m[4 * r + 2] * d2;   // R^T (p - t)
		colors[3 * j + r] = gt_image[r * plane + idx];
	}
	const float s = z * cam.scale;
	dist2[j] = s * s;
}

// ------------------------------------------------------------------------------------------------------------------------
// Bounded-budget densification (3DGS-MCMC, Kheradmand et al., NeurIPS 2024; gsplat's MCMCStrategy — no counterpart in the reference):
// psb_relocate moves dead rows onto live ones, psb_grow appends copies of sampled rows. Both are
//   reloc_weight_kernel   per block of 128 rows: weight o = sigmoid(opacity) of the candidates (0 for the others), inclusive prefix sum
//                         inside the block in double and in a fixed order, the block's sum and its number of dead rows;
//   reloc_scan_kernel     one block: exclusive scan of the block sums (double) and of the dead counts -> the total weight, the dead count;
//   reloc_draw_kernel     one thread per draw: u in [0, 1) -> the first row whose cumulative weight exceeds u * total (binary search),
//                         integer histogram of the picks (atomicAdd on ints: order-independent);
//   reloc_correct_kernel  per block of 128 rows: every picked row gets (o', s') for its multiplicity and zero moments, in place;
//   reloc_copy_kernel     per block of 128 targets: target row <- its (corrected) source row, zero moments and statistics.
// No float atomics anywhere: the result is bit-identical from run to run and on every data-parallel replica.
// ------------------------------------------------------------------------------------------------------------------------
constexpr int RL_MAXN = 51;   // multiplicities are clamped here (gsplat's n_max)

// C(n, k) for n, k < 51, exact in double (C(50, 25) < 2^53)
struct BinomTable {
	double c[RL_MAXN][RL_MAXN];
	constexpr BinomTable() : c()
	{
		for (int n = 0; n < RL_MAXN; n++)
			for (int k = 0; k < RL_MAXN; k++) c[n][k] = k == 0 ? 1.0 : (n == 0 || k > n ? 0.0 : c[n - 1][k - 1] + c[n - 1][k]);
	}
};
__constant__ BinomTable c_binom = BinomTable();

// A row of opacity o and scale s that stands for N co-located copies (the paper's Eq. 9, gsplat compute_relocation):
//   o' = 1 - (1 - o)^(1/N);  D = sum_{a=1..N} sum_{k=0..a-1} C(a-1, k) (-1)^k o'^(k+1) / sqrt(k+1);  s' = s o / D.
// Returns o' clamped to [min_opacity, 1 - 1e-7] and the scale factor o / D of the unclamped o'. The alternating sum cancels up to 1e4
// of its terms at N = 51, so it is formed in double (a few hundred picked rows per thousand: not on any hot path).
__device__ __forceinline__ void relocation(float o, int N, float min_opacity, float& o_new, float& scale_factor)
{
	const double od = (double)o;
	const double on = 1.0 - pow(1.0 - od, 1.0 / (double)N);
	double D = 0.0;
	for (int a = 1; a <= N; a++) {
		double pw = on, sgn = 1.0;
		for (int k = 0; k < a; k++) {
			D += c_binom.c[a - 1][k] * sgn * pw * rsqrt((double)(k + 1));
			pw *= on; sgn = -sgn;
		}
	}
	scale_factor = (float)(od / D);
	o_new = fminf(fmaxf((float)on, min_opacity), 1.0f - 1e-7f);
}

struct RelocTotals {
	double total;       // sum of the candidates' weights
	uint32_t n_dead;    // rows with sigmoid(opacity) <= min_opacity
	uint32_t pad;
};

// flags[i]: bit 0 = dead. all_rows: every row is a candidate (grow), else the alive rows (relocate)
__global__ void __launch_bounds__(DN_TB) reloc_weight_kernel(int P, const float* __restrict__ opacity, float min_opacity, int all_rows,
                                                           uint8_t* __restrict__ flags, double* __restrict__ cum, int* __restrict__ mult,
                                                           double* __restrict__ block_sum, uint32_t* __restrict__ block_dead)
{
	__shared__ double s_w[DN_TB / 32];
	__shared__ uint32_t s_d[DN_TB / 32];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int i = blockIdx.x * DN_TB + tid;
	bool dead = false;
	double w = 0.0;
	if (i < P) {
		const float o = sigmoidf(opacity[i]);
		dead = o <= min_opacity;
		if (all_rows || !dead) w = (double)o;
		flags[i] = dead ? 1 : 0;
		mult[i] = 0;
	}
	double inc = w;
#pragma unroll
	for (int d = 1; d < 32; d <<= 1) {
		const double u = __shfl_up_sync(0xffffffffu, inc, d);
		if (lane >= d) inc += u;
	}
	const uint32_t b = __ballot_sync(0xffffffffu, dead);
	if (lane == 31) s_w[warp] = inc;
	if (lane == 0) s_d[warp] = __popc(b);
	__syncthreads();
	for (int k = 0; k < warp; k++) inc += s_w[k];
	if (i < P) cum[i] = inc;
	if (tid == DN_TB - 1) {
		block_sum[blockIdx.x] = inc;
		uint32_t nd = 0;
		for (int k = 0; k < DN_TB / 32; k++) nd += s_d[k];
		block_dead[blockIdx.x] = nd;
	}
}

__global__ void __launch_bounds__(1024) reloc_scan_kernel(int nblocks, const double* __restrict__ block_sum, const uint32_t* __restrict__ block_dead,
                                                        double* __restrict__ sum_off, uint32_t* __restrict__ dead_off, RelocTotals* __restrict__ totals)
{
	__shared__ double s_w[32];
	__shared__ uint32_t s_d[32];
	__shared__ double s_run;
	__shared__ uint32_t s_rund;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (tid == 0) { s_run = 0.0; s_rund = 0u; }
	__syncthreads();
	for (int b0 = 0; b0 < nblocks; b0 += 1024) {
		const int b = b0 + tid;
		const double w = b < nblocks ? block_sum[b] : 0.0;
		const uint32_t d = b < nblocks ? block_dead[b] : 0u;
		double inc = w;
		uint32_t incd = d;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) {
			const double u = __shfl_up_sync(0xffffffffu, inc, o);
			const uint32_t ud = __shfl_up_sync(0xffffffffu, incd, o);
			if (lane >= o) { inc += u; incd += ud; }
		}
		if (lane == 31) { s_w[warp] = inc; s_d[warp] = incd; }
		__syncthreads();
		double base = s_run;
		uint32_t based = s_rund;
		for (int k = 0; k < warp; k++) { base += s_w[k]; based += s_d[k]; }
		if (b < nblocks) { sum_off[b] = base + inc - w; dead_off[b] = based + incd - d; }
		__syncthreads();
		if (tid == 1023) { s_run = base + inc; s_rund = based + incd; }
		__syncthreads();
	}
	if (tid == 0) { totals->total = s_run; totals->n_dead = s_rund; totals->pad = 0u; }
}

// u of draw j: injected, or the first word of Philox(counter = (j, sub, offset), key = seed) as (word + 0.5) 2^-32 in float, at most
// 1 - 2^-24. sub = 1 (relocate) or 2 (grow) keeps the two draws of one refinement, and the normals of normal3 (sub 0), on streams of their own.
__device__ __forceinline__ float uniform1(const float* __restrict__ uniforms, unsigned long long seed, unsigned long long offset, uint32_t sub, uint32_t j)
{
	if (uniforms) return uniforms[j];
	const uint4 r = philox4x32_10(make_uint4(j, sub, (uint32_t)offset, (uint32_t)(offset >> 32)), make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
	return fminf(((float)r.x + 0.5f) * 2.3283064365386963e-10f, 0.99999994f);
}

// n_host < 0: one draw per dead row (totals->n_dead)
__global__ void __launch_bounds__(256) reloc_draw_kernel(int P, int n_host, const RelocTotals* __restrict__ totals, const double* __restrict__ cum,
                                                       const double* __restrict__ sum_off, const float* __restrict__ uniforms, unsigned long long seed,
                                                       unsigned long long offset, uint32_t sub, int* __restrict__ pick, int* __restrict__ mult)
{
	const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t n = n_host < 0 ? totals->n_dead : (uint32_t)n_host;
	const double total = totals->total;
	if (j >= n || (n_host < 0 && !(total > 0.0))) return;   // relocate without an alive row: nothing to draw from
	const float u = uniform1(uniforms, seed, offset, sub, j);
	const double target = (double)u * total;
	int lo = 0, hi = P - 1;   // first row whose cumulative weight exceeds the target (the last row's equals the total > target)
	if (!(total > 0.0)) lo = hi = min((int)(u * (float)P), P - 1);   // grow over rows whose opacities all underflowed: uniform picks
	while (lo < hi) {
		const int mid = (lo + hi) >> 1;
		if (sum_off[mid / DN_TB] + cum[mid] > target) hi = mid; else lo = mid + 1;
	}
	pick[j] = lo;
	atomicAdd(&mult[lo], 1);
}

// a model's tensors as the row kernels take them (rows_of); relocate and grow write them in place
struct RelocTensors {
	float* p[6]; float* m[6]; float* v[6];
	float* stat[3];            // max_radii2D, xyz_gradient_accum, denom (any may be null)
	int* exist;                // or null
	unsigned char* live;       // psb_model.adam_live or null
};

__global__ void __launch_bounds__(DN_TB) reloc_correct_kernel(int P, RelocTensors t, const int* __restrict__ mult, float min_opacity)
{
	__shared__ int s_picked[DN_TB];
	const int tid = threadIdx.x;
	const int base = blockIdx.x * DN_TB;
	const int rows = min(DN_TB, P - base);
	const int i = base + tid;
	const int cnt = i < P ? mult[i] : 0;
	s_picked[tid] = cnt;
	if (cnt > 0) {
		float o_new, f;
		relocation(sigmoidf(t.p[3][i]), min(cnt + 1, RL_MAXN), min_opacity, o_new, f);
		// a corrected row is alive: where o' was clamped to min_opacity, the stored logit is nudged until its sigmoid clears the threshold
		float lo = logf(o_new / (1.0f - o_new));
		for (int k = 0; k < 16 && !(sigmoidf(lo) > min_opacity * 1.000001f); k++) lo = nextafterf(lo, 100.f);
		t.p[3][i] = lo;
#pragma unroll
		for (int c = 0; c < 3; c++) t.p[4][3 * i + c] = logf(expf(t.p[4][3 * i + c]) * f);
		if (t.live) t.live[i] = 0;
	}
	__syncthreads();
#pragma unroll
	for (int ti = 0; ti < 6; ti++) {
		const int k = row_floats(ti);
		float* __restrict__ dm = t.m[ti] + (size_t)base * k;
		float* __restrict__ dv = t.v[ti] + (size_t)base * k;
		for (int e = tid; e < rows * k; e += DN_TB)
			if (s_picked[e / k] > 0) { dm[e] = 0.f; dv[e] = 0.f; }
	}
}

// Targets of block b are rows tbase + [b * 128, ...). flags != null (relocate): row i is a target when it is dead, its source is the
// pick of its rank among the dead rows; flags == null (grow): target n_old + j is draw j's.
__global__ void __launch_bounds__(DN_TB) reloc_copy_kernel(int n_targets, int tbase, RelocTensors t, const uint8_t* __restrict__ flags,
                                                         const uint32_t* __restrict__ dead_off, const RelocTotals* __restrict__ totals,
                                                         const int* __restrict__ pick, int iteration)
{
	__shared__ int s_src[DN_TB];
	__shared__ uint32_t s_wcnt[DN_TB / 32];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int base = blockIdx.x * DN_TB;
	const int rows = min(DN_TB, n_targets - base);
	const int j = base + tid;
	const bool go = !flags || totals->total > 0.0;
	int src = -1;
	if (flags) {
		const bool dead = j < n_targets && flags[j] != 0;
		const uint32_t b = __ballot_sync(0xffffffffu, dead);
		if (lane == 0) s_wcnt[warp] = __popc(b);
		__syncthreads();
		uint32_t rank = dead_off[blockIdx.x] + __popc(b & ((1u << lane) - 1u));
		for (int w = 0; w < warp; w++) rank += s_wcnt[w];
		if (dead && go) src = pick[rank];
	} else if (j < n_targets && go) {
		src = pick[j];
	}
	s_src[tid] = src;
	if (src >= 0) {
		const size_t d = (size_t)tbase + j;
#pragma unroll
		for (int q = 0; q < 3; q++) if (t.stat[q]) t.stat[q][d] = 0.f;
		if (t.exist) t.exist[d] = iteration;
		if (t.live) t.live[d] = 0;
	}
	__syncthreads();
#pragma unroll
	for (int ti = 0; ti < 6; ti++) {
		const int k = row_floats(ti);
		const size_t o = ((size_t)tbase + base) * k;
		for (int e = tid; e < rows * k; e += DN_TB) {
			const int r = e / k, s = s_src[r];
			if (s < 0) continue;
			t.p[ti][o + e] = t.p[ti][(size_t)s * k + (e - r * k)];
			t.m[ti][o + e] = 0.f; t.v[ti][o + e] = 0.f;
		}
	}
}

// Position noise of 3DGS-MCMC (gsplat inject_noise_to_position): xyz += Sigma xi lr g(o), Sigma = R(q) diag(exp(scaling)^2) R(q)^T with q
// the normalised quaternion, g(o) = 1 / (1 + exp(-100 ((1 - o) - 0.995))), xi = normal3(seed, step, row). One thread per row, no atomics.
// Nothing moves when the pass overflowed the binning arena; visible_only: only rows the pass saw (tile_info.z != 0).
__global__ void __launch_bounds__(256) position_noise_kernel(int P, float* __restrict__ xyz, const float* __restrict__ opacity, const float* __restrict__ scaling,
                                                           const float* __restrict__ rotation, float lr, unsigned long long seed, unsigned long long step,
                                                           const uint4* __restrict__ tile_info, const uint32_t* __restrict__ counters, uint32_t capacity)
{
	if (counters[0] > capacity) return;
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P || (tile_info && tile_info[i].z == 0)) return;
	const float o = sigmoidf(opacity[i]);
	const float g = 1.0f / (1.0f + expf(-100.0f * ((1.0f - o) - 0.995f)));
	const float4 qr = reinterpret_cast<const float4*>(rotation)[i];
	const float n = fmaxf(sqrtf(qr.x * qr.x + qr.y * qr.y + qr.z * qr.z + qr.w * qr.w), 1e-12f);
	const float r = qr.x / n, x = qr.y / n, y = qr.z / n, z = qr.w / n;
	const float R00 = 1.f - 2.f * (y * y + z * z), R01 = 2.f * (x * y - r * z), R02 = 2.f * (x * z + r * y);
	const float R10 = 2.f * (x * y + r * z), R11 = 1.f - 2.f * (x * x + z * z), R12 = 2.f * (y * z - r * x);
	const float R20 = 2.f * (x * z - r * y), R21 = 2.f * (y * z + r * x), R22 = 1.f - 2.f * (x * x + y * y);
	const float s0 = expf(scaling[3 * i]), s1 = expf(scaling[3 * i + 1]), s2 = expf(scaling[3 * i + 2]);
	const float3 xi = normal3(seed, step, (uint32_t)i);
	// Sigma xi = R (s^2 * (R^T xi))
	const float a = (R00 * xi.x + R10 * xi.y + R20 * xi.z) * s0 * s0;
	const float b = (R01 * xi.x + R11 * xi.y + R21 * xi.z) * s1 * s1;
	const float c = (R02 * xi.x + R12 * xi.y + R22 * xi.z) * s2 * s2;
	const float k = lr * g;
	xyz[3 * i] += (R00 * a + R01 * b + R02 * c) * k;
	xyz[3 * i + 1] += (R10 * a + R11 * b + R12 * c) * k;
	xyz[3 * i + 2] += (R20 * a + R21 * b + R22 * c) * k;
}

struct RelocWorkspace {
	uint8_t* flags; double* cum; int* mult; int* pick; double* block_sum; double* sum_off; uint32_t* block_dead; uint32_t* dead_off; RelocTotals* totals;
};
size_t reloc_ws_bytes(int P)
{
	const size_t nb = ((size_t)P + DN_TB - 1) / DN_TB, p = (size_t)P;
	return align_up(p, 256) + align_up(p * 8, 256) + 2 * align_up(p * 4, 256) + 2 * align_up(nb * 8, 256) + 2 * align_up(nb * 4, 256) + 256;
}
RelocWorkspace reloc_ws_carve(void* w, int P)
{
	const size_t nb = ((size_t)P + DN_TB - 1) / DN_TB, p = (size_t)P;
	char* c = static_cast<char*>(w);
	RelocWorkspace s;
	s.cum = reinterpret_cast<double*>(c); c += align_up(p * 8, 256);
	s.block_sum = reinterpret_cast<double*>(c); c += align_up(nb * 8, 256);
	s.sum_off = reinterpret_cast<double*>(c); c += align_up(nb * 8, 256);
	s.totals = reinterpret_cast<RelocTotals*>(c); c += 256;
	s.mult = reinterpret_cast<int*>(c); c += align_up(p * 4, 256);
	s.pick = reinterpret_cast<int*>(c); c += align_up(p * 4, 256);
	s.block_dead = reinterpret_cast<uint32_t*>(c); c += align_up(nb * 4, 256);
	s.dead_off = reinterpret_cast<uint32_t*>(c); c += align_up(nb * 4, 256);
	s.flags = reinterpret_cast<uint8_t*>(c);
	return s;
}
// the tensors of a model (all null for a null model)
RelocTensors rows_of(const psb_model* m)
{
	RelocTensors t = {};
	if (!m) return t;
	for (int i = 0; i < 6; i++) { t.p[i] = m->param[i]; t.m[i] = m->exp_avg[i]; t.v[i] = m->exp_avg_sq[i]; }
	t.stat[0] = m->max_radii2D; t.stat[1] = m->xyz_gradient_accum; t.stat[2] = m->denom;
	t.exist = m->exist_since_iter;
	t.live = m->adam_live;
	return t;
}
// all 18 parameter / moment tensors are given
bool has_rows(const RelocTensors& t)
{
	for (int i = 0; i < 6; i++)
		if (!t.p[i] || !t.m[i] || !t.v[i]) return false;
	return true;
}
// rows [0, P) of dst := those of src: the 18 parameter / moment tensors, and exist_since_iter when both models have it
int copy_rows(int P, const RelocTensors& s, const RelocTensors& d, cudaStream_t stream)
{
	for (int i = 0; i < 6; i++) {
		const size_t bytes = (size_t)P * row_floats(i) * sizeof(float);
		PSB_CUDA_OK(cudaMemcpyAsync(d.p[i], s.p[i], bytes, cudaMemcpyDeviceToDevice, stream));
		PSB_CUDA_OK(cudaMemcpyAsync(d.m[i], s.m[i], bytes, cudaMemcpyDeviceToDevice, stream));
		PSB_CUDA_OK(cudaMemcpyAsync(d.v[i], s.v[i], bytes, cudaMemcpyDeviceToDevice, stream));
	}
	if (d.exist && s.exist) PSB_CUDA_OK(cudaMemcpyAsync(d.exist, s.exist, (size_t)P * sizeof(int), cudaMemcpyDeviceToDevice, stream));
	return 0;
}
// rows [0, n) of the statistics the model has := 0 (reference densificationPostfix :709-711)
int zero_stats(const RelocTensors& t, size_t n, cudaStream_t stream)
{
	for (int q = 0; q < 3; q++)
		if (t.stat[q]) PSB_CUDA_OK(cudaMemsetAsync(t.stat[q], 0, n * sizeof(float), stream));
	return 0;
}
bool reloc_cfg_ok(const psb_relocate_cfg* c)
{
	return c && c->min_opacity >= 0.f && c->min_opacity < 1.f;   // (also false for a NaN)
}
// weights, scan and n draws (n < 0: one per dead row) over the P rows of `opacity` into the workspace
int reloc_sample(int P, const float* opacity, const psb_relocate_cfg* cfg, int all_rows, int n, const RelocWorkspace& w, const float* uniforms,
                 cudaStream_t stream)
{
	const int nb = (P + DN_TB - 1) / DN_TB;
	reloc_weight_kernel<<<nb, DN_TB, 0, stream>>>(P, opacity, cfg->min_opacity, all_rows, w.flags, w.cum, w.mult, w.block_sum, w.block_dead);
	PSB_LAUNCH_OK();
	reloc_scan_kernel<<<1, 1024, 0, stream>>>(nb, w.block_sum, w.block_dead, w.sum_off, w.dead_off, w.totals);
	PSB_LAUNCH_OK();
	reloc_draw_kernel<<<((n < 0 ? P : n) + 255) / 256, 256, 0, stream>>>(P, n, w.totals, w.cum, w.sum_off, uniforms, cfg->seed, cfg->offset, all_rows ? 2u : 1u, w.pick, w.mult);
	PSB_LAUNCH_OK();
	return 0;
}

struct Workspace {
	uint8_t* flags; uint32_t* counts; uint32_t* offsets; uint32_t* totals;
};
size_t ws_bytes(int P)
{
	const size_t nb = ((size_t)P + DN_TB - 1) / DN_TB;
	return align_up((size_t)P, 256) + 2 * align_up(nb * 4 * sizeof(uint32_t), 256) + 256;
}
Workspace ws_carve(void* w, int P)
{
	const size_t nb = ((size_t)P + DN_TB - 1) / DN_TB;
	char* c = static_cast<char*>(w);
	Workspace s;
	s.flags = reinterpret_cast<uint8_t*>(c); c += align_up((size_t)P, 256);
	s.counts = reinterpret_cast<uint32_t*>(c); c += align_up(nb * 4 * sizeof(uint32_t), 256);
	s.offsets = reinterpret_cast<uint32_t*>(c); c += align_up(nb * 4 * sizeof(uint32_t), 256);
	s.totals = reinterpret_cast<uint32_t*>(c);
	return s;
}
DensifyCfg to_cfg(const psb_densify_cfg* c)
{
	DensifyCfg d;
	d.tau = c->max_grad; d.min_opacity = c->min_opacity;
	d.size_thr = c->percent_dense * c->extent;   // float * float like percentDense() * scene_extent
	d.ws_thr = 0.1f * c->extent;
	d.ws_prune = c->max_screen_size != 0;
	return d;
}

// the plans' tail: scan of the block counts, then the one host round trip (the caller sizes the output tensors from the totals)
int plan_totals(int P, const Workspace& w, uint32_t tot[4], cudaStream_t stream)
{
	densify_scan_kernel<<<1, 1024, 0, stream>>>((P + DN_TB - 1) / DN_TB, w.counts, w.offsets, w.totals);
	PSB_LAUNCH_OK();
	PSB_CUDA_OK(cudaMemcpyAsync(tot, w.totals, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
	PSB_CUDA_OK(cudaStreamSynchronize(stream));
	return 0;
}

// psb_densify_apply and psb_prune_apply: dst's P_new rows from src's P rows by the plan in the workspace. keep_stats: the statistics
// of the surviving originals are compacted (when both models have all three); otherwise those of dst are zeroed.
int scatter_apply(const char* fn, int P, const psb_model* src, const psb_model* dst, int P_new, const psb_densify_cfg* cfg,
                  const void* workspace, bool keep_stats, const float* normal_samples, cudaStream_t stream)
{
	const RelocTensors s = rows_of(src), d = rows_of(dst);
	const bool rows = P > 0 && P_new > 0;
	const char* err = nullptr;
	if (P < 0 || P_new < 0 || !cfg || (P > 0 && (!src || !workspace)) || (P_new > 0 && !dst)) err = ": bad argument";
	else if (rows && (!has_rows(s) || !has_rows(d))) err = ": null tensor";
	else if (rows && (reinterpret_cast<uintptr_t>(s.p[5]) & 15)) err = ": rotation tensor must be 16-byte aligned";
	if (err) { set_error_msg((std::string(fn) + err).c_str()); return PSB_ERR_ARG; }
	int rc;
	if (!keep_stats && P_new > 0 && (rc = zero_stats(d, (size_t)P_new, stream))) return rc;
	if (!rows) return 0;
	const bool stats = keep_stats && s.stat[0] && s.stat[1] && s.stat[2] && d.stat[0] && d.stat[1] && d.stat[2];
	DensifyTensors t;
	for (int i = 0; i < 6; i++) {
		t.p[i] = s.p[i]; t.m[i] = s.m[i]; t.v[i] = s.v[i];
		t.dp[i] = d.p[i]; t.dm[i] = d.m[i]; t.dv[i] = d.v[i];
	}
	t.exist = s.exist && d.exist ? s.exist : nullptr;
	t.dexist = d.exist;
	for (int q = 0; q < 3; q++) { t.stat[q] = stats ? s.stat[q] : nullptr; t.dstat[q] = stats ? d.stat[q] : nullptr; }
	const Workspace w = ws_carve(const_cast<void*>(workspace), P);
	densify_scatter_kernel<<<(P + DN_TB - 1) / DN_TB, DN_TB, 0, stream>>>(P, t, w.flags, w.offsets, w.totals, normal_samples, cfg->seed, cfg->offset);
	PSB_LAUNCH_OK();
	return 0;
}

// psb_insert_points' argument checks (messages prefixed with fn) and its body; seeding runs the same two with its emitted points
int insert_check(const char* fn, int P, const psb_model* src, const psb_model* dst, int n, const float* points, const float* colors, const float* dist2)
{
	const RelocTensors s = rows_of(src), d = rows_of(dst);
	const size_t Q = (size_t)P + n;
	const char* err = nullptr;
	if (P < 0 || n < 0 || !dst || (P > 0 && !src) || (n > 0 && (!points || !colors || !dist2))) err = ": bad argument";
	else if ((Q > 0 && !has_rows(d)) || (P > 0 && !has_rows(s))) err = ": null tensor";
	else if (n > 0 && (reinterpret_cast<uintptr_t>(d.p[5]) & 15)) err = ": rotation tensor must be 16-byte aligned";
	if (err) { set_error_msg((std::string(fn) + err).c_str()); return PSB_ERR_ARG; }
	return 0;
}
int insert_run(int P, const psb_model* src, const psb_model* dst, int n, const float* points, const float* colors, const float* dist2, int iteration,
               cudaStream_t stream)
{
	const RelocTensors s = rows_of(src), d = rows_of(dst);
	const size_t Q = (size_t)P + n;
	int rc;
	if (P > 0 && (rc = copy_rows(P, s, d, stream))) return rc;
	for (int i = 0; i < 6 && n > 0; i++) {   // moments of the new rows: zeros (cat(..., zeros_like(extension)), :675-676)
		const size_t k = (size_t)row_floats(i);
		PSB_CUDA_OK(cudaMemsetAsync(d.m[i] + (size_t)P * k, 0, (size_t)n * k * sizeof(float), stream));
		PSB_CUDA_OK(cudaMemsetAsync(d.v[i] + (size_t)P * k, 0, (size_t)n * k * sizeof(float), stream));
	}
	if (Q > 0 && (rc = zero_stats(d, Q, stream))) return rc;
	if (n > 0) {
		DensifyTensors t = {};
		for (int i = 0; i < 6; i++) t.dp[i] = d.p[i];
		t.dexist = d.exist;
		insert_fill_kernel<<<(n + 127) / 128, 128, 0, stream>>>(P, n, points, colors, dist2, iteration, t);
		PSB_LAUNCH_OK();
	}
	return 0;
}

// ---- seeding: the workspace is the densify workspace of the ng grid pixels (flags, counts, offsets, totals), then points [ng,3],
//      colours [ng,3] and dist2 [ng]
bool seed_grid(int W, int H, int stride, SeedGrid& g)
{
	if (W <= 0 || H <= 0 || stride < 1 || (long long)W * H > INT_MAX) return false;
	g.W = W; g.H = H; g.stride = stride;
	g.gw = (W + stride - 1) / stride;
	g.ng = g.gw * ((H + stride - 1) / stride);
	return true;
}
size_t seed_ws_bytes(const SeedGrid& g)
{
	const size_t n = (size_t)g.ng;
	return ws_bytes(g.ng) + 2 * align_up(n * 3 * sizeof(float), 256) + align_up(n * sizeof(float), 256);
}
struct SeedOut { float* points; float* colors; float* dist2; };
SeedOut seed_out(void* w, const SeedGrid& g)
{
	const size_t n = (size_t)g.ng;
	char* c = static_cast<char*>(w) + ws_bytes(g.ng);
	SeedOut o;
	o.points = reinterpret_cast<float*>(c); c += align_up(n * 3 * sizeof(float), 256);
	o.colors = reinterpret_cast<float*>(c); c += align_up(n * 3 * sizeof(float), 256);
	o.dist2 = reinterpret_cast<float*>(c);
	return o;
}
bool seed_cfg_ok(const psb_seed_cfg* c)
{
	// written so that a NaN fails every test
	return c && c->alpha_min > 0.f && c->alpha_min <= 1.f && c->depth_rel >= 0.f && c->depth_rel <= 1.f && c->min_depth >= 0.f &&
	       c->min_depth < c->max_depth && c->stride >= 1 && c->max_new >= 0;
}

// What a plan left in a workspace, kept on the host so that psb_seed_apply can refuse an n above the selected count before it enqueues
// anything: the last kSeedPlans workspaces planned, each with the grid it was planned on.
struct SeedPlan { const void* ws; int W, H, stride, selected; };
constexpr int kSeedPlans = 16;
std::mutex g_seed_mu;
SeedPlan g_seed_plans[kSeedPlans];
int g_seed_next = 0;

void seed_record(const void* ws, const SeedGrid& g, int selected)
{
	std::lock_guard<std::mutex> lk(g_seed_mu);
	for (SeedPlan& p : g_seed_plans)
		if (p.ws == ws) p.ws = nullptr;
	g_seed_plans[g_seed_next] = {ws, g.W, g.H, g.stride, selected};
	g_seed_next = (g_seed_next + 1) % kSeedPlans;
}
// the selected count of the plan in ws on grid g, or -1
int seed_lookup(const void* ws, const SeedGrid& g)
{
	std::lock_guard<std::mutex> lk(g_seed_mu);
	for (const SeedPlan& p : g_seed_plans)
		if (p.ws == ws && p.W == g.W && p.H == g.H && p.stride == g.stride) return p.selected;
	return -1;
}
void seed_forget(const void* ws)
{
	std::lock_guard<std::mutex> lk(g_seed_mu);
	for (SeedPlan& p : g_seed_plans)
		if (p.ws == ws) p.ws = nullptr;
}

}  // namespace

int launch_position_noise(int P, float* xyz, const float* opacity, const float* scaling, const float* rotation, float lr, unsigned long long seed,
                          unsigned long long step, const uint4* tile_info, const uint32_t* counters, uint32_t capacity, cudaStream_t stream)
{
	if (P <= 0) return 0;
	position_noise_kernel<<<(P + 255) / 256, 256, 0, stream>>>(P, xyz, opacity, scaling, rotation, lr, seed, step, tile_info, counters, capacity);
	PSB_LAUNCH_OK();
	return 0;
}

}  // namespace psb

using namespace psb;

extern "C" {

size_t psb_relocate_workspace_bytes(int P) { return P > 0 ? reloc_ws_bytes(P) : 256; }

int psb_relocate(int P, const psb_model* model, const psb_relocate_cfg* cfg, void* workspace, const float* uniforms, int* counts_host, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	const RelocTensors t = rows_of(model);
	if (P < 0 || !reloc_cfg_ok(cfg) || (P > 0 && (!workspace || !has_rows(t)))) {
		set_error_msg("psb_relocate: bad argument (P >= 0, min_opacity in [0, 1), a model with parameters and moments, and a workspace required)");
		return PSB_ERR_ARG;
	}
	if (P > 0 && (reinterpret_cast<uintptr_t>(workspace) & 7)) { set_error_msg("psb_relocate: workspace must be 8-byte aligned"); return PSB_ERR_ARG; }
	if (counts_host) counts_host[0] = counts_host[1] = 0;
	if (P == 0) return 0;
	const RelocWorkspace w = reloc_ws_carve(workspace, P);
	int rc;
	if ((rc = reloc_sample(P, t.p[3], cfg, 0, -1, w, uniforms, stream))) return rc;
	const int nb = (P + DN_TB - 1) / DN_TB;
	reloc_correct_kernel<<<nb, DN_TB, 0, stream>>>(P, t, w.mult, cfg->min_opacity);
	PSB_LAUNCH_OK();
	reloc_copy_kernel<<<nb, DN_TB, 0, stream>>>(P, 0, t, w.flags, w.dead_off, w.totals, w.pick, cfg->iteration);
	PSB_LAUNCH_OK();
	if (counts_host) {   // the one host round trip, only for a caller that wants the count
		RelocTotals tot;
		PSB_CUDA_OK(cudaMemcpyAsync(&tot, w.totals, sizeof(tot), cudaMemcpyDeviceToHost, stream));
		PSB_CUDA_OK(cudaStreamSynchronize(stream));
		counts_host[1] = (int)tot.n_dead;
		counts_host[0] = tot.total > 0.0 ? (int)tot.n_dead : 0;
	}
	return 0;
}

int psb_grow(int P, const psb_model* src, const psb_model* dst, int P_new, const psb_relocate_cfg* cfg, void* workspace, const float* uniforms,
             void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	const RelocTensors ts = rows_of(src);
	RelocTensors t = rows_of(dst);
	const long long n = (long long)P_new - P;
	if (P < 0 || n < 0 || n > P || !reloc_cfg_ok(cfg) || (P_new > 0 && (!workspace || !has_rows(ts) || !has_rows(t)))) {
		set_error_msg("psb_grow: bad argument (P <= P_new <= 2 P, min_opacity in [0, 1), two models with parameters and moments, and a workspace required)");
		return PSB_ERR_ARG;
	}
	if (P_new > 0 && (reinterpret_cast<uintptr_t>(workspace) & 7)) { set_error_msg("psb_grow: workspace must be 8-byte aligned"); return PSB_ERR_ARG; }
	if (P == 0) return 0;
	// the P old rows as they are (statistics and exist_since_iter included), then the picked ones are corrected in place in dst
	int rc;
	if ((rc = copy_rows(P, ts, t, stream))) return rc;
	for (int q = 0; q < 3; q++)
		if (t.stat[q] && ts.stat[q]) PSB_CUDA_OK(cudaMemcpyAsync(t.stat[q], ts.stat[q], (size_t)P * sizeof(float), cudaMemcpyDeviceToDevice, stream));
	t.live = nullptr;   // dst is a new model: its live bytes are the caller's to rebuild
	if (n == 0) return 0;
	const RelocWorkspace w = reloc_ws_carve(workspace, P);
	if ((rc = reloc_sample(P, t.p[3], cfg, 1, (int)n, w, uniforms, stream))) return rc;
	reloc_correct_kernel<<<(P + DN_TB - 1) / DN_TB, DN_TB, 0, stream>>>(P, t, w.mult, cfg->min_opacity);
	PSB_LAUNCH_OK();
	reloc_copy_kernel<<<((int)n + DN_TB - 1) / DN_TB, DN_TB, 0, stream>>>((int)n, P, t, nullptr, nullptr, w.totals, w.pick, cfg->iteration);
	PSB_LAUNCH_OK();
	return 0;
}

size_t psb_densify_workspace_bytes(int P) { return P > 0 ? ws_bytes(P) : 256; }

int psb_densify_plan(int P, const psb_model* src, const psb_densify_cfg* cfg, void* workspace, int* counts_host, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	if (P < 0 || !cfg || !counts_host || (P > 0 && (!src || !workspace || !src->param[3] || !src->param[4] || !src->xyz_gradient_accum || !src->denom))) {
		set_error_msg("psb_densify_plan: bad argument (model with opacity, scaling, xyz_gradient_accum, denom and a workspace required)");
		return PSB_ERR_ARG;
	}
	for (int k = 0; k < 5; k++) counts_host[k] = 0;
	if (P == 0) return 0;
	const Workspace w = ws_carve(workspace, P);
	densify_mask_kernel<<<(P + DN_TB - 1) / DN_TB, DN_TB, 0, stream>>>(P, src->param[4], src->param[3], src->xyz_gradient_accum, src->denom, to_cfg(cfg), w.flags, w.counts);
	PSB_LAUNCH_OK();
	uint32_t tot[4];
	int rc;
	if ((rc = plan_totals(P, w, tot, stream))) return rc;
	counts_host[0] = (int)(tot[0] + tot[1] + 2 * tot[2]);
	counts_host[1] = (int)tot[0]; counts_host[2] = (int)tot[1]; counts_host[3] = (int)tot[2]; counts_host[4] = (int)tot[3];
	return 0;
}

int psb_densify_apply(int P, const psb_model* src, const psb_model* dst, int P_new, const psb_densify_cfg* cfg, const void* workspace,
                      const float* normal_samples, void* stream_)
{
	return scatter_apply("psb_densify_apply", P, src, dst, P_new, cfg, workspace, false, normal_samples, (cudaStream_t)stream_);
}

int psb_prune_plan(int P, const unsigned char* mask, void* workspace, int* counts_host, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	if (P < 0 || !counts_host || (P > 0 && (!mask || !workspace))) { set_error_msg("psb_prune_plan: bad argument"); return PSB_ERR_ARG; }
	for (int k = 0; k < 5; k++) counts_host[k] = 0;
	if (P == 0) return 0;
	const Workspace w = ws_carve(workspace, P);
	prune_mask_kernel<<<(P + DN_TB - 1) / DN_TB, DN_TB, 0, stream>>>(P, mask, w.flags, w.counts);
	PSB_LAUNCH_OK();
	uint32_t tot[4];
	int rc;
	if ((rc = plan_totals(P, w, tot, stream))) return rc;
	counts_host[0] = counts_host[1] = (int)tot[0];
	return 0;
}

int psb_prune_apply(int P, const psb_model* src, const psb_model* dst, int P_new, const void* workspace, int keep_stats, void* stream_)
{
	static const psb_densify_cfg no_draw = {};   // a prune draws nothing: no samples, seed 0, offset 0
	return scatter_apply("psb_prune_apply", P, src, dst, P_new, &no_draw, workspace, keep_stats != 0, nullptr, (cudaStream_t)stream_);
}

int psb_insert_points(int P, const psb_model* src, const psb_model* dst, int n, const float* points, const float* colors, const float* dist2,
                      int iteration, void* stream_)
{
	int rc;
	if ((rc = insert_check("psb_insert_points", P, src, dst, n, points, colors, dist2))) return rc;
	return insert_run(P, src, dst, n, points, colors, dist2, iteration, (cudaStream_t)stream_);
}

size_t psb_seed_workspace_bytes(int width, int height, int stride)
{
	SeedGrid g;
	return seed_grid(width, height, stride, g) ? seed_ws_bytes(g) : 0;
}

int psb_seed_plan(const psb_camera* camera, const float* alpha, const float* depth, const float* gt_depth, const float* mask, const psb_seed_cfg* cfg,
                  void* workspace, int* counts_host, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	SeedGrid g;
	if (!camera || !seed_cfg_ok(cfg) || !seed_grid(camera->width, camera->height, cfg->stride, g) || !alpha || !depth || !gt_depth || !workspace ||
	    !counts_host) {
		set_error_msg("psb_seed_plan: bad argument (a camera of positive size, the alpha, depth and gt_depth planes, alpha_min in (0, 1], depth_rel "
		              "in [0, 1], 0 <= min_depth < max_depth, stride >= 1, max_new >= 0, a workspace and counts_host required)");
		return PSB_ERR_ARG;
	}
	for (int k = 0; k < 3; k++) counts_host[k] = 0;
	seed_forget(workspace);   // a plan that fails below leaves no plan behind
	const SeedTest s = {cfg->alpha_min, 1.0f - cfg->depth_rel, cfg->min_depth, cfg->max_depth};
	const Workspace w = ws_carve(workspace, g.ng);
	seed_mask_kernel<<<(g.ng + DN_TB - 1) / DN_TB, DN_TB, 0, stream>>>(g, s, alpha, depth, gt_depth, mask, w.flags, w.counts);
	PSB_LAUNCH_OK();
	uint32_t tot[4];
	int rc;
	if ((rc = plan_totals(g.ng, w, tot, stream))) return rc;
	counts_host[0] = (int)tot[0]; counts_host[1] = (int)tot[1]; counts_host[2] = (int)tot[2];
	seed_record(workspace, g, (int)tot[0]);
	return 0;
}

int psb_seed_apply(int P, const psb_model* src, const psb_model* dst, int n, const psb_camera* camera, const float* gt_image, const float* gt_depth,
                   const psb_seed_cfg* cfg, const void* workspace, int iteration, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	SeedGrid g;
	if (!camera || !camera->viewmatrix || !seed_cfg_ok(cfg) || !seed_grid(camera->width, camera->height, cfg->stride, g) ||
	    !(camera->tan_fovx > 0.f) || !(camera->tan_fovy > 0.f) || !std::isfinite(camera->tan_fovx) || !std::isfinite(camera->tan_fovy) ||
	    !gt_image || !gt_depth || !workspace || n < 0 || n > cfg->max_new) {
		set_error_msg("psb_seed_apply: bad argument (a camera with a view matrix, positive size and finite positive tan_fov, gt_image, gt_depth, "
		              "a valid cfg, the plan's workspace and 0 <= n <= max_new required)");
		return PSB_ERR_ARG;
	}
	const int selected = seed_lookup(workspace, g);
	if (selected < 0) { set_error_msg("psb_seed_apply: the workspace holds no psb_seed_plan of this camera size and stride"); return PSB_ERR_ARG; }
	if (n > selected) { set_error_msg("psb_seed_apply: n exceeds the number of pixels the plan selected"); return PSB_ERR_ARG; }
	const SeedOut o = seed_out(const_cast<void*>(workspace), g);
	int rc;
	if ((rc = insert_check("psb_seed_apply", P, src, dst, n, o.points, o.colors, o.dist2))) return rc;
	if (n > 0) {
		const Workspace w = ws_carve(const_cast<void*>(workspace), g.ng);
		SeedCam c;
		c.view = camera->viewmatrix;
		c.fx = (float)g.W / (2.0f * camera->tan_fovx);
		c.fy = (float)g.H / (2.0f * camera->tan_fovy);
		c.half_w = 0.5f * (float)g.W; c.half_h = 0.5f * (float)g.H;
		c.scale = (float)g.stride / (0.5f * (c.fx + c.fy));
		seed_emit_kernel<<<(g.ng + DN_TB - 1) / DN_TB, DN_TB, 0, stream>>>(g, c, n, w.flags, w.offsets, w.totals, gt_image, gt_depth, o.points,
		                                                                  o.colors, o.dist2);
		PSB_LAUNCH_OK();
	}
	return insert_run(P, src, dst, n, o.points, o.colors, o.dist2, iteration, stream);
}

int psb_reset_opacity(int P, float* opacity, float* exp_avg, float* exp_avg_sq, void* stream_)
{
	if (P < 0 || (P > 0 && (!opacity || !exp_avg || !exp_avg_sq))) { set_error_msg("psb_reset_opacity: bad argument"); return PSB_ERR_ARG; }
	if (P == 0) return 0;
	reset_opacity_kernel<<<(P + 255) / 256, 256, 0, (cudaStream_t)stream_>>>(P, opacity, exp_avg, exp_avg_sq);
	PSB_LAUNCH_OK();
	return 0;
}

}  // extern "C"
