// Fused photometric loss of the training step:  L = (1 - lambda) * mean|I - G| + lambda * (1 - mean SSIM(I, G))
// with I = rendered * mask (or, with exposure compensation, mask * the rendered image through the keyframe's 3x4 affine row), SSIM over an 11x11 Gaussian window (sigma 1.5), zero padding, per channel —
// the loss of reference gaussian_mapper.cpp:692-698 / include/loss_utils.h:28-124, which the reference runs
// as five grouped cuDNN convolutions plus ~20 elementwise kernels forward and the autograd mirror backward.
// Here: two kernels. Forward computes the five windowed moments with a separable filter in shared memory,
// the SSIM map, the two loss sums, and stores the three partial derivatives of the map that the backward
// needs; backward filters those three maps (the window is symmetric, so the adjoint of the zero-padded
// convolution is the same convolution) and writes dL/d(rendered) directly.
#include "psb_common.cuh"
#include "psb_normals.cuh"
#include "psb_train.h"

namespace psb {

namespace {

constexpr int LT = 16;          // output tile edge
constexpr int LH = 5;           // window half width
constexpr int LS = LT + 2 * LH; // staged tile edge (26)

struct Win { float w[11]; };

__device__ __forceinline__ float block_sum_256(float v, float* s_red)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	__syncthreads();
	if (lane == 0) s_red[warp] = v;
	__syncthreads();
	float t = 0.f;
#pragma unroll
	for (int i = 0; i < 8; i++) t += s_red[i];
	return t;
}

// The two block sums of a block: added to sums[0..1] (double atomics, in whatever order the blocks finish) or, DET, stored as the
// block's partials at sums[2 * block ..] for reduce_partials_kernel.
template <bool DET>
__device__ __forceinline__ void block_sums_out(float a, float b, double* __restrict__ sums)
{
	if (threadIdx.x != 0) return;
	if (DET) {
		const size_t blk = ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
		sums[2 * blk] = (double)a;
		sums[2 * blk + 1] = (double)b;
	} else {
		atomicAdd(&sums[0], (double)a);
		atomicAdd(&sums[1], (double)b);
	}
}

// Exposure compensation: the column of the 3x4 row E (row-major, E[r][j] = E[4 r + j]) that makes channel c of the compensated image,
// I'(c) = sum_k E[k][c] I(k) + E[c][3]. Loaded once per thread: E is the device copy the previous queued step may have updated.
struct ExpCol { float e0, e1, e2, eb; };
__device__ __forceinline__ ExpCol exp_col(const float* __restrict__ E, int c) { return {E[c], E[4 + c], E[8 + c], E[4 * c + 3]}; }
// I'(c, q) at pixel q of the planar [3][HW] image; with the identity row it is I(c, q) exactly (products with 1 and sums with 0)
__device__ __forceinline__ float exposed(const ExpCol& e, const float* __restrict__ img, size_t HW, size_t q)
{
	return e.e0 * img[q] + e.e1 * img[HW + q] + e.e2 * img[2 * HW + q] + e.eb;
}

// grid (tiles_x, tiles_y, 3), block 256 (16x16). EXP: the loss of X = mask * I' (E: the device row, see ExpCol) instead of mask * I.
template <bool DET, bool EXP>
__global__ void __launch_bounds__(256) loss_fwd_kernel(int H, int W, const float* __restrict__ img, const float* __restrict__ gt,
                                                       const float* __restrict__ mask, Win win, float g_ssim,
                                                       float* __restrict__ dmap /* [3 maps][3][H][W] */,
                                                       double* __restrict__ sums /* [2] | DET: [blocks][2] */, const float* __restrict__ E)
{
	__shared__ float s_x[LS][LS + 1], s_y[LS][LS + 1];
	__shared__ float s_h[5][LS][LT + 1];
	__shared__ float s_red[8];
	const int ch = blockIdx.z;
	const size_t HW = (size_t)H * W;
	const int x0 = blockIdx.x * LT, y0 = blockIdx.y * LT;
	const int tid = threadIdx.x;
	ExpCol e{};
	if (EXP) e = exp_col(E, ch);
	for (int i = tid; i < LS * LS; i += 256) {
		const int ly = i / LS, lx = i % LS;
		const int gy = y0 + ly - LH, gx = x0 + lx - LH;
		float a = 0.f, b = 0.f;
		if (gx >= 0 && gx < W && gy >= 0 && gy < H) {
			const size_t p = ch * HW + (size_t)gy * W + gx;
			a = EXP ? exposed(e, img, HW, (size_t)gy * W + gx) : img[p];
			if (mask) a *= mask[p];
			b = gt[p];
		}
		s_x[ly][lx] = a;
		s_y[ly][lx] = b;
	}
	__syncthreads();
	// horizontal pass: 26 rows x 16 columns x 5 moments
	for (int i = tid; i < LS * LT; i += 256) {
		const int ly = i / LT, lx = i % LT;
		float m1 = 0.f, m2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
		for (int k = 0; k < 11; k++) {
			const float a = s_x[ly][lx + k], b = s_y[ly][lx + k], wk = win.w[k];
			m1 += wk * a; m2 += wk * b; e11 += wk * a * a; e22 += wk * b * b; e12 += wk * a * b;
		}
		s_h[0][ly][lx] = m1; s_h[1][ly][lx] = m2; s_h[2][ly][lx] = e11; s_h[3][ly][lx] = e22; s_h[4][ly][lx] = e12;
	}
	__syncthreads();
	const int lx = tid % LT, ly = tid / LT;
	const int gx = x0 + lx, gy = y0 + ly;
	float l1 = 0.f, ss = 0.f;
	if (gx < W && gy < H) {
		float m1 = 0.f, m2 = 0.f, e11 = 0.f, e22 = 0.f, e12 = 0.f;
#pragma unroll
		for (int k = 0; k < 11; k++) {
			const float wk = win.w[k];
			m1 += wk * s_h[0][ly + k][lx]; m2 += wk * s_h[1][ly + k][lx]; e11 += wk * s_h[2][ly + k][lx];
			e22 += wk * s_h[3][ly + k][lx]; e12 += wk * s_h[4][ly + k][lx];
		}
		const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
		const float s1 = e11 - m1 * m1, s2 = e22 - m2 * m2, s12 = e12 - m1 * m2;
		const float A1 = 2.f * m1 * m2 + C1, A2 = 2.f * s12 + C2, B1 = m1 * m1 + m2 * m2 + C1, B2 = s1 + s2 + C2;
		const float inv = 1.f / (B1 * B2);
		const float map = A1 * A2 * inv;
		// partials of the map w.r.t. the three windowed moments that depend on the rendered image
		const float dm_dm1 = (2.f * m2 * A2 - 2.f * m2 * A1) * inv - map * (2.f * m1 / B1 - 2.f * m1 / B2);
		const float dm_de11 = -map / B2;
		const float dm_de12 = 2.f * A1 * inv;
		const size_t p = ch * HW + (size_t)gy * W + gx;
		dmap[p] = g_ssim * dm_dm1;
		dmap[3 * HW + p] = g_ssim * dm_de11;
		dmap[6 * HW + p] = g_ssim * dm_de12;
		ss = map;
		l1 = fabsf(s_x[ly + LH][lx + LH] - s_y[ly + LH][lx + LH]);
	}
	const float tl1 = block_sum_256(l1, s_red);
	const float tss = block_sum_256(ss, s_red);
	block_sums_out<DET>(tl1, tss, sums);
}

// Deterministic mode: sums[c] = the n block partials partials[2 b + c] (c = 0, 1) added in a fixed order (one block: strided
// per-thread sums, then a fixed tree), whatever order the blocks that wrote them ran in.
__global__ void __launch_bounds__(256) reduce_partials_kernel(int n, const double* __restrict__ partials, double* __restrict__ sums)
{
	__shared__ double s[2][256];
	const int tid = threadIdx.x;
	double a = 0.0, b = 0.0;
	for (int i = tid; i < n; i += 256) { a += partials[2 * i]; b += partials[2 * i + 1]; }
	s[0][tid] = a;
	s[1][tid] = b;
	__syncthreads();
	for (int o = 128; o > 0; o >>= 1) {
		if (tid < o) { s[0][tid] += s[0][tid + o]; s[1][tid] += s[1][tid + o]; }
		__syncthreads();
	}
	if (tid == 0) { sums[0] = s[0][0]; sums[1] = s[1][0]; }
}

// The double sums of a block (the distortion term): as above, with the block's value in double.
template <bool DET>
__device__ __forceinline__ void block_sums_out(double a, double b, double* __restrict__ sums)
{
	if (threadIdx.x != 0) return;
	if (DET) {
		const size_t blk = ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
		sums[2 * blk] = a;
		sums[2 * blk + 1] = b;
	} else {
		atomicAdd(&sums[0], a);
		atomicAdd(&sums[1], b);
	}
}

__device__ __forceinline__ double block_sum_256(double v, double* s_red)
{
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	__syncthreads();
	if (lane == 0) s_red[warp] = v;
	__syncthreads();
	double t = 0.0;
#pragma unroll
	for (int i = 0; i < 8; i++) t += s_red[i];
	return t;
}

// EXP: evaluated at x = X = mask * I' (see loss_fwd_kernel); dL_dimg then receives g = dL/dI' (mask factor applied), which
// exposure_mix_kernel turns into dL/dI.
template <bool EXP>
__global__ void __launch_bounds__(256) loss_bwd_kernel(int H, int W, const float* __restrict__ img, const float* __restrict__ gt,
                                                       const float* __restrict__ mask, Win win, float g_l1,
                                                       const float* __restrict__ dmap, float* __restrict__ dL_dimg, const float* __restrict__ E)
{
	__shared__ float s_d[3][LS][LS + 1];
	__shared__ float s_h[3][LS][LT + 1];
	const int ch = blockIdx.z;
	const size_t HW = (size_t)H * W;
	const int x0 = blockIdx.x * LT, y0 = blockIdx.y * LT;
	const int tid = threadIdx.x;
	for (int i = tid; i < LS * LS; i += 256) {
		const int ly = i / LS, lx = i % LS;
		const int gy = y0 + ly - LH, gx = x0 + lx - LH;
		float a = 0.f, b = 0.f, c = 0.f;
		if (gx >= 0 && gx < W && gy >= 0 && gy < H) {
			const size_t p = ch * HW + (size_t)gy * W + gx;
			a = dmap[p]; b = dmap[3 * HW + p]; c = dmap[6 * HW + p];
		}
		s_d[0][ly][lx] = a; s_d[1][ly][lx] = b; s_d[2][ly][lx] = c;
	}
	__syncthreads();
	for (int i = tid; i < LS * LT; i += 256) {
		const int ly = i / LT, lx = i % LT;
		float a = 0.f, b = 0.f, c = 0.f;
#pragma unroll
		for (int k = 0; k < 11; k++) {
			const float wk = win.w[k];
			a += wk * s_d[0][ly][lx + k]; b += wk * s_d[1][ly][lx + k]; c += wk * s_d[2][ly][lx + k];
		}
		s_h[0][ly][lx] = a; s_h[1][ly][lx] = b; s_h[2][ly][lx] = c;
	}
	__syncthreads();
	const int lx = tid % LT, ly = tid / LT;
	const int gx = x0 + lx, gy = y0 + ly;
	if (gx < W && gy < H) {
		float c1 = 0.f, c2 = 0.f, c3 = 0.f;
#pragma unroll
		for (int k = 0; k < 11; k++) {
			const float wk = win.w[k];
			c1 += wk * s_h[0][ly + k][lx]; c2 += wk * s_h[1][ly + k][lx]; c3 += wk * s_h[2][ly + k][lx];
		}
		const size_t p = ch * HW + (size_t)gy * W + gx;
		const float mk = mask ? mask[p] : 1.f;
		const float x = (EXP ? exposed(exp_col(E, ch), img, HW, (size_t)gy * W + gx) : img[p]) * mk, y = gt[p];
		const float d = x - y;
		const float sgn = (d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f);
		dL_dimg[p] = (g_l1 * sgn + c1 + 2.f * x * c2 + y * c3) * mk;
	}
}

// Exposure, pass 1 (grid-stride over the n = H W pixels, 256 threads): g = dL/dI' in dL_dpix (loss_bwd_kernel<true>) becomes
// dL/dI(k) = sum_c E[k][c] g(c) in place, the plane the tile backward reads; the block's 12 sums
// dL/dE[k][c] = sum_p g(c) I(k) (k < 3) and dL/dE[c][3] = sum_p g(c) go to partials[12 block + 4 r + j] (the layout of E) in double.
__global__ void __launch_bounds__(256) exposure_mix_kernel(int n, const float* __restrict__ E, const float* __restrict__ img,
                                                           float* __restrict__ dL_dpix, double* __restrict__ partials)
{
	__shared__ double s_red[8][12];
	float e[12];
#pragma unroll
	for (int j = 0; j < 12; j++) e[j] = E[j];
	double acc[12];
#pragma unroll
	for (int j = 0; j < 12; j++) acc[j] = 0.0;
	for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
		const float g[3] = {dL_dpix[i], dL_dpix[n + i], dL_dpix[2 * n + i]};
		const float x[3] = {img[i], img[n + i], img[2 * n + i]};
#pragma unroll
		for (int k = 0; k < 3; k++) dL_dpix[(size_t)k * n + i] = e[4 * k] * g[0] + e[4 * k + 1] * g[1] + e[4 * k + 2] * g[2];
#pragma unroll
		for (int c = 0; c < 3; c++) {
#pragma unroll
			for (int k = 0; k < 3; k++) acc[4 * k + c] += (double)g[c] * (double)x[k];
			acc[4 * c + 3] += (double)g[c];
		}
	}
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
	for (int j = 0; j < 12; j++) {
		double v = acc[j];
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
		if (lane == 0) s_red[warp][j] = v;
	}
	__syncthreads();
	if (threadIdx.x < 12) {
		double t = 0.0;
#pragma unroll
		for (int w = 0; w < 8; w++) t += s_red[w][threadIdx.x];
		partials[12 * (size_t)blockIdx.x + threadIdx.x] = t;
	}
}

// Exposure, pass 2 (one block): the 12 sums = the n block partials added in a fixed order (strided per-thread sums, then a fixed tree,
// as reduce_partials_kernel), so the gradient is the same every run. Then, unless the pass overflowed the binning arena
// (counters[0] > capacity: the step is a no-op and is repeated, so the row must not move), either the Adam step of the row with its
// own device step count (grad == null), or the gradient -> grad[12] (zeros for an overflowing pass, like the raw-parameter gradients).
// rec.rec != null: the gradient goes to the data-parallel record instead (header id, lr, K, valid; valid = 0 for an overflowing pass).

// One element of an exposure row's Adam step with step count t (the single-GPU update and exposure_apply_kernel share it).
__device__ __forceinline__ void exposure_adam(float* __restrict__ param, float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq, int t, float g,
                                              float lr, float beta1, float beta2, float eps)
{
	const double bc1 = 1.0 - pow((double)beta1, t), bc2 = 1.0 - pow((double)beta2, t);
	float m = *exp_avg, v = *exp_avg_sq;
	m = m * beta1 + (1.f - beta1) * g;
	v = v * beta2 + (1.f - beta2) * g * g;
	*exp_avg = m;
	*exp_avg_sq = v;
	const float denom = sqrtf(v) / (float)sqrt(bc2) + eps;
	*param -= (float)(lr / bc1) * (m / denom);
}

__global__ void __launch_bounds__(256) exposure_update_kernel(int n, const double* __restrict__ partials, const uint32_t* __restrict__ counters,
                                                              uint32_t capacity, ExposureUpdate u, float* __restrict__ grad, ExposureRecordOut rec)
{
	__shared__ double s[12][256];
	const int tid = threadIdx.x;
	const bool overflow = counters && counters[0] > capacity;   // (null: a pass without Gaussians, which cannot overflow)
	if (rec.rec) {
		grad = rec.rec + 4;
		if (tid == 0) { rec.rec[0] = (float)rec.id; rec.rec[1] = rec.lr; rec.rec[2] = (float)rec.K; rec.rec[3] = overflow ? 0.f : 1.f; }
	}
	if (overflow && !grad) return;
	double a[12];
#pragma unroll
	for (int j = 0; j < 12; j++) a[j] = 0.0;
	for (int i = tid; i < n; i += 256)
#pragma unroll
		for (int j = 0; j < 12; j++) a[j] += partials[12 * (size_t)i + j];
#pragma unroll
	for (int j = 0; j < 12; j++) s[j][tid] = a[j];
	__syncthreads();
	for (int o = 128; o > 0; o >>= 1) {
		if (tid < o)
#pragma unroll
			for (int j = 0; j < 12; j++) s[j][tid] += s[j][tid + o];
		__syncthreads();
	}
	if (grad) {
		if (tid < 12) grad[tid] = overflow ? 0.f : (float)s[tid][0];
		return;
	}
	const int t = u.step[0] + 1;   // read by every thread before thread 0 stores it
	__syncthreads();
	if (tid < 12) exposure_adam(u.param + tid, u.exp_avg + tid, u.exp_avg_sq + tid, t, (float)s[tid][0], u.lr, u.beta1, u.beta2, u.eps);
	if (tid == 0) u.step[0] = t;
}

// The data-parallel exposure update (launch_exposure_apply): one block, thread 12 s + j handles element j of the row record s names,
// when s leads its id (the lowest valid rank with that id). Every rank runs it on the same records, so every replica of the table ends
// bit-identical.
constexpr int EXP_APPLY_THREADS = 12 * DP_MAX_WORLD;
__global__ void __launch_bounds__(EXP_APPLY_THREADS) exposure_apply_kernel(const float* __restrict__ recs, int stride, int world, ExposureTable tab,
                                                                           float beta1, float beta2, float eps, float grad_scale,
                                                                           uint32_t* __restrict__ status)
{
	__shared__ int s_id[DP_MAX_WORLD];   // the row record s updates, or -1 (not valid, or refused)
	const int tid = threadIdx.x, s = tid / 12, j = tid - 12 * s;
	if (tid < world) {
		const float* r = recs + (size_t)tid * stride;
		int id = -1;
		if (r[3] != 0.f) {
			const float k = r[0];
			if (r[2] == (float)tab.K && k >= 0.f && k < (float)tab.K) id = (int)k;
			else if (status) atomicCAS(status, 0u, 2u);
		}
		s_id[tid] = id;
	}
	__syncthreads();
	const int k = s < world ? s_id[s] : -1;
	bool lead = k >= 0;
	for (int r = 0; r < s && lead; r++) lead = s_id[r] != k;
	const int t = lead ? tab.step[k] + 1 : 0;   // read by the row's 12 threads before its thread 0 stores it
	__syncthreads();
	if (!lead) return;
	const float* rs = recs + (size_t)s * stride;
	float g = rs[4 + j];
	for (int r = s + 1; r < world; r++)
		if (s_id[r] == k) g += recs[(size_t)r * stride + 4 + j];
	g *= grad_scale;
	const size_t e = 12 * (size_t)k + j;
	exposure_adam(tab.param + e, tab.exp_avg + e, tab.exp_avg_sq + e, t, g, rs[1], beta1, beta2, eps);
	if (j == 0) tab.step[k] = t;
}

// Depth L1, pass 1 (grid-stride, 256 threads): per valid pixel |D - G| and sign(D - G) (-> dL_dD, scaled by pass 2); block sums of
// |D - G| and of the valid count go to sums[0], sums[1] in double (the count is exact); DET: to the block's partials.
template <bool DET>
__global__ void __launch_bounds__(256) depth_loss_kernel(int n, const float* __restrict__ D, const float* __restrict__ G, const float* __restrict__ mask,
                                                         float* __restrict__ dL_dD, double* __restrict__ sums)
{
	__shared__ float s_red[8];
	float acc = 0.f, cnt = 0.f;
	for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
		const float g = G[i];
		const bool valid = g > 0.f && (!mask || mask[i] != 0.f);
		float sgn = 0.f;
		if (valid) {
			const float d = D[i] - g;
			acc += fabsf(d);
			cnt += 1.f;
			sgn = (d > 0.f) ? 1.f : ((d < 0.f) ? -1.f : 0.f);
		}
		dL_dD[i] = sgn;
	}
	const float tacc = block_sum_256(acc, s_red);
	const float tcnt = block_sum_256(cnt, s_red);
	block_sums_out<DET>(tacc, tcnt, sums);
}

// Depth L1, pass 2: dL_dD *= lambda / max(N_valid, 1), N_valid read on the device (no host round trip).
__global__ void __launch_bounds__(256) depth_grad_scale_kernel(int n, float lambda, const double* __restrict__ sums, float* __restrict__ dL_dD)
{
	const float scale = lambda / (float)fmax(sums[1], 1.0);
	for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) dL_dD[i] *= scale;
}

// Normal L1, pass 1 (as depth_loss_kernel, over the three planes of N and G): a pixel is valid when G(p) != (0, 0, 0) and, with a mask,
// mask[0, p] != 0; per valid pixel sum_c |N_c - G_c| and sign(N_c - G_c) (-> dL_dN, scaled by pass 2).
template <bool DET>
__global__ void __launch_bounds__(256) normal_loss_kernel(int n, const float* __restrict__ N, const float* __restrict__ G, const float* __restrict__ mask,
                                                          float* __restrict__ dL_dN, double* __restrict__ sums)
{
	__shared__ float s_red[8];
	float acc = 0.f, cnt = 0.f;
	for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
		const float g0 = G[i], g1 = G[n + i], g2 = G[2 * n + i];
		const bool valid = (g0 != 0.f || g1 != 0.f || g2 != 0.f) && (!mask || mask[i] != 0.f);
		float sg[3] = {0.f, 0.f, 0.f};
		if (valid) {
			const float d[3] = {N[i] - g0, N[n + i] - g1, N[2 * n + i] - g2};
#pragma unroll
			for (int c = 0; c < 3; c++) {
				acc += fabsf(d[c]);
				sg[c] = (d[c] > 0.f) ? 1.f : ((d[c] < 0.f) ? -1.f : 0.f);
			}
			cnt += 1.f;
		}
#pragma unroll
		for (int c = 0; c < 3; c++) dL_dN[c * n + i] = sg[c];
	}
	const float tacc = block_sum_256(acc, s_red);
	const float tcnt = block_sum_256(cnt, s_red);
	block_sums_out<DET>(tacc, tcnt, sums);
}

// Normal L1, pass 2: dL_dN [3, n] *= lambda / max(N_valid, 1), N_valid read on the device.
__global__ void __launch_bounds__(256) normal_grad_scale_kernel(int n, float lambda, const double* __restrict__ sums, float* __restrict__ dL_dN)
{
	const float scale = lambda / (float)fmax(sums[1], 1.0);
	for (int i = blockIdx.x * 256 + threadIdx.x; i < 3 * n; i += gridDim.x * 256) dL_dN[i] *= scale;
}

// Depth-normal consistency (include/psb200.h, psb_dn). The planes of one pass and its camera; D-bar(q) = D(q) / A(q) where
// A(q) >= alpha_min, else 0 (a hole to the stencil).
struct DnPlanes {
	NormalCam c;
	const float* __restrict__ D;
	const float* __restrict__ A;
	const float* __restrict__ N;
	const float* __restrict__ mask;
	float alpha_min, max_rel_jump;
};

__device__ __forceinline__ float dn_dbar(const DnPlanes& p, int q)
{
	const float a = p.A[q];
	return a >= p.alpha_min ? p.D[q] / a : 0.f;
}

// n_d at pixel (u, v), which may lie outside the image ((0,0,0) there and on the border); its stencil -> st (st.s = 0 where n_d = 0)
__device__ __forceinline__ float3 dn_normal(const DnPlanes& p, int u, int v, Stencil& st)
{
	float3 nrm = make_float3(0.f, 0.f, 0.f);
	st.s = 0.f;
	if (u > 0 && v > 0 && u < p.c.W - 1 && v < p.c.H - 1) {
		const int i = v * p.c.W + u;
		stencil_normal(p.c, u, v, dn_dbar(p, i), dn_dbar(p, i - 1), dn_dbar(p, i + 1), dn_dbar(p, i - p.c.W), dn_dbar(p, i + p.c.W), p.max_rel_jump,
		               nrm, st);
	}
	return nrm;
}

__device__ __forceinline__ bool dn_valid(const DnPlanes& p, int i, float3 nd)
{
	return (nd.x != 0.f || nd.y != 0.f || nd.z != 0.f) && (!p.mask || p.mask[i] != 0.f);
}

// Pass 1 (the geometry of depth_loss_kernel): per valid pixel 1 - n_d . N; block sums of it and of the valid count -> sums[0..1]
// (DET: the block's partials); n_d -> out_dn when given. (The minimum of 4 blocks lets ptxas keep the DET variant out of local memory:
// without it it picks 32 registers and spills.)
template <bool DET>
__global__ void __launch_bounds__(256, 4) dn_loss_kernel(DnPlanes p, float* __restrict__ out_dn, double* __restrict__ sums)
{
	__shared__ float s_red[8];
	const int n = p.c.W * p.c.H;
	float acc = 0.f, cnt = 0.f;
	for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
		Stencil st;
		const float3 nd = dn_normal(p, i % p.c.W, i / p.c.W, st);
		if (dn_valid(p, i, nd)) {
			acc += 1.f - (nd.x * p.N[i] + nd.y * p.N[n + i] + nd.z * p.N[2 * n + i]);
			cnt += 1.f;
		}
		if (out_dn) {
			out_dn[i] = nd.x;
			out_dn[n + i] = nd.y;
			out_dn[2 * n + i] = nd.z;
		}
	}
	const float tacc = block_sum_256(acc, s_red);
	const float tcnt = block_sum_256(cnt, s_red);
	block_sums_out<DET>(tacc, tcnt, sums);
}

// dL/dc of the stencil of pixel (u, v) per unit of lambda / max(N_valid, 1), for n_d = s c and the term -n_d . N:
// -s (N - n_d (n_d . N)). False where (u, v) is not a valid pixel.
__device__ __forceinline__ bool dn_dc(const DnPlanes& p, int u, int v, Stencil& st, float3& g)
{
	const float3 nd = dn_normal(p, u, v, st);
	const int n = p.c.W * p.c.H, i = v * p.c.W + u;
	if (!dn_valid(p, i, nd)) return false;
	const float N0 = p.N[i], N1 = p.N[n + i], N2 = p.N[2 * n + i];
	const float nN = nd.x * N0 + nd.y * N1 + nd.z * N2;
	g = make_float3(-st.s * (N0 - nd.x * nN), -st.s * (N1 - nd.y * nN), -st.s * (N2 - nd.z * nN));
	return true;
}

__device__ __forceinline__ float3 cross3(float3 a, float3 b)
{
	return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

// Pass 2, one thread per pixel q, no atomics: with k = lambda / max(N_valid, 1) read on the device, dL/dN(q) += -k n_d(q) on a valid q;
// dL/dD-bar(q) gathers, in a fixed order, the dL/dX(q) of the four stencils that read q (c = a x b: dL/da = b x dL/dc, dL/db = dL/dc x a;
// q is X(u-1) of its right neighbour, X(u+1) of its left one, X(v-1) of the one below and X(v+1) of the one above), each recomputed
// here, times dX/dD-bar = the ray of q. Then dL/dD(q) += dL/dD-bar / A and dL/dA(q) += -dL/dD-bar D-bar / A where A >= alpha_min.
__global__ void __launch_bounds__(256) dn_grad_kernel(DnPlanes p, float lambda, const double* __restrict__ sums, float* __restrict__ dL_dD,
                                                      float* __restrict__ dL_dA, float* __restrict__ dL_dN)
{
	const int n = p.c.W * p.c.H;
	const int i = blockIdx.x * 256 + threadIdx.x;
	if (i >= n) return;
	const int u = i % p.c.W, v = i / p.c.W;
	const float k = lambda / (float)fmax(sums[1], 1.0);
	Stencil st;
	const float3 nd = dn_normal(p, u, v, st);
	if (dn_valid(p, i, nd)) {
		dL_dN[i] += -k * nd.x;
		dL_dN[n + i] += -k * nd.y;
		dL_dN[2 * n + i] += -k * nd.z;
	}
	const float a = p.A[i];
	if (!(a >= p.alpha_min)) return;
	const float rx = ((float)u + 0.5f - p.c.half_w) / p.c.fx, ry = ((float)v + 0.5f - p.c.half_h) / p.c.fy;
	float g = 0.f;
	float3 gc;
	if (dn_dc(p, u + 1, v, st, gc)) { const float3 d = cross3(st.b, gc); g -= rx * d.x + ry * d.y + d.z; }
	if (dn_dc(p, u - 1, v, st, gc)) { const float3 d = cross3(st.b, gc); g += rx * d.x + ry * d.y + d.z; }
	if (dn_dc(p, u, v + 1, st, gc)) { const float3 d = cross3(gc, st.a); g -= rx * d.x + ry * d.y + d.z; }
	if (dn_dc(p, u, v - 1, st, gc)) { const float3 d = cross3(gc, st.a); g += rx * d.x + ry * d.y + d.z; }
	g *= k;
	const float dbar = p.D[i] / a;
	dL_dD[i] += g / a;
	dL_dA[i] += -g * dbar / a;
}

// Depth distortion, pass 1 (the geometry of depth_loss_kernel): per valid pixel A M - D^2 in double (the products of two floats are
// exact there, so the difference is rounded once); block sums of it and of the valid count -> sums[0..1] (DET: the block's partials).
template <bool DET>
__global__ void __launch_bounds__(256) dist_loss_kernel(int n, const float* __restrict__ D, const float* __restrict__ A, const float* __restrict__ M,
                                                        const float* __restrict__ mask, double* __restrict__ sums)
{
	__shared__ double s_red[8];
	double acc = 0.0, cnt = 0.0;
	for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
		if (!mask || mask[i] != 0.f) {
			const double d = (double)D[i];
			acc += __dadd_rn(__dmul_rn((double)A[i], (double)M[i]), -__dmul_rn(d, d));
			cnt += 1.0;
		}
	}
	const double tacc = block_sum_256(acc, s_red);
	const double tcnt = block_sum_256(cnt, s_red);
	block_sums_out<DET>(tacc, tcnt, sums);
}

// Depth distortion, pass 2: k = lambda / max(N_valid, 1) read on the device (an IEEE float division); on valid pixels dL/dA += k M and
// dL/dD += (-2k) D, and dL/dM = k A (0 elsewhere). Explicit roundings, no contraction: torch float32 reproduces the planes bit for bit.
__global__ void __launch_bounds__(256) dist_grad_kernel(int n, float lambda, const double* __restrict__ sums, const float* __restrict__ D,
                                                        const float* __restrict__ A, const float* __restrict__ M, const float* __restrict__ mask,
                                                        float* __restrict__ dL_dD, float* __restrict__ dL_dA, float* __restrict__ dL_dM)
{
	const float k = __fdiv_rn(lambda, (float)fmax(sums[1], 1.0));
	const float m2k = __fmul_rn(-2.f, k);
	for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) {
		float gM = 0.f;
		if (!mask || mask[i] != 0.f) {
			dL_dA[i] = __fadd_rn(dL_dA[i], __fmul_rn(k, M[i]));
			dL_dD[i] = __fadd_rn(dL_dD[i], __fmul_rn(m2k, D[i]));
			gM = __fmul_rn(k, A[i]);
		}
		dL_dM[i] = gM;
	}
}

}  // namespace

int launch_dist_loss(int H, int W, const float* depth, const float* alpha, const float* depth2, const float* mask, float lambda, double* sums,
                     float* dL_dD, float* dL_dA, float* dL_dM, cudaStream_t stream, double* partials)
{
	const int n = H * W;
	const int grid = depth_loss_blocks(H, W);
	const bool det = partials != nullptr;
	if (!det) PSB_CUDA_OK(cudaMemsetAsync(sums, 0, 2 * sizeof(double), stream));
	(det ? dist_loss_kernel<true> : dist_loss_kernel<false>)<<<grid, 256, 0, stream>>>(n, depth, alpha, depth2, mask, det ? partials : sums);
	PSB_LAUNCH_OK();
	if (det) {
		reduce_partials_kernel<<<1, 256, 0, stream>>>(grid, partials, sums);
		PSB_LAUNCH_OK();
	}
	dist_grad_kernel<<<grid, 256, 0, stream>>>(n, lambda, sums, depth, alpha, depth2, mask, dL_dD, dL_dA, dL_dM);
	PSB_LAUNCH_OK();
	return 0;
}

int launch_dn_loss(int W, int H, float tan_fovx, float tan_fovy, const float* depth, const float* alpha, const float* normal, const float* mask,
                   float lambda, float alpha_min, float max_rel_jump, float* out_dn, double* sums, float* dL_dD, float* dL_dA, float* dL_dN,
                   cudaStream_t stream, double* partials)
{
	const DnPlanes p{normal_cam(W, H, tan_fovx, tan_fovy), depth, alpha, normal, mask, alpha_min, max_rel_jump};
	const int n = H * W;
	const int grid = depth_loss_blocks(H, W);
	const bool det = partials != nullptr;
	if (!det) PSB_CUDA_OK(cudaMemsetAsync(sums, 0, 2 * sizeof(double), stream));
	(det ? dn_loss_kernel<true> : dn_loss_kernel<false>)<<<grid, 256, 0, stream>>>(p, out_dn, det ? partials : sums);
	PSB_LAUNCH_OK();
	if (det) {
		reduce_partials_kernel<<<1, 256, 0, stream>>>(grid, partials, sums);
		PSB_LAUNCH_OK();
	}
	dn_grad_kernel<<<cdiv(n, 256), 256, 0, stream>>>(p, lambda, sums, dL_dD, dL_dA, dL_dN);
	PSB_LAUNCH_OK();
	return 0;
}

int launch_normal_loss(int H, int W, const float* normal, const float* gt_normal, const float* mask, float lambda_normal, double* sums, float* dL_dN,
                       cudaStream_t stream, double* partials)
{
	const int n = H * W;
	const int grid = depth_loss_blocks(H, W);
	const bool det = partials != nullptr;
	if (!det) PSB_CUDA_OK(cudaMemsetAsync(sums, 0, 2 * sizeof(double), stream));
	(det ? normal_loss_kernel<true> : normal_loss_kernel<false>)<<<grid, 256, 0, stream>>>(n, normal, gt_normal, mask, dL_dN, det ? partials : sums);
	PSB_LAUNCH_OK();
	if (det) {
		reduce_partials_kernel<<<1, 256, 0, stream>>>(grid, partials, sums);
		PSB_LAUNCH_OK();
	}
	normal_grad_scale_kernel<<<grid, 256, 0, stream>>>(n, lambda_normal, sums, dL_dN);
	PSB_LAUNCH_OK();
	return 0;
}

int launch_depth_loss(int H, int W, const float* depth, const float* gt_depth, const float* mask, float lambda_depth, double* sums, float* dL_dD,
                      cudaStream_t stream, double* partials)
{
	const int n = H * W;
	const int grid = depth_loss_blocks(H, W);
	const bool det = partials != nullptr;
	if (!det) PSB_CUDA_OK(cudaMemsetAsync(sums, 0, 2 * sizeof(double), stream));
	(det ? depth_loss_kernel<true> : depth_loss_kernel<false>)<<<grid, 256, 0, stream>>>(n, depth, gt_depth, mask, dL_dD, det ? partials : sums);
	PSB_LAUNCH_OK();
	if (det) {
		reduce_partials_kernel<<<1, 256, 0, stream>>>(grid, partials, sums);
		PSB_LAUNCH_OK();
	}
	depth_grad_scale_kernel<<<grid, 256, 0, stream>>>(n, lambda_depth, sums, dL_dD);
	PSB_LAUNCH_OK();
	return 0;
}

// sums: device double[2] (zeroed here); after the launch sums[0] = sum|I-G|, sums[1] = sum ssim_map.
// dmap: device float[9*H*W] scratch. dL_dimg may be null (loss value only).
int launch_loss(int H, int W, const float* img, const float* gt, const float* mask, float lambda_dssim, float* dmap, double* sums,
                float* dL_dimg, cudaStream_t stream, double* partials, const float* E)
{
	Win win;
	float s = 0.f;
	for (int x = 0; x < 11; x++) { const int t = x - 5; win.w[x] = expf(-(float)(t * t) / (2.0f * 1.5f * 1.5f)); s += win.w[x]; }
	for (int x = 0; x < 11; x++) win.w[x] /= s;
	const float inv_n = 1.0f / (3.0f * (float)H * (float)W);
	dim3 grid((W + LT - 1) / LT, (H + LT - 1) / LT, 3);
	const bool det = partials != nullptr;
	const auto fwd = det ? (E ? loss_fwd_kernel<true, true> : loss_fwd_kernel<true, false>)
	                     : (E ? loss_fwd_kernel<false, true> : loss_fwd_kernel<false, false>);
	if (!det) PSB_CUDA_OK(cudaMemsetAsync(sums, 0, 2 * sizeof(double), stream));
	fwd<<<grid, 256, 0, stream>>>(H, W, img, gt, mask, win, -lambda_dssim * inv_n, dmap, det ? partials : sums, E);
	PSB_LAUNCH_OK();
	if (det) {
		reduce_partials_kernel<<<1, 256, 0, stream>>>((int)(grid.x * grid.y * grid.z), partials, sums);
		PSB_LAUNCH_OK();
	}
	if (dL_dimg) {
		(E ? loss_bwd_kernel<true> : loss_bwd_kernel<false>)<<<grid, 256, 0, stream>>>(H, W, img, gt, mask, win, (1.0f - lambda_dssim) * inv_n, dmap,
		                                                                              dL_dimg, E);
		PSB_LAUNCH_OK();
	}
	return 0;
}

int launch_exposure(int H, int W, const float* img, const float* E, float* dL_dpix, double* partials, const uint32_t* counters, uint32_t capacity,
                    const ExposureUpdate* update, float* grad, const ExposureRecordOut* record, cudaStream_t stream)
{
	const int n = H * W;
	const int grid = exposure_blocks(H, W);
	exposure_mix_kernel<<<grid, 256, 0, stream>>>(n, E, img, dL_dpix, partials);
	PSB_LAUNCH_OK();
	ExposureUpdate u{};
	if (update) u = *update;
	ExposureRecordOut rec{};
	if (record && !update) rec = *record;
	exposure_update_kernel<<<1, 256, 0, stream>>>(grid, partials, counters, capacity, u, update || rec.rec ? nullptr : grad, rec);
	PSB_LAUNCH_OK();
	return 0;
}

int launch_exposure_apply(const float* recs, int stride, int world, const ExposureTable& table, float beta1, float beta2, float eps, float grad_scale,
                          uint32_t* status, cudaStream_t stream)
{
	if (world < 1 || world > DP_MAX_WORLD) { set_error_msg("launch_exposure_apply: world must lie in 1..8"); return -1; }
	exposure_apply_kernel<<<1, EXP_APPLY_THREADS, 0, stream>>>(recs, stride, world, table, beta1, beta2, eps, grad_scale, status);
	PSB_LAUNCH_OK();
	return 0;
}

}  // namespace psb
