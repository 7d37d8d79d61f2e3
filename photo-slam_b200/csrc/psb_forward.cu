// Forward pipeline up to the per-tile instance lists:
//   preprocess (project, covariance -> conic, SH -> RGB, tile rectangle)          [per Gaussian]
//   depth sort of the Gaussians (4 x 8-bit onesweep passes on the float bits)     [per Gaussian]
//   exclusive scan of tiles_touched in depth order  -> instance offsets, num_rendered
//   emit (tile id, Gaussian) instances in depth order
//   stable sort of the instances by tile id (ceil(log2 #tiles) bits, 1-2 onesweep passes)
//   tile ranges
//
// The reference sorts every instance on a 64-bit (tile | depth) key in ~6 radix passes
// (reference rasterizer_impl.cu:70-111, 300-308). Sorting the P Gaussians by depth ONCE and then
// stably partitioning the N instances by tile yields exactly the same order — ties on (tile, depth)
// stay in ascending Gaussian index in both — with 4 passes over P plus 2 passes over N of 8-byte
// records instead of 6 passes over N of 12-byte records.
#include "psb_geom.cuh"
#include "psb_state.h"
#include "psb_kernels.h"

namespace psb {

// ------------------------------------------------------------------------------------------------
// Preprocess. One thread per Gaussian. Mirrors the per-Gaussian contract of reference
// forward.cu:155-256 (near cull at view z <= 0.2, det == 0 cull, zero-area rect cull; culled
// Gaussians only get radii = tiles_touched = 0).
// RAW = true: inputs are the raw trainer parameters (log-scales, unnormalised quaternions, opacity
// logits, SH split into dc/rest); the activations of reference gaussian_model.cpp:48-71 are applied
// here instead of by five separate elementwise kernels and a 192 B/Gaussian concatenation.
// AA = true: anti-aliasing (Mip-Splatting's 2D filter, upstream diff-gaussian-rasterization's `antialiasing`): the splat blends with
// opacity o' = o h, h = sqrt(max(det0 / det1, 2.5e-5)), det0 / det1 the determinants of the 2D covariance before / after the 0.3 px^2
// dilation. Conic, radius, tile rectangle, depth key, colour and clamp bits are those of AA = false; the record, pmin and the tight
// tile cull all see o'.
// F3D = true (trainer variant only, RAW): the 3D smoothing filter of Mip-Splatting (psb_filter3d): the covariance is built from
// s' = sqrt(s^2 + f^2) and the opacity is o c, c = sqrt(prod s^2 / prod s'^2), f = f3d[idx]; with AA the blend opacity is o c h, h taken
// from the 2D covariance of the widened splat. Radius, rectangle, the record, pmin and the tight tile cull all see the filtered splat.
// ------------------------------------------------------------------------------------------------
constexpr int PRE_TB = 128;  // Gaussians per block

template <bool RAW, bool AA = false, bool F3D = false>
__global__ void __launch_bounds__(PRE_TB) preprocess_fwd_kernel(GaussIn in, Camera cam, int* __restrict__ radii_out, GeomState geom, int tight,
                                                                const float* __restrict__ f3d)
{
	static_assert(RAW || !F3D, "the 3D filter is applied to the raw trainer parameters only");
	// SH rows of this block's Gaussians ([128][45] raw f_rest rows or [128][48] activated rows), one TMA bulk copy per block:
	// they are consumed last (after both culls), so the copy hides behind the projection / covariance arithmetic and each
	// thread then walks its own row in shared memory (odd / 48-word row stride: at most 2-way bank conflicts on the 48 case).
	__shared__ __align__(128) float s_sh[PRE_TB * 48];
	__shared__ __align__(8) uint64_t s_bar;

	const int tid = threadIdx.x;
	const int base = blockIdx.x * PRE_TB;
	const int idx = base + tid;
	const int rows = min(PRE_TB, in.P - base);
	const bool want_sh = in.colors_precomp == nullptr;
	const int row_floats = RAW ? (in.M - 1) * 3 : in.M * 3;
	const float* sh_src = RAW ? in.sh_rest : in.shs;
	// staged only for full-degree storage (M == 16) and 16-byte aligned tensors; otherwise rows are read directly
	const bool staged = want_sh && in.M == 16 && (reinterpret_cast<uintptr_t>(sh_src) & 15) == 0;
	if (staged) {
		const size_t goff = (size_t)base * row_floats;
		const uint32_t row_bytes = (uint32_t)rows * row_floats * sizeof(float);
		const uint32_t bulk_bytes = row_bytes & ~15u;
		if (tid == 0) {
			mbar_init(&s_bar, 1);
			mbar_fence_init();
			mbar_arrive_expect_tx(&s_bar, bulk_bytes);
			bulk_g2s(s_sh, sh_src + goff, bulk_bytes, &s_bar);
			for (uint32_t i = bulk_bytes / 4; i < row_bytes / 4; i++) s_sh[i] = sh_src[goff + i];  // < 16 trailing bytes (last block)
		}
		__syncthreads();  // the mbarrier must be initialised before any other thread waits on it
	}

	// every small per-Gaussian input is loaded up front (one memory round trip instead of a chain across the culls)
	bool alive = idx < in.P;
	float3 p_orig = make_float3(0, 0, 1), s = make_float3(0, 0, 0), dc = make_float3(0, 0, 0);
	float4 q = make_float4(1, 0, 0, 0);
	float opacity = 0.f;
	float f3d_f = 0.f;  // F3D: this row's filter
	float cov3D[6] = {0, 0, 0, 0, 0, 0};
	if (alive) {
		if (F3D) f3d_f = f3d[idx];
		p_orig = make_float3(in.means3D[3 * idx], in.means3D[3 * idx + 1], in.means3D[3 * idx + 2]);
		if (in.cov3D_precomp != nullptr) {
#pragma unroll
			for (int i = 0; i < 6; i++) cov3D[i] = in.cov3D_precomp[6 * idx + i];
		} else {
			s = make_float3(in.scales[3 * idx], in.scales[3 * idx + 1], in.scales[3 * idx + 2]);
			q = reinterpret_cast<const float4*>(in.rotations)[idx];
		}
		opacity = in.opacities[idx];
		if (RAW) dc = make_float3(in.sh_dc[3 * idx], in.sh_dc[3 * idx + 1], in.sh_dc[3 * idx + 2]);
		else if (!want_sh) dc = make_float3(in.colors_precomp[3 * idx], in.colors_precomp[3 * idx + 1], in.colors_precomp[3 * idx + 2]);
		if (radii_out) radii_out[idx] = 0;
		geom.tile_info[idx] = make_uint4(0u, 0u, 0u, 0u);
		geom.depth_key[0][idx] = 0xFFFFFFFFu;
	}

	float3 p_view = make_float3(0, 0, 0), conic = make_float3(0, 0, 0);
	float2 point_image = make_float2(0, 0);
	float my_radius = 0.f;
	float aa_h = 1.f;  // AA: the opacity factor h
	float f3d_c = 1.f; // F3D: the opacity factor c
	int x0 = 0, y0 = 0, x1 = 0, y1 = 0;
	if (alive) {
		p_view = xform4x3(p_orig, cam.view);
		alive = p_view.z > 0.2f;
	}
	if (alive) {
		const float4 p_hom = xform4x4(p_orig, cam.proj);
		const float p_w = 1.0f / (p_hom.w + 0.0000001f);
		const float3 p_proj = make_float3(p_hom.x * p_w, p_hom.y * p_w, p_hom.z * p_w);

		if (in.cov3D_precomp == nullptr) {
			if (RAW) {
				s = make_float3(expf(s.x), expf(s.y), expf(s.z));
				const float n = fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f);
				q = make_float4(q.x / n, q.y / n, q.z / n, q.w / n);
			}
			if (F3D) f3d_c = filter3d_widen(s, f3d_f);
			cov3d_from_scale_rot(s, in.scale_modifier, q, cov3D);
		}

		Cov2DTerms ct;
		cov2d_terms(p_orig, cam.focal_x, cam.focal_y, cam.tan_fovx, cam.tan_fovy, cov3D, cam.view, ct);
		const float det0 = AA ? aa_det0(ct) : 0.f;
		ct.cov(0, 0) += 0.3f;
		ct.cov(1, 1) += 0.3f;
		const float3 cov = make_float3(float(ct.cov(0, 0)), float(ct.cov(0, 1)), float(ct.cov(1, 1)));

		const float det = (cov.x * cov.z - cov.y * cov.y);
		alive = det != 0.0f;
		if (alive) {
			if (AA) aa_h = aa_factor(det0, det);
			const float det_inv = 1.f / det;
			conic = make_float3(cov.z * det_inv, -cov.y * det_inv, cov.x * det_inv);

			const float mid = 0.5f * (cov.x + cov.z);
			const float lambda1 = mid + sqrt(max(0.1f, mid * mid - det));
			const float lambda2 = mid - sqrt(max(0.1f, mid * mid - det));
			my_radius = ceil(3.f * sqrt(max(lambda1, lambda2)));
			point_image = make_float2(ndc_to_pix(p_proj.x, cam.W), ndc_to_pix(p_proj.y, cam.H));
			tile_rect(point_image.x, point_image.y, (int)my_radius, cam.grid_x, cam.grid_y, x0, y0, x1, y1);
			alive = (x1 - x0) * (y1 - y0) != 0;
		}
	}

	if (staged) mbar_wait(&s_bar, 0);  // every thread waits: the block must not retire while the copy is in flight
	if (staged) __syncthreads();       // (also publishes thread 0's trailing plain stores)
	if (!alive) return;

	float3 rgb;
	uint32_t clamp_bits = 0;
	if (!want_sh) {
		rgb = dc;
	} else {
		const float3 campos = make_float3(cam.campos[0], cam.campos[1], cam.campos[2]);
		float sh[48];
		const int ncoef = (in.D + 1) * (in.D + 1);
		const float* row = staged ? s_sh + tid * row_floats : sh_src + (size_t)idx * row_floats;
		if (RAW) {
			sh[0] = dc.x; sh[1] = dc.y; sh[2] = dc.z;
#pragma unroll
			for (int k = 3; k < 48; k++) sh[k] = (k < ncoef * 3) ? row[k - 3] : 0.f;
		} else if (staged || in.sh_vec4) {
#pragma unroll
			for (int k = 0; k < 12; k++) {
				float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
				if (k * 4 < ncoef * 3) v = reinterpret_cast<const float4*>(row)[k];
				sh[4 * k] = v.x; sh[4 * k + 1] = v.y; sh[4 * k + 2] = v.z; sh[4 * k + 3] = v.w;
			}
		} else {
#pragma unroll
			for (int k = 0; k < 48; k++) sh[k] = (k < ncoef * 3) ? row[k] : 0.f;
		}
		rgb = sh_to_rgb(in.D, p_orig, campos, sh, clamp_bits);
	}

	if (RAW) opacity = 1.0f / (1.0f + expf(-opacity));
	if (F3D) opacity *= f3d_c;
	if (AA) opacity *= aa_h;

	const int radius_i = (int)my_radius;
	GaussRec r;
	r.q0 = make_float4(point_image.x, point_image.y, conic.x, conic.y);
	r.q1 = make_float4(conic.z, opacity, -(__logf(255.0f * opacity) + 1e-3f), p_view.z);
	r.q2 = make_float4(rgb.x, rgb.y, rgb.z, __uint_as_float(((uint32_t)radius_i << 3) | clamp_bits));
	geom.rec[idx] = r;
	geom.depth_key[0][idx] = __float_as_uint(p_view.z);
	if (radii_out) radii_out[idx] = radius_i;
	uint32_t count = (uint32_t)((y1 - y0) * (x1 - x0)), mask = 0xffffffffu;
	if (tight) {
		// Tight instance lists (trainer path): only the tiles of the rectangle on which the splat can reach alpha >= 1/255
		// get an instance. The blend skips such instances anyway (reference forward.cu:338-339 `alpha < 1/255 -> continue`),
		// so the image and every gradient are unchanged; the lists the sort and the blend walk shrink by about a third.
		if ((int)count <= TIGHT_MAX_AREA) {
			mask = TileCull(r.q0, r.q1).rect_mask(x0, y0, x1, y1, cam.W, cam.H);
			count = (uint32_t)__popc(mask);
		}
		count |= TT_VISIBLE;
	}
	geom.tile_info[idx] = make_uint4((uint32_t)x0 | ((uint32_t)y0 << 16), (uint32_t)x1 | ((uint32_t)y1 << 16), count, mask);
}

// z > 0.2 visibility test only (reference rasterizer_impl.cu:54-66, auxiliary.h:139-164).
__global__ void mark_visible_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ view, uint8_t* __restrict__ present)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= P) return;
	const float3 p = make_float3(means3D[3 * idx], means3D[3 * idx + 1], means3D[3 * idx + 2]);
	const float3 pv = xform4x3(p, view);
	present[idx] = pv.z > 0.2f ? 1 : 0;
}

// Warp-wide decoupled look-back (called by warp 0 of a tile, tiles taken in ticket order): publishes this tile's
// aggregate, returns the exclusive prefix of the tile, then publishes the inclusive prefix.
// status word: 2 flag bits (1 = aggregate, 2 = inclusive) | 30-bit value; 32 predecessors per round trip.
__device__ __forceinline__ uint32_t lookback_exclusive(uint32_t* status, uint32_t tile, uint32_t block_total, int lane)
{
	uint32_t excl = 0;
	volatile uint32_t* st = status;
	if (tile == 0) {
		if (lane == 0) st[0] = (2u << 30) | block_total;
		return 0;
	}
	if (lane == 0) st[tile] = (1u << 30) | block_total;
	int p = (int)tile - 1;
	while (true) {
		const int q = p - lane;
		uint32_t s = (q >= 0) ? st[q] : (2u << 30);
		// lanes closer to the tile must be published before a farther inclusive value can be used
		uint32_t unpublished = __ballot_sync(0xffffffffu, (s >> 30) == 0u);
		uint32_t incl = __ballot_sync(0xffffffffu, (s >> 30) == 2u);
		const int first_incl = incl ? (__ffs(incl) - 1) : 32;
		const int first_unpub = unpublished ? (__ffs(unpublished) - 1) : 32;
		if (first_unpub < first_incl) continue;  // poll again (same window)
		const int upto = min(first_incl, 31);
		uint32_t contrib = (lane <= upto) ? (s & ((1u << 30) - 1u)) : 0u;
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
		excl += contrib;
		if (first_incl < 32) break;
		p -= 32;
	}
	if (lane == 0) st[tile] = (2u << 30) | ((excl + block_total) & ((1u << 30) - 1u));
	return excl;
}

// ------------------------------------------------------------------------------------------------
// Single-pass exclusive scan (decoupled look-back) of tiles_touched taken in depth-sorted order.
// status word: 2 flag bits | 30-bit value. counters[0] <- total (num_rendered).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SCAN_THREADS) scan_offsets_kernel(int P, const uint32_t* __restrict__ order, const uint4* __restrict__ tile_info,
                                                                    uint32_t* __restrict__ offsets, uint32_t* __restrict__ counters,
                                                                    uint32_t* __restrict__ status)
{
	__shared__ uint32_t s_warp[SCAN_THREADS / 32];
	__shared__ uint32_t s_tile, s_prefix;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (tid == 0) s_tile = atomicAdd(&counters[1], 1u);
	__syncthreads();
	const uint32_t tile = s_tile;
	const int base = (int)tile * SCAN_TILE + tid * SCAN_ITEMS;
	uint32_t v[SCAN_ITEMS];
	uint32_t sum = 0;
#pragma unroll
	for (int i = 0; i < SCAN_ITEMS; i++) {
		const int j = base + i;
		v[i] = (j < P) ? (tile_info[order[j]].z & TT_COUNT) : 0u;
		sum += v[i];
	}
	uint32_t inc = sum;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
		if (lane >= o) inc += u;
	}
	if (lane == 31) s_warp[warp] = inc;
	__syncthreads();
	uint32_t wb = 0, block_total = 0;
#pragma unroll
	for (int i = 0; i < SCAN_THREADS / 32; i++) {
		if (i < warp) wb += s_warp[i];
		block_total += s_warp[i];
	}
	if (warp == 0) {
		const uint32_t excl = lookback_exclusive(status, tile, block_total, lane);
		if (lane == 0) {
			s_prefix = excl;
			if ((int)(tile + 1) * SCAN_TILE >= P) counters[0] = excl + block_total;
		}
	}
	__syncthreads();
	uint32_t run = s_prefix + wb + inc - sum;
#pragma unroll
	for (int i = 0; i < SCAN_ITEMS; i++) {
		const int j = base + i;
		if (j < P) offsets[j] = run;
		run += v[i];
	}
}

// ------------------------------------------------------------------------------------------------
// Emit one (tile id, Gaussian) instance per overlapped tile, Gaussians taken in depth order, tiles of
// one Gaussian row-major (y outer, x inner) like reference rasterizer_impl.cu:95-108. Small rectangles
// are written by the owning lane, large ones cooperatively by the warp.
// ------------------------------------------------------------------------------------------------
// All 32 lanes call with their own Gaussian (tt = 0: nothing to write). TIGHT: rectangles of up to 32 tiles carry the mask
// of the tiles that get an instance (popc(mask) == tt). put(k, key, g) stores instance k (counted from `off`).
template <bool TIGHT, typename Put>
__device__ __forceinline__ void emit_warp(uint32_t g, uint32_t tt, uint32_t off, const uint4 info, int grid_x, int lane, Put put)
{
	const InstRect r(info, TIGHT, tt);
	const uint32_t x0 = r.x0, y0 = r.y0, w = r.w, mask = r.mask;
	const bool masked = r.masked;
	constexpr uint32_t SMALL = 6;
	if (tt > 0 && tt <= SMALL) {
		if (masked) {
			uint32_t m = mask;
			for (uint32_t k = 0; k < tt; k++) {  // the k-th set bit of the mask has rank k
				const uint32_t a = (uint32_t)__ffs(m) - 1u;
				m &= m - 1u;
				put(off + k, (y0 + a / w) * grid_x + x0 + a % w, g);
			}
		} else {
			uint32_t tx = x0, ty = y0;
			for (uint32_t k = 0; k < tt; k++) {
				put(off + k, ty * grid_x + tx, g);
				if (++tx == x0 + w) { tx = x0; ty++; }
			}
		}
	}
	uint32_t big = __ballot_sync(0xffffffffu, tt > SMALL);
	while (big) {
		const int src = __ffs(big) - 1;
		big &= big - 1;
		const uint32_t bg = __shfl_sync(0xffffffffu, g, src);
		const uint32_t btt = __shfl_sync(0xffffffffu, tt, src);
		const uint32_t boff = __shfl_sync(0xffffffffu, off, src);
		const uint32_t bx0 = __shfl_sync(0xffffffffu, x0, src);
		const uint32_t by0 = __shfl_sync(0xffffffffu, y0, src);
		const uint32_t bw = __shfl_sync(0xffffffffu, w, src);
		const uint32_t bmask = __shfl_sync(0xffffffffu, mask, src);
		const bool bmasked = __shfl_sync(0xffffffffu, (int)masked, src) != 0;
		if (bmasked) {  // masked rectangle (<= 32 tiles): lane k owns tile k
			if ((bmask >> lane) & 1u) put(boff + InstRect::rank(true, bmask, lane), (by0 + lane / bw) * grid_x + bx0 + lane % bw, bg);
			continue;
		}
		for (uint32_t k = lane; k < btt; k += 32) put(boff + k, (by0 + k / bw) * grid_x + bx0 + k % bw, bg);
	}
}

// B1/B2 path: offsets come from scan_offsets_kernel, the instance count is known on the host (capacity = num_rendered).
__global__ void __launch_bounds__(256) emit_instances_kernel(int P, const uint32_t* __restrict__ order, const uint4* __restrict__ tile_info,
                                                             const uint32_t* __restrict__ offsets, uint32_t* __restrict__ tile_key,
                                                             uint32_t* __restrict__ inst, int grid_x, uint32_t capacity)
{
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	uint32_t g = 0, tt = 0, off = 0;
	uint4 info = make_uint4(0u, 0u, 0u, 0u);
	if (j < P) {
		g = order[j];
		info = tile_info[g];
		tt = info.z & TT_COUNT;
		off = offsets[j];
	}
	emit_warp<false>(g, tt, off, info, grid_x, threadIdx.x & 31, [&](uint32_t pos, uint32_t key, uint32_t gg) {
		if (pos < capacity) { tile_key[pos] = key; inst[pos] = gg; }
	});
}

// Trainer path: exclusive scan of the instance counts in depth order (single pass, decoupled look-back) and emission in
// ONE kernel — one 16-byte gather per Gaussian, no offsets array. The block's instances are laid out in shared memory at
// their block-local offsets (which need no look-back: warp 0 resolves the block's global prefix meanwhile) and leave as
// one contiguous, coalesced run. counters[0] <- total instance count; instances beyond `capacity` are not written (the
// step then degrades to a no-op, see psb_trainer.cu).
// DET (deterministic mode): also base[g] <- emission offset of every Gaussian with instances (its first instance's index).
constexpr int EM_THREADS = 256, EM_ITEMS = 4, EM_TILE = EM_THREADS * EM_ITEMS;
constexpr int EM_STAGE = 5120;  // instances staged per block (40 KB); a block with more writes to global memory directly
template <bool TIGHT, bool DET = false>
__global__ void __launch_bounds__(EM_THREADS) emit_scan_kernel(int P, const uint32_t* __restrict__ order, const uint4* __restrict__ tile_info,
                                                               uint32_t* __restrict__ tile_key, uint32_t* __restrict__ inst, int grid_x,
                                                               uint32_t capacity, uint32_t* __restrict__ counters, uint32_t* __restrict__ status,
                                                               uint32_t* __restrict__ base_out = nullptr)
{
	__shared__ uint32_t s_key[EM_STAGE], s_ins[EM_STAGE];
	__shared__ uint32_t s_warp[EM_THREADS / 32];
	__shared__ uint32_t s_tile, s_prefix;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (tid == 0) s_tile = atomicAdd(&counters[1], 1u);
	__syncthreads();
	const uint32_t tile = s_tile;
	const int base = (int)tile * EM_TILE + tid * EM_ITEMS;
	uint32_t g[EM_ITEMS], cnt[EM_ITEMS];
	uint4 info[EM_ITEMS];
	if (base + EM_ITEMS <= P) {
		const uint4 o = *reinterpret_cast<const uint4*>(order + base);
		g[0] = o.x; g[1] = o.y; g[2] = o.z; g[3] = o.w;
	} else {
#pragma unroll
		for (int i = 0; i < EM_ITEMS; i++) g[i] = (base + i < P) ? order[base + i] : 0u;
	}
	uint32_t sum = 0;
#pragma unroll
	for (int i = 0; i < EM_ITEMS; i++) {
		info[i] = (base + i < P) ? tile_info[g[i]] : make_uint4(0u, 0u, 0u, 0u);
		cnt[i] = info[i].z & TT_COUNT;
		sum += cnt[i];
	}
	uint32_t inc = sum;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) {
		const uint32_t u = __shfl_up_sync(0xffffffffu, inc, o);
		if (lane >= o) inc += u;
	}
	if (lane == 31) s_warp[warp] = inc;
	__syncthreads();
	uint32_t wb = 0, block_total = 0;
#pragma unroll
	for (int i = 0; i < EM_THREADS / 32; i++) {
		if (i < warp) wb += s_warp[i];
		block_total += s_warp[i];
	}
	const bool staged = block_total <= (uint32_t)EM_STAGE;
	if (warp == 0) {  // publish the aggregate right away, resolve the prefix while the other warps lay out their instances
		const uint32_t excl = lookback_exclusive(status, tile, block_total, lane);
		if (lane == 0) {
			s_prefix = excl;
			if ((int)(tile + 1) * EM_TILE >= P) counters[0] = excl + block_total;
		}
	}
	if (!staged) __syncthreads();  // direct emission needs the global prefix first
	uint32_t run = (staged ? 0u : s_prefix) + wb + inc - sum;
#pragma unroll
	for (int i = 0; i < EM_ITEMS; i++) {
		if (staged)
			emit_warp<TIGHT>(g[i], cnt[i], run, info[i], grid_x, lane, [&](uint32_t pos, uint32_t key, uint32_t gg) { s_key[pos] = key; s_ins[pos] = gg; });
		else
			emit_warp<TIGHT>(g[i], cnt[i], run, info[i], grid_x, lane, [&](uint32_t pos, uint32_t key, uint32_t gg) {
				if (pos < capacity) { tile_key[pos] = key; inst[pos] = gg; }
			});
		run += cnt[i];
	}
	auto write_base = [&](uint32_t prefix) {
		uint32_t o = prefix + wb + inc - sum;
#pragma unroll
		for (int i = 0; i < EM_ITEMS; i++) {
			if (cnt[i] > 0) base_out[g[i]] = o;
			o += cnt[i];
		}
	};
	if (!staged) {
		if (DET) write_base(s_prefix);
		return;
	}
	__syncthreads();
	const uint32_t prefix = s_prefix;
	if (DET) write_base(prefix);
	for (uint32_t k = tid; k < block_total; k += EM_THREADS) {
		const uint32_t pos = prefix + k;
		if (pos < capacity) { tile_key[pos] = s_key[k]; inst[pos] = s_ins[k]; }
	}
}

// B1/B2 path, deterministic backward: scan_offsets_kernel left the emission offset of depth rank j in offsets[j]; the tile backward
// and the gather index by Gaussian, so invert the permutation for the Gaussians that have instances.
__global__ void __launch_bounds__(256) det_base_kernel(int P, const uint32_t* __restrict__ order, const uint4* __restrict__ tile_info,
                                                       const uint32_t* __restrict__ offsets, uint32_t* __restrict__ base)
{
	const int j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= P) return;
	const uint32_t g = order[j];
	if (tile_info[g].z & TT_COUNT) base[g] = offsets[j];
}

// Start/end of every tile in the tile-sorted instance list (semantics of reference
// rasterizer_impl.cu:116-138; ranges must be zeroed beforehand so untouched tiles read {0,0}).
// ovf (trainer path, may be null): sticky record of overflowing views {count, first sequence number, largest instance count}
// kept across steps until the host collects it (psb_trainer_result) — a queued step that degraded to a no-op stays detectable.
__global__ void __launch_bounds__(256) tile_ranges_kernel(const uint32_t* __restrict__ n_dev, uint32_t n_host, const uint32_t* __restrict__ tile_key_sorted,
                                                          uint2* __restrict__ ranges, uint32_t* __restrict__ ovf, uint32_t seq)
{
	const uint32_t n = n_dev ? (*n_dev > n_host ? 0u : *n_dev) : n_host;
	if (ovf && n_dev && blockIdx.x == 0 && threadIdx.x == 0 && *n_dev > n_host) {
		atomicAdd(&ovf[0], 1u);
		atomicMin(&ovf[1], seq);
		atomicMax(&ovf[2], *n_dev);
	}
	for (uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x; idx < n; idx += gridDim.x * blockDim.x) {
		const uint32_t cur = tile_key_sorted[idx];
		if (idx == 0) ranges[cur].x = 0;
		else {
			const uint32_t prev = tile_key_sorted[idx - 1];
			if (cur != prev) { ranges[prev].y = idx; ranges[cur].x = idx; }
		}
		if (idx == n - 1) ranges[cur].y = n;
	}
}

// n_i (normal_axis) of every visible row behind the preprocess. RAW: the trainer's raw parameters (log-scales; the quaternion normalised
// as the preprocess does); otherwise the operator's inputs (activated scales, whose arg-min is that of the log-scales and of the
// modified scales; the rotation as given). The view-space mean is formed exactly as the preprocess does.
template <bool RAW>
__device__ __forceinline__ void normals_body(int P, const float* __restrict__ xyz, const float* __restrict__ scaling,
                                             const float4* __restrict__ rotation, const float* __restrict__ view,
                                             const uint4* __restrict__ tile_info, float4* __restrict__ normals)
{
	const int idx = blockIdx.x * 256 + threadIdx.x;
	if (idx >= P || tile_info[idx].z == 0) return;
	const float3 p = make_float3(xyz[3 * idx], xyz[3 * idx + 1], xyz[3 * idx + 2]);
	const float3 sraw = make_float3(scaling[3 * idx], scaling[3 * idx + 1], scaling[3 * idx + 2]);
	float4 q = rotation[idx];
	if (RAW) {
		const float n = fmaxf(sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w), 1e-12f);
		q = make_float4(q.x / n, q.y / n, q.z / n, q.w / n);
	}
	const NormalAxis a = normal_axis(q, sraw, xform4x3(p, view), view);
	normals[idx] = make_float4(a.n.x, a.n.y, a.n.z, 0.f);
}

// The normal pass's n_i from the raw trainer parameters: a kernel of its own, so the preprocess variants keep their code.
__global__ void __launch_bounds__(256) normals_kernel(int P, const float* __restrict__ xyz, const float* __restrict__ scaling,
                                                      const float4* __restrict__ rotation, const float* __restrict__ view,
                                                      const uint4* __restrict__ tile_info, float4* __restrict__ normals)
{
	normals_body<true>(P, xyz, scaling, rotation, view, tile_info, normals);
}

// The operator's n_i (psb_rasterize_forward_planes / psb_rasterize_backward_planes) from its activated scales and rotations.
__global__ void __launch_bounds__(256) op_normals_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ scales,
                                                         const float4* __restrict__ rotations, const float* __restrict__ view,
                                                         const uint4* __restrict__ tile_info, float4* __restrict__ normals)
{
	normals_body<false>(P, means3D, scales, rotations, view, tile_info, normals);
}

// ------------------------------------------------------------------------------------------------
// Host orchestration
// ------------------------------------------------------------------------------------------------
int launch_preprocess(const GaussIn& in, const Camera& cam, int* radii_out, const GeomState& geom, bool raw, bool tight, cudaStream_t stream, bool aa,
                      const float* f3d)
{
	if (in.P == 0) return 0;
	if (f3d && !raw) { set_error_msg("launch_preprocess: the 3D filter needs the raw trainer parameters"); return -1; }
	const int grid = cdiv(in.P, PRE_TB);
	const int tt = tight ? 1 : 0;
	if (f3d && aa) preprocess_fwd_kernel<true, true, true><<<grid, PRE_TB, 0, stream>>>(in, cam, radii_out, geom, tt, f3d);
	else if (f3d) preprocess_fwd_kernel<true, false, true><<<grid, PRE_TB, 0, stream>>>(in, cam, radii_out, geom, tt, f3d);
	else if (aa && raw) preprocess_fwd_kernel<true, true><<<grid, PRE_TB, 0, stream>>>(in, cam, radii_out, geom, tt, nullptr);
	else if (aa) preprocess_fwd_kernel<false, true><<<grid, PRE_TB, 0, stream>>>(in, cam, radii_out, geom, tt, nullptr);
	else if (raw) preprocess_fwd_kernel<true><<<grid, PRE_TB, 0, stream>>>(in, cam, radii_out, geom, tt, nullptr);
	else preprocess_fwd_kernel<false><<<grid, PRE_TB, 0, stream>>>(in, cam, radii_out, geom, tt, nullptr);
	PSB_LAUNCH_OK();
	return 0;
}

int launch_normals(int P, const float* xyz, const float* scaling, const float* rotation, const Camera& cam, const uint4* tile_info, float4* normals,
                   cudaStream_t stream)
{
	if (P == 0) return 0;
	normals_kernel<<<cdiv(P, 256), 256, 0, stream>>>(P, xyz, scaling, reinterpret_cast<const float4*>(rotation), cam.view, tile_info, normals);
	PSB_LAUNCH_OK();
	return 0;
}

int launch_op_normals(const GaussIn& in, const Camera& cam, const uint4* tile_info, float4* normals, cudaStream_t stream)
{
	if (in.P == 0) return 0;
	op_normals_kernel<<<cdiv(in.P, 256), 256, 0, stream>>>(in.P, in.means3D, in.scales, reinterpret_cast<const float4*>(in.rotations), cam.view,
	                                                      tile_info, normals);
	PSB_LAUNCH_OK();
	return 0;
}

int launch_mark_visible(int P, const float* means3D, const float* view, uint8_t* present, cudaStream_t stream)
{
	if (P == 0) return 0;
	mark_visible_kernel<<<cdiv(P, 256), 256, 0, stream>>>(P, means3D, view, present);
	PSB_LAUNCH_OK();
	return 0;
}

// Depth sort (+ offsets scan when `scan`: the B1/B2 path needs the instance count on the host before it can size the
// binning buffer; the trainer path scans inside emit_scan_kernel). After this geom.order[0] is the depth-sorted
// permutation; with `scan`, geom.offsets holds the instance offsets and geom.counters[0] = num_rendered.
int launch_depth_sort_and_scan(int P, GeomState& geom, bool scan, cudaStream_t stream)
{
	if (P == 0) return 0;
	PSB_CUDA_OK(cudaMemsetAsync(geom.counters, 0, 32 * sizeof(uint32_t), stream));
	PSB_CUDA_OK(cudaMemsetAsync(geom.scan_status, 0, scan_status_words((size_t)P) * sizeof(uint32_t), stream));
	const SortPlan plan = make_sort_plan(32);
	int rc = radix_sort_pairs(geom.depth_key, geom.order, /*iota_vals=*/true, nullptr, (size_t)P, plan, geom.sort_scratch,
	                          geom.sort_scratch_bytes, stream);
	if (rc) return rc;
	// 4 passes -> result back in buffer 0
	if (scan) {
		scan_offsets_kernel<<<cdiv(P, SCAN_TILE), SCAN_THREADS, 0, stream>>>(P, geom.order[0], geom.tile_info, geom.offsets, geom.counters,
		                                                                    geom.scan_status);
		PSB_LAUNCH_OK();
	}
	return 0;
}

int launch_det_base(int P, const GeomState& geom, uint32_t* base, cudaStream_t stream)
{
	if (P == 0) return 0;
	det_base_kernel<<<cdiv(P, 256), 256, 0, stream>>>(P, geom.order[0], geom.tile_info, geom.offsets, base);
	PSB_LAUNCH_OK();
	return 0;
}

static int ranges_grid(size_t n_host)
{
	const size_t want = (n_host + 255) / 256;
	return (int)(want < kNumSMs * 16 ? (want ? want : 1) : kNumSMs * 16);
}

// B1/B2 path: emit + tile sort + ranges for a known instance count R (= n_host; the binning chunk was carved for it).
int launch_binning(int P, const Camera& cam, const GeomState& geom, BinState& bin, const ImgState& img, size_t n_host, cudaStream_t stream)
{
	const int num_tiles = cam.grid_x * cam.grid_y;
	PSB_CUDA_OK(cudaMemsetAsync(img.ranges, 0, (size_t)num_tiles * sizeof(uint2), stream));
	if (P == 0 || n_host == 0) return 0;
	emit_instances_kernel<<<cdiv(P, 256), 256, 0, stream>>>(P, geom.order[0], geom.tile_info, geom.offsets, bin.tile_key[0], bin.inst[0], cam.grid_x,
	                                                       (uint32_t)n_host);
	PSB_LAUNCH_OK();
	const SortPlan plan = make_sort_plan(tile_id_bits(num_tiles));
	int rc = radix_sort_pairs(bin.tile_key, bin.inst, false, nullptr, n_host, plan, bin.sort_scratch, bin.sort_scratch_bytes, stream);
	if (rc) return rc;
	tile_ranges_kernel<<<ranges_grid(n_host), 256, 0, stream>>>(nullptr, (uint32_t)n_host, bin.tile_key[plan.result()], img.ranges, nullptr, 0u);
	PSB_LAUNCH_OK();
	return 0;
}

// Trainer path: scan + emit in one kernel, tile sort, ranges. The instance count stays on the device
// (geom.counters[0]); `capacity` = size the binning chunk was carved for.
int launch_scan_binning(int P, const Camera& cam, const GeomState& geom, BinState& bin, const ImgState& img, size_t capacity, bool tight,
                        uint32_t* ovf, uint32_t seq, cudaStream_t stream, uint32_t* base)
{
	const int num_tiles = cam.grid_x * cam.grid_y;
	PSB_CUDA_OK(cudaMemsetAsync(img.ranges, 0, (size_t)num_tiles * sizeof(uint2), stream));
	if (P == 0 || capacity == 0) return 0;
	const SortPlan plan = make_sort_plan(tile_id_bits(num_tiles));
	if (base) {
		if (tight)
			emit_scan_kernel<true, true><<<cdiv(P, EM_TILE), EM_THREADS, 0, stream>>>(P, geom.order[0], geom.tile_info, bin.tile_key[0], bin.inst[0], cam.grid_x,
			                                                                        (uint32_t)capacity, geom.counters, geom.scan_status, base);
		else
			emit_scan_kernel<false, true><<<cdiv(P, EM_TILE), EM_THREADS, 0, stream>>>(P, geom.order[0], geom.tile_info, bin.tile_key[0], bin.inst[0], cam.grid_x,
			                                                                         (uint32_t)capacity, geom.counters, geom.scan_status, base);
	} else if (tight)
		emit_scan_kernel<true><<<cdiv(P, EM_TILE), EM_THREADS, 0, stream>>>(P, geom.order[0], geom.tile_info, bin.tile_key[0], bin.inst[0], cam.grid_x,
		                                                                  (uint32_t)capacity, geom.counters, geom.scan_status);
	else
		emit_scan_kernel<false><<<cdiv(P, EM_TILE), EM_THREADS, 0, stream>>>(P, geom.order[0], geom.tile_info, bin.tile_key[0], bin.inst[0], cam.grid_x,
		                                                                   (uint32_t)capacity, geom.counters, geom.scan_status);
	PSB_LAUNCH_OK();
	int rc = radix_sort_pairs(bin.tile_key, bin.inst, false, geom.counters, capacity, plan, bin.sort_scratch, bin.sort_scratch_bytes, stream);
	if (rc) return rc;
	tile_ranges_kernel<<<ranges_grid(capacity), 256, 0, stream>>>(geom.counters, (uint32_t)capacity, bin.tile_key[plan.result()], img.ranges, ovf, seq);
	PSB_LAUNCH_OK();
	return 0;
}

}  // namespace psb
