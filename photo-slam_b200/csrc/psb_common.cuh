// psb200 — Hopper-native Gaussian-splatting rasterizer / trainer step (sm_90a, H100).
// Shared device helpers. Nothing here depends on torch; everything is plain CUDA.
#pragma once
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <cuda_runtime.h>

#define PSB_TILE_X 16
#define PSB_TILE_Y 16
#define PSB_TILE_PIX (PSB_TILE_X * PSB_TILE_Y)

// Error plumbing: every host entry point returns 0 on success or a negative psb error code and keeps
// the CUDA error string retrievable through psb_last_error().
namespace psb {

void set_error(const char* what, cudaError_t e, const char* file, int line);
void set_error_msg(const char* what);

#define PSB_CUDA_OK(expr)                                              \
	do {                                                               \
		cudaError_t _e = (expr);                                       \
		if (_e != cudaSuccess) {                                       \
			psb::set_error(#expr, _e, __FILE__, __LINE__);             \
			return -2;                                                 \
		}                                                              \
	} while (0)

#define PSB_LAUNCH_OK()                                                \
	do {                                                               \
		cudaError_t _e = cudaGetLastError();                           \
		if (_e != cudaSuccess) {                                       \
			psb::set_error("kernel launch", _e, __FILE__, __LINE__);   \
			return -2;                                                 \
		}                                                              \
	} while (0)

// ---- Owned CUDA memory: nothing is freed by hand ----
// How CudaBuffer::grow treats a buffer that already exists: keep it only at exactly the requested count, or at any count at least that
// large.
enum class Fit { exact, at_least };

// The bytes of `count` elements of T. A chunk that one scratch state is carved from counts rows of that state instead (StateBytes,
// psb_state.h).
template <typename T>
struct ElementBytes {
	static size_t of(size_t count) { return count * sizeof(T); }
};

// One allocation and the count of elements it was made for: device memory, or page-locked host memory when `Pinned`, with `Slack`
// bytes past the elements. Not copyable; the destructor frees it.
template <typename T, size_t Slack = 0, bool Pinned = false, typename Bytes = ElementBytes<T>>
class CudaBuffer {
public:
	CudaBuffer() = default;
	CudaBuffer(const CudaBuffer&) = delete;
	CudaBuffer& operator=(const CudaBuffer&) = delete;
	~CudaBuffer() { release(); }

	T* get() const { return p_; }
	size_t count() const { return count_; }

	// Keeps the buffer if it holds `count` elements (Fit::exact) or at least that many (Fit::at_least). Otherwise drains `stream` (work
	// on it may still use the old buffer), frees the old buffer, allocates Bytes::of(count) + Slack bytes and, when `zero`, zeroes the
	// elements on `stream` (pinned memory: on the host). After a failed allocation the buffer is empty (null, count 0), so the next call
	// allocates again, and the error is reported only through the return value: it is taken off the runtime's last error, where a later
	// launch check would find it.
	cudaError_t grow(size_t count, Fit fit, bool zero, cudaStream_t stream)
	{
		if (fit == Fit::exact ? p_ && count_ == count : count_ >= count) return cudaSuccess;
		cudaError_t e;
		if (p_) {
			if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
			release();
		}
		const size_t bytes = Bytes::of(count);
		void* p = nullptr;
		e = Pinned ? cudaMallocHost(&p, bytes + Slack) : cudaMalloc(&p, bytes + Slack);
		if (e != cudaSuccess) {
			cudaGetLastError();
			return e;
		}
		p_ = static_cast<T*>(p);
		count_ = count;
		if (zero) {
			if (Pinned) memset(p, 0, bytes);
			else if ((e = cudaMemsetAsync(p, 0, bytes, stream)) != cudaSuccess) release();
		}
		return e;
	}

private:
	void release()
	{
		if (p_) Pinned ? cudaFreeHost(p_) : cudaFree(p_);
		p_ = nullptr;
		count_ = 0;
	}
	T* p_ = nullptr;
	size_t count_ = 0;
};

// Stream-ordered scratch of one call: alloc() takes it with cudaMallocAsync on `stream`, and it goes back with cudaFreeAsync on the
// same stream when the scope ends, on every path out of it.
template <typename T>
class StreamScratch {
public:
	explicit StreamScratch(cudaStream_t stream) : stream_(stream) {}
	StreamScratch(const StreamScratch&) = delete;
	StreamScratch& operator=(const StreamScratch&) = delete;
	~StreamScratch()
	{
		if (p_) cudaFreeAsync(p_, stream_);
	}

	// once per scope
	cudaError_t alloc(size_t count)
	{
		void* p = nullptr;
		const cudaError_t e = cudaMallocAsync(&p, count * sizeof(T), stream_);
		if (e == cudaSuccess) p_ = static_cast<T*>(p);
		return e;
	}
	T* get() const { return p_; }

private:
	cudaStream_t stream_;
	T* p_ = nullptr;
};

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// SMs of an H100 SXM: caps the grids of the grid-stride kernels at a few resident blocks per SM.
constexpr int kNumSMs = 132;

// Floats per Gaussian row of the six parameter tensors, in psb_model.param order: xyz, features_dc, features_rest (15 SH coefficients
// x 3 channels: every entry point that moves rows or steps Adam requires all 16 coefficients), opacity, scaling, rotation. The Adam
// moments have the same rows.
__host__ __device__ constexpr int row_floats(int tensor)
{
	constexpr int k[6] = {3, 3, 45, 1, 3, 4};
	return k[tensor];
}
constexpr int kRestFloats = row_floats(2);

// ---------------------------------------------------------------------------------------------
// Per-Gaussian screen-space record produced by the forward preprocess and consumed (as one
// 48-byte bulk copy) by the tile kernels. 16-byte aligned, three float4 lanes:
//   q0 = (mean2D.x, mean2D.y, conic.a, conic.b)
//   q1 = (conic.c,  opacity,  pmin,    depth)      pmin = -(ln(255 * opacity) + 1e-3): a pixel whose exponent
//                                                   `power` is below pmin cannot reach alpha >= 1/255, so the tile
//                                                   kernels skip exp() for it (the exact alpha test still decides
//                                                   everything at or above pmin)
//   q2 = (rgb.r,    rgb.g,    rgb.b,   meta)       meta bits: radius << 3 | SH clamp flag per channel (bits 0..2)
// ---------------------------------------------------------------------------------------------
struct __align__(16) GaussRec {
	float4 q0, q1, q2;
};
static_assert(sizeof(GaussRec) == 48, "GaussRec must be 48 bytes");
__host__ __device__ __forceinline__ int rec_radius(uint32_t meta) { return (int)(meta >> 3); }
__host__ __device__ __forceinline__ uint32_t rec_clamp_bits(uint32_t meta) { return meta & 7u; }

// Camera block passed by value to the per-Gaussian kernels. The 4x4 matrices stay where the caller put
// them (device memory, column-major m[4*c + r] exactly as the reference passes them, e.g.
// reference rasterize_points.cu:104-106) so that no host round trip is needed at the boundary.
struct Camera {
	const float* view;    // world -> view, 16 floats
	const float* proj;    // world -> clip (view * projection), 16 floats
	const float* campos;  // camera centre, 3 floats
	float tan_fovx, tan_fovy;
	float focal_x, focal_y;
	int W, H;
	int grid_x, grid_y;
};

// Spherical-harmonics basis constants (real SH up to degree 3, the standard 3DGS convention; same
// values as reference cuda_rasterizer/auxiliary.h:22-39). constexpr scalars: usable in device code.
constexpr float kSH_C0 = 0.28209479177387814f;
constexpr float kSH_C1 = 0.4886025119029199f;
constexpr float kSH_C2_0 = 1.0925484305920792f;
constexpr float kSH_C2_1 = -1.0925484305920792f;
constexpr float kSH_C2_2 = 0.31539156525252005f;
constexpr float kSH_C2_3 = -1.0925484305920792f;
constexpr float kSH_C2_4 = 0.5462742152960396f;
constexpr float kSH_C3_0 = -0.5900435899266435f;
constexpr float kSH_C3_1 = 2.890611442640554f;
constexpr float kSH_C3_2 = -0.4570457994644658f;
constexpr float kSH_C3_3 = 0.3731763325901154f;
constexpr float kSH_C3_4 = -0.4570457994644658f;
constexpr float kSH_C3_5 = 1.445305721320277f;
constexpr float kSH_C3_6 = -0.5900435899266435f;

// ---- tiny column-major 3x3 (M[c][r] at m[3c+r]); products are written as three-term sums in the
// order  a[0][r]*b[c][0] + a[1][r]*b[c][1] + a[2][r]*b[c][2]  so nvcc contracts them exactly like the
// reference's glm expressions (bit-exact radii / tile rects depend on it; checked against the
// reference's outputs by tests/test_parity_ref_gpu.py).
struct Mat3 {
	float m[9];
	__device__ __forceinline__ float& operator()(int c, int r) { return m[3 * c + r]; }
	__device__ __forceinline__ float operator()(int c, int r) const { return m[3 * c + r]; }
};
__device__ __forceinline__ Mat3 mat3_mul(const Mat3& a, const Mat3& b)
{
	Mat3 r;
#pragma unroll
	for (int c = 0; c < 3; c++)
#pragma unroll
		for (int rr = 0; rr < 3; rr++)
			r(c, rr) = a(0, rr) * b(c, 0) + a(1, rr) * b(c, 1) + a(2, rr) * b(c, 2);
	return r;
}
__device__ __forceinline__ Mat3 mat3_transpose(const Mat3& a)
{
	Mat3 r;
#pragma unroll
	for (int c = 0; c < 3; c++)
#pragma unroll
		for (int rr = 0; rr < 3; rr++) r(c, rr) = a(rr, c);
	return r;
}

__device__ __forceinline__ float3 xform4x3(const float3 p, const float* m)
{
	return make_float3(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12],
	                   m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
	                   m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14]);
}
__device__ __forceinline__ float4 xform4x4(const float3 p, const float* m)
{
	return make_float4(m[0] * p.x + m[4] * p.y + m[8] * p.z + m[12],
	                   m[1] * p.x + m[5] * p.y + m[9] * p.z + m[13],
	                   m[2] * p.x + m[6] * p.y + m[10] * p.z + m[14],
	                   m[3] * p.x + m[7] * p.y + m[11] * p.z + m[15]);
}

// Pixel centre from NDC. Evaluated in double like the reference (cuda_rasterizer/auxiliary.h:41-44):
// the tile rectangle, and therefore every (tile|depth) key, depends on this rounding.
__device__ __forceinline__ float ndc_to_pix(float v, int S) { return ((v + 1.0) * S - 1.0) * 0.5; }

// Tile rectangle of a splat (reference semantics, cuda_rasterizer/auxiliary.h:46-56): truncation toward
// zero, then clamp to [0, grid].
__device__ __forceinline__ void tile_rect(float px, float py, int max_radius, int gx, int gy,
                                          int& x0, int& y0, int& x1, int& y1)
{
	x0 = min(gx, max(0, (int)((px - max_radius) / PSB_TILE_X)));
	y0 = min(gy, max(0, (int)((py - max_radius) / PSB_TILE_Y)));
	x1 = min(gx, max(0, (int)((px + max_radius + PSB_TILE_X - 1) / PSB_TILE_X)));
	y1 = min(gy, max(0, (int)((py + max_radius + PSB_TILE_Y - 1) / PSB_TILE_Y)));
}

// Exponent of a splat at offset d = mean - pixel:  power = -0.5 (A dx^2 + C dy^2) - B dx dy.
// Which products get fused decides the last bit of `power`, hence (rarely) whether alpha passes 1/255 or T passes
// 1e-4, hence n_contrib. The operation order below is the one the reference's kernels compile to (SASS of reference
// forward.cu:336 and backward.cu:489: FFMA(dx, A*dx, (C*dy)*dy), then FFMA(sum, -0.5, -((B*dx)*dy))); explicit
// intrinsics keep it independent of how the surrounding code is unrolled.
__device__ __forceinline__ float splat_power(float A, float B, float C, float dx, float dy)
{
	const float s = __fmaf_rn(dx, __fmul_rn(A, dx), __fmul_rn(dy, __fmul_rn(C, dy)));
	return __fmaf_rn(s, -0.5f, -__fmul_rn(dy, __fmul_rn(B, dx)));
}

// Can this splat reach alpha >= 1/255 on any pixel of the pixel rectangle [px0,px1] x [py0,py1]?
// q(d) = 0.5 (A dx^2 + C dy^2) + B dx dy, d = mean - pixel; a contribution needs q <= ln(255 * opacity) = -(pmin + 1e-3)
// (GaussRec.q1.z). Returns false only when q exceeds that bound (+ a rounding pad) on the WHOLE rectangle, so dropping
// the splat for that rectangle never changes a pixel.
// q is a convex quadratic with its minimum (0) at d = 0. If the box does not contain 0, q(t p) = t^2 q(p) shrinks along
// the segment from any box point p towards 0, so the box minimum sits on an edge FACING the origin: the edge
// dx = dxlo when dxlo > 0 (dx = dxhi when dxhi < 0), and the same in y — at most two edges, and on each the 1-D minimum
// is q at the clamped stationary point (corners included by the clamp).
__device__ __forceinline__ float splat_q(float A, float B, float C, float dx, float dy)
{
	const float s = __fmaf_rn(__fmul_rn(A, dx), dx, __fmul_rn(__fmul_rn(C, dy), dy));
	return __fmaf_rn(__fmul_rn(B, dx), dy, __fmul_rn(0.5f, s));
}
struct TileCull {
	float mx, my, A, B, C, thr, nbc, nba;
	bool none, all;  // opacity below 1/255: never; conic not positive definite (numerically): always keep
	__device__ __forceinline__ TileCull(const float4 q0, const float4 q1)
	{
		mx = q0.x; my = q0.y; A = q0.z; B = q0.w; C = q1.x; thr = -q1.z;
		nbc = __fdividef(-B, C); nba = __fdividef(-B, A);  // approximate: a displaced edge point only raises q in second order
		none = q1.y < (1.0f / 255.0f);
		all = !(A > 0.f && C > 0.f && A * C > B * B);
	}
	__device__ __forceinline__ bool reaches(float px0, float py0, float px1, float py1) const
	{
		if (none) return false;
		const float dxlo = mx - px1, dxhi = mx - px0, dylo = my - py1, dyhi = my - py0;
		const bool xin = dxlo <= 0.f && dxhi >= 0.f, yin = dylo <= 0.f && dyhi >= 0.f;
		if ((xin && yin) || all) return true;  // centre inside: q = 0 reachable
		const float dxm = fmaxf(fabsf(dxlo), fabsf(dxhi)), dym = fmaxf(fabsf(dylo), fabsf(dyhi));
		const float pad = __fmaf_rn(1e-5f, splat_q(A, fabsf(B), C, dxm, dym), 1e-4f);
		float qmin = 3.0e38f;
		if (!xin) {  // vertical edge facing the centre
			const float ex = dxlo > 0.f ? dxlo : dxhi;
			qmin = splat_q(A, B, C, ex, fminf(fmaxf(nbc * ex, dylo), dyhi));
		}
		if (!yin) {  // horizontal edge facing the centre
			const float ey = dylo > 0.f ? dylo : dyhi;
			qmin = fminf(qmin, splat_q(A, B, C, fminf(fmaxf(nba * ey, dxlo), dxhi), ey));
		}
		return !(qmin > thr + pad);
	}
	// Bit k (row-major) = tile k of the tile rectangle [x0,x1) x [y0,y1) (at most 32 tiles) of a W x H image can be reached.
	// O(rows), not O(tiles): the level set {q <= t} is an ellipse; over a band of tile rows dy in [lo, hi] its dx-extent is the
	// interval [xl, xr] with the closed form  dx = (-B dy +- sqrt(2 t A - det dy^2)) / A  evaluated where the band is widest (the
	// ellipse's own dx-extremes sit at dy = -+B sqrt(2t / (det C)), clamped into the band). A tile of the row is kept iff its
	// pixel columns meet the interval: a contiguous run of tiles -> a run of mask bits, no per-tile loop. One rounding pad (t) for the
	// whole rectangle plus a relative pad on the interval: always a superset of the tiles with a pixel at alpha >= 1/255
	// (numpy restatement checked against brute-force per-pixel evaluation: tests/test_cull_cpu.py).
	__device__ __forceinline__ uint32_t rect_mask(int x0, int y0, int x1, int y1, int W, int H) const
	{
		const int w = x1 - x0, area = w * (y1 - y0);
		const uint32_t full = area >= 32 ? 0xffffffffu : ((1u << area) - 1u);
		if (none) return 0u;
		const float det = __fsub_rn(__fmul_rn(A, C), __fmul_rn(B, B));
		if (all || !(det > 0.f)) return full;
		const float DX = fmaxf(fabsf(mx - (float)(x0 * PSB_TILE_X)), fabsf(mx - (float)(min(x1 * PSB_TILE_X, W) - 1)));
		const float DY = fmaxf(fabsf(my - (float)(y0 * PSB_TILE_Y)), fabsf(my - (float)(min(y1 * PSB_TILE_Y, H) - 1)));
		const float t = thr + __fmaf_rn(1e-5f, splat_q(A, fabsf(B), C, DX, DY), 1e-4f);
		const float t2 = 2.f * t;
		const float Y = sqrtf(__fdiv_rn(__fmul_rn(t2, A), det));                       // |dy| extent of the ellipse
		const float dyr = __fmul_rn(-B, sqrtf(__fdiv_rn(t2, __fmul_rn(det, C))));      // dy at which dx is largest
		const float invA = __fdiv_rn(1.f, A), t2A = __fmul_rn(t2, A);
		uint32_t mask = 0u;
		for (int ty = y0; ty < y1; ty++) {
			const int py0 = ty * PSB_TILE_Y;
			const float dylo = my - (float)(min(py0 + PSB_TILE_Y, H) - 1), dyhi = my - (float)py0;
			const float lo = fmaxf(dylo, -Y), hi = fminf(dyhi, Y);
			if (lo > hi) continue;                                                       // the band misses the ellipse
			const float ya = fminf(fmaxf(dyr, lo), hi), yb = fminf(fmaxf(-dyr, lo), hi);
			const float Da = fmaxf(__fsub_rn(t2A, __fmul_rn(__fmul_rn(det, ya), ya)), 0.f);
			const float Db = fmaxf(__fsub_rn(t2A, __fmul_rn(__fmul_rn(det, yb), yb)), 0.f);
			float xr = __fmul_rn(__fadd_rn(__fmul_rn(-B, ya), sqrtf(Da)), invA);
			float xl = __fmul_rn(__fsub_rn(__fmul_rn(-B, yb), sqrtf(Db)), invA);
			const float e = __fmul_rn(1e-4f, __fadd_rn(fmaxf(fabsf(xl), fabsf(xr)), 1.f));
			xr = __fadd_rn(xr, e); xl = __fsub_rn(xl, e);
			// tile tx holds pixel columns [16 tx, 16 tx + 15] (the image edge only shortens it: treating it as full keeps a superset);
			// dx = mx - column: kept iff  mx - xr <= 16 tx + 15  and  16 tx <= mx - xl
			const int tlo = max(x0, (int)ceilf(__fmul_rn(__fsub_rn(__fsub_rn(mx, xr), 15.f), 0.0625f)));
			const int thi = min(x1 - 1, (int)floorf(__fmul_rn(__fsub_rn(mx, xl), 0.0625f)));
			if (tlo <= thi) mask |= ((2u << (thi - tlo)) - 1u) << ((ty - y0) * w + (tlo - x0));
		}
		return mask;
	}
};
__device__ __forceinline__ bool splat_reaches_tile(const float4 q0, const float4 q1, float px0, float py0, float px1, float py1)
{
	return TileCull(q0, q1).reaches(px0, py0, px1, py1);
}
constexpr uint32_t TT_VISIBLE = 0x80000000u;  // tight lists: tiles_touched = exact count | this flag (Gaussian passed the culls)
constexpr uint32_t TT_COUNT = 0x7FFFFFFFu;
constexpr int TIGHT_MAX_AREA = 32;             // larger rectangles keep every tile (one 32-bit mask per Gaussian, bounded loop)

// The instances of one Gaussian (tile_info = GeomState::tile_info[g], tt = its instance count): the tiles of its rectangle,
// row-major, and on a tight list over at most TIGHT_MAX_AREA tiles only those of the mask. emit_warp emits them in this order and
// the deterministic tile backward stores the flush of (Gaussian, tile) at the same rank, so both take the order from here.
struct InstRect {
	uint32_t x0, y0, w, mask;
	bool masked;
	__device__ __forceinline__ InstRect(const uint4 info, bool tight, uint32_t tt)
	{
		x0 = info.x & 0xFFFFu;
		y0 = info.x >> 16;
		w = max((info.y & 0xFFFFu) - x0, 1u);
		masked = tight && tt > 0 && w * ((info.y >> 16) - y0) <= (uint32_t)TIGHT_MAX_AREA;
		mask = masked ? info.w : 0xffffffffu;
	}
	// rank among the Gaussian's instances of tile a (row-major in the rectangle), which must be one of its instances
	static __device__ __forceinline__ uint32_t rank(bool masked, uint32_t mask, uint32_t a)
	{
		return masked ? (uint32_t)__popc(mask & ((1u << a) - 1u)) : a;
	}
	__device__ __forceinline__ uint32_t rank_of(uint32_t tx, uint32_t ty) const { return rank(masked, mask, (ty - y0) * w + (tx - x0)); }
};

// ---- async-copy / mbarrier PTX wrappers (TMA 1-D bulk copies) ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init()
{
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
	asm volatile(
		"{\n"
		".reg .pred p;\n"
		"WAIT_LOOP:\n"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
		"@p bra DONE;\n"
		"bra WAIT_LOOP;\n"
		"DONE:\n"
		"}\n" ::"r"(smem_u32(bar)),
		"r"(parity)
		: "memory");
}
// 1-D bulk async copy global -> shared (TMA engine, SASS UBLKCP); bytes must be a multiple of 16 and
// both addresses 16-byte aligned. Completion is signalled on the mbarrier as transaction bytes.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
	             "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
	             : "memory");
}
// 4-byte asynchronous copy global -> shared (SASS LDGSTS): no register staging; complete (for the issuing thread) after cp_async_wait_all
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gmem_src)
{
	asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gmem_src) : "memory");
}
// brings the 128-byte line holding `gmem` into L2 with the evict-last priority (a later load of it hits L2); no register, no wait
__device__ __forceinline__ void prefetch_l2_evict_last(const void* gmem)
{
	asm volatile("prefetch.global.L2::evict_last [%0];" ::"l"(gmem));
}
__device__ __forceinline__ void cp_async_wait_all()
{
	asm volatile("cp.async.wait_all;" ::: "memory");
}

}  // namespace psb
