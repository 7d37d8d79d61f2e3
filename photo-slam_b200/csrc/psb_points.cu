// Point-cloud helpers that live in the same shared objects as the rasterizer in the reference:
//   psb_dist_cuda2                  mean squared distance to the 3 nearest neighbours (scale initialisation of new
//                                   Gaussians) — reference third_party/simple-knn/simple_knn.cu:185-221, spatial.cu:15-26
//   psb_transform_points            p' = M p                          — reference src/operate_points.cu:38-50, 73-93
//   psb_scale_transform_points      masked p' = M (s p), q' = quat(M3x3 R(q)) — src/operate_points.cu:52-71,
//                                   cuda_rasterizer/operate_points.h:55-178
// simple-knn here: no cudaMalloc / thrust vectors / blocking copies per call (the reference does 7 allocations and 2
// host round trips): bounds are reduced on the device, scratch comes from the stream-ordered allocator, the Morton
// sort is the library's own onesweep radix sort.
#include <cfloat>
#include "psb_kernels.h"
#include "../../include/psb200.h"

namespace psb {

namespace {


__device__ __forceinline__ uint32_t f2ord(float f) { const uint32_t u = __float_as_uint(f); return (u & 0x80000000u) ? ~u : (u | 0x80000000u); }
__device__ __forceinline__ float ord2f(uint32_t o) { return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o); }

// bounds[0..2] = min xyz, bounds[3..5] = max xyz as order-preserving uints
__global__ void knn_bounds_kernel(int P, const float* __restrict__ pts, uint32_t* __restrict__ bounds)
{
	float mn[3] = {FLT_MAX, FLT_MAX, FLT_MAX}, mx[3] = {-FLT_MAX, -FLT_MAX, -FLT_MAX};
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < P; i += gridDim.x * blockDim.x) {
#pragma unroll
		for (int c = 0; c < 3; c++) { const float v = pts[3 * i + c]; mn[c] = fminf(mn[c], v); mx[c] = fmaxf(mx[c], v); }
	}
#pragma unroll
	for (int c = 0; c < 3; c++) {
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) { mn[c] = fminf(mn[c], __shfl_xor_sync(0xffffffffu, mn[c], o)); mx[c] = fmaxf(mx[c], __shfl_xor_sync(0xffffffffu, mx[c], o)); }
	}
	if ((threadIdx.x & 31) == 0) {
#pragma unroll
		for (int c = 0; c < 3; c++) { atomicMin(&bounds[c], f2ord(mn[c])); atomicMax(&bounds[3 + c], f2ord(mx[c])); }
	}
}

__device__ __forceinline__ uint32_t prep_morton(uint32_t x)
{
	x = (x | (x << 16)) & 0x030000FF;
	x = (x | (x << 8)) & 0x0300F00F;
	x = (x | (x << 4)) & 0x030C30C3;
	x = (x | (x << 2)) & 0x09249249;
	return x;
}

__global__ void knn_morton_kernel(int P, const float* __restrict__ pts, const uint32_t* __restrict__ bounds, uint32_t* __restrict__ codes)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	uint32_t code = 0;
#pragma unroll
	for (int c = 0; c < 3; c++) {
		const float mn = ord2f(bounds[c]), mx = ord2f(bounds[3 + c]);
		const float ext = mx - mn;
		const float n = ext > 0.f ? (pts[3 * i + c] - mn) / ext : 0.f;
		code |= prep_morton((uint32_t)(n * 1023.0f)) << c;
	}
	codes[i] = code;
}

// ------------------------------------------------------------------------------------------------------------------------
// Exact 3-nearest-neighbour search, block-cooperative (the reference, simple_knn.cu:147-183, lets every thread walk all boxes
// of 1024 points on its own, gathering candidates one by one from global memory through the Morton permutation).
//
//   * the points are copied once into Morton order as float4 (xyz + original index): candidate tiles are contiguous;
//   * a block owns one tile of 256 queries (one per thread, in registers) and visits the candidate tiles outwards from its own
//     (b, b+1, b-1, b+2, ...: Morton neighbours first, so the 3rd-best distances shrink early);
//   * a tile is skipped for the WHOLE block when the gap between the two tiles' bounding boxes exceeds the largest 3rd-best
//     distance any query of the block still has (one uniform test per tile pair instead of 256 per-thread box tests);
//   * a tile that survives is staged in shared memory once (coalesced 16-byte loads) and every query that its own point-to-box
//     test lets through scans it there: all lanes read the same candidate -> shared-memory broadcasts instead of gathers;
//   * the three smallest squared distances are kept by a branch-free min/max insertion network.
// The result is the exact 3-NN mean of squared distances like the reference's (any exact search returns the same three values).
// ------------------------------------------------------------------------------------------------------------------------
constexpr int KNN_TILE = 256;
struct Box { float mn[3], mx[3]; };

__global__ void knn_gather_kernel(int P, const float* __restrict__ pts, const uint32_t* __restrict__ order, float4* __restrict__ sorted)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const uint32_t g = order[i];
	sorted[i] = make_float4(pts[3 * g], pts[3 * g + 1], pts[3 * g + 2], __uint_as_float(g));
}

__global__ void __launch_bounds__(KNN_TILE) knn_tile_box_kernel(int P, const float4* __restrict__ sorted, Box* __restrict__ boxes)
{
	__shared__ float s_red[6][KNN_TILE / 32];
	const int i = blockIdx.x * KNN_TILE + threadIdx.x;
	float v[6] = {FLT_MAX, FLT_MAX, FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX};
	if (i < P) {
		const float4 p = sorted[i];
		v[0] = v[3] = p.x; v[1] = v[4] = p.y; v[2] = v[5] = p.z;
	}
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
	for (int c = 0; c < 6; c++) {
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) {
			const float u = __shfl_xor_sync(0xffffffffu, v[c], o);
			v[c] = c < 3 ? fminf(v[c], u) : fmaxf(v[c], u);
		}
		if (lane == 0) s_red[c][warp] = v[c];
	}
	__syncthreads();
	if (threadIdx.x < 6) {
		const int c = threadIdx.x;
		float r = s_red[c][0];
#pragma unroll
		for (int w = 1; w < KNN_TILE / 32; w++) r = c < 3 ? fminf(r, s_red[c][w]) : fmaxf(r, s_red[c][w]);
		if (c < 3) boxes[blockIdx.x].mn[c] = r;
		else boxes[blockIdx.x].mx[c - 3] = r;
	}
}

__device__ __forceinline__ float axis_gap(float lo_a, float hi_a, float lo_b, float hi_b) { return fmaxf(0.f, fmaxf(lo_b - hi_a, lo_a - hi_b)); }

__global__ void __launch_bounds__(KNN_TILE) knn_search_kernel(int P, int ntile, const float4* __restrict__ sorted, const Box* __restrict__ boxes,
                                                            float* __restrict__ dists)
{
	__shared__ float4 s_tile[KNN_TILE];
	__shared__ float s_wmax[KNN_TILE / 32];
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int my = blockIdx.x;
	const int qi = my * KNN_TILE + tid;
	const bool valid = qi < P;
	const float4 q = valid ? sorted[qi] : make_float4(0.f, 0.f, 0.f, 0.f);
	const Box Q = boxes[my];
	float b0 = FLT_MAX, b1 = FLT_MAX, b2 = FLT_MAX;   // three smallest squared distances, ascending
	float rmax = FLT_MAX;                              // largest b2 over the block's queries (uniform)
	const int reach = max(my, ntile - 1 - my);
	for (int k = 0; k <= reach; k++) {
#pragma unroll
		for (int side = 0; side < 2; side++) {
			const int t = side == 0 ? my + k : my - k;
			if ((side == 1 && k == 0) || t < 0 || t >= ntile) continue;   // uniform
			const Box B = boxes[t];
			const float gx = axis_gap(Q.mn[0], Q.mx[0], B.mn[0], B.mx[0]), gy = axis_gap(Q.mn[1], Q.mx[1], B.mn[1], B.mx[1]),
			            gz = axis_gap(Q.mn[2], Q.mx[2], B.mn[2], B.mx[2]);
			if (gx * gx + gy * gy + gz * gz > rmax) continue;             // no query of this block can gain from that tile (uniform)
			__syncthreads();                                               // previous tile fully consumed
			const int ci = t * KNN_TILE + tid;
			s_tile[tid] = ci < P ? sorted[ci] : make_float4(FLT_MAX, FLT_MAX, FLT_MAX, 0.f);
			__syncthreads();
			if (valid) {
				const float px = axis_gap(q.x, q.x, B.mn[0], B.mx[0]), py = axis_gap(q.y, q.y, B.mn[1], B.mx[1]), pz = axis_gap(q.z, q.z, B.mn[2], B.mx[2]);
				if (!(px * px + py * py + pz * pz > b2)) {
					const int self = t == my ? tid : -1;
					const int cnt = min(KNN_TILE, P - t * KNN_TILE);
					for (int j = 0; j < cnt; j++) {
						const float4 c = s_tile[j];
						const float dx = c.x - q.x, dy = c.y - q.y, dz = c.z - q.z;
						float d = dx * dx + dy * dy + dz * dz;
						if (j == self) d = FLT_MAX;
						const float t0 = fmaxf(b0, d); b0 = fminf(b0, d);
						const float t1 = fmaxf(b1, t0); b1 = fminf(b1, t0);
						b2 = fminf(b2, t1);
					}
				}
			}
			// refresh the block-wide bound
			float m = valid ? b2 : 0.f;
#pragma unroll
			for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
			__syncthreads();
			if (lane == 0) s_wmax[warp] = m;
			__syncthreads();
			rmax = s_wmax[0];
#pragma unroll
			for (int w = 1; w < KNN_TILE / 32; w++) rmax = fmaxf(rmax, s_wmax[w]);
		}
	}
	if (valid) dists[__float_as_uint(q.w)] = (b0 + b1 + b2) / 3.0f;
}

__global__ void transform_points_kernel(int P, const float* __restrict__ pts, const float* __restrict__ m, float* __restrict__ out)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const float3 p = xform4x3(make_float3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]), m);
	out[3 * i] = p.x; out[3 * i + 1] = p.y; out[3 * i + 2] = p.z;
}

__global__ void scale_transform_points_kernel(int P, float scale, const float* __restrict__ pts, const float* __restrict__ rots,
                                              const float* __restrict__ m, const uint8_t* __restrict__ mask, float* __restrict__ out_pts,
                                              float* __restrict__ out_rots, int fix_quaternion_write)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P || !mask[i]) return;
	float3 p = make_float3(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
	p.x *= scale; p.y *= scale; p.z *= scale;
	const float3 pt = xform4x3(p, m);
	out_pts[3 * i] = pt.x; out_pts[3 * i + 1] = pt.y; out_pts[3 * i + 2] = pt.z;

	// rotation of the (w,x,y,z) quaternion by the 3x3 block of m, back to a quaternion (Shoemake 1987)
	const float qx = rots[4 * i + 1], qy = rots[4 * i + 2], qz = rots[4 * i + 3], qw = rots[4 * i];
	const float tx = 2.0f * qx, ty = 2.0f * qy, tz = 2.0f * qz;
	const float twx = tx * qw, twy = ty * qw, twz = tz * qw, txx = tx * qx, txy = ty * qx, txz = tz * qx, tyy = ty * qy, tyz = tz * qy, tzz = tz * qz;
	const float R0[3][3] = {{1.0f - (tyy + tzz), txy - twz, txz + twy}, {txy + twz, 1.0f - (txx + tzz), tyz - twx}, {txz - twy, tyz + twx, 1.0f - (txx + tyy)}};
	float R[3][3];
#pragma unroll
	for (int r = 0; r < 3; r++)
#pragma unroll
		for (int c = 0; c < 3; c++) R[r][c] = m[r] * R0[0][c] + m[4 + r] * R0[1][c] + m[8 + r] * R0[2][c];
	float q[4];  // x y z w
	float t = R[0][0] + R[1][1] + R[2][2];
	if (t > 0.0f) {
		t = sqrt(t + 1.0f);
		q[3] = 0.5f * t;
		t = 0.5f / t;
		q[0] = (R[2][1] - R[1][2]) * t; q[1] = (R[0][2] - R[2][0]) * t; q[2] = (R[1][0] - R[0][1]) * t;
	} else {
		int a = 0;
		if (R[1][1] > R[0][0]) a = 1;
		if (R[2][2] > R[a][a]) a = 2;
		const int b = (a + 1) % 3, c = (b + 1) % 3;
		t = sqrt(R[a][a] - R[b][b] - R[c][c] + 1.0f);
		float xyz[3];
		xyz[a] = 0.5f * t;
		t = 0.5f / t;
		q[3] = (R[c][b] - R[b][c]) * t;
		xyz[b] = (R[b][a] + R[a][b]) * t;
		xyz[c] = (R[c][a] + R[a][c]) * t;
		q[0] = xyz[0]; q[1] = xyz[1]; q[2] = xyz[2];
	}
	out_rots[4 * i] = q[3];
	out_rots[4 * i + 1] = q[0];
	if (fix_quaternion_write) { out_rots[4 * i + 2] = q[1]; out_rots[4 * i + 3] = q[2]; }
	else out_rots[4 * i + 2] = q[2];  // the reference writes z into slot +2 and never writes slot +3 (operate_points.h:170-178)
}

// (u, v, depth) -> camera-space point; u, v truncated to int like the reference helper
// (cuda_rasterizer/stereo_vision.h:40-55 takes `const int u, const int v`).
__device__ __forceinline__ float3 reproject_pinhole(int u, int v, float depth, float fx, float fy, float cx, float cy)
{
	return make_float3((u - cx) * depth / fx, (v - cy) * depth / fy, depth);
}

__global__ void reproject_depths_kernel(int P, int width, float fx, float fy, float cx, float cy, const float* __restrict__ depths,
                                        const uint8_t* __restrict__ mask, float* __restrict__ points)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= P || !mask[idx]) return;
	const int v = idx / width, u = idx - v * width;
	const float3 p = reproject_pinhole(u, v, depths[idx], fx, fy, cx, cy);
	points[3 * idx] = p.x; points[3 * idx + 1] = p.y; points[3 * idx + 2] = p.z;
}

// Keypoints without a 3-D point borrow the depth of the nearest keypoint (in pixels) that has one. One warp per
// keypoint scans the N candidates cooperatively (the reference runs an O(N) loop per thread); ties on the distance keep
// the lowest index like the reference's strict `dist >= min_dist` rejection.
__global__ void neighbour_depth_kernel(int N, int width, float fx, float fy, float cx, float cy, float max_pixel_dist,
                                       const float* __restrict__ pixels, const uint8_t* __restrict__ has3D, const float* __restrict__ p3d,
                                       const float* __restrict__ colors, float* __restrict__ out_p3d, float* __restrict__ out_col)
{
	const int idx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
	const int lane = threadIdx.x & 31;
	if (idx >= N) return;
	const float u = pixels[2 * idx], v = pixels[2 * idx + 1];
	const int pix = (int)(v * width + u);  // reference: `int pxidx_in_image = v * width + u;` (src/stereo_vision.cu:86)
	if (has3D[idx]) {
		if (lane < 3) { out_p3d[3 * idx + lane] = p3d[3 * idx + lane]; out_col[3 * idx + lane] = colors[pix + lane]; }
		return;
	}
	float best = 3.402823466e+38f;
	int best_i = 0x7fffffff;
	for (int i = lane; i < N; i += 32) {
		if (!has3D[i] || i == idx) continue;
		const float du = u - pixels[2 * i], dv = v - pixels[2 * i + 1];
		const float dist = du * du + dv * dv;
		if (dist > max_pixel_dist) continue;
		if (dist < best) { best = dist; best_i = i; }  // ascending i within a lane: first minimum kept
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) {
		const float ob = __shfl_xor_sync(0xffffffffu, best, o);
		const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
		if (ob < best || (ob == best && oi < best_i)) { best = ob; best_i = oi; }
	}
	if (lane == 0) {
		const float depth = (best_i != 0x7fffffff) ? p3d[3 * best_i + 2] : -1.0f;
		if (depth > 0.0f) {
			const float3 p = reproject_pinhole((int)u, (int)v, depth, fx, fy, cx, cy);
			out_p3d[3 * idx] = p.x; out_p3d[3 * idx + 1] = p.y; out_p3d[3 * idx + 2] = p.z;
			out_col[3 * idx] = colors[pix]; out_col[3 * idx + 1] = colors[pix + 1]; out_col[3 * idx + 2] = colors[pix + 2];
		} else {
			out_p3d[3 * idx + 2] = -1.0f;
		}
	}
}

__global__ void init_bounds_kernel(uint32_t* bounds)
{
	if (threadIdx.x < 3) bounds[threadIdx.x] = 0xFFFFFFFFu;
	else if (threadIdx.x < 6) bounds[threadIdx.x] = 0u;
}

}  // namespace

}  // namespace psb

using namespace psb;

extern "C" {

int psb_dist_cuda2(int P, const float* points, float* mean_dists, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	if (P < 0 || (P > 0 && (!points || !mean_dists))) { set_error_msg("psb_dist_cuda2: bad argument"); return PSB_ERR_ARG; }
	if (P == 0) return 0;
	const SortPlan plan = make_sort_plan(30);
	const size_t sb = sort_scratch_bytes((size_t)P, plan.npass);
	const int nbox = (P + KNN_TILE - 1) / KNN_TILE;
	const size_t bytes = align_up((size_t)P * 4, 256) * 4 + align_up(sb, 256) + align_up((size_t)nbox * sizeof(Box), 256) + align_up((size_t)P * sizeof(float4), 256) + 512;
	StreamScratch<char> mem(stream);
	PSB_CUDA_OK(mem.alloc(bytes));
	char* c = mem.get();
	uint32_t* keys[2]; uint32_t* vals[2];
	keys[0] = carve<uint32_t>(c, P, 256); keys[1] = carve<uint32_t>(c, P, 256);
	vals[0] = carve<uint32_t>(c, P, 256); vals[1] = carve<uint32_t>(c, P, 256);
	char* scratch = carve<char>(c, sb, 256);
	Box* boxes = carve<Box>(c, nbox, 256);
	float4* sorted = carve<float4>(c, P, 256);
	uint32_t* bounds = carve<uint32_t>(c, 8, 32);
	init_bounds_kernel<<<1, 32, 0, stream>>>(bounds);
	int grid = cdiv(P, 256);
	if (grid > kNumSMs * 8) grid = kNumSMs * 8;
	knn_bounds_kernel<<<grid, 256, 0, stream>>>(P, points, bounds);
	knn_morton_kernel<<<cdiv(P, 256), 256, 0, stream>>>(P, points, bounds, keys[0]);
	PSB_LAUNCH_OK();
	int rc;
	if ((rc = radix_sort_pairs(keys, vals, /*iota_vals=*/true, nullptr, (size_t)P, plan, scratch, sb, stream))) return rc;
	const uint32_t* order = vals[plan.result()];
	knn_gather_kernel<<<cdiv(P, 256), 256, 0, stream>>>(P, points, order, sorted);
	knn_tile_box_kernel<<<nbox, KNN_TILE, 0, stream>>>(P, sorted, boxes);
	knn_search_kernel<<<nbox, KNN_TILE, 0, stream>>>(P, nbox, sorted, boxes, mean_dists);
	const cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) { set_error("knn kernels", e, __FILE__, __LINE__); return PSB_ERR_CUDA; }
	return 0;
}

int psb_reproject_depth_pinhole(int P, int width, float fx, float fy, float cx, float cy, const float* depths, const unsigned char* mask,
                                float* points, void* stream_)
{
	if (P < 0 || width <= 0 || (P > 0 && (!depths || !mask || !points))) { set_error_msg("psb_reproject_depth_pinhole: bad argument"); return PSB_ERR_ARG; }
	if (P == 0) return 0;
	reproject_depths_kernel<<<cdiv(P, 256), 256, 0, (cudaStream_t)stream_>>>(P, width, fx, fy, cx, cy, depths, mask, points);
	PSB_LAUNCH_OK();
	return 0;
}

int psb_neighbour_depth_pinhole(int N, int width, float fx, float fy, float cx, float cy, float max_pixel_dist, const float* pixels,
                                const unsigned char* has3D, const float* points_local, const float* colors, float* out_points, float* out_colors,
                                void* stream_)
{
	if (N < 0 || (N > 0 && (!pixels || !has3D || !points_local || !colors || !out_points || !out_colors))) { set_error_msg("psb_neighbour_depth_pinhole: bad argument"); return PSB_ERR_ARG; }
	if (N == 0) return 0;
	neighbour_depth_kernel<<<cdiv(N * 32, 256), 256, 0, (cudaStream_t)stream_>>>(N, width, fx, fy, cx, cy, max_pixel_dist, pixels, has3D, points_local,
	                                                                            colors, out_points, out_colors);
	PSB_LAUNCH_OK();
	return 0;
}

int psb_transform_points(int P, const float* points, const float* transform, float* out_points, void* stream_)
{
	if (P < 0 || (P > 0 && (!points || !transform || !out_points))) { set_error_msg("psb_transform_points: bad argument"); return PSB_ERR_ARG; }
	if (P == 0) return 0;
	transform_points_kernel<<<cdiv(P, 256), 256, 0, (cudaStream_t)stream_>>>(P, points, transform, out_points);
	PSB_LAUNCH_OK();
	return 0;
}

int psb_scale_transform_points(int P, float scale, const float* points, const float* rots, const float* transform, const unsigned char* mask,
                               float* out_points, float* out_rots, int fix_quaternion_write, void* stream_)
{
	if (P < 0 || (P > 0 && (!points || !rots || !transform || !mask || !out_points || !out_rots))) { set_error_msg("psb_scale_transform_points: bad argument"); return PSB_ERR_ARG; }
	if (P == 0) return 0;
	scale_transform_points_kernel<<<cdiv(P, 256), 256, 0, (cudaStream_t)stream_>>>(P, scale, points, rots, transform, mask, out_points, out_rots,
	                                                                             fix_quaternion_write);
	PSB_LAUNCH_OK();
	return 0;
}

}  // extern "C"
