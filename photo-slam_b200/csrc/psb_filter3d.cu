// The 3D smoothing filter of Mip-Splatting (include/psb200.h, psb_filter3d): per row, the finest sampling interval any keyframe sees it at.
// Two launches, no host round trip unless the caller asks for the number of rows seen:
//   filter3d_kernel         one thread per row, the cameras staged in shared memory F3D_CHUNK at a time: d = min view-space z over the
//                           cameras that see the row (+inf: none), written to `filter`; the largest d of a seen row, the number of seen rows
//                           and F = max focal_x go to a 16-byte scratch as integer maxima and sums (non-negative float bits order like
//                           unsigned integers), so the result is the same on every run;
//   filter3d_finish_kernel  unseen rows take the largest d; every row becomes d / F * sqrt(0.2) (all zeros when no row is seen).
#include "psb_kernels.h"
#include "../../include/psb200.h"

namespace psb {
namespace {

constexpr int F3D_TB = 256;       // rows per block
constexpr int F3D_CHUNK = 64;     // cameras per shared-memory round (5 KB)
constexpr int CAM_FLOATS = 20;    // view matrix (16, column-major), focal_x, focal_y, W, H

struct Filter3dScratch {
	uint32_t max_d;   // bits of the largest d of a seen row
	uint32_t seen;    // rows seen by at least one camera
	uint32_t focal;   // bits of F = max focal_x
	uint32_t pad;
};

__global__ void __launch_bounds__(F3D_TB) filter3d_kernel(int P, const float* __restrict__ xyz, int K, const float* __restrict__ cams,
                                                          float* __restrict__ dist, Filter3dScratch* __restrict__ sc)
{
	__shared__ float s_cam[F3D_CHUNK * CAM_FLOATS];
	const int i = blockIdx.x * F3D_TB + threadIdx.x;
	const bool valid = i < P;
	float3 p = make_float3(0.f, 0.f, 0.f);
	if (valid) p = make_float3(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
	float d = INFINITY, F = 0.f;
	for (int k0 = 0; k0 < K; k0 += F3D_CHUNK) {
		const int n = min(F3D_CHUNK, K - k0);
		__syncthreads();  // every thread is done with the previous chunk
		for (int j = threadIdx.x; j < n * CAM_FLOATS; j += F3D_TB) s_cam[j] = cams[(size_t)k0 * CAM_FLOATS + j];
		__syncthreads();
		for (int k = 0; k < n; k++) {
			const float* c = s_cam + k * CAM_FLOATS;
			const float fx = c[16], fy = c[17], W = c[18], H = c[19];
			F = fmaxf(F, fx);
			const float3 v = xform4x3(p, c);   // the forward's near cull, bit for bit (preprocess_fwd_kernel)
			if (!(v.z > 0.2f)) continue;
			const float u = v.x / v.z * fx + 0.5f * W;
			const float w = v.y / v.z * fy + 0.5f * H;
			if (u >= -0.15f * W && u <= 1.15f * W && w >= -0.15f * H && w <= 1.15f * H) d = fminf(d, v.z);
		}
	}
	const bool seen = valid && d != INFINITY;
	if (valid) dist[i] = d;
	const uint32_t ball = __ballot_sync(0xffffffffu, seen);
	const uint32_t mx = __reduce_max_sync(0xffffffffu, seen ? __float_as_uint(d) : 0u);
	if ((threadIdx.x & 31) == 0 && ball) {
		atomicMax(&sc->max_d, mx);
		atomicAdd(&sc->seen, (uint32_t)__popc(ball));
	}
	if (blockIdx.x == 0 && threadIdx.x == 0) sc->focal = __float_as_uint(F);
}

__global__ void __launch_bounds__(F3D_TB) filter3d_finish_kernel(int P, float* __restrict__ filter, const Filter3dScratch* __restrict__ sc)
{
	const int i = blockIdx.x * F3D_TB + threadIdx.x;
	if (i >= P) return;
	if (sc->seen == 0) { filter[i] = 0.f; return; }
	float d = filter[i];
	if (d == INFINITY) d = __uint_as_float(sc->max_d);
	filter[i] = d / __uint_as_float(sc->focal) * 0.44721359549995793f;   // sqrt(0.2)
}

}  // namespace
}  // namespace psb

using namespace psb;

extern "C" int psb_filter3d(int P, const float* xyz, int K, const float* cams, float* filter, int* seen_host, void* stream_)
{
	if (P < 0 || K < 0 || (P > 0 && (!xyz || !filter)) || (K > 0 && !cams)) {
		set_error_msg("psb_filter3d: need P >= 0, K >= 0, xyz and filter when P > 0, cams when K > 0");
		return PSB_ERR_ARG;
	}
	cudaStream_t stream = (cudaStream_t)stream_;
	if (P == 0) {
		if (seen_host) *seen_host = 0;
		return 0;
	}
	StreamScratch<Filter3dScratch> sc(stream);
	PSB_CUDA_OK(sc.alloc(1));
	if (cudaMemsetAsync(sc.get(), 0, sizeof(Filter3dScratch), stream) != cudaSuccess) return PSB_ERR_CUDA;
	const int grid = cdiv(P, F3D_TB);
	filter3d_kernel<<<grid, F3D_TB, 0, stream>>>(P, xyz, K, cams, filter, sc.get());
	filter3d_finish_kernel<<<grid, F3D_TB, 0, stream>>>(P, filter, sc.get());
	cudaError_t e = cudaGetLastError();
	if (e != cudaSuccess) { set_error("psb_filter3d: kernel launch", e, __FILE__, __LINE__); return PSB_ERR_CUDA; }
	if (seen_host) {
		uint32_t seen = 0;
		e = cudaMemcpyAsync(&seen, &sc.get()->seen, sizeof(seen), cudaMemcpyDeviceToHost, stream);
		if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
		if (e != cudaSuccess) { set_error("psb_filter3d", e, __FILE__, __LINE__); return PSB_ERR_CUDA; }
		*seen_host = (int)seen;
	}
	return 0;
}
