// Sensor normals of a depth image (psb_depth_normals, include/psb200.h): one thread per pixel, central differences of the back-projected
// neighbours, no atomics (bit-identical from run to run).
#include <cmath>
#include "psb_common.cuh"
#include "../../include/psb200.h"

namespace psb {
namespace {

struct NormalCam {
	int W, H;
	float fx, fy, half_w, half_h;  // the seeding rule's back-projection (psb_seed_apply)
};

__device__ __forceinline__ float3 back_project(const NormalCam& c, int u, int v, float z)
{
	return make_float3(((float)u + 0.5f - c.half_w) * z / c.fx, ((float)v + 0.5f - c.half_h) * z / c.fy, z);
}

__device__ __forceinline__ bool usable(float z) { return isfinite(z) && z > 0.f; }

__global__ void __launch_bounds__(256) depth_normals_kernel(NormalCam c, const float* __restrict__ depth, float max_rel_jump, float* __restrict__ out)
{
	const int i = blockIdx.x * 256 + threadIdx.x;
	const int n = c.W * c.H;
	if (i >= n) return;
	const int u = i % c.W, v = i / c.W;
	float3 nrm = make_float3(0.f, 0.f, 0.f);
	if (u > 0 && v > 0 && u < c.W - 1 && v < c.H - 1) {
		const float z = depth[i], zl = depth[i - 1], zr = depth[i + 1], zu = depth[i - c.W], zd = depth[i + c.W];
		const float jump = max_rel_jump * z;
		if (usable(z) && usable(zl) && usable(zr) && usable(zu) && usable(zd) && !(fabsf(zl - z) > jump) && !(fabsf(zr - z) > jump) &&
		    !(fabsf(zu - z) > jump) && !(fabsf(zd - z) > jump)) {
			const float3 X = back_project(c, u, v, z);
			const float3 L = back_project(c, u - 1, v, zl), R = back_project(c, u + 1, v, zr);
			const float3 U = back_project(c, u, v - 1, zu), D = back_project(c, u, v + 1, zd);
			const float3 a = make_float3(R.x - L.x, R.y - L.y, R.z - L.z), b = make_float3(D.x - U.x, D.y - U.y, D.z - U.z);
			const float3 cr = make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
			const float len = sqrtf(cr.x * cr.x + cr.y * cr.y + cr.z * cr.z);
			if (len > 0.f) {
				const float s = (cr.x * X.x + cr.y * X.y + cr.z * X.z < 0.f ? 1.f : -1.f) / len;
				nrm = make_float3(cr.x * s, cr.y * s, cr.z * s);
			}
		}
	}
	out[i] = nrm.x;
	out[n + i] = nrm.y;
	out[2 * n + i] = nrm.z;
}

}  // namespace
}  // namespace psb

using namespace psb;

extern "C" int psb_depth_normals(const psb_camera* camera, const float* depth, float max_rel_jump, float* out_normal, void* stream_)
{
	if (!camera || !depth || !out_normal) { set_error_msg("psb_depth_normals: null argument"); return PSB_ERR_ARG; }
	if (camera->width <= 0 || camera->height <= 0 || (long long)camera->width * camera->height > (long long)INT32_MAX) {
		set_error_msg("psb_depth_normals: the camera needs a positive size");
		return PSB_ERR_ARG;
	}
	if (!std::isfinite(camera->tan_fovx) || !std::isfinite(camera->tan_fovy) || !(camera->tan_fovx > 0.f) || !(camera->tan_fovy > 0.f)) {
		set_error_msg("psb_depth_normals: tan_fovx and tan_fovy must be finite and positive");
		return PSB_ERR_ARG;
	}
	if (!std::isfinite(max_rel_jump) || !(max_rel_jump > 0.f)) { set_error_msg("psb_depth_normals: max_rel_jump must be finite and positive"); return PSB_ERR_ARG; }
	NormalCam c;
	c.W = camera->width; c.H = camera->height;
	c.fx = (float)c.W / (2.0f * camera->tan_fovx);
	c.fy = (float)c.H / (2.0f * camera->tan_fovy);
	c.half_w = 0.5f * (float)c.W; c.half_h = 0.5f * (float)c.H;
	const int n = c.W * c.H;
	depth_normals_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream_>>>(c, depth, max_rel_jump, out_normal);
	PSB_LAUNCH_OK();
	return 0;
}
