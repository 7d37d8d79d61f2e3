// Sensor normals of a depth image (psb_depth_normals, include/psb200.h): one thread per pixel, central differences of the back-projected
// neighbours, no atomics (bit-identical from run to run).
#include <cmath>
#include <string>
#include "psb_normals.cuh"
#include "psb_train.h"
#include "../../include/psb200.h"

namespace psb {
namespace {

__global__ void __launch_bounds__(256) depth_normals_kernel(NormalCam c, const float* __restrict__ depth, float max_rel_jump, float* __restrict__ out)
{
	const int i = blockIdx.x * 256 + threadIdx.x;
	const int n = c.W * c.H;
	if (i >= n) return;
	const int u = i % c.W, v = i / c.W;
	float3 nrm = make_float3(0.f, 0.f, 0.f);
	if (u > 0 && v > 0 && u < c.W - 1 && v < c.H - 1) {
		Stencil st;
		stencil_normal(c, u, v, depth[i], depth[i - 1], depth[i + 1], depth[i - c.W], depth[i + c.W], max_rel_jump, nrm, st);
	}
	out[i] = nrm.x;
	out[n + i] = nrm.y;
	out[2 * n + i] = nrm.z;
}

}  // namespace
}  // namespace psb

using namespace psb;

namespace {
// The camera checks of psb_depth_normals and psb_dn_loss (before any CUDA call)
int check_normal_camera(const psb_camera* camera, const char* fn)
{
	if (camera->width <= 0 || camera->height <= 0 || (long long)camera->width * camera->height > (long long)INT32_MAX) {
		set_error_msg(std::string(fn).append(": the camera needs a positive size").c_str());
		return PSB_ERR_ARG;
	}
	if (!std::isfinite(camera->tan_fovx) || !std::isfinite(camera->tan_fovy) || !(camera->tan_fovx > 0.f) || !(camera->tan_fovy > 0.f)) {
		set_error_msg(std::string(fn).append(": tan_fovx and tan_fovy must be finite and positive").c_str());
		return PSB_ERR_ARG;
	}
	return 0;
}
}  // namespace

extern "C" int psb_depth_normals(const psb_camera* camera, const float* depth, float max_rel_jump, float* out_normal, void* stream_)
{
	int rc;
	if (!camera || !depth || !out_normal) { set_error_msg("psb_depth_normals: null argument"); return PSB_ERR_ARG; }
	if ((rc = check_normal_camera(camera, "psb_depth_normals"))) return rc;
	if (!std::isfinite(max_rel_jump) || !(max_rel_jump > 0.f)) { set_error_msg("psb_depth_normals: max_rel_jump must be finite and positive"); return PSB_ERR_ARG; }
	const NormalCam c = normal_cam(camera->width, camera->height, camera->tan_fovx, camera->tan_fovy);
	const int n = c.W * c.H;
	depth_normals_kernel<<<cdiv(n, 256), 256, 0, (cudaStream_t)stream_>>>(c, depth, max_rel_jump, out_normal);
	PSB_LAUNCH_OK();
	return 0;
}

extern "C" int psb_dn_loss(const psb_camera* camera, const float* depth, const float* alpha, const float* normal, const float* mask, const psb_dn* dn,
                           float* dL_ddepth, float* dL_dalpha, float* dL_dnormal, float* out2_host, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	int rc;
	if (!camera || !depth || !alpha || !normal || !dn || !dL_ddepth || !dL_dalpha || !dL_dnormal) {
		set_error_msg("psb_dn_loss: null argument");
		return PSB_ERR_ARG;
	}
	if ((rc = check_normal_camera(camera, "psb_dn_loss"))) return rc;
	if (!std::isfinite(dn->lambda_dn) || !(dn->lambda_dn > 0.f)) { set_error_msg("psb_dn_loss: lambda_dn must be finite and > 0"); return PSB_ERR_ARG; }
	if (!(dn->alpha_min > 0.f && dn->alpha_min <= 1.f)) { set_error_msg("psb_dn_loss: alpha_min must lie in (0, 1]"); return PSB_ERR_ARG; }
	if (!std::isfinite(dn->max_rel_jump) || !(dn->max_rel_jump > 0.f)) { set_error_msg("psb_dn_loss: max_rel_jump must be finite and > 0"); return PSB_ERR_ARG; }
	const int W = camera->width, H = camera->height;
	// stream-ordered scratch; the sums are reduced in a fixed order, so the result is the same every run
	StreamScratch<double> sums(stream), partials(stream);
	if (sums.alloc(2) != cudaSuccess || partials.alloc(2 * (size_t)depth_loss_blocks(H, W)) != cudaSuccess) {
		set_error_msg("psb_dn_loss: out of device memory");
		return PSB_ERR_CUDA;
	}
	if ((rc = launch_dn_loss(W, H, camera->tan_fovx, camera->tan_fovy, depth, alpha, normal, mask, dn->lambda_dn, dn->alpha_min, dn->max_rel_jump,
	                         dn->out_depth_normal, sums.get(), dL_ddepth, dL_dalpha, dL_dnormal, stream, partials.get())))
		return rc;
	double h[2] = {0, 0};
	PSB_CUDA_OK(cudaMemcpyAsync(h, sums.get(), sizeof(h), cudaMemcpyDeviceToHost, stream));
	PSB_CUDA_OK(cudaStreamSynchronize(stream));
	if (out2_host) {
		out2_host[0] = (float)(h[0] / (h[1] > 1.0 ? h[1] : 1.0));
		out2_host[1] = (float)h[1];
	}
	return 0;
}
