// Per-Gaussian backward: gradients of the 9 screen-space sums produced by the tile kernel
// (dL/dmean2D.xy, dL/dconic.xyw, dL/dopacity, dL/drgb) with respect to the 3D parameters.
// ONE kernel for what the reference runs as computeCov2DCUDA + preprocessCUDA
// (reference cuda_rasterizer/backward.cu:144-274, 346-396, SH part :20-139, cov3D part :278-341):
// the 3D covariance is recomputed in registers instead of being written in forward and re-read, and
// dL/dcov3D never round-trips through memory unless the caller asks for it.
#include "psb_backward.cuh"

namespace psb {

// DEPTH: dL/dz (view-space depth, the depth tile backward's tenth sum) joins dL/dmean3D through the view matrix's z row,
// z = V[2] x + V[6] y + V[10] z + V[14] (column-major), as in gaussian_backward_kernel<MODE_DEPTH>.
// AA: the forward blended o' = o h (preprocess_fwd_kernel<false, true>, o' in the record). dL_dopacity [P] holds dL/do' from the tile
// backward (atomic or gathered); the h-term joins the covariance gradient and dL_dopacity[g] is rescaled in place to dL/do = h dL/do'.
// NORMAL (scales + rotations): dL_dn [P,3] holds dL/dn of the operator's n_i (op_normals_kernel: activated scales, the rotation as given);
// its rotation gradient, through column k of R(q), the sign and V (normal_axis_backward), joins dL/drot. The arg-min k and the sign are
// piecewise constant, so nothing reaches the scales or the mean.
// One entry for the eight variants: dL_dz is read only when DEPTH, dL_dopacity only when AA, dL_dn only when NORMAL.
template <bool DEPTH, bool AA, bool NORMAL>
__global__ void __launch_bounds__(128) preprocess_bwd_kernel(GaussIn in, Camera cam, GeomState geom, const float* __restrict__ dL_dmean2D,
                                                             int mean2D_stride, const float* __restrict__ dL_dconic, int conic_stride,
                                                             const float* __restrict__ dL_dcolor, int color_stride, GaussGradOut out,
                                                             const float* __restrict__ dL_dz, float* __restrict__ dL_dopacity,
                                                             const float* __restrict__ dL_dn)
{
	const int idx = blockIdx.x * blockDim.x + threadIdx.x;
	if (idx >= in.P || geom.tile_info[idx].z == 0) return;

	const float3 mean = make_float3(in.means3D[3 * idx], in.means3D[3 * idx + 1], in.means3D[3 * idx + 2]);
	float cov3D[6];
	float3 scale = make_float3(0, 0, 0);
	float4 rot = make_float4(0, 0, 0, 0);
	if (in.cov3D_precomp != nullptr) {
#pragma unroll
		for (int i = 0; i < 6; i++) cov3D[i] = in.cov3D_precomp[6 * idx + i];
	} else {
		scale = make_float3(in.scales[3 * idx], in.scales[3 * idx + 1], in.scales[3 * idx + 2]);
		rot = reinterpret_cast<const float4*>(in.rotations)[idx];
		cov3d_from_scale_rot(scale, in.scale_modifier, rot, cov3D);
	}
	const uint32_t clamp_bits = rec_clamp_bits(__float_as_uint(geom.rec[idx].q2.w));
	const float2 g2 = make_float2(dL_dmean2D[(size_t)idx * mean2D_stride], dL_dmean2D[(size_t)idx * mean2D_stride + 1]);
	const float3 gc = make_float3(dL_dconic[(size_t)idx * conic_stride], dL_dconic[(size_t)idx * conic_stride + 1],
	                              dL_dconic[(size_t)idx * conic_stride + 3]);
	const float3 gcol = make_float3(dL_dcolor[(size_t)idx * color_stride], dL_dcolor[(size_t)idx * color_stride + 1],
	                                dL_dcolor[(size_t)idx * color_stride + 2]);
	const float* sh_row = in.shs ? in.shs + (size_t)idx * in.M * 3 : nullptr;
	float* dsh_row = (in.shs && out.dL_dsh) ? out.dL_dsh + (size_t)idx * in.M * 3 : nullptr;

	float3 dL_dmean, dL_dscale = make_float3(0, 0, 0);
	float4 dL_drot = make_float4(0, 0, 0, 0);
	float dL_dcov[6];
	float aa_h = 1.f;
	const float dL_dop = AA ? dL_dopacity[idx] : 0.f;
	gaussian_backward<AA>(in, cam, idx, mean, cov3D, scale, rot, sh_row, clamp_bits, g2, gc, gcol, dsh_row, dL_dmean, dL_dcov, dL_dscale, dL_drot,
	                      AA ? geom.rec[idx].q1.y : 0.f, dL_dop, &aa_h);
	if (AA) dL_dopacity[idx] = aa_h * dL_dop;
	if (DEPTH) {
		const float dz = dL_dz[idx];
		dL_dmean.x += dz * cam.view[2]; dL_dmean.y += dz * cam.view[6]; dL_dmean.z += dz * cam.view[10];
	}
	if constexpr (NORMAL) {
		const NormalAxis a = normal_axis(rot, scale, xform4x3(mean, cam.view), cam.view);
		const float3 gn = make_float3(dL_dn[3 * idx], dL_dn[3 * idx + 1], dL_dn[3 * idx + 2]);
		const float4 gq = normal_axis_backward(rot, a, gn, cam.view);
		dL_drot.x += gq.x; dL_drot.y += gq.y; dL_drot.z += gq.z; dL_drot.w += gq.w;
	}

	if (out.dL_dmeans3D) { out.dL_dmeans3D[3 * idx] = dL_dmean.x; out.dL_dmeans3D[3 * idx + 1] = dL_dmean.y; out.dL_dmeans3D[3 * idx + 2] = dL_dmean.z; }
	if (out.dL_dcov3D) {
#pragma unroll
		for (int i = 0; i < 6; i++) out.dL_dcov3D[6 * idx + i] = dL_dcov[i];
	}
	if (in.scales) {
		if (out.dL_dscales) { out.dL_dscales[3 * idx] = dL_dscale.x; out.dL_dscales[3 * idx + 1] = dL_dscale.y; out.dL_dscales[3 * idx + 2] = dL_dscale.z; }
		if (out.dL_drots) reinterpret_cast<float4*>(out.dL_drots)[idx] = dL_drot;
	}
}

int launch_preprocess_backward(const GaussIn& in, const Camera& cam, const GeomState& geom, const float* dL_dmean2D, int mean2D_stride,
                               const float* dL_dconic, int conic_stride, const float* dL_dcolor, int color_stride,
                               const GaussGradOut& out, cudaStream_t stream, const float* dL_dz, float* aa_dL_dopacity, const float* dL_dn)
{
	if (in.P == 0) return 0;
	if (dL_dn && (!in.scales || !in.rotations)) { set_error_msg("launch_preprocess_backward: the normal gradient needs scales and rotations"); return -1; }
	const int v = (dL_dz ? 1 : 0) | (aa_dL_dopacity ? 2 : 0) | (dL_dn ? 4 : 0);
	using Kernel = decltype(&preprocess_bwd_kernel<false, false, false>);
	static const Kernel VARIANTS[8] = {preprocess_bwd_kernel<false, false, false>, preprocess_bwd_kernel<true, false, false>,
	                                   preprocess_bwd_kernel<false, true, false>,  preprocess_bwd_kernel<true, true, false>,
	                                   preprocess_bwd_kernel<false, false, true>,  preprocess_bwd_kernel<true, false, true>,
	                                   preprocess_bwd_kernel<false, true, true>,   preprocess_bwd_kernel<true, true, true>};
	VARIANTS[v]<<<cdiv(in.P, 128), 128, 0, stream>>>(in, cam, geom, dL_dmean2D, mean2D_stride, dL_dconic, conic_stride, dL_dcolor, color_stride, out, dL_dz,
	                                                 aa_dL_dopacity, dL_dn);
	PSB_LAUNCH_OK();
	return 0;
}

}  // namespace psb
