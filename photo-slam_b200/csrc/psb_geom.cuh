// Per-Gaussian geometry shared by the forward and backward preprocess kernels:
// quaternion+scale -> 3D covariance, EWA projection -> 2D covariance, SH -> RGB.
// Semantics follow reference cuda_rasterizer/forward.cu:20-152 (cited per function); the code is
// written from those formulas, with expression shapes kept so rounding matches bit for bit.
#pragma once
#include "psb_common.cuh"

namespace psb {

// Rotation matrix of a (w,x,y,z) quaternion, stored the way the reference fills its glm::mat3
// (forward.cu:134-138: constructor arguments fill columns). NOT normalised here (forward.cu:127).
__device__ __forceinline__ Mat3 quat_to_mat3(const float4 q)
{
	const float r = q.x, x = q.y, y = q.z, z = q.w;
	Mat3 R;
	R(0, 0) = 1.f - 2.f * (y * y + z * z); R(0, 1) = 2.f * (x * y - r * z); R(0, 2) = 2.f * (x * z + r * y);
	R(1, 0) = 2.f * (x * y + r * z); R(1, 1) = 1.f - 2.f * (x * x + z * z); R(1, 2) = 2.f * (y * z - r * x);
	R(2, 0) = 2.f * (x * z - r * y); R(2, 1) = 2.f * (y * z + r * x); R(2, 2) = 1.f - 2.f * (x * x + y * y);
	return R;
}

__device__ __forceinline__ Mat3 diag3(float a, float b, float c)
{
	Mat3 S;
#pragma unroll
	for (int i = 0; i < 9; i++) S.m[i] = 0.f;
	S(0, 0) = a; S(1, 1) = b; S(2, 2) = c;
	return S;
}

// Sigma = (S R)^T (S R), upper triangle [00,01,02,11,12,22]   (forward.cu:118-152)
__device__ __forceinline__ void cov3d_from_scale_rot(const float3 scale, float mod, const float4 rot, float* cov3D)
{
	Mat3 S = diag3(mod * scale.x, mod * scale.y, mod * scale.z);
	Mat3 R = quat_to_mat3(rot);
	Mat3 M = mat3_mul(S, R);
	Mat3 Sigma = mat3_mul(mat3_transpose(M), M);
	cov3D[0] = Sigma(0, 0); cov3D[1] = Sigma(0, 1); cov3D[2] = Sigma(0, 2);
	cov3D[3] = Sigma(1, 1); cov3D[4] = Sigma(1, 2); cov3D[5] = Sigma(2, 2);
}

// EWA splatting Jacobian chain (forward.cu:74-113 / backward.cu:163-197). Returns T = W*J, the
// symmetric Vrk, the clamped view-space mean t and the clamp masks; cov = T^T Vrk^T T.
struct Cov2DTerms {
	Mat3 T, Vrk, cov;
	float3 t;
	float x_grad_mul, y_grad_mul;
};
__device__ __forceinline__ void cov2d_terms(const float3 mean, float focal_x, float focal_y, float tan_fovx, float tan_fovy,
                                            const float* cov3D, const float* vm, Cov2DTerms& o)
{
	float3 t = xform4x3(mean, vm);
	const float limx = 1.3f * tan_fovx;
	const float limy = 1.3f * tan_fovy;
	const float txtz = t.x / t.z;
	const float tytz = t.y / t.z;
	t.x = min(limx, max(-limx, txtz)) * t.z;
	t.y = min(limy, max(-limy, tytz)) * t.z;
	o.x_grad_mul = txtz < -limx || txtz > limx ? 0 : 1;
	o.y_grad_mul = tytz < -limy || tytz > limy ? 0 : 1;

	Mat3 J;
	J(0, 0) = focal_x / t.z; J(0, 1) = 0.0f; J(0, 2) = -(focal_x * t.x) / (t.z * t.z);
	J(1, 0) = 0.0f; J(1, 1) = focal_y / t.z; J(1, 2) = -(focal_y * t.y) / (t.z * t.z);
	J(2, 0) = 0; J(2, 1) = 0; J(2, 2) = 0;
	Mat3 W;
	W(0, 0) = vm[0]; W(0, 1) = vm[4]; W(0, 2) = vm[8];
	W(1, 0) = vm[1]; W(1, 1) = vm[5]; W(1, 2) = vm[9];
	W(2, 0) = vm[2]; W(2, 1) = vm[6]; W(2, 2) = vm[10];
	o.T = mat3_mul(W, J);
	Mat3 V;
	V(0, 0) = cov3D[0]; V(0, 1) = cov3D[1]; V(0, 2) = cov3D[2];
	V(1, 0) = cov3D[1]; V(1, 1) = cov3D[3]; V(1, 2) = cov3D[4];
	V(2, 0) = cov3D[2]; V(2, 1) = cov3D[4]; V(2, 2) = cov3D[5];
	o.Vrk = V;
	o.cov = mat3_mul(mat3_mul(mat3_transpose(o.T), mat3_transpose(V)), o.T);
	o.t = t;
}

// Anti-aliasing (2D Mip filter): the splat's opacity is scaled by h = sqrt(max(det0 / det1, 2.5e-5)), in [0.005, 1], where det0 is the
// determinant of the 2D covariance before the 0.3 px^2 dilation (this function, on cov2d_terms' output) and det1 the one after it.
__device__ __forceinline__ float aa_det0(const Cov2DTerms& ct) { return ct.cov(0, 0) * ct.cov(1, 1) - ct.cov(0, 1) * ct.cov(0, 1); }
constexpr float kAaMinRatio = 2.5e-5f;
__device__ __forceinline__ float aa_factor(float det0, float det1) { return sqrtf(fmaxf(det0 / det1, kAaMinRatio)); }

// 3D smoothing filter (Mip-Splatting; include/psb200.h, psb_filter3d): s <- s' = sqrt(s^2 + f^2) per axis, and returns the opacity factor
// c = sqrt(prod_c s_c^2 / s'_c^2), formed as the product of the per-axis ratios (the products of three squares can underflow). IEEE sqrt and
// division: f = 0 leaves s bit for bit (sqrt(fl(s^2)) = s) and returns exactly 1.
__device__ __forceinline__ float filter3d_widen(float3& s, float f)
{
	const float f2 = f * f;
	const float sx2 = s.x * s.x, sy2 = s.y * s.y, sz2 = s.z * s.z;
	const float px2 = sx2 + f2, py2 = sy2 + f2, pz2 = sz2 + f2;
	const float r = (px2 > 0.f ? sx2 / px2 : 1.f) * (py2 > 0.f ? sy2 / py2 : 1.f) * (pz2 > 0.f ? sz2 / pz2 : 1.f);
	s = make_float3(sqrtf(px2), sqrtf(py2), sqrtf(pz2));
	return sqrtf(r);
}

// Rendered normals (include/psb200.h): the camera-facing shortest axis n of a Gaussian in view space. q = the normalised (w, x, y, z)
// quaternion the covariance is built from, sraw = the raw log-scales, t = the view-space mean (xform4x3 of the mean, as the forward forms
// it), vm the view matrix. k = argmin_c sraw[c] (ties: lowest index), r = column k of R(q) (the world-space axis the covariance scales by
// exp(sraw[k])), m = V r; n = m if m . t <= 0, else -m (sign = +1 / -1). The backward forms the same k and sign from the same inputs.
struct NormalAxis {
	float3 n;
	int k;
	float sign;
};
__device__ __forceinline__ NormalAxis normal_axis(const float4 q, const float3 sraw, const float3 t, const float* vm)
{
	const float w = q.x, x = q.y, y = q.z, z = q.w;
	int k = 0;
	float smin = sraw.x;
	if (sraw.y < smin) { k = 1; smin = sraw.y; }
	if (sraw.z < smin) k = 2;
	float3 r;
	if (k == 0) r = make_float3(1.f - 2.f * (y * y + z * z), 2.f * (x * y + w * z), 2.f * (x * z - w * y));
	else if (k == 1) r = make_float3(2.f * (x * y - w * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z + w * x));
	else r = make_float3(2.f * (x * z + w * y), 2.f * (y * z - w * x), 1.f - 2.f * (x * x + y * y));
	const float3 m = make_float3(vm[0] * r.x + vm[4] * r.y + vm[8] * r.z, vm[1] * r.x + vm[5] * r.y + vm[9] * r.z,
	                             vm[2] * r.x + vm[6] * r.y + vm[10] * r.z);
	const float sign = (m.x * t.x + m.y * t.y + m.z * t.z <= 0.f) ? 1.f : -1.f;
	return {make_float3(sign * m.x, sign * m.y, sign * m.z), k, sign};
}

// dL/dq (of the normalised quaternion) of n = sign V r_k(q), given dL/dn: dL/dr = sign V^T dL/dn, then the derivative of column k of R(q).
// k and the sign are piecewise constant: they pass no gradient to the scales or the mean.
__device__ __forceinline__ float4 normal_axis_backward(const float4 q, const NormalAxis& a, const float3 dL_dn, const float* vm)
{
	const float w = q.x, x = q.y, y = q.z, z = q.w;
	const float g0 = a.sign * (vm[0] * dL_dn.x + vm[1] * dL_dn.y + vm[2] * dL_dn.z);
	const float g1 = a.sign * (vm[4] * dL_dn.x + vm[5] * dL_dn.y + vm[6] * dL_dn.z);
	const float g2 = a.sign * (vm[8] * dL_dn.x + vm[9] * dL_dn.y + vm[10] * dL_dn.z);
	if (a.k == 0)
		return make_float4(2.f * (z * g1 - y * g2), 2.f * (y * g1 + z * g2), 2.f * (x * g1 - w * g2) - 4.f * y * g0, 2.f * (w * g1 + x * g2) - 4.f * z * g0);
	if (a.k == 1)
		return make_float4(2.f * (x * g2 - z * g0), 2.f * (y * g0 + w * g2) - 4.f * x * g1, 2.f * (x * g0 + z * g2), 2.f * (y * g2 - w * g0) - 4.f * z * g1);
	return make_float4(2.f * (y * g0 - x * g1), 2.f * (z * g0 - w * g1) - 4.f * x * g2, 2.f * (w * g0 + z * g1) - 4.f * y * g2, 2.f * (x * g0 + y * g1));
}

// SH (degree <= 3) -> RGB for one Gaussian, all three channels; sh points at this Gaussian's
// [M][3] coefficient row (forward.cu:20-71). Returns colour after +0.5 and clamp at 0; `clamp_bits`
// bit c set when channel c was clamped.
__device__ __forceinline__ float3 sh_to_rgb(int deg, const float3 pos, const float3 campos, const float* __restrict__ sh, uint32_t& clamp_bits)
{
	float3 dir = make_float3(pos.x - campos.x, pos.y - campos.y, pos.z - campos.z);
	const float len = sqrtf(dir.x * dir.x + dir.y * dir.y + dir.z * dir.z);
	dir.x = dir.x / len; dir.y = dir.y / len; dir.z = dir.z / len;
	const float x = dir.x, y = dir.y, z = dir.z;
	float res[3];
#pragma unroll
	for (int ch = 0; ch < 3; ch++) {
		float result = kSH_C0 * sh[ch];
		if (deg > 0) {
			result = result - kSH_C1 * y * sh[3 + ch] + kSH_C1 * z * sh[6 + ch] - kSH_C1 * x * sh[9 + ch];
			if (deg > 1) {
				const float xx = x * x, yy = y * y, zz = z * z;
				const float xy = x * y, yz = y * z, xz = x * z;
				result = result + kSH_C2_0 * xy * sh[12 + ch] + kSH_C2_1 * yz * sh[15 + ch] +
				         kSH_C2_2 * (2.0f * zz - xx - yy) * sh[18 + ch] + kSH_C2_3 * xz * sh[21 + ch] +
				         kSH_C2_4 * (xx - yy) * sh[24 + ch];
				if (deg > 2) {
					result = result + kSH_C3_0 * y * (3.0f * xx - yy) * sh[27 + ch] + kSH_C3_1 * xy * z * sh[30 + ch] +
					         kSH_C3_2 * y * (4.0f * zz - xx - yy) * sh[33 + ch] +
					         kSH_C3_3 * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * sh[36 + ch] +
					         kSH_C3_4 * x * (4.0f * zz - xx - yy) * sh[39 + ch] + kSH_C3_5 * z * (xx - yy) * sh[42 + ch] +
					         kSH_C3_6 * x * (xx - 3.0f * yy) * sh[45 + ch];
				}
			}
		}
		result += 0.5f;
		if (result < 0) clamp_bits |= (1u << ch);
		res[ch] = fmaxf(result, 0.0f);
	}
	return make_float3(res[0], res[1], res[2]);
}

}  // namespace psb
