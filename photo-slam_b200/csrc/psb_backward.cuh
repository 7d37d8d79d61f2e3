// Device functions of the per-Gaussian backward, shared by the stand-alone backward kernel (psb_backward.cu)
// and the per-Gaussian backward + Adam kernel of the trainer step (psb_train.cu).
// Math follows reference cuda_rasterizer/backward.cu:20-139 (SH), :144-274 (cov2D), :278-341 (cov3D), :346-396.
#pragma once
#include "psb_geom.cuh"
#include "psb_kernels.h"

namespace psb {


// d(normalize(v))/dv applied to dv  (reference auxiliary.h:107-117)
__device__ __forceinline__ float3 dnormvdv(float3 v, float3 dv)
{
	const float sum2 = v.x * v.x + v.y * v.y + v.z * v.z;
	const float invsum32 = 1.0f / sqrt(sum2 * sum2 * sum2);
	float3 o;
	o.x = ((+sum2 - v.x * v.x) * dv.x - v.y * v.x * dv.y - v.z * v.x * dv.z) * invsum32;
	o.y = (-v.x * v.y * dv.x + (sum2 - v.y * v.y) * dv.y - v.z * v.y * dv.z) * invsum32;
	o.z = (-v.x * v.z * dv.x - v.y * v.z * dv.y + (sum2 - v.z * v.z) * dv.z) * invsum32;
	return o;
}

// Unit view direction of dir = pos - campos: the direction the SH colour of a Gaussian at pos is evaluated at.
__device__ __forceinline__ float3 sh_dir(const float3 dir)
{
	const float len = sqrtf(dir.x * dir.x + dir.y * dir.y + dir.z * dir.z);
	return make_float3(dir.x / len, dir.y / len, dir.z / len);
}

// SH basis weights w_k = dRGB/dsh_k of the unit direction d, k < 16. The NVLink owner rank re-evaluates them from its copy of xyz
// and the sender's camera centre: both sides go through sh_dir and this function, so the weights agree bit for bit.
__device__ __forceinline__ void sh_basis(const float3 d, float* w /*[16]*/)
{
	const float x = d.x, y = d.y, z = d.z;
	const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
	w[0] = kSH_C0;
	w[1] = -kSH_C1 * y; w[2] = kSH_C1 * z; w[3] = -kSH_C1 * x;
	w[4] = kSH_C2_0 * xy; w[5] = kSH_C2_1 * yz; w[6] = kSH_C2_2 * (2.f * zz - xx - yy); w[7] = kSH_C2_3 * xz; w[8] = kSH_C2_4 * (xx - yy);
	w[9] = kSH_C3_0 * y * (3.f * xx - yy); w[10] = kSH_C3_1 * xy * z; w[11] = kSH_C3_2 * y * (4.f * zz - xx - yy);
	w[12] = kSH_C3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy); w[13] = kSH_C3_4 * x * (4.f * zz - xx - yy); w[14] = kSH_C3_5 * z * (xx - yy);
	w[15] = kSH_C3_6 * x * (xx - 3.f * yy);
}

// SH backward for one Gaussian. `get(k, ch)` returns SH coefficient k of channel ch, `put(k, ch, g)` receives
// dL/dsh[k][ch] (called for the coefficients of the active degree only). All reads happen before the
// first put, so `put` may update the coefficient in place. Returns the view-direction contribution to dL/dmean.
template <typename Get, typename Put>
__device__ __forceinline__ float3 sh_backward_t(int deg, const float3 pos, const float3 campos, uint32_t clamp_bits,
                                                const float3 dL_dcolor, Get get, Put put, float* w_out = nullptr)
{
	const float3 dir_orig = make_float3(pos.x - campos.x, pos.y - campos.y, pos.z - campos.z);
	const float3 d = sh_dir(dir_orig);
	const float x = d.x, y = d.y, z = d.z;
	float g[3] = {dL_dcolor.x, dL_dcolor.y, dL_dcolor.z};
#pragma unroll
	for (int ch = 0; ch < 3; ch++) g[ch] *= ((clamp_bits >> ch) & 1u) ? 0 : 1;
	const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
	float dx[3] = {0, 0, 0}, dy[3] = {0, 0, 0}, dz[3] = {0, 0, 0};
#define SHC(k) get(k, ch)
#pragma unroll
	for (int ch = 0; ch < 3; ch++) {
		if (deg > 0) {
			dx[ch] = -kSH_C1 * SHC(3); dy[ch] = -kSH_C1 * SHC(1); dz[ch] = kSH_C1 * SHC(2);
			if (deg > 1) {
				dx[ch] += kSH_C2_0 * y * SHC(4) + kSH_C2_2 * 2.f * -x * SHC(6) + kSH_C2_3 * z * SHC(7) + kSH_C2_4 * 2.f * x * SHC(8);
				dy[ch] += kSH_C2_0 * x * SHC(4) + kSH_C2_1 * z * SHC(5) + kSH_C2_2 * 2.f * -y * SHC(6) + kSH_C2_4 * 2.f * -y * SHC(8);
				dz[ch] += kSH_C2_1 * y * SHC(5) + kSH_C2_2 * 2.f * 2.f * z * SHC(6) + kSH_C2_3 * x * SHC(7);
				if (deg > 2) {
					dx[ch] += (kSH_C3_0 * SHC(9) * 3.f * 2.f * xy + kSH_C3_1 * SHC(10) * yz + kSH_C3_2 * SHC(11) * -2.f * xy +
					           kSH_C3_3 * SHC(12) * -3.f * 2.f * xz + kSH_C3_4 * SHC(13) * (-3.f * xx + 4.f * zz - yy) +
					           kSH_C3_5 * SHC(14) * 2.f * xz + kSH_C3_6 * SHC(15) * 3.f * (xx - yy));
					dy[ch] += (kSH_C3_0 * SHC(9) * 3.f * (xx - yy) + kSH_C3_1 * SHC(10) * xz +
					           kSH_C3_2 * SHC(11) * (-3.f * yy + 4.f * zz - xx) + kSH_C3_3 * SHC(12) * -3.f * 2.f * yz +
					           kSH_C3_4 * SHC(13) * -2.f * xy + kSH_C3_5 * SHC(14) * -2.f * yz + kSH_C3_6 * SHC(15) * -3.f * 2.f * xy);
					dz[ch] += (kSH_C3_1 * SHC(10) * xy + kSH_C3_2 * SHC(11) * 4.f * 2.f * yz +
					           kSH_C3_3 * SHC(12) * 3.f * (2.f * zz - xx - yy) + kSH_C3_4 * SHC(13) * 4.f * 2.f * xz +
					           kSH_C3_5 * SHC(14) * (xx - yy));
				}
			}
		}
	}
#undef SHC
	float w[16];
	sh_basis(d, w);
	if (w_out) {
#pragma unroll
		for (int k = 0; k < 16; k++) w_out[k] = w[k];
	}
	const int ncoef = (deg + 1) * (deg + 1);
#pragma unroll
	for (int k = 0; k < 16; k++) {
		if (k < ncoef) {
#pragma unroll
			for (int ch = 0; ch < 3; ch++) put(k, ch, w[k] * g[ch]);
		}
	}
	const float3 dL_ddir = make_float3(dx[0] * g[0] + dx[1] * g[1] + dx[2] * g[2], dy[0] * g[0] + dy[1] * g[1] + dy[2] * g[2],
	                                   dz[0] * g[0] + dz[1] * g[1] + dz[2] * g[2]);
	return dnormvdv(dir_orig, dL_ddir);
}

// Row-pointer flavour: sh / dL_dsh point at this Gaussian's [M][3] rows (dL_dsh may be null).
__device__ __forceinline__ float3 sh_backward(int deg, const float3 pos, const float3 campos, const float* __restrict__ sh,
                                              uint32_t clamp_bits, const float3 dL_dcolor, float* __restrict__ dL_dsh)
{
	return sh_backward_t(deg, pos, campos, clamp_bits, dL_dcolor,
	                     [&](int k, int ch) { return sh[3 * k + ch]; },
	                     [&](int k, int ch, float g) { if (dL_dsh) dL_dsh[3 * k + ch] = g; });
}

// (scale, quaternion) <- dL/dSigma  (reference backward.cu:278-341)
__device__ __forceinline__ void cov3d_backward(const float3 scale, float mod, const float4 rot, const float* dL_dcov3D, float3& dL_dscale,
                                               float4& dL_drot)
{
	const float r = rot.x, x = rot.y, y = rot.z, z = rot.w;
	const Mat3 R = quat_to_mat3(rot);
	const float3 s = make_float3(mod * scale.x, mod * scale.y, mod * scale.z);
	const Mat3 S = diag3(s.x, s.y, s.z);
	const Mat3 M = mat3_mul(S, R);
	Mat3 dL_dSigma;
	dL_dSigma(0, 0) = dL_dcov3D[0]; dL_dSigma(0, 1) = 0.5f * dL_dcov3D[1]; dL_dSigma(0, 2) = 0.5f * dL_dcov3D[2];
	dL_dSigma(1, 0) = 0.5f * dL_dcov3D[1]; dL_dSigma(1, 1) = dL_dcov3D[3]; dL_dSigma(1, 2) = 0.5f * dL_dcov3D[4];
	dL_dSigma(2, 0) = 0.5f * dL_dcov3D[2]; dL_dSigma(2, 1) = 0.5f * dL_dcov3D[4]; dL_dSigma(2, 2) = dL_dcov3D[5];
	Mat3 M2;
#pragma unroll
	for (int i = 0; i < 9; i++) M2.m[i] = M.m[i] * 2.0f;
	const Mat3 dL_dM = mat3_mul(M2, dL_dSigma);
	const Mat3 Rt = mat3_transpose(R);
	Mat3 dL_dMt = mat3_transpose(dL_dM);
	dL_dscale.x = Rt(0, 0) * dL_dMt(0, 0) + Rt(0, 1) * dL_dMt(0, 1) + Rt(0, 2) * dL_dMt(0, 2);
	dL_dscale.y = Rt(1, 0) * dL_dMt(1, 0) + Rt(1, 1) * dL_dMt(1, 1) + Rt(1, 2) * dL_dMt(1, 2);
	dL_dscale.z = Rt(2, 0) * dL_dMt(2, 0) + Rt(2, 1) * dL_dMt(2, 1) + Rt(2, 2) * dL_dMt(2, 2);
#pragma unroll
	for (int rr = 0; rr < 3; rr++) { dL_dMt(0, rr) *= s.x; dL_dMt(1, rr) *= s.y; dL_dMt(2, rr) *= s.z; }
	dL_drot.x = 2 * z * (dL_dMt(0, 1) - dL_dMt(1, 0)) + 2 * y * (dL_dMt(2, 0) - dL_dMt(0, 2)) + 2 * x * (dL_dMt(1, 2) - dL_dMt(2, 1));
	dL_drot.y = 2 * y * (dL_dMt(1, 0) + dL_dMt(0, 1)) + 2 * z * (dL_dMt(2, 0) + dL_dMt(0, 2)) + 2 * r * (dL_dMt(1, 2) - dL_dMt(2, 1)) -
	            4 * x * (dL_dMt(2, 2) + dL_dMt(1, 1));
	dL_drot.z = 2 * x * (dL_dMt(1, 0) + dL_dMt(0, 1)) + 2 * r * (dL_dMt(2, 0) - dL_dMt(0, 2)) + 2 * z * (dL_dMt(1, 2) + dL_dMt(2, 1)) -
	            4 * y * (dL_dMt(2, 2) + dL_dMt(0, 0));
	dL_drot.w = 2 * r * (dL_dMt(0, 1) - dL_dMt(1, 0)) + 2 * x * (dL_dMt(2, 0) + dL_dMt(0, 2)) + 2 * y * (dL_dMt(1, 2) + dL_dMt(2, 1)) -
	            4 * z * (dL_dMt(1, 1) + dL_dMt(0, 0));
}

// Projection part of the per-Gaussian backward: (dL/dmean2D, dL/dconic) -> dL/dcov3D[6] and the covariance- and
// projection-induced parts of dL/dmean3D (reference backward.cu:155-273 and :366-387).
// AA (anti-aliasing, see preprocess_fwd_kernel): the blend used o' = o h. With aa_dL_dop = dL/do' and aa_o = o (or o' when aa_o_is_prime),
// dL/dh = o dL/do' joins dL/d(a, b, c) through dh/d(a0, b, c0) (0 where the clamp of h is active); *aa_h receives h, so the caller can
// form dL/do = h dL/do'.
template <bool AA = false>
__device__ __forceinline__ void gaussian_backward_geom(const Camera& cam, const float3 mean, const float* cov3D, const float2 dL_dmean2D,
                                                       const float3 dL_dconic, float3& dL_dmean, float* dL_dcov, float aa_o = 0.f,
                                                       float aa_dL_dop = 0.f, bool aa_o_is_prime = false, float* aa_h = nullptr)
{
	Cov2DTerms ct;
	cov2d_terms(mean, cam.focal_x, cam.focal_y, cam.tan_fovx, cam.tan_fovy, cov3D, cam.view, ct);
	const Mat3& T = ct.T;
	const Mat3& Vrk = ct.Vrk;
	const float3 t = ct.t;
	const float h_x = cam.focal_x, h_y = cam.focal_y;
	const float a = ct.cov(0, 0) + 0.3f;
	const float b = ct.cov(0, 1);
	const float c = ct.cov(1, 1) + 0.3f;
	const float denom = a * c - b * b;
	float dL_da = 0, dL_db = 0, dL_dc = 0;
	const float denom2inv = 1.0f / ((denom * denom) + 0.0000001f);
	if (denom2inv != 0) {
		dL_da = denom2inv * (-c * c * dL_dconic.x + 2 * b * c * dL_dconic.y + (denom - a * c) * dL_dconic.z);
		dL_dc = denom2inv * (-a * a * dL_dconic.z + 2 * a * b * dL_dconic.y + (denom - a * c) * dL_dconic.x);
		dL_db = denom2inv * 2 * (b * c * dL_dconic.x - (denom + 2 * b * b) * dL_dconic.y + a * b * dL_dconic.z);
		if (AA) {
			// h = sqrt(det0 / det1): dh/da0 = h/2 (c0/det0 - c1/det1), dh/dc0 = h/2 (a0/det0 - a1/det1), dh/db = h b (1/det1 - 1/det0)
			const float a0 = ct.cov(0, 0), c0 = ct.cov(1, 1);
			const float det0 = aa_det0(ct);
			const float h = aa_factor(det0, denom);
			*aa_h = h;
			if (det0 / denom > kAaMinRatio) {
				const float dL_dh = (aa_o_is_prime ? aa_o / h : aa_o) * aa_dL_dop;
				const float i0 = 1.f / det0, i1 = 1.f / denom;
				dL_da += dL_dh * (0.5f * h * (c0 * i0 - c * i1));
				dL_dc += dL_dh * (0.5f * h * (a0 * i0 - a * i1));
				dL_db += dL_dh * (h * b * (i1 - i0));
			}
		}
		dL_dcov[0] = (T(0, 0) * T(0, 0) * dL_da + T(0, 0) * T(1, 0) * dL_db + T(1, 0) * T(1, 0) * dL_dc);
		dL_dcov[3] = (T(0, 1) * T(0, 1) * dL_da + T(0, 1) * T(1, 1) * dL_db + T(1, 1) * T(1, 1) * dL_dc);
		dL_dcov[5] = (T(0, 2) * T(0, 2) * dL_da + T(0, 2) * T(1, 2) * dL_db + T(1, 2) * T(1, 2) * dL_dc);
		dL_dcov[1] = 2 * T(0, 0) * T(0, 1) * dL_da + (T(0, 0) * T(1, 1) + T(0, 1) * T(1, 0)) * dL_db + 2 * T(1, 0) * T(1, 1) * dL_dc;
		dL_dcov[2] = 2 * T(0, 0) * T(0, 2) * dL_da + (T(0, 0) * T(1, 2) + T(0, 2) * T(1, 0)) * dL_db + 2 * T(1, 0) * T(1, 2) * dL_dc;
		dL_dcov[4] = 2 * T(0, 2) * T(0, 1) * dL_da + (T(0, 1) * T(1, 2) + T(0, 2) * T(1, 1)) * dL_db + 2 * T(1, 1) * T(1, 2) * dL_dc;
	} else {
#pragma unroll
		for (int i = 0; i < 6; i++) dL_dcov[i] = 0;
	}
	const float dL_dT00 = 2 * (T(0, 0) * Vrk(0, 0) + T(0, 1) * Vrk(0, 1) + T(0, 2) * Vrk(0, 2)) * dL_da +
	                      (T(1, 0) * Vrk(0, 0) + T(1, 1) * Vrk(0, 1) + T(1, 2) * Vrk(0, 2)) * dL_db;
	const float dL_dT01 = 2 * (T(0, 0) * Vrk(1, 0) + T(0, 1) * Vrk(1, 1) + T(0, 2) * Vrk(1, 2)) * dL_da +
	                      (T(1, 0) * Vrk(1, 0) + T(1, 1) * Vrk(1, 1) + T(1, 2) * Vrk(1, 2)) * dL_db;
	const float dL_dT02 = 2 * (T(0, 0) * Vrk(2, 0) + T(0, 1) * Vrk(2, 1) + T(0, 2) * Vrk(2, 2)) * dL_da +
	                      (T(1, 0) * Vrk(2, 0) + T(1, 1) * Vrk(2, 1) + T(1, 2) * Vrk(2, 2)) * dL_db;
	const float dL_dT10 = 2 * (T(1, 0) * Vrk(0, 0) + T(1, 1) * Vrk(0, 1) + T(1, 2) * Vrk(0, 2)) * dL_dc +
	                      (T(0, 0) * Vrk(0, 0) + T(0, 1) * Vrk(0, 1) + T(0, 2) * Vrk(0, 2)) * dL_db;
	const float dL_dT11 = 2 * (T(1, 0) * Vrk(1, 0) + T(1, 1) * Vrk(1, 1) + T(1, 2) * Vrk(1, 2)) * dL_dc +
	                      (T(0, 0) * Vrk(1, 0) + T(0, 1) * Vrk(1, 1) + T(0, 2) * Vrk(1, 2)) * dL_db;
	const float dL_dT12 = 2 * (T(1, 0) * Vrk(2, 0) + T(1, 1) * Vrk(2, 1) + T(1, 2) * Vrk(2, 2)) * dL_dc +
	                      (T(0, 0) * Vrk(2, 0) + T(0, 1) * Vrk(2, 1) + T(0, 2) * Vrk(2, 2)) * dL_db;
	// W(c, r): c-th column of the view rotation as filled in cov2d_terms
	const float* vm = cam.view;
	const float W00 = vm[0], W01 = vm[4], W02 = vm[8], W10 = vm[1], W11 = vm[5], W12 = vm[9], W20 = vm[2], W21 = vm[6], W22 = vm[10];
	const float dL_dJ00 = W00 * dL_dT00 + W01 * dL_dT01 + W02 * dL_dT02;
	const float dL_dJ02 = W20 * dL_dT00 + W21 * dL_dT01 + W22 * dL_dT02;
	const float dL_dJ11 = W10 * dL_dT10 + W11 * dL_dT11 + W12 * dL_dT12;
	const float dL_dJ12 = W20 * dL_dT10 + W21 * dL_dT11 + W22 * dL_dT12;
	const float tz = 1.f / t.z;
	const float tz2 = tz * tz;
	const float tz3 = tz2 * tz;
	const float dL_dtx = ct.x_grad_mul * -h_x * tz2 * dL_dJ02;
	const float dL_dty = ct.y_grad_mul * -h_y * tz2 * dL_dJ12;
	const float dL_dtz = -h_x * tz2 * dL_dJ00 - h_y * tz2 * dL_dJ11 + (2 * h_x * t.x) * tz3 * dL_dJ02 + (2 * h_y * t.y) * tz3 * dL_dJ12;
	dL_dmean = make_float3(vm[0] * dL_dtx + vm[1] * dL_dty + vm[2] * dL_dtz, vm[4] * dL_dtx + vm[5] * dL_dty + vm[6] * dL_dtz,
	                       vm[8] * dL_dtx + vm[9] * dL_dty + vm[10] * dL_dtz);

	const float* proj = cam.proj;
	const float3 m = mean;
	const float4 m_hom = xform4x4(m, proj);
	const float m_w = 1.0f / (m_hom.w + 0.0000001f);
	const float mul1 = (proj[0] * m.x + proj[4] * m.y + proj[8] * m.z + proj[12]) * m_w * m_w;
	const float mul2 = (proj[1] * m.x + proj[5] * m.y + proj[9] * m.z + proj[13]) * m_w * m_w;
	float3 dm2;
	dm2.x = (proj[0] * m_w - proj[3] * mul1) * dL_dmean2D.x + (proj[1] * m_w - proj[3] * mul2) * dL_dmean2D.y;
	dm2.y = (proj[4] * m_w - proj[7] * mul1) * dL_dmean2D.x + (proj[5] * m_w - proj[7] * mul2) * dL_dmean2D.y;
	dm2.z = (proj[8] * m_w - proj[11] * mul1) * dL_dmean2D.x + (proj[9] * m_w - proj[11] * mul2) * dL_dmean2D.y;
	dL_dmean.x += dm2.x; dL_dmean.y += dm2.y; dL_dmean.z += dm2.z;

}

// Everything between the 9 screen-space sums and the activated 3D parameters, for one visible Gaussian
// (row-pointer SH layout [M][3]; dL/dsh written through the pointer if non-null). AA: as gaussian_backward_geom, with aa_o = o'.
template <bool AA = false>
__device__ __forceinline__ void gaussian_backward(const GaussIn& in, const Camera& cam, int idx, const float3 mean, const float* cov3D,
                                                  const float3 scale, const float4 rot, const float* __restrict__ sh_row,
                                                  uint32_t clamp_bits, const float2 dL_dmean2D, const float3 dL_dconic,
                                                  const float3 dL_dcolor, float* __restrict__ dL_dsh_row, float3& dL_dmean, float* dL_dcov,
                                                  float3& dL_dscale, float4& dL_drot, float aa_o_prime = 0.f, float aa_dL_dop = 0.f,
                                                  float* aa_h = nullptr)
{
	(void)idx;
	gaussian_backward_geom<AA>(cam, mean, cov3D, dL_dmean2D, dL_dconic, dL_dmean, dL_dcov, aa_o_prime, aa_dL_dop, true, aa_h);
	if (sh_row) {
		const float3 campos = make_float3(cam.campos[0], cam.campos[1], cam.campos[2]);
		const float3 dsh = sh_backward(in.D, mean, campos, sh_row, clamp_bits, dL_dcolor, dL_dsh_row);
		dL_dmean.x += dsh.x; dL_dmean.y += dsh.y; dL_dmean.z += dsh.z;
	}
	if (in.scales) cov3d_backward(scale, in.scale_modifier, rot, dL_dcov, dL_dscale, dL_drot);
}

}  // namespace psb
