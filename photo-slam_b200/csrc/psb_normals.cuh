// The depth-normal stencil of include/psb200.h (psb_depth_normals), shared by depth_normals_kernel (psb_normals.cu) and the depth-normal
// consistency term (psb_loss.cu), so both give the same n_d from the same five depths.
#pragma once
#include "psb_common.cuh"

namespace psb {

struct NormalCam {
	int W, H;
	float fx, fy, half_w, half_h;  // the seeding rule's back-projection (psb_seed_apply)
};

inline NormalCam normal_cam(int W, int H, float tan_fovx, float tan_fovy)
{
	NormalCam c;
	c.W = W; c.H = H;
	c.fx = (float)c.W / (2.0f * tan_fovx);
	c.fy = (float)c.H / (2.0f * tan_fovy);
	c.half_w = 0.5f * (float)c.W; c.half_h = 0.5f * (float)c.H;
	return c;
}

__device__ __forceinline__ float3 back_project(const NormalCam& c, int u, int v, float z)
{
	return make_float3(((float)u + 0.5f - c.half_w) * z / c.fx, ((float)v + 0.5f - c.half_h) * z / c.fy, z);
}

__device__ __forceinline__ bool usable(float z) { return isfinite(z) && z > 0.f; }

// The pieces of the stencil the consistency term differentiates: a = X(u+1,v) - X(u-1,v), b = X(u,v+1) - X(u,v-1), c = a x b and
// s = +-1 / |c| (the camera-facing flip over the length), so n = s c. s = 0 where n is (0,0,0); a, b and c are then unspecified.
struct Stencil {
	float3 a, b, c;
	float s;
};

// n_d at an interior pixel (u, v) with depth z and neighbours zl = z(u-1,v), zr = z(u+1,v), zu = z(u,v-1), zd = z(u,v+1) -> nrm, which
// is left as the caller set it ((0,0,0)) at a hole, across a depth edge and where |c| = 0. The caller handles the border and loads the
// five depths.
__device__ __forceinline__ void stencil_normal(const NormalCam& c, int u, int v, float z, float zl, float zr, float zu, float zd, float max_rel_jump,
                                               float3& nrm, Stencil& st)
{
	st.s = 0.f;
	const float jump = max_rel_jump * z;
	if (usable(z) && usable(zl) && usable(zr) && usable(zu) && usable(zd) && !(fabsf(zl - z) > jump) && !(fabsf(zr - z) > jump) &&
	    !(fabsf(zu - z) > jump) && !(fabsf(zd - z) > jump)) {
		const float3 X = back_project(c, u, v, z);
		const float3 L = back_project(c, u - 1, v, zl), R = back_project(c, u + 1, v, zr);
		const float3 U = back_project(c, u, v - 1, zu), D = back_project(c, u, v + 1, zd);
		const float3 a = make_float3(R.x - L.x, R.y - L.y, R.z - L.z), b = make_float3(D.x - U.x, D.y - U.y, D.z - U.z);
		const float3 cr = make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
		const float len = sqrtf(cr.x * cr.x + cr.y * cr.y + cr.z * cr.z);
		st.a = a; st.b = b; st.c = cr;
		if (len > 0.f) {
			const float s = (cr.x * X.x + cr.y * X.y + cr.z * X.z < 0.f ? 1.f : -1.f) / len;
			st.s = s;
			nrm = make_float3(cr.x * s, cr.y * s, cr.z * s);
		}
	}
}

}  // namespace psb
