// C-ABI entry points of libpsb200 (declared in include/psb200.h) and the host orchestration of one
// rasterization: scratch carving through the caller's allocator callbacks, kernel sequence, error checks.
#include <cstdio>
#include <cstring>
#include <string>
#include "psb_kernels.h"
#include "../../include/psb200.h"

namespace psb {

static thread_local std::string g_last_error;

void set_error(const char* what, cudaError_t e, const char* file, int line)
{
	char buf[512];
	snprintf(buf, sizeof(buf), "%s failed: %s (%s:%d)", what, cudaGetErrorString(e), file, line);
	g_last_error = buf;
}
void set_error_msg(const char* what) { g_last_error = what; }

static GaussIn make_input(int P, int D, int M, const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
                          const float* scales, float scale_modifier, const float* rotations, const float* cov3D_precomp)
{
	GaussIn in;
	memset(&in, 0, sizeof(in));
	in.P = P; in.D = D; in.M = M;
	in.means3D = means3D; in.scales = scales; in.rotations = rotations; in.opacities = opacities;
	in.shs = shs; in.cov3D_precomp = cov3D_precomp; in.colors_precomp = colors_precomp;
	in.scale_modifier = scale_modifier;
	in.sh_vec4 = (shs != nullptr && M == 16 && (reinterpret_cast<uintptr_t>(shs) & 15) == 0) ? 1 : 0;
	return in;
}

// ---- debug export kernels ------------------------------------------------------------------------
__global__ void export_geom_kernel(int P, GeomState geom, float* depths, float* means2D, float* conic_opacity, float* rgb, uint8_t* clamped,
                                   uint32_t* tiles_touched)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P) return;
	const uint32_t tt = geom.tile_info[i].z;
	GaussRec r;
	r.q0 = r.q1 = r.q2 = make_float4(0, 0, 0, 0);
	if (tt) r = geom.rec[i];
	if (tiles_touched) tiles_touched[i] = tt;
	if (depths) depths[i] = r.q1.w;
	if (means2D) { means2D[2 * i] = r.q0.x; means2D[2 * i + 1] = r.q0.y; }
	if (conic_opacity) { conic_opacity[4 * i] = r.q0.z; conic_opacity[4 * i + 1] = r.q0.w; conic_opacity[4 * i + 2] = r.q1.x; conic_opacity[4 * i + 3] = r.q1.y; }
	if (rgb) { rgb[3 * i] = r.q2.x; rgb[3 * i + 1] = r.q2.y; rgb[3 * i + 2] = r.q2.z; }
	if (clamped) {
		const uint32_t cb = rec_clamp_bits(__float_as_uint(r.q2.w));
		clamped[3 * i] = cb & 1u; clamped[3 * i + 1] = (cb >> 1) & 1u; clamped[3 * i + 2] = (cb >> 2) & 1u;
	}
}
__global__ void export_keys_kernel(int R, const uint32_t* tile_key, const uint32_t* inst, const GaussRec* rec, uint64_t* keys, uint32_t* values)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= R) return;
	const uint32_t g = inst[i];
	if (keys) keys[i] = ((uint64_t)tile_key[i] << 32) | (uint64_t)__float_as_uint(rec[g].q1.w);
	if (values) values[i] = g;
}

static int arg_error(const char* fn, const char* what)
{
	g_last_error = std::string(fn) + ": " + what;
	return PSB_ERR_ARG;
}

// Scratch bytes of the operator's normal plane; 0 for a negative size.
static size_t op_plane_bytes(int P, int R) { return (P < 0 || R < 0) ? 0 : OpPlaneState::required_bytes((size_t)P, (size_t)R); }

// Body of psb_rasterize_forward[_depth|_aa|_planes]; fn names the entry point in error messages. pl: the planes beyond colour
// (include/psb200.h psb_raster_planes; pl.normals is filled in here); plane_scratch / plane_bytes: the caller's scratch of
// psb_rasterize_planes_bytes(P, 0) bytes, read only with the normal plane; aa: the 2D Mip filter.
static int rasterize_forward(const char* fn, psb_alloc_fn geometry_buffer, void* geometry_user, psb_alloc_fn binning_buffer, void* binning_user,
                             psb_alloc_fn image_buffer, void* image_user, int P, int D, int M, const float* background, int width, int height,
                             const float* means3D, const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                             float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                             const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                             int* radii, FwdPlanes pl, void* plane_scratch, size_t plane_bytes, bool aa, void* stream_)
{
	(void)prefiltered;  // the reference only uses it for a device-side assert (auxiliary.h:156-160)
	cudaStream_t stream = (cudaStream_t)stream_;
	if (P < 0 || width <= 0 || height <= 0 || !geometry_buffer || !binning_buffer || !image_buffer) return arg_error(fn, "bad argument");
	if (P > 0 && (!means3D || !opacities || !viewmatrix || !projmatrix || !background || !out_color)) return arg_error(fn, "null required pointer");
	if (P > 0 && ((shs == nullptr) == (colors_precomp == nullptr))) return arg_error(fn, "provide exactly one of shs / colors_precomp");
	if (P > 0 && (((scales == nullptr) || (rotations == nullptr)) == (cov3D_precomp == nullptr))) return arg_error(fn, "provide exactly one of scales+rotations / cov3D_precomp");
	if (P > 0 && shs && (M < (D + 1) * (D + 1) || D > 3 || D < 0)) return arg_error(fn, "SH degree / coefficient count mismatch");
	if (P > 0 && shs && !cam_pos) return arg_error(fn, "cam_pos required with shs");
	if (width > 65535 * 16 || height > 65535 * 16) return arg_error(fn, "image too large");
	if (pl.out_normal && cov3D_precomp) return arg_error(fn, "the normal plane needs scales and rotations, not cov3D_precomp");
	if (pl.out_normal && (!plane_scratch || plane_bytes < op_plane_bytes(P, 0)))
		return arg_error(fn, ("the normal plane needs a plane_scratch of psb_rasterize_planes_bytes(P, 0) = " + std::to_string(op_plane_bytes(P, 0)) +
		                      " bytes").c_str());

	const Camera cam = make_camera(width, height, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy);
	if ((size_t)cam.grid_x * cam.grid_y >= (1u << 24)) return arg_error(fn, "more than 2^24 tiles");

	char* geom_chunk = geometry_buffer(required_bytes<GeomState>((size_t)P), geometry_user);
	char* img_chunk = image_buffer(required_bytes<ImgState>((size_t)width * height), image_user);
	if (!geom_chunk || !img_chunk) return arg_error(fn, "allocator returned null");
	GeomState geom = GeomState::from_chunk(geom_chunk, (size_t)P);
	ImgState img = ImgState::from_chunk(img_chunk, (size_t)width * height);

	const GaussIn in = make_input(P, D, M, means3D, shs, colors_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp);
	int rc;
	if ((rc = launch_preprocess(in, cam, radii, geom, /*raw=*/false, /*tight=*/false, stream, aa))) return rc;
	pl.normals = nullptr;
	if (pl.out_normal) {
		char* chunk = static_cast<char*>(plane_scratch);
		float4* normals = OpPlaneState::from_chunk(chunk, (size_t)P, 0).normals;
		if ((rc = launch_op_normals(in, cam, geom.tile_info, normals, stream))) return rc;
		pl.normals = normals;
	}
	if ((rc = launch_depth_sort_and_scan(P, geom, /*scan=*/true, stream))) return rc;

	uint32_t num_rendered = 0;
	if (P > 0) {
		PSB_CUDA_OK(cudaMemcpyAsync(&num_rendered, geom.counters, sizeof(uint32_t), cudaMemcpyDeviceToHost, stream));
		PSB_CUDA_OK(cudaStreamSynchronize(stream));
	}
	if (num_rendered >= (1u << 30)) { g_last_error = std::string(fn) + ": more than 2^30 instances"; return PSB_ERR_SIZE; }

	char* bin_chunk = binning_buffer(required_bytes<BinState>((size_t)num_rendered), binning_user);
	if (!bin_chunk) return arg_error(fn, "allocator returned null");
	BinState bin = BinState::from_chunk(bin_chunk, (size_t)num_rendered);
	if ((rc = launch_binning(P, cam, geom, bin, img, (size_t)num_rendered, stream))) return rc;

	if ((rc = launch_render_forward(cam, img.ranges, bin.inst[sorted_slot(width, height)], geom.rec, background, out_color, img.final_T, img.n_contrib, pl,
	                                stream)))
		return rc;
	return (int)num_rendered;
}

// Scratch bytes of the deterministic operator backward; 0 for a negative size.
static size_t op_det_bytes(int P, int R) { return (P < 0 || R < 0) ? 0 : OpDetState::required_bytes((size_t)P, (size_t)R); }

// What an entry point adds to the plain backward. dL_ddepth [H,W] or NULL; with it, dL_dz [P] receives dL/dz and the depth variants
// run. det: the deterministic variant over det_scratch (det_bytes: its size). aa: the forward was anti-aliased. dL_dalpha, dL_dnormal,
// dL_ddepth2: the gradients of the other planes (psb_raster_plane_grads); dL_ddepth2 also needs dL_dz, dL_dnormal a plane_scratch of
// psb_rasterize_planes_bytes(P, det ? R : 0) bytes (plane_bytes: its size).
struct BwdVariant {
	const float* dL_ddepth;
	float* dL_dz;
	void* det_scratch;
	size_t det_bytes;
	bool det, aa;
	const float *dL_dalpha, *dL_dnormal, *dL_ddepth2;
	void* plane_scratch;
	size_t plane_bytes;
};

// Body of psb_rasterize_backward[_depth|_deterministic|_aa|_planes]; fn names the entry point in error messages. Every argument check comes
// before any CUDA call.
static int rasterize_backward(const char* fn, int P, int D, int M, int R, const float* background, int width, int height, const float* means3D,
                              const float* shs, const float* colors_precomp, const float* scales, float scale_modifier, const float* rotations,
                              const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                              float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
                              float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D,
                              float* dL_dsh, float* dL_dscale, float* dL_drot, const BwdVariant& v, void* stream_)
{
	(void)radii;  // visibility is re-derived from the private geometry state (tiles_touched), identical to radii > 0
	cudaStream_t stream = (cudaStream_t)stream_;
	const float* dL_ddepth = v.dL_ddepth;
	float* dL_dz = v.dL_dz;
	const bool normal = v.dL_dnormal != nullptr;
	if (dL_ddepth && !dL_dz) return arg_error(fn, "dL_ddepth needs a dL_dz array");
	if (v.dL_ddepth2 && !dL_dz) return arg_error(fn, "dL_ddepth2 needs a dL_dz array");
	if (normal && cov3D_precomp) return arg_error(fn, "dL_dnormal needs scales and rotations, not cov3D_precomp");
	if (normal && !dL_drot) return arg_error(fn, "dL_dnormal needs a dL_drot array");
	if (P == 0) return 0;
	if (P < 0 || R < 0 || !geom_buffer || !binning_buffer || !image_buffer || !dL_dpix || !dL_dmean2D || !dL_dconic || !dL_dopacity || !dL_dcolor)
		return arg_error(fn, "bad argument");
	if (normal && (!scales || !rotations)) return arg_error(fn, "dL_dnormal needs scales and rotations");
	const int plane_R = v.det ? R : 0;
	if (normal && (!v.plane_scratch || v.plane_bytes < op_plane_bytes(P, plane_R)))
		return arg_error(fn, ("dL_dnormal needs a plane_scratch of psb_rasterize_planes_bytes(P, " + std::string(v.det ? "R" : "0") + ") = " +
		                      std::to_string(op_plane_bytes(P, plane_R)) + " bytes").c_str());
	if (v.det && !v.det_scratch) return arg_error(fn, "det_scratch is NULL");
	if (v.det && v.det_bytes < op_det_bytes(P, R))
		return arg_error(fn, ("det_scratch holds " + std::to_string(v.det_bytes) + " bytes, psb_rasterize_backward_det_bytes(P, R) = " +
		                      std::to_string(op_det_bytes(P, R))).c_str());
	const Camera cam = make_camera(width, height, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy);
	GeomState geom = GeomState::from_chunk(geom_buffer, (size_t)P);
	BinState bin = BinState::from_chunk(binning_buffer, (size_t)R);
	ImgState img = ImgState::from_chunk(image_buffer, (size_t)width * height);

	GradSink sink;
	sink.mean2D = dL_dmean2D; sink.mean2D_stride = 3;
	sink.conic = dL_dconic; sink.conic_stride = 4;
	sink.opacity = dL_dopacity; sink.opacity_stride = 1;
	sink.color = dL_dcolor; sink.color_stride = 3;
	sink.packed = 0;
	const bool depth = dL_ddepth || v.dL_ddepth2;
	if (depth) { sink.z = dL_dz; sink.z_stride = 1; }
	const GaussIn in = make_input(P, D, M, means3D, shs, colors_precomp, nullptr, scales, scale_modifier, rotations, cov3D_precomp);
	OpPlaneState ps{};
	int rc;
	if (normal) {
		// n_i is a function of the inputs: recomputed here rather than kept from the forward (the scratch sizes stay functions of P / R / W H)
		char* chunk = static_cast<char*>(v.plane_scratch);
		ps = OpPlaneState::from_chunk(chunk, (size_t)P, (size_t)plane_R);
		PSB_CUDA_OK(cudaMemsetAsync(ps.dn, 0, (size_t)P * 3 * sizeof(float), stream));
		if ((rc = launch_op_normals(in, cam, geom.tile_info, ps.normals, stream))) return rc;
	}
	if (R > 0) {
		DetSlots slots{};
		if (v.det) {
			// Every (Gaussian, tile) sum goes to the slot of its instance, base[g] + the tile's row-major rank in g's full rectangle (the
			// emission order of emit_instances_kernel), and the gather adds each Gaussian's slots in that order. The slots are zeroed on
			// every call: a block handed back by the caller's allocator may hold tags of an earlier call, which the fixed seq would accept.
			char* chunk = static_cast<char*>(v.det_scratch);
			const OpDetState ds = OpDetState::from_chunk(chunk, (size_t)P, (size_t)R);
			// (the normal variant's 64-byte slots live in the plane scratch; ds.slots is then unused)
			float4* slot_rows = normal ? ps.slots : ds.slots;
			PSB_CUDA_OK(cudaMemsetAsync(slot_rows, 0, (size_t)R * (normal ? 4 : 3) * sizeof(float4), stream));
			if ((rc = launch_det_base(P, geom, ds.base, stream))) return rc;
			slots.slots = slot_rows; slots.base = ds.base; slots.tile_info = geom.tile_info; slots.counters = geom.counters;
			slots.capacity = (uint32_t)R; slots.seq = 1u; slots.P = P; slots.tight = 0;
		}
		const BwdPlanes planes{dL_ddepth, v.det ? &slots : nullptr, v.dL_dalpha, ps.normals, v.dL_dnormal, v.dL_ddepth2, ps.dn};
		if ((rc = launch_render_backward(cam, img.ranges, bin.inst[sorted_slot(width, height)], geom.rec, background, img.final_T, img.n_contrib, dL_dpix,
		                                 sink, planes, stream)))
			return rc;
	}

	GaussGradOut out;
	out.dL_dmeans3D = dL_dmean3D; out.dL_dcov3D = dL_dcov3D; out.dL_dsh = dL_dsh; out.dL_dscales = dL_dscale; out.dL_drots = dL_drot;
	// (AA: dL_dopacity holds dL/do' here, the per-Gaussian kernel turns it into dL/do)
	if ((rc = launch_preprocess_backward(in, cam, geom, dL_dmean2D, 3, dL_dconic, 4, dL_dcolor, 3, out, stream, depth ? dL_dz : nullptr,
	                                     v.aa ? dL_dopacity : nullptr, normal ? ps.dn : nullptr)))
		return rc;
	return 0;
}

}  // namespace psb

using namespace psb;

extern "C" {

int psb_version(void) { return 100; }
const char* psb_last_error(void) { return g_last_error.c_str(); }

size_t psb_geometry_bytes(int P) { return required_bytes<GeomState>((size_t)P); }
size_t psb_binning_bytes(int R) { return required_bytes<BinState>((size_t)R); }
size_t psb_image_bytes(int N) { return required_bytes<ImgState>((size_t)N); }

int psb_rasterize_forward(psb_alloc_fn geometry_buffer, void* geometry_user, psb_alloc_fn binning_buffer, void* binning_user,
                          psb_alloc_fn image_buffer, void* image_user, int P, int D, int M, const float* background, int width, int height,
                          const float* means3D, const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                          float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                          const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                          int* radii, void* stream)
{
	return rasterize_forward("psb_rasterize_forward", geometry_buffer, geometry_user, binning_buffer, binning_user, image_buffer, image_user, P, D, M,
	                         background, width, height, means3D, shs, colors_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp,
	                         viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, prefiltered, out_color, radii, FwdPlanes{}, nullptr, 0, /*aa=*/false, stream);
}

int psb_rasterize_forward_depth(psb_alloc_fn geometry_buffer, void* geometry_user, psb_alloc_fn binning_buffer, void* binning_user,
                                psb_alloc_fn image_buffer, void* image_user, int P, int D, int M, const float* background, int width, int height,
                                const float* means3D, const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                                float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                                const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                                int* radii, float* out_depth, void* stream)
{
	return rasterize_forward("psb_rasterize_forward_depth", geometry_buffer, geometry_user, binning_buffer, binning_user, image_buffer, image_user, P,
	                         D, M, background, width, height, means3D, shs, colors_precomp, opacities, scales, scale_modifier, rotations,
	                         cov3D_precomp, viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, prefiltered, out_color, radii, FwdPlanes{out_depth}, nullptr, 0, /*aa=*/false, stream);
}

int psb_rasterize_backward(int P, int D, int M, int R, const float* background, int width, int height, const float* means3D, const float* shs,
                           const float* colors_precomp, const float* scales, float scale_modifier, const float* rotations,
                           const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                           float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
                           float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D,
                           float* dL_dsh, float* dL_dscale, float* dL_drot, void* stream)
{
	return rasterize_backward("psb_rasterize_backward", P, D, M, R, background, width, height, means3D, shs, colors_precomp, scales, scale_modifier,
	                          rotations, cov3D_precomp, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, radii, geom_buffer, binning_buffer,
	                          image_buffer, dL_dpix, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale,
	                          dL_drot, BwdVariant{}, stream);
}

int psb_rasterize_backward_depth(int P, int D, int M, int R, const float* background, int width, int height, const float* means3D,
                                 const float* shs, const float* colors_precomp, const float* scales, float scale_modifier, const float* rotations,
                                 const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                                 float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer,
                                 const float* dL_dpix, float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor,
                                 float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh, float* dL_dscale, float* dL_drot, const float* dL_ddepth,
                                 float* dL_dz, void* stream)
{
	BwdVariant v{};
	v.dL_ddepth = dL_ddepth; v.dL_dz = dL_dz;
	return rasterize_backward("psb_rasterize_backward_depth", P, D, M, R, background, width, height, means3D, shs, colors_precomp, scales,
	                          scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, radii, geom_buffer,
	                          binning_buffer, image_buffer, dL_dpix, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh,
	                          dL_dscale, dL_drot, v, stream);
}

size_t psb_rasterize_backward_det_bytes(int P, int R) { return op_det_bytes(P, R); }

int psb_rasterize_backward_deterministic(int P, int D, int M, int R, const float* background, int width, int height, const float* means3D,
                                         const float* shs, const float* colors_precomp, const float* scales, float scale_modifier,
                                         const float* rotations, const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix,
                                         const float* campos, float tan_fovx, float tan_fovy, const int* radii, char* geom_buffer,
                                         char* binning_buffer, char* image_buffer, const float* dL_dpix, float* dL_dmean2D, float* dL_dconic,
                                         float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                                         float* dL_dscale, float* dL_drot, const float* dL_ddepth, float* dL_dz, void* det_scratch,
                                         size_t det_scratch_bytes, void* stream)
{
	BwdVariant v{};
	v.dL_ddepth = dL_ddepth; v.dL_dz = dL_dz;
	v.det = true; v.det_scratch = det_scratch; v.det_bytes = det_scratch_bytes;
	return rasterize_backward("psb_rasterize_backward_deterministic", P, D, M, R, background, width, height, means3D, shs, colors_precomp, scales,
	                          scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, radii, geom_buffer,
	                          binning_buffer, image_buffer, dL_dpix, dL_dmean2D, dL_dconic, dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh,
	                          dL_dscale, dL_drot, v, stream);
}

int psb_rasterize_forward_aa(psb_alloc_fn geometry_buffer, void* geometry_user, psb_alloc_fn binning_buffer, void* binning_user,
                             psb_alloc_fn image_buffer, void* image_user, int P, int D, int M, const float* background, int width, int height,
                             const float* means3D, const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                             float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                             const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                             int* radii, float* out_depth, int antialiasing, void* stream)
{
	if (antialiasing != 0 && antialiasing != 1) return arg_error("psb_rasterize_forward_aa", "antialiasing must be 0 or 1");
	return rasterize_forward("psb_rasterize_forward_aa", geometry_buffer, geometry_user, binning_buffer, binning_user, image_buffer, image_user, P, D,
	                         M, background, width, height, means3D, shs, colors_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp,
	                         viewmatrix, projmatrix, cam_pos, tan_fovx, tan_fovy, prefiltered, out_color, radii, FwdPlanes{out_depth}, nullptr, 0, antialiasing != 0, stream);
}

int psb_rasterize_backward_aa(int P, int D, int M, int R, const float* background, int width, int height, const float* means3D, const float* shs,
                              const float* colors_precomp, const float* scales, float scale_modifier, const float* rotations,
                              const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                              float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
                              float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D,
                              float* dL_dsh, float* dL_dscale, float* dL_drot, const float* dL_ddepth, float* dL_dz, void* det_scratch,
                              size_t det_scratch_bytes, int antialiasing, void* stream)
{
	const char* fn = "psb_rasterize_backward_aa";
	if (antialiasing != 0 && antialiasing != 1) return arg_error(fn, "antialiasing must be 0 or 1");
	BwdVariant v{};
	v.dL_ddepth = dL_ddepth; v.dL_dz = dL_dz;
	v.det = det_scratch != nullptr; v.det_scratch = det_scratch; v.det_bytes = det_scratch_bytes;
	v.aa = antialiasing != 0;
	return rasterize_backward(fn, P, D, M, R, background, width, height, means3D, shs, colors_precomp, scales, scale_modifier, rotations, cov3D_precomp,
	                          viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, dL_dmean2D,
	                          dL_dconic, dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, v, stream);
}

size_t psb_rasterize_planes_bytes(int P, int R) { return op_plane_bytes(P, R); }

int psb_rasterize_forward_planes(psb_alloc_fn geometry_buffer, void* geometry_user, psb_alloc_fn binning_buffer, void* binning_user,
                                 psb_alloc_fn image_buffer, void* image_user, int P, int D, int M, const float* background, int width, int height,
                                 const float* means3D, const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                                 float scale_modifier, const float* rotations, const float* cov3D_precomp, const float* viewmatrix,
                                 const float* projmatrix, const float* cam_pos, float tan_fovx, float tan_fovy, int prefiltered, float* out_color,
                                 int* radii, const psb_raster_planes* planes, void* plane_scratch, size_t plane_scratch_bytes, int antialiasing,
                                 void* stream)
{
	const char* fn = "psb_rasterize_forward_planes";
	if (antialiasing != 0 && antialiasing != 1) return arg_error(fn, "antialiasing must be 0 or 1");
	FwdPlanes pl{};
	if (planes) { pl.out_depth = planes->out_depth; pl.out_alpha = planes->out_alpha; pl.out_normal = planes->out_normal; pl.out_depth2 = planes->out_depth2; }
	return rasterize_forward(fn, geometry_buffer, geometry_user, binning_buffer, binning_user, image_buffer, image_user, P, D, M, background, width,
	                         height, means3D, shs, colors_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix,
	                         cam_pos, tan_fovx, tan_fovy, prefiltered, out_color, radii, pl, plane_scratch, plane_scratch_bytes, antialiasing != 0, stream);
}

int psb_rasterize_backward_planes(int P, int D, int M, int R, const float* background, int width, int height, const float* means3D, const float* shs,
                                  const float* colors_precomp, const float* scales, float scale_modifier, const float* rotations,
                                  const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* campos, float tan_fovx,
                                  float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
                                  float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D,
                                  float* dL_dsh, float* dL_dscale, float* dL_drot, const psb_raster_plane_grads* grads, float* dL_dz,
                                  void* det_scratch, size_t det_scratch_bytes, void* plane_scratch, size_t plane_scratch_bytes, int antialiasing,
                                  int deterministic, void* stream)
{
	const char* fn = "psb_rasterize_backward_planes";
	if (antialiasing != 0 && antialiasing != 1) return arg_error(fn, "antialiasing must be 0 or 1");
	if (deterministic != 0 && deterministic != 1) return arg_error(fn, "deterministic must be 0 or 1");
	BwdVariant v{};
	if (grads) { v.dL_ddepth = grads->dL_ddepth; v.dL_dalpha = grads->dL_dalpha; v.dL_dnormal = grads->dL_dnormal; v.dL_ddepth2 = grads->dL_ddepth2; }
	v.dL_dz = dL_dz;
	v.det = deterministic != 0; v.det_scratch = det_scratch; v.det_bytes = det_scratch_bytes;
	v.aa = antialiasing != 0;
	v.plane_scratch = plane_scratch; v.plane_bytes = plane_scratch_bytes;
	return rasterize_backward(fn, P, D, M, R, background, width, height, means3D, shs, colors_precomp, scales, scale_modifier, rotations, cov3D_precomp,
	                          viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, dL_dmean2D,
	                          dL_dconic, dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, v, stream);
}

int psb_mark_visible(int P, const float* means3D, const float* viewmatrix, const float* projmatrix, unsigned char* present, void* stream_)
{
	(void)projmatrix;
	if (P < 0 || (P > 0 && (!means3D || !viewmatrix || !present))) { set_error_msg("psb_mark_visible: bad argument"); return PSB_ERR_ARG; }
	return launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)stream_);
}

int psb_debug_export(int P, int R, int width, int height, char* geom_buffer, char* binning_buffer, char* image_buffer, float* depths,
                     float* means2D, float* conic_opacity, float* rgb, unsigned char* clamped, uint32_t* tiles_touched, uint64_t* keys_sorted,
                     uint32_t* values_sorted, uint32_t* ranges, uint32_t* n_contrib, float* final_T, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	if (P <= 0) return 0;
	GeomState geom = GeomState::from_chunk(geom_buffer, (size_t)P);
	export_geom_kernel<<<cdiv(P, 256), 256, 0, stream>>>(P, geom, depths, means2D, conic_opacity, rgb, clamped, tiles_touched);
	PSB_LAUNCH_OK();
	if (binning_buffer && R > 0 && (keys_sorted || values_sorted)) {
		BinState bin = BinState::from_chunk(binning_buffer, (size_t)R);
		const int res = sorted_slot(width, height);
		export_keys_kernel<<<cdiv(R, 256), 256, 0, stream>>>(R, bin.tile_key[res], bin.inst[res], geom.rec, keys_sorted, values_sorted);
		PSB_LAUNCH_OK();
	}
	if (image_buffer) {
		ImgState img = ImgState::from_chunk(image_buffer, (size_t)width * height);
		const int2 grid = tile_grid(width, height);
		if (ranges) PSB_CUDA_OK(cudaMemcpyAsync(ranges, img.ranges, (size_t)grid.x * grid.y * sizeof(uint2), cudaMemcpyDeviceToDevice, stream));
		if (n_contrib) PSB_CUDA_OK(cudaMemcpyAsync(n_contrib, img.n_contrib, (size_t)width * height * sizeof(uint32_t), cudaMemcpyDeviceToDevice, stream));
		if (final_T) PSB_CUDA_OK(cudaMemcpyAsync(final_T, img.final_T, (size_t)width * height * sizeof(float), cudaMemcpyDeviceToDevice, stream));
	}
	return 0;
}

int psb_debug_sort_pairs(uint32_t* keys, uint32_t* vals, size_t n, int nbits, void* stream_)
{
	cudaStream_t stream = (cudaStream_t)stream_;
	if (n == 0) return 0;
	const SortPlan plan = make_sort_plan(nbits);
	CudaBuffer<uint32_t> k1, v1;
	CudaBuffer<char> scratch;
	const size_t sb = sort_scratch_bytes(n, plan.npass);
	PSB_CUDA_OK(k1.grow(n, Fit::exact, false, stream));
	PSB_CUDA_OK(v1.grow(n, Fit::exact, false, stream));
	PSB_CUDA_OK(scratch.grow(sb, Fit::exact, false, stream));
	uint32_t* kk[2] = {keys, k1.get()};
	uint32_t* vv[2] = {vals, v1.get()};
	int rc = radix_sort_pairs(kk, vv, false, nullptr, n, plan, scratch.get(), sb, stream);
	if (rc == 0 && plan.result() == 1) {
		cudaMemcpyAsync(keys, k1.get(), n * 4, cudaMemcpyDeviceToDevice, stream);
		cudaMemcpyAsync(vals, v1.get(), n * 4, cudaMemcpyDeviceToDevice, stream);
	}
	cudaStreamSynchronize(stream);
	return rc;
}

}  // extern "C"
