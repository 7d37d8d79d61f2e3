// Internal kernel-launch interface shared by the translation units of libpsb200 (not installed).
#pragma once
#include "psb_common.cuh"
#include "psb_state.h"

namespace psb {

// Per-Gaussian inputs of the forward/backward preprocess. Exactly one of {shs | sh_dc+sh_rest | colors_precomp}
// and one of {scales+rotations | cov3D_precomp} is non-null ("None" = nullptr, the reference's empty-tensor
// convention, reference gaussian_rasterizer.cpp:209-219).
struct GaussIn {
	int P, D, M;
	const float* means3D;        // [P,3]
	const float* scales;         // [P,3]
	const float* rotations;      // [P,4] (w,x,y,z)
	const float* opacities;      // [P]
	const float* shs;            // [P,M,3]
	const float* sh_dc;          // [P,1,3]   (raw trainer layout)
	const float* sh_rest;        // [P,M-1,3] (raw trainer layout)
	const float* cov3D_precomp;  // [P,6]
	const float* colors_precomp; // [P,3]
	float scale_modifier;
	int sh_vec4;                 // shs rows are 16-byte aligned and M == 16: use 128-bit loads
};

// Where the tile backward kernel adds its 9 per-Gaussian sums. Strides in floats.
struct GradSink {
	float* mean2D;  int mean2D_stride;   // .x .y at +0 +1
	float* conic;   int conic_stride;    // .x .y .w at +0 +1 +3
	float* opacity; int opacity_stride;
	float* color;   int color_stride;    // rgb at +0..2
	int packed;                          // != 0: one 16-byte aligned [P][12] row layout (mean2D base), vector reductions
	float* z = nullptr; int z_stride = 0;  // unpacked sink with a depth gradient: the tenth sum, dL/dz (the packed row keeps it in slot 11)
};

// The operator's unpacked sink with a normal gradient: GradSink plus the dL/dn destination (three sums at +0..2). A type of its own
// rather than two more GradSink fields, so that the kernels taking a GradSink keep their parameter layout and code.
struct GradSinkN : GradSink {
	float* n = nullptr; int n_stride = 0;
};

// Deterministic mode of the tile backward (the trainer's packed sink, or the operator's unpacked one). Float atomics from tiles that finish in any order would
// sum a Gaussian's (Gaussian, tile) flushes in a different order every run; instead each flush is STORED in the slot of its
// instance's emission index, base[g] + (rank of the tile among g's instances, InstRect), and gather_slots_kernel then sums every
// Gaussian's slots in emission order and writes its sink row(s). A slot counts only when tagged with this pass's `seq`: entries the
// tile backward does not flush (behind a tile's deepest contributor, culled by the reach tests) keep an older tag and read as zero.
struct DetSlots {
	float4* slots;              // [capacity][3]: one packed sink row per instance; lane 2 (padding) = seq of the pass that wrote it
	const uint32_t* base;       // [P] emission offset of each Gaussian with instances (emit_scan_kernel, DET; operator path: launch_det_base)
	const uint4* tile_info;     // GeomState::tile_info
	const uint32_t* counters;   // GeomState::counters: an overflowing pass (counters[0] > capacity) gathers nothing
	uint32_t capacity, seq;
	int P, tight;
};

// Where the score pass of the forward tile kernel adds its contribution scores (include/psb200.h, psb_trainer_contribution): [P] each.
struct ScoreSink {
	uint32_t* max;             // largest blending weight, as the bits of a non-negative float (atomicMax)
	unsigned long long* sum;   // summed blending weight in units of 2^-kScoreFracBits, each pixel's weight truncated (atomicAdd)
};
constexpr int kScoreFracBits = 26;   // PSB_CONTRIB_SUM_FRAC_BITS
constexpr float kScoreUnitsPerWeight = (float)(1u << kScoreFracBits);

// What the forward tile pass renders beyond colour, final T and n_contrib (launch_render_forward); a null pointer leaves its plane out.
// The set of planes picks the render_fwd_kernel<F> instantiation.
struct FwdPlanes {
	float* out_depth;       // [H,W] the expected depth D
	float* out_alpha;       // [H,W] the accumulated opacity 1 - final_T
	const float4* normals;  // [P] n_i of the pass (launch_normals); read with out_normal only
	float* out_normal;      // [3,H,W] the normal plane
	float* out_depth2;      // [H,W] the second depth moment sum z^2 alpha T; a depth variant, in which out_depth may be null
	ScoreSink score;        // score.max != null: also add the contribution scores (colour only: no other plane)
};

// What the tile backward takes beyond dL/dpix (launch_render_backward); a null pointer leaves its plane out. The set of planes and the sink
// pick the render_bwd_kernel<F, Sink> instantiation.
struct BwdPlanes {
	const float* dL_ddepth;   // [H,W] depth variant: dL/dz of every Gaussian lands in slot 11 of its packed sink row, or at sink.z
	                          // (unpacked sink; refused without either destination)
	const DetSlots* det;      // the deterministic variant: slot stores, then the ordered gather, which WRITES the sink rows
	const float* dL_dalpha;   // [H,W] opacity variant: the gradient of the accumulated opacity 1 - final_T joins dL/dalpha of every splat
	const float4* normals;    // [P] n_i of the forward pass; with dL_dnormal only
	const float* dL_dnormal;  // [3,H,W] normal variant: packed 16-float sink rows and 64-byte deterministic slots, or with an unpacked sink
	                          // (the operator) the GradSinkN variant, which sends dL/dn to dL_dn
	const float* dL_ddepth2;  // [H,W] moment variant (a depth variant; dL_ddepth may be null): its dL/dz (slot 11 of a packed sink, sink.z
	                          // of an unpacked one) includes 2 z dL/dM
	float* dL_dn;             // [P,3] (unpacked sink with dL_dnormal) receives dL/dn
};

// Outputs of the per-Gaussian backward (any pointer may be null = not wanted).
struct GaussGradOut {
	float* dL_dmeans3D;  // [P,3]
	float* dL_dcov3D;    // [P,6]
	float* dL_dsh;       // [P,M,3]
	float* dL_dscales;   // [P,3]
	float* dL_drots;     // [P,4]
};

// tiles of an image of width x height pixels in x and y
inline int2 tile_grid(int width, int height) { return make_int2(cdiv(width, PSB_TILE_X), cdiv(height, PSB_TILE_Y)); }

inline Camera make_camera(int width, int height, const float* view, const float* proj, const float* campos, float tan_fovx, float tan_fovy)
{
	Camera cam;
	cam.view = view; cam.proj = proj; cam.campos = campos;
	cam.tan_fovx = tan_fovx; cam.tan_fovy = tan_fovy;
	cam.focal_y = height / (2.0f * tan_fovy);
	cam.focal_x = width / (2.0f * tan_fovx);
	cam.W = width; cam.H = height;
	const int2 grid = tile_grid(width, height);
	cam.grid_x = grid.x; cam.grid_y = grid.y;
	return cam;
}

// The half of a BinState's ping-pong buffers (tile_key / inst) that holds the instance list sorted by tile, for an image of
// width x height pixels (the plan launch_binning / launch_scan_binning sort with).
inline int sorted_slot(int width, int height)
{
	const int2 grid = tile_grid(width, height);
	return make_sort_plan(tile_id_bits(grid.x * grid.y)).result();
}

// tight: instance lists hold only the tiles a splat can reach (trainer path; see preprocess_fwd_kernel) — pass the same flag to launch_scan_binning
// aa: anti-aliasing (the 2D Mip filter: the record holds o' = o h, see preprocess_fwd_kernel); pair it with the AA variant of the
// per-Gaussian backward that follows
// f3d [P] (raw only; null = off): the 3D smoothing filter (psb_filter3d) per row, see preprocess_fwd_kernel; pair it with the F3D variant of the
// per-Gaussian backward that follows
int launch_preprocess(const GaussIn& in, const Camera& cam, int* radii_out, const GeomState& geom, bool raw, bool tight, cudaStream_t stream,
                      bool aa = false, const float* f3d = nullptr);
int launch_mark_visible(int P, const float* means3D, const float* view, uint8_t* present, cudaStream_t stream);
int launch_depth_sort_and_scan(int P, GeomState& geom, bool scan, cudaStream_t stream);
int launch_binning(int P, const Camera& cam, const GeomState& geom, BinState& bin, const ImgState& img, size_t n_host, cudaStream_t stream);
// B1/B2 path after launch_depth_sort_and_scan(scan = true): base[order[0][j]] <- offsets[j] for every Gaussian with instances, the
// emission offsets by Gaussian index that the deterministic tile backward needs (DetSlots::base); other entries are not written
int launch_det_base(int P, const GeomState& geom, uint32_t* base, cudaStream_t stream);
// base != null (deterministic mode): base[g] <- emission offset of every Gaussian with instances (DetSlots::base)
int launch_scan_binning(int P, const Camera& cam, const GeomState& geom, BinState& bin, const ImgState& img, size_t capacity, bool tight,
                        uint32_t* ovf, uint32_t seq, cudaStream_t stream, uint32_t* base = nullptr);
int launch_render_forward(const Camera& cam, const uint2* ranges, const uint32_t* point_list, const GaussRec* rec, const float* bg,
                          float* out_color, float* final_T, uint32_t* n_contrib, const FwdPlanes& planes, cudaStream_t stream);
// n_i of include/psb200.h (the camera-facing shortest axis in view space) of every visible row of the pass -> normals [P]; raw trainer
// parameters (xyz, scaling, rotation), after launch_preprocess (tile_info says which rows are visible)
int launch_normals(int P, const float* xyz, const float* scaling, const float* rotation, const Camera& cam, const uint4* tile_info, float4* normals,
                   cudaStream_t stream);
// The same n_i from the operator's inputs: activated scales (the arg-min ignores the scale modifier) and the rotation as given, not
// normalised (the operator's covariance does not normalise it either)
int launch_op_normals(const GaussIn& in, const Camera& cam, const uint4* tile_info, float4* normals, cudaStream_t stream);
int launch_render_backward(const Camera& cam, const uint2* ranges, const uint32_t* point_list, const GaussRec* rec, const float* bg,
                           const float* final_T, const uint32_t* n_contrib, const float* dL_dpix, const GradSink& sink, const BwdPlanes& planes,
                           cudaStream_t stream);
// dL_dz [P] (non-null: depth variant): dL/dmean3D += dL/dz (V[2], V[6], V[10]) for every visible Gaussian
// aa_dL_dopacity [P] (non-null: AA variant, after an anti-aliased forward): holds dL/do' on entry, dL/do on return
// dL_dn [P,3] (non-null: normal variant, scales + rotations only): dL/drot += the rotation gradient of n_i (launch_op_normals' n_i)
int launch_preprocess_backward(const GaussIn& in, const Camera& cam, const GeomState& geom, const float* dL_dmean2D, int mean2D_stride,
                               const float* dL_dconic, int conic_stride, const float* dL_dcolor, int color_stride,
                               const GaussGradOut& out, cudaStream_t stream, const float* dL_dz = nullptr, float* aa_dL_dopacity = nullptr,
                               const float* dL_dn = nullptr);

}  // namespace psb
