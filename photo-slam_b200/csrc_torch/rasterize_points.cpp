// libcuda_rasterizer drop-in: the reference's torch-typed glue (B1) and raw-pointer class (B2) re-exported with
// the reference's exact C++ signatures, implemented on the psb200 C-ABI.
//
//   RasterizeGaussiansCUDA / RasterizeGaussiansBackwardCUDA / markVisible
//        reference include/rasterize_points.h:18-65 (definitions src/rasterize_points.cu:36-214)
//   CudaRasterizer::Rasterizer::{forward, backward, markVisible}
//        reference cuda_rasterizer/rasterizer.h:24-82
//
// libgaussian_mapper.so links against exactly these symbols (SURVEY.md §8b); building this file into
// libcuda_rasterizer.so (+ libpsb200.so) swaps the rasterizer without touching any caller. Pure C++/LibTorch host
// code: no kernels here. Every RasterizeGaussians*CUDA forward is forward_impl and every backward is backward_impl (below), which
// differ per export only in the C entry point they call; the planes pair (RasterizeGaussians[Backward]PlanesCUDA) calls the one C entry
// point that takes every plane in a record. The TORCH_LIBRARY block at the end only exists so the Python test-suite can call the
// C++ entry points (torch.ops.psb200.*).
#include <functional>
#include <optional>
#include <stdexcept>
#include <tuple>
#include <vector>
#include <torch/torch.h>
#include <torch/library.h>
#include <c10/cuda/CUDAStream.h>
#include "../../include/psb200.h"

namespace {

char* resize_cb(size_t n, void* user)
{
	// reference resizeFunctional (src/rasterize_points.cu:28-34)
	auto* t = static_cast<torch::Tensor*>(user);
	t->resize_({(long long)n});
	return reinterpret_cast<char*>(t->contiguous().data_ptr());
}

const float* fptr(const torch::Tensor& t) { return t.numel() ? t.contiguous().data_ptr<float>() : nullptr; }

void* current_stream() { return (void*)c10::cuda::getCurrentCUDAStream().stream(); }

char* fn_cb(size_t n, void* user) { return (*static_cast<std::function<char*(size_t)>*>(user))(n); }

using Fwd7 = std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>;
using Bwd8 = std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>;

// The one forward behind RasterizeGaussians[Depth|Antialiased]CUDA -> (rendered, out_color, out_depth, radii, geomBuffer, binningBuffer,
// imgBuffer). depth: also the [H,W] depth image (out_depth stays undefined without it); aa: the 2D Mip filter. Each combination calls
// the narrowest C entry point that has it.
Fwd7 forward_impl(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors, const torch::Tensor& opacity,
                  const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                  const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                  const int image_height, const int image_width, const torch::Tensor& sh, const int degree, const torch::Tensor& campos,
                  const bool prefiltered, const bool depth, const bool aa)
{
	if (means3D.ndimension() != 2 || means3D.size(1) != 3) { AT_ERROR("means3D must have dimensions (num_points, 3)"); }
	const int P = means3D.size(0);
	const int H = image_height, W = image_width;
	auto float_opts = means3D.options().dtype(torch::kFloat32);
	torch::Tensor out_color = torch::full({3, H, W}, 0.0, float_opts);
	torch::Tensor out_depth;
	if (depth) out_depth = torch::full({H, W}, 0.0, float_opts);
	torch::Tensor radii = torch::full({P}, 0, means3D.options().dtype(torch::kInt32));
	torch::TensorOptions options(torch::kByte);
	torch::Tensor geomBuffer = torch::empty({0}, options.device(means3D.device()));
	torch::Tensor binningBuffer = torch::empty({0}, options.device(means3D.device()));
	torch::Tensor imgBuffer = torch::empty({0}, options.device(means3D.device()));
	int rendered = 0;
	if (P != 0) {
		int M = 0;
		if (sh.size(0) != 0) M = sh.size(1);
		// keep contiguous copies alive for the duration of the call
		const auto bg = background.contiguous(), m3 = means3D.contiguous(), shc = sh.contiguous(), col = colors.contiguous(), op = opacity.contiguous(),
		           sc = scales.contiguous(), rot = rotations.contiguous(), cov = cov3D_precomp.contiguous(), vm = viewmatrix.contiguous(),
		           pm = projmatrix.contiguous(), cp = campos.contiguous();
		// the arguments every forward entry point starts with
		const auto args = std::make_tuple(&resize_cb, (void*)&geomBuffer, &resize_cb, (void*)&binningBuffer, &resize_cb, (void*)&imgBuffer, P, degree, M,
		                                  fptr(bg), W, H, fptr(m3), fptr(shc), fptr(col), fptr(op), fptr(sc), scale_modifier, fptr(rot), fptr(cov),
		                                  fptr(vm), fptr(pm), fptr(cp), tan_fovx, tan_fovy, prefiltered ? 1 : 0, out_color.data_ptr<float>(),
		                                  radii.data_ptr<int>());
		float* dep = depth ? out_depth.data_ptr<float>() : nullptr;
		void* stream = current_stream();
		if (aa) {
			rendered = std::apply([&](auto... a) { return psb_rasterize_forward_aa(a..., dep, 1, stream); }, args);
			if (rendered < 0) { AT_ERROR("psb_rasterize_forward_aa: ", psb_last_error()); }
		} else if (depth) {
			rendered = std::apply([&](auto... a) { return psb_rasterize_forward_depth(a..., dep, stream); }, args);
			if (rendered < 0) { AT_ERROR("psb_rasterize_forward_depth: ", psb_last_error()); }
		} else {
			rendered = std::apply([&](auto... a) { return psb_rasterize_forward(a..., stream); }, args);
			if (rendered < 0) { AT_ERROR("psb_rasterize_forward: ", psb_last_error()); }
		}
	}
	return std::make_tuple(rendered, out_color, out_depth, radii, geomBuffer, binningBuffer, imgBuffer);
}

// Which C entry point a backward export calls: each the previous one plus one thing (a depth gradient; the fixed-order sums over a
// scratch; the h-term of an anti-aliased forward, deterministic or not).
enum class Bwd { Plain, Depth, Deterministic, Antialiased };

// The one backward behind RasterizeGaussiansBackward[Depth|Deterministic|Antialiased]CUDA. dL_dout_depth [H,W]; undefined or empty is
// colour only (and all Bwd::Plain takes). `deterministic` is read by Bwd::Antialiased alone.
Bwd8 backward_impl(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii, const torch::Tensor& colors,
                   const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                   const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                   const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_depth, const torch::Tensor& sh, const int degree,
                   const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R, const torch::Tensor& binningBuffer,
                   const torch::Tensor& imageBuffer, const Bwd mode, const bool deterministic)
{
	const int P = means3D.size(0);
	const int H = dL_dout_color.size(1), W = dL_dout_color.size(2);
	const bool depth = dL_dout_depth.defined() && dL_dout_depth.numel() != 0;
	if (depth && (dL_dout_depth.ndimension() != 2 || dL_dout_depth.size(0) != H || dL_dout_depth.size(1) != W)) {
		AT_ERROR("dL_dout_depth must have dimensions (", H, ", ", W, ")");
	}
	int M = 0;
	if (sh.size(0) != 0) M = sh.size(1);
	torch::Tensor dL_dmeans3D = torch::zeros({P, 3}, means3D.options());
	torch::Tensor dL_dmeans2D = torch::zeros({P, 3}, means3D.options());
	torch::Tensor dL_dcolors = torch::zeros({P, 3}, means3D.options());
	torch::Tensor dL_dconic = torch::zeros({P, 2, 2}, means3D.options());
	torch::Tensor dL_dopacity = torch::zeros({P, 1}, means3D.options());
	torch::Tensor dL_dcov3D = torch::zeros({P, 6}, means3D.options());
	torch::Tensor dL_dsh = torch::zeros({P, M, 3}, means3D.options());
	torch::Tensor dL_dscales = torch::zeros({P, 3}, means3D.options());
	torch::Tensor dL_drotations = torch::zeros({P, 4}, means3D.options());
	if (P != 0) {
		const auto bg = background.contiguous(), m3 = means3D.contiguous(), shc = sh.contiguous(), col = colors.contiguous(), sc = scales.contiguous(),
		           rot = rotations.contiguous(), cov = cov3D_precomp.contiguous(), vm = viewmatrix.contiguous(), pm = projmatrix.contiguous(),
		           cp = campos.contiguous(), dpix = dL_dout_color.contiguous(), rad = radii.contiguous();
		// the arguments every backward entry point starts with
		const auto args = std::make_tuple(
			P, degree, M, R, fptr(bg), W, H, fptr(m3), fptr(shc), fptr(col), fptr(sc), scale_modifier, fptr(rot), fptr(cov), fptr(vm), fptr(pm), fptr(cp),
			tan_fovx, tan_fovy, (const int*)rad.data_ptr<int>(), reinterpret_cast<char*>(geomBuffer.contiguous().data_ptr()),
			reinterpret_cast<char*>(binningBuffer.contiguous().data_ptr()), reinterpret_cast<char*>(imageBuffer.contiguous().data_ptr()), fptr(dpix),
			dL_dmeans2D.data_ptr<float>(), dL_dconic.data_ptr<float>(), dL_dopacity.data_ptr<float>(), dL_dcolors.data_ptr<float>(),
			dL_dmeans3D.data_ptr<float>(), dL_dcov3D.data_ptr<float>(), M ? dL_dsh.data_ptr<float>() : nullptr, dL_dscales.data_ptr<float>(),
			dL_drotations.data_ptr<float>());
		const torch::Tensor ddep_t = depth ? dL_dout_depth.contiguous() : torch::Tensor();
		torch::Tensor dL_dz, det_t;
		if (depth) dL_dz = torch::zeros({P}, means3D.options());
		const float* ddep = depth ? ddep_t.data_ptr<float>() : nullptr;
		float* dz = depth ? dL_dz.data_ptr<float>() : nullptr;
		const bool det = mode == Bwd::Deterministic || (mode == Bwd::Antialiased && deterministic);
		const size_t det_bytes = det ? psb_rasterize_backward_det_bytes(P, R) : 0;
		if (det) det_t = torch::empty({(long long)det_bytes}, means3D.options().dtype(torch::kByte));
		void* det_scratch = det ? det_t.data_ptr() : nullptr;
		void* stream = current_stream();
		int rc = 0;
		switch (mode) {
		case Bwd::Plain:
			rc = std::apply([&](auto... a) { return psb_rasterize_backward(a..., stream); }, args);
			if (rc < 0) { AT_ERROR("psb_rasterize_backward: ", psb_last_error()); }
			break;
		case Bwd::Depth:
			rc = std::apply([&](auto... a) { return psb_rasterize_backward_depth(a..., ddep, dz, stream); }, args);
			if (rc < 0) { AT_ERROR("psb_rasterize_backward_depth: ", psb_last_error()); }
			break;
		case Bwd::Deterministic:
			rc = std::apply([&](auto... a) { return psb_rasterize_backward_deterministic(a..., ddep, dz, det_scratch, det_bytes, stream); }, args);
			if (rc < 0) { AT_ERROR("psb_rasterize_backward_deterministic: ", psb_last_error()); }
			break;
		case Bwd::Antialiased:
			rc = std::apply([&](auto... a) { return psb_rasterize_backward_aa(a..., ddep, dz, det_scratch, det_bytes, 1, stream); }, args);
			if (rc < 0) { AT_ERROR("psb_rasterize_backward_aa: ", psb_last_error()); }
			break;
		}
	}
	return std::make_tuple(dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations);
}

}  // namespace

std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors, const torch::Tensor& opacity,
                       const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                       const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                       const int image_height, const int image_width, const torch::Tensor& sh, const int degree, const torch::Tensor& campos,
                       const bool prefiltered)
{
	const Fwd7 r = forward_impl(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
	                            tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, /*depth=*/false, /*aa=*/false);
	return std::make_tuple(std::get<0>(r), std::get<1>(r), std::get<3>(r), std::get<4>(r), std::get<5>(r), std::get<6>(r));
}

std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansBackwardCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii, const torch::Tensor& colors,
                               const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier,
                               const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix,
                               const float tan_fovx, const float tan_fovy, const torch::Tensor& dL_dout_color, const torch::Tensor& sh,
                               const int degree, const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R,
                               const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer)
{
	return backward_impl(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
	                     dL_dout_color, torch::Tensor(), sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, Bwd::Plain, false);
}

// ---- rendered depth D(p) = sum_i z_i alpha_i T_i (include/psb200.h), which the reference has no symbol for: the two functions
// above with the depth image added, for a GaussianRasterizerFunction that returns and back-propagates depth (INTEGRATION.md §1)
std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansDepthCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors, const torch::Tensor& opacity,
                            const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                            const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                            const int image_height, const int image_width, const torch::Tensor& sh, const int degree, const torch::Tensor& campos,
                            const bool prefiltered)
{
	return forward_impl(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
	                    image_height, image_width, sh, degree, campos, prefiltered, /*depth=*/true, /*aa=*/false);
}

// dL_dout_depth [H,W]; an undefined tensor is the plain backward. dL/dz is folded into dL_dmeans3D, and dL_dmeans2D includes the depth term.
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansBackwardDepthCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii, const torch::Tensor& colors,
                                    const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier,
                                    const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix,
                                    const float tan_fovx, const float tan_fovy, const torch::Tensor& dL_dout_color,
                                    const torch::Tensor& dL_dout_depth, const torch::Tensor& sh, const int degree, const torch::Tensor& campos,
                                    const torch::Tensor& geomBuffer, const int R, const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer)
{
	return backward_impl(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
	                     dL_dout_color, dL_dout_depth, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, Bwd::Depth, false);
}

// RasterizeGaussiansBackwardDepthCUDA whose outputs are bit-identical from call to call (psb_rasterize_backward_deterministic): the
// (Gaussian, tile) sums are added in a fixed order instead of with float atomics. An undefined or empty dL_dout_depth is colour only.
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansBackwardDeterministicCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii,
                                            const torch::Tensor& colors, const torch::Tensor& scales, const torch::Tensor& rotations,
                                            const float scale_modifier, const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix,
                                            const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                                            const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_depth, const torch::Tensor& sh,
                                            const int degree, const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R,
                                            const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer)
{
	return backward_impl(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
	                     dL_dout_color, dL_dout_depth, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, Bwd::Deterministic, true);
}

// ---- anti-aliasing (the 2D Mip filter, upstream diff-gaussian-rasterization's `antialiasing`; include/psb200.h psb_rasterize_forward_aa):
// every splat blends with opacity o' = o h, h = sqrt(max(det0 / det1, 2.5e-5)) of its 2D covariance before / after the 0.3 px^2 dilation.
// RasterizeGaussiansAntialiasedCUDA: the signature and 7-tuple of RasterizeGaussiansDepthCUDA (colour, depth, radii, buffers), anti-aliased.
std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansAntialiasedCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors,
                                  const torch::Tensor& opacity, const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier,
                                  const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix,
                                  const float tan_fovx, const float tan_fovy, const int image_height, const int image_width, const torch::Tensor& sh,
                                  const int degree, const torch::Tensor& campos, const bool prefiltered)
{
	return forward_impl(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
	                    image_height, image_width, sh, degree, campos, prefiltered, /*depth=*/true, /*aa=*/true);
}

// The backward of RasterizeGaussiansAntialiasedCUDA: the signature of RasterizeGaussiansBackwardDeterministicCUDA plus `deterministic`
// (true: bit-identical from call to call; false: the float-atomic backward). dL_dopacity is dL/do; an undefined or empty dL_dout_depth is
// colour only.
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansBackwardAntialiasedCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii,
                                          const torch::Tensor& colors, const torch::Tensor& scales, const torch::Tensor& rotations,
                                          const float scale_modifier, const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix,
                                          const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                                          const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_depth, const torch::Tensor& sh,
                                          const int degree, const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R,
                                          const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const bool deterministic)
{
	return backward_impl(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx, tan_fovy,
	                     dL_dout_color, dL_dout_depth, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, Bwd::Antialiased, deterministic);
}

// ---- opacity, normals and the second depth moment (include/psb200.h psb_rasterize_forward_planes): A = 1 - T_final, N = sum n alpha T,
// M = sum z^2 alpha T beside colour and depth, for a GaussianRasterizerFunction that returns and back-propagates them (INTEGRATION.md §1).
// -> (rendered, out_color, out_depth, out_alpha, out_normal, out_depth2, radii, geomBuffer, binningBuffer, imgBuffer); a plane that is not
// requested comes back undefined. Colour, depth, radii and the buffers are bit-identical to RasterizeGaussiansAntialiasedCUDA's (with the
// same antialiasing flag). The normal plane needs scales and rotations.
std::tuple<int, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansPlanesCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& colors, const torch::Tensor& opacity,
                             const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier, const torch::Tensor& cov3D_precomp,
                             const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix, const float tan_fovx, const float tan_fovy,
                             const int image_height, const int image_width, const torch::Tensor& sh, const int degree, const torch::Tensor& campos,
                             const bool prefiltered, const bool depth, const bool alpha, const bool normal, const bool depth2, const bool antialiasing)
{
	if (means3D.ndimension() != 2 || means3D.size(1) != 3) { AT_ERROR("means3D must have dimensions (num_points, 3)"); }
	if (normal && cov3D_precomp.defined() && cov3D_precomp.numel() != 0) { AT_ERROR("the normal plane needs scales and rotations, not cov3D_precomp"); }
	const int P = means3D.size(0);
	const int H = image_height, W = image_width;
	auto float_opts = means3D.options().dtype(torch::kFloat32);
	torch::Tensor out_color = torch::full({3, H, W}, 0.0, float_opts);
	torch::Tensor out_depth, out_alpha, out_normal, out_depth2;
	if (depth) out_depth = torch::full({H, W}, 0.0, float_opts);
	if (alpha) out_alpha = torch::full({H, W}, 0.0, float_opts);
	if (normal) out_normal = torch::full({3, H, W}, 0.0, float_opts);
	if (depth2) out_depth2 = torch::full({H, W}, 0.0, float_opts);
	torch::Tensor radii = torch::full({P}, 0, means3D.options().dtype(torch::kInt32));
	torch::TensorOptions options(torch::kByte);
	torch::Tensor geomBuffer = torch::empty({0}, options.device(means3D.device()));
	torch::Tensor binningBuffer = torch::empty({0}, options.device(means3D.device()));
	torch::Tensor imgBuffer = torch::empty({0}, options.device(means3D.device()));
	int rendered = 0;
	if (P != 0) {
		int M = 0;
		if (sh.size(0) != 0) M = sh.size(1);
		const auto bg = background.contiguous(), m3 = means3D.contiguous(), shc = sh.contiguous(), col = colors.contiguous(), op = opacity.contiguous(),
		           sc = scales.contiguous(), rot = rotations.contiguous(), cov = cov3D_precomp.contiguous(), vm = viewmatrix.contiguous(),
		           pm = projmatrix.contiguous(), cp = campos.contiguous();
		psb_raster_planes planes{depth ? out_depth.data_ptr<float>() : nullptr, alpha ? out_alpha.data_ptr<float>() : nullptr,
		                         normal ? out_normal.data_ptr<float>() : nullptr, depth2 ? out_depth2.data_ptr<float>() : nullptr};
		const size_t plane_bytes = normal ? psb_rasterize_planes_bytes(P, 0) : 0;
		torch::Tensor plane_t;
		if (normal) plane_t = torch::empty({(long long)plane_bytes}, means3D.options().dtype(torch::kByte));
		rendered = psb_rasterize_forward_planes(resize_cb, &geomBuffer, resize_cb, &binningBuffer, resize_cb, &imgBuffer, P, degree, M, fptr(bg), W, H,
		                                        fptr(m3), fptr(shc), fptr(col), fptr(op), fptr(sc), scale_modifier, fptr(rot), fptr(cov), fptr(vm), fptr(pm),
		                                        fptr(cp), tan_fovx, tan_fovy, prefiltered ? 1 : 0, out_color.data_ptr<float>(), radii.data_ptr<int>(),
		                                        &planes, normal ? plane_t.data_ptr() : nullptr, plane_bytes, antialiasing ? 1 : 0, current_stream());
		if (rendered < 0) { AT_ERROR("psb_rasterize_forward_planes: ", psb_last_error()); }
	}
	return std::make_tuple(rendered, out_color, out_depth, out_alpha, out_normal, out_depth2, radii, geomBuffer, binningBuffer, imgBuffer);
}

// The backward of RasterizeGaussiansPlanesCUDA: the signature of RasterizeGaussiansBackwardAntialiasedCUDA plus the gradients of the
// opacity, normal and second-moment planes after dL_dout_depth, and `antialiasing` (the forward's flag) before `deterministic`. An
// undefined or empty gradient is none; without any it is RasterizeGaussiansBackwardAntialiasedCUDA's backward. Returns the same 8-tuple;
// dL/dz (depth and second moment) is folded into dL_dmeans3D and dL/dn into dL_drotations.
std::tuple<torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor, torch::Tensor>
RasterizeGaussiansBackwardPlanesCUDA(const torch::Tensor& background, const torch::Tensor& means3D, const torch::Tensor& radii, const torch::Tensor& colors,
                                     const torch::Tensor& scales, const torch::Tensor& rotations, const float scale_modifier,
                                     const torch::Tensor& cov3D_precomp, const torch::Tensor& viewmatrix, const torch::Tensor& projmatrix,
                                     const float tan_fovx, const float tan_fovy, const torch::Tensor& dL_dout_color, const torch::Tensor& dL_dout_depth,
                                     const torch::Tensor& dL_dout_alpha, const torch::Tensor& dL_dout_normal, const torch::Tensor& dL_dout_depth2,
                                     const torch::Tensor& sh, const int degree, const torch::Tensor& campos, const torch::Tensor& geomBuffer, const int R,
                                     const torch::Tensor& binningBuffer, const torch::Tensor& imageBuffer, const bool antialiasing,
                                     const bool deterministic)
{
	const int P = means3D.size(0);
	const int H = dL_dout_color.size(1), W = dL_dout_color.size(2);
	auto given = [&](const torch::Tensor& t, int C, const char* name) {
		if (!t.defined() || t.numel() == 0) return false;
		const bool ok = C == 1 ? (t.ndimension() == 2 && t.size(0) == H && t.size(1) == W)
		                       : (t.ndimension() == 3 && t.size(0) == C && t.size(1) == H && t.size(2) == W);
		if (!ok) { AT_ERROR(name, " must have dimensions (", C == 1 ? "" : "3, ", H, ", ", W, ")"); }
		return true;
	};
	const bool depth = given(dL_dout_depth, 1, "dL_dout_depth"), alpha = given(dL_dout_alpha, 1, "dL_dout_alpha");
	const bool normal = given(dL_dout_normal, 3, "dL_dout_normal"), depth2 = given(dL_dout_depth2, 1, "dL_dout_depth2");
	if (normal && cov3D_precomp.defined() && cov3D_precomp.numel() != 0) { AT_ERROR("dL_dout_normal needs scales and rotations, not cov3D_precomp"); }
	int M = 0;
	if (sh.size(0) != 0) M = sh.size(1);
	torch::Tensor dL_dmeans3D = torch::zeros({P, 3}, means3D.options());
	torch::Tensor dL_dmeans2D = torch::zeros({P, 3}, means3D.options());
	torch::Tensor dL_dcolors = torch::zeros({P, 3}, means3D.options());
	torch::Tensor dL_dconic = torch::zeros({P, 2, 2}, means3D.options());
	torch::Tensor dL_dopacity = torch::zeros({P, 1}, means3D.options());
	torch::Tensor dL_dcov3D = torch::zeros({P, 6}, means3D.options());
	torch::Tensor dL_dsh = torch::zeros({P, M, 3}, means3D.options());
	torch::Tensor dL_dscales = torch::zeros({P, 3}, means3D.options());
	torch::Tensor dL_drotations = torch::zeros({P, 4}, means3D.options());
	if (P != 0) {
		const auto bg = background.contiguous(), m3 = means3D.contiguous(), shc = sh.contiguous(), col = colors.contiguous(), sc = scales.contiguous(),
		           rot = rotations.contiguous(), cov = cov3D_precomp.contiguous(), vm = viewmatrix.contiguous(), pm = projmatrix.contiguous(),
		           cp = campos.contiguous(), dpix = dL_dout_color.contiguous(), rad = radii.contiguous();
		const torch::Tensor gd = depth ? dL_dout_depth.contiguous() : torch::Tensor(), ga = alpha ? dL_dout_alpha.contiguous() : torch::Tensor(),
		                    gn = normal ? dL_dout_normal.contiguous() : torch::Tensor(), gm = depth2 ? dL_dout_depth2.contiguous() : torch::Tensor();
		const psb_raster_plane_grads grads{depth ? gd.data_ptr<float>() : nullptr, alpha ? ga.data_ptr<float>() : nullptr,
		                                   normal ? gn.data_ptr<float>() : nullptr, depth2 ? gm.data_ptr<float>() : nullptr};
		torch::Tensor dL_dz, det_t, plane_t;
		if (depth || depth2) dL_dz = torch::zeros({P}, means3D.options());
		const size_t det_bytes = deterministic ? psb_rasterize_backward_det_bytes(P, R) : 0;
		if (deterministic) det_t = torch::empty({(long long)det_bytes}, means3D.options().dtype(torch::kByte));
		const size_t plane_bytes = normal ? psb_rasterize_planes_bytes(P, deterministic ? R : 0) : 0;
		if (normal) plane_t = torch::empty({(long long)plane_bytes}, means3D.options().dtype(torch::kByte));
		const int rc = psb_rasterize_backward_planes(
			P, degree, M, R, fptr(bg), W, H, fptr(m3), fptr(shc), fptr(col), fptr(sc), scale_modifier, fptr(rot), fptr(cov), fptr(vm), fptr(pm), fptr(cp),
			tan_fovx, tan_fovy, rad.data_ptr<int>(), reinterpret_cast<char*>(geomBuffer.contiguous().data_ptr()),
			reinterpret_cast<char*>(binningBuffer.contiguous().data_ptr()), reinterpret_cast<char*>(imageBuffer.contiguous().data_ptr()), fptr(dpix),
			dL_dmeans2D.data_ptr<float>(), dL_dconic.data_ptr<float>(), dL_dopacity.data_ptr<float>(), dL_dcolors.data_ptr<float>(),
			dL_dmeans3D.data_ptr<float>(), dL_dcov3D.data_ptr<float>(), M ? dL_dsh.data_ptr<float>() : nullptr, dL_dscales.data_ptr<float>(),
			dL_drotations.data_ptr<float>(), &grads, (depth || depth2) ? dL_dz.data_ptr<float>() : nullptr, deterministic ? det_t.data_ptr() : nullptr,
			det_bytes, normal ? plane_t.data_ptr() : nullptr, plane_bytes, antialiasing ? 1 : 0, deterministic ? 1 : 0, current_stream());
		if (rc < 0) { AT_ERROR("psb_rasterize_backward_planes: ", psb_last_error()); }
	}
	return std::make_tuple(dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations);
}

torch::Tensor markVisible(torch::Tensor& means3D, torch::Tensor& viewmatrix, torch::Tensor& projmatrix)
{
	const int P = means3D.size(0);
	torch::Tensor present = torch::full({P}, false, means3D.options().dtype(at::kBool));
	if (P != 0) {
		const int rc = psb_mark_visible(P, means3D.contiguous().data_ptr<float>(), viewmatrix.contiguous().data_ptr<float>(),
		                                projmatrix.contiguous().data_ptr<float>(), reinterpret_cast<unsigned char*>(present.data_ptr<bool>()),
		                                current_stream());
		if (rc < 0) { AT_ERROR("psb_mark_visible: ", psb_last_error()); }
	}
	return present;
}

// ---- the other torch-typed exports of the reference's libcuda_rasterizer.so / libsimple_knn.so ----
//   transformPoints, scaleAndTransformThenMarkVisiblePoints   include/operate_points.h:27-40, src/operate_points.cu:73-143
//   reprojectDepthPinhole, monocularPinholeInactiveGeoDensifyBySearchingNeighborhoodKeypoints
//                                                              include/stereo_vision.h:26-40, src/stereo_vision.cu:138-215
//   distCUDA2                                                  third_party/simple-knn/spatial.h:14, spatial.cu:15-26
void transformPoints(torch::Tensor& points, torch::Tensor& transformmatrix)
{
	if (points.ndimension() != 2 || points.size(1) != 3) { AT_ERROR("points must have dimensions (num_points, 3)"); }
	const int P = points.size(0);
	torch::Tensor transformed_points = torch::zeros_like(points);
	if (P != 0) {
		if (psb_transform_points(P, points.contiguous().data_ptr<float>(), transformmatrix.contiguous().data_ptr<float>(),
		                         transformed_points.data_ptr<float>(), current_stream()) < 0) { AT_ERROR(psb_last_error()); }
		points = transformed_points;
	}
}

void scaleAndTransformThenMarkVisiblePoints(torch::Tensor& points, torch::Tensor& rots, torch::Tensor& point_not_transformed_mask,
                                            torch::Tensor& point_unstable_mask, torch::Tensor& transformmatrix, torch::Tensor& viewmatrix,
                                            torch::Tensor& projmatrix, int& num_transformed, const float scale)
{
	if (points.ndimension() != 2 || points.size(1) != 3) { AT_ERROR("points must have dimensions (num_points, 3)"); }
	torch::Tensor present = markVisible(points, viewmatrix, projmatrix);
	auto num_points = present.size(0);
	if (point_not_transformed_mask.size(0) != num_points || point_unstable_mask.size(0) != num_points) { AT_ERROR("points_mask must have dimensions (num_points)"); }
	torch::Tensor final_mask = torch::logical_and(torch::logical_and(point_not_transformed_mask, point_unstable_mask), present);
	num_transformed += final_mask.sum().item<int>();
	const int P = points.size(0);
	if (P != 0) {
		torch::Tensor transformed_points = torch::zeros_like(points);
		torch::Tensor transformed_rots = torch::zeros_like(rots);
		const auto fm = final_mask.contiguous();
		if (psb_scale_transform_points(P, scale, points.contiguous().data_ptr<float>(), rots.contiguous().data_ptr<float>(),
		                               transformmatrix.contiguous().data_ptr<float>(), reinterpret_cast<const unsigned char*>(fm.data_ptr<bool>()),
		                               transformed_points.data_ptr<float>(), transformed_rots.data_ptr<float>(), /*fix_quaternion_write=*/0,
		                               current_stream()) < 0) { AT_ERROR(psb_last_error()); }
		points.index_put_({final_mask}, transformed_points.index({final_mask}));
		rots.index_put_({final_mask}, transformed_rots.index({final_mask}));
		point_not_transformed_mask.index_put_({final_mask}, torch::full({P}, false, point_not_transformed_mask.options()).index({final_mask}));
	}
}

torch::Tensor reprojectDepthPinhole(torch::Tensor& depth, torch::Tensor& mask, std::vector<float>& intr, int width)
{
	if (depth.ndimension() != 1) { AT_ERROR("points must have dimensions (num_points)"); }
	const int P = depth.size(0);
	torch::Tensor points;
	if (P != 0) {
		points = torch::zeros({P, 3}, depth.options());
		const auto mk = mask.contiguous();
		if (psb_reproject_depth_pinhole(P, width, intr[0], intr[1], intr[2], intr[3], depth.contiguous().data_ptr<float>(),
		                                reinterpret_cast<const unsigned char*>(mk.data_ptr<bool>()), points.data_ptr<float>(), current_stream()) < 0) { AT_ERROR(psb_last_error()); }
	}
	return points;
}

std::tuple<torch::Tensor, torch::Tensor> monocularPinholeInactiveGeoDensifyBySearchingNeighborhoodKeypoints(
	torch::Tensor& kps_pixel, torch::Tensor& kps_has3D, torch::Tensor& kps_point_local, torch::Tensor& colors, float max_pixel_dist,
	std::vector<float>& intr, int width)
{
	if (kps_pixel.ndimension() != 2 || kps_pixel.size(1) != 2) AT_ERROR("kps_pixel must have dimensions (num_points, 2)");
	if (kps_has3D.ndimension() != 1) AT_ERROR("kps_has3D must have dimensions (num_points)");
	if (kps_point_local.ndimension() != 2 || kps_point_local.size(1) != 3) AT_ERROR("kps_point_local must have dimensions (num_points, 3)");
	const int N = kps_pixel.size(0);
	torch::Tensor result_pt, result_color;
	if (N != 0) {
		result_pt = torch::zeros_like(kps_point_local);
		result_color = torch::zeros_like(kps_point_local);
		const auto h3 = kps_has3D.contiguous();
		if (psb_neighbour_depth_pinhole(N, width, intr[0], intr[1], intr[2], intr[3], max_pixel_dist, kps_pixel.contiguous().data_ptr<float>(),
		                                reinterpret_cast<const unsigned char*>(h3.data_ptr<bool>()), kps_point_local.contiguous().data_ptr<float>(),
		                                colors.contiguous().data_ptr<float>(), result_pt.data_ptr<float>(), result_color.data_ptr<float>(),
		                                current_stream()) < 0) { AT_ERROR(psb_last_error()); }
		torch::Tensor depth_valid_flags = torch::where(result_pt.index({torch::indexing::Slice(), 2}) > 0.0f, true, false);
		result_pt = result_pt.index({depth_valid_flags});
		result_color = result_color.index({depth_valid_flags});
	}
	return std::make_tuple(result_pt, result_color);
}

torch::Tensor distCUDA2(const torch::Tensor& points)
{
	const int P = points.size(0);
	auto float_opts = points.options().dtype(torch::kFloat32);
	torch::Tensor means = torch::full({P}, 0.0, float_opts);
	if (P != 0) {
		const auto pts = points.contiguous();
		if (psb_dist_cuda2(P, pts.data_ptr<float>(), means.data_ptr<float>(), current_stream()) < 0) { AT_ERROR(psb_last_error()); }
	}
	return means;
}

// ---- B2: the raw-pointer class of cuda_rasterizer/rasterizer.h, same static members, same argument lists ----
namespace CudaRasterizer {
class Rasterizer {
public:
	static void markVisible(int P, float* means3D, float* viewmatrix, float* projmatrix, bool* present);
	static int forward(std::function<char*(size_t)> geometryBuffer, std::function<char*(size_t)> binningBuffer, std::function<char*(size_t)> imageBuffer,
	                   const int P, int D, int M, const float* background, const int width, int height, const float* means3D, const float* shs,
	                   const float* colors_precomp, const float* opacities, const float* scales, const float scale_modifier, const float* rotations,
	                   const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* cam_pos, const float tan_fovx,
	                   float tan_fovy, const bool prefiltered, float* out_color, int* radii = nullptr);
	static void backward(const int P, int D, int M, int R, const float* background, const int width, int height, const float* means3D, const float* shs,
	                     const float* colors_precomp, const float* scales, const float scale_modifier, const float* rotations,
	                     const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* campos, const float tan_fovx,
	                     float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
	                     float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
	                     float* dL_dscale, float* dL_drot);
};

void Rasterizer::markVisible(int P, float* means3D, float* viewmatrix, float* projmatrix, bool* present)
{
	if (psb_mark_visible(P, means3D, viewmatrix, projmatrix, reinterpret_cast<unsigned char*>(present), nullptr) < 0) throw std::runtime_error(psb_last_error());
}

int Rasterizer::forward(std::function<char*(size_t)> geometryBuffer, std::function<char*(size_t)> binningBuffer, std::function<char*(size_t)> imageBuffer,
                        const int P, int D, int M, const float* background, const int width, int height, const float* means3D, const float* shs,
                        const float* colors_precomp, const float* opacities, const float* scales, const float scale_modifier, const float* rotations,
                        const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* cam_pos, const float tan_fovx,
                        float tan_fovy, const bool prefiltered, float* out_color, int* radii)
{
	// the reference launches on the legacy default stream (no stream argument anywhere): keep that here
	const int r = psb_rasterize_forward(fn_cb, &geometryBuffer, fn_cb, &binningBuffer, fn_cb, &imageBuffer, P, D, M, background, width, height, means3D,
	                                    shs, colors_precomp, opacities, scales, scale_modifier, rotations, cov3D_precomp, viewmatrix, projmatrix, cam_pos,
	                                    tan_fovx, tan_fovy, prefiltered ? 1 : 0, out_color, radii, nullptr);
	if (r < 0) throw std::runtime_error(psb_last_error());  // reference throws std::runtime_error too (rasterizer_impl.cu:241-244)
	return r;
}

void Rasterizer::backward(const int P, int D, int M, int R, const float* background, const int width, int height, const float* means3D, const float* shs,
                          const float* colors_precomp, const float* scales, const float scale_modifier, const float* rotations,
                          const float* cov3D_precomp, const float* viewmatrix, const float* projmatrix, const float* campos, const float tan_fovx,
                          float tan_fovy, const int* radii, char* geom_buffer, char* binning_buffer, char* image_buffer, const float* dL_dpix,
                          float* dL_dmean2D, float* dL_dconic, float* dL_dopacity, float* dL_dcolor, float* dL_dmean3D, float* dL_dcov3D, float* dL_dsh,
                          float* dL_dscale, float* dL_drot)
{
	if (psb_rasterize_backward(P, D, M, R, background, width, height, means3D, shs, colors_precomp, scales, scale_modifier, rotations, cov3D_precomp,
	                           viewmatrix, projmatrix, campos, tan_fovx, tan_fovy, radii, geom_buffer, binning_buffer, image_buffer, dL_dpix, dL_dmean2D,
	                           dL_dconic, dL_dopacity, dL_dcolor, dL_dmean3D, dL_dcov3D, dL_dsh, dL_dscale, dL_drot, nullptr) < 0)
		throw std::runtime_error(psb_last_error());
}
}  // namespace CudaRasterizer

// ---- test hook: expose the C++ entry points to Python without pybind ----
namespace {
using T = torch::Tensor;
std::tuple<int64_t, T, T, T, T, T> op_fwd(const T& bg, const T& m3, const T& col, const T& op, const T& sc, const T& rot, double smod, const T& cov,
                                          const T& vm, const T& pm, double tfx, double tfy, int64_t H, int64_t W, const T& sh, int64_t deg, const T& cp,
                                          bool pre)
{
	auto r = RasterizeGaussiansCUDA(bg, m3, col, op, sc, rot, (float)smod, cov, vm, pm, (float)tfx, (float)tfy, (int)H, (int)W, sh, (int)deg, cp, pre);
	return std::make_tuple((int64_t)std::get<0>(r), std::get<1>(r), std::get<2>(r), std::get<3>(r), std::get<4>(r), std::get<5>(r));
}
std::tuple<T, T, T, T, T, T, T, T> op_bwd(const T& bg, const T& m3, const T& radii, const T& col, const T& sc, const T& rot, double smod, const T& cov,
                                          const T& vm, const T& pm, double tfx, double tfy, const T& dpix, const T& sh, int64_t deg, const T& cp,
                                          const T& gb, int64_t R, const T& bb, const T& ib)
{
	return RasterizeGaussiansBackwardCUDA(bg, m3, radii, col, sc, rot, (float)smod, cov, vm, pm, (float)tfx, (float)tfy, dpix, sh, (int)deg, cp, gb, (int)R, bb, ib);
}
std::tuple<int64_t, T, T, T, T, T, T> op_fwd_depth(const T& bg, const T& m3, const T& col, const T& op, const T& sc, const T& rot, double smod,
                                                   const T& cov, const T& vm, const T& pm, double tfx, double tfy, int64_t H, int64_t W, const T& sh,
                                                   int64_t deg, const T& cp, bool pre)
{
	auto r = RasterizeGaussiansDepthCUDA(bg, m3, col, op, sc, rot, (float)smod, cov, vm, pm, (float)tfx, (float)tfy, (int)H, (int)W, sh, (int)deg, cp, pre);
	return std::make_tuple((int64_t)std::get<0>(r), std::get<1>(r), std::get<2>(r), std::get<3>(r), std::get<4>(r), std::get<5>(r), std::get<6>(r));
}
std::tuple<T, T, T, T, T, T, T, T> op_bwd_depth(const T& bg, const T& m3, const T& radii, const T& col, const T& sc, const T& rot, double smod,
                                                const T& cov, const T& vm, const T& pm, double tfx, double tfy, const T& dpix,
                                                const std::optional<T>& ddep, const T& sh, int64_t deg, const T& cp, const T& gb, int64_t R, const T& bb,
                                                const T& ib)
{
	return RasterizeGaussiansBackwardDepthCUDA(bg, m3, radii, col, sc, rot, (float)smod, cov, vm, pm, (float)tfx, (float)tfy, dpix, ddep.value_or(T()), sh,
	                                           (int)deg, cp, gb, (int)R, bb, ib);
}
std::tuple<T, T, T, T, T, T, T, T> op_bwd_det(const T& bg, const T& m3, const T& radii, const T& col, const T& sc, const T& rot, double smod,
                                              const T& cov, const T& vm, const T& pm, double tfx, double tfy, const T& dpix,
                                              const std::optional<T>& ddep, const T& sh, int64_t deg, const T& cp, const T& gb, int64_t R, const T& bb,
                                              const T& ib)
{
	return RasterizeGaussiansBackwardDeterministicCUDA(bg, m3, radii, col, sc, rot, (float)smod, cov, vm, pm, (float)tfx, (float)tfy, dpix, ddep.value_or(T()),
	                                                   sh, (int)deg, cp, gb, (int)R, bb, ib);
}
std::tuple<int64_t, T, T, T, T, T, T> op_fwd_aa(const T& bg, const T& m3, const T& col, const T& op, const T& sc, const T& rot, double smod,
                                                const T& cov, const T& vm, const T& pm, double tfx, double tfy, int64_t H, int64_t W, const T& sh,
                                                int64_t deg, const T& cp, bool pre)
{
	auto r = RasterizeGaussiansAntialiasedCUDA(bg, m3, col, op, sc, rot, (float)smod, cov, vm, pm, (float)tfx, (float)tfy, (int)H, (int)W, sh, (int)deg, cp,
	                                           pre);
	return std::make_tuple((int64_t)std::get<0>(r), std::get<1>(r), std::get<2>(r), std::get<3>(r), std::get<4>(r), std::get<5>(r), std::get<6>(r));
}
std::tuple<T, T, T, T, T, T, T, T> op_bwd_aa(const T& bg, const T& m3, const T& radii, const T& col, const T& sc, const T& rot, double smod,
                                             const T& cov, const T& vm, const T& pm, double tfx, double tfy, const T& dpix,
                                             const std::optional<T>& ddep, const T& sh, int64_t deg, const T& cp, const T& gb, int64_t R, const T& bb,
                                             const T& ib, bool deterministic)
{
	return RasterizeGaussiansBackwardAntialiasedCUDA(bg, m3, radii, col, sc, rot, (float)smod, cov, vm, pm, (float)tfx, (float)tfy, dpix, ddep.value_or(T()),
	                                                 sh, (int)deg, cp, gb, (int)R, bb, ib, deterministic);
}
std::tuple<int64_t, T, T, T, T, T, T, T, T, T> op_fwd_planes(const T& bg, const T& m3, const T& col, const T& op, const T& sc, const T& rot, double smod,
                                                            const T& cov, const T& vm, const T& pm, double tfx, double tfy, int64_t H, int64_t W,
                                                            const T& sh, int64_t deg, const T& cp, bool pre, bool depth, bool alpha, bool normal,
                                                            bool depth2, bool aa)
{
	auto r = RasterizeGaussiansPlanesCUDA(bg, m3, col, op, sc, rot, (float)smod, cov, vm, pm, (float)tfx, (float)tfy, (int)H, (int)W, sh, (int)deg, cp, pre,
	                                      depth, alpha, normal, depth2, aa);
	return std::make_tuple((int64_t)std::get<0>(r), std::get<1>(r), std::get<2>(r), std::get<3>(r), std::get<4>(r), std::get<5>(r), std::get<6>(r),
	                       std::get<7>(r), std::get<8>(r), std::get<9>(r));
}
std::tuple<T, T, T, T, T, T, T, T> op_bwd_planes(const T& bg, const T& m3, const T& radii, const T& col, const T& sc, const T& rot, double smod,
                                                 const T& cov, const T& vm, const T& pm, double tfx, double tfy, const T& dpix,
                                                 const std::optional<T>& ddep, const std::optional<T>& dalpha, const std::optional<T>& dnormal,
                                                 const std::optional<T>& ddep2, const T& sh, int64_t deg, const T& cp, const T& gb, int64_t R,
                                                 const T& bb, const T& ib, bool aa, bool deterministic)
{
	return RasterizeGaussiansBackwardPlanesCUDA(bg, m3, radii, col, sc, rot, (float)smod, cov, vm, pm, (float)tfx, (float)tfy, dpix, ddep.value_or(T()),
	                                            dalpha.value_or(T()), dnormal.value_or(T()), ddep2.value_or(T()), sh, (int)deg, cp, gb, (int)R, bb, ib, aa,
	                                            deterministic);
}
T op_vis(T m3, T vm, T pm) { return markVisible(m3, vm, pm); }
T op_dist(const T& p) { return distCUDA2(p); }
T op_xform(T p, T m) { transformPoints(p, m); return p; }
T op_reproject(T d, T mk, double fx, double fy, double cx, double cy, int64_t w)
{
	std::vector<float> intr{(float)fx, (float)fy, (float)cx, (float)cy};
	return reprojectDepthPinhole(d, mk, intr, (int)w);
}
std::tuple<T, T> op_neigh(T px, T h3, T pl, T col, double maxd, double fx, double fy, double cx, double cy, int64_t w)
{
	std::vector<float> intr{(float)fx, (float)fy, (float)cx, (float)cy};
	return monocularPinholeInactiveGeoDensifyBySearchingNeighborhoodKeypoints(px, h3, pl, col, (float)maxd, intr, (int)w);
}
// B2 through std::function allocators, for the test of the raw-pointer class
std::tuple<int64_t, T, T> op_b2_fwd(const T& bg, const T& m3, const T& op, const T& sc, const T& rot, const T& vm, const T& pm, double tfx, double tfy,
                                    int64_t H, int64_t W, const T& sh, int64_t deg, const T& cp)
{
	const int P = m3.size(0);
	T out = torch::zeros({3, H, W}, m3.options()), radii = torch::zeros({P}, m3.options().dtype(torch::kInt32));
	T g = torch::empty({0}, m3.options().dtype(torch::kByte)), b = g.clone(), i = g.clone();
	auto mk = [](T& t) { return std::function<char*(size_t)>([&t](size_t n) { t.resize_({(long long)n}); return reinterpret_cast<char*>(t.data_ptr()); }); };
	const int R = CudaRasterizer::Rasterizer::forward(mk(g), mk(b), mk(i), P, (int)deg, (int)sh.size(1), bg.data_ptr<float>(), (int)W, (int)H,
	                                                  m3.data_ptr<float>(), sh.data_ptr<float>(), nullptr, op.data_ptr<float>(), sc.data_ptr<float>(), 1.0f,
	                                                  rot.data_ptr<float>(), nullptr, vm.data_ptr<float>(), pm.data_ptr<float>(), cp.data_ptr<float>(),
	                                                  (float)tfx, (float)tfy, false, out.data_ptr<float>(), radii.data_ptr<int>());
	return std::make_tuple((int64_t)R, out, radii);
}
}  // namespace

TORCH_LIBRARY(psb200, m)
{
	m.def("rasterize_gaussians", &op_fwd);
	m.def("rasterize_gaussians_backward", &op_bwd);
	m.def("rasterize_gaussians_depth", &op_fwd_depth);
	m.def("rasterize_gaussians_backward_depth", &op_bwd_depth);
	m.def("rasterize_gaussians_backward_deterministic", &op_bwd_det);
	m.def("rasterize_gaussians_antialiased", &op_fwd_aa);
	m.def("rasterize_gaussians_backward_antialiased", &op_bwd_aa);
	m.def("rasterize_gaussians_planes", &op_fwd_planes);
	m.def("rasterize_gaussians_backward_planes", &op_bwd_planes);
	m.def("mark_visible", &op_vis);
	m.def("b2_forward", &op_b2_fwd);
	m.def("dist_cuda2", &op_dist);
	m.def("transform_points", &op_xform);
	m.def("reproject_depth_pinhole", &op_reproject);
	m.def("neighbour_depth_pinhole", &op_neigh);
}
