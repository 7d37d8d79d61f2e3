"""Host-side mirror of the reference's rasterizer operator interface, calling the psb200 C-ABI.

Mirrors, name for name and argument for argument:
  RasterizeGaussiansCUDA / RasterizeGaussiansBackwardCUDA / markVisible
      reference include/rasterize_points.h:18-65, src/rasterize_points.cu:36-214
  GaussianRasterizationSettings, GaussianRasterizerFunction (here _RasterizeGaussians),
  rasterizeGaussians, GaussianRasterizer
      reference include/gaussian_rasterizer.h:25-127, src/gaussian_rasterizer.cpp:28-234

Rendered depth D(p) = sum_i z_i alpha_i T_i (include/psb200.h), which the reference does not have:
  RasterizeGaussiansDepthCUDA / RasterizeGaussiansBackwardDepthCUDA   the two functions above plus the depth image and its gradient
  _RasterizeGaussians(..., depth=True), GaussianRasterizer.forward(..., return_depth=True)   autograd through colour and depth

Opacity A = 1 - T_final, normals N = sum n alpha T and the second depth moment M = sum z^2 alpha T (include/psb200.h), the planes the
fused training step renders:
  RasterizeGaussiansPlanesCUDA / RasterizeGaussiansBackwardPlanesCUDA   colour plus any of D, A, N, M and their gradients
  GaussianRasterizer.forward(..., return_alpha=True, return_normal=True, return_depth2=True)   autograd through every requested plane
N needs scales and rotations (not cov3D_precomp).

deterministic=True (keyword) on the backward functions, rasterize_gaussians and GaussianRasterizer.forward selects
psb_rasterize_backward_deterministic: the same gradients, bit-identical from run to run. The default keeps the float-atomic backward.

GaussianRasterizationSettings.antialiasing=True (upstream diff-gaussian-rasterization's field) selects the 2D Mip filter: every splat blends
with opacity o' = o * sqrt(max(det0 / det1, 2.5e-5)), det0 / det1 the determinants of its 2D covariance before / after the 0.3 px^2
dilation (psb_rasterize_forward_aa / psb_rasterize_backward_aa). The B1 functions take it as the keyword antialiasing=False, the
autograd functions read it from the settings.

PyTorch is used only for device memory, streams and autograd bookkeeping.
"""
import ctypes as C
from dataclasses import dataclass

import torch

from . import _lib


def _ptr(t):
    """None / empty tensor -> NULL (the reference's "None" convention, gaussian_rasterizer.cpp:209-219)."""
    if t is None or t.numel() == 0:
        return None
    return t.data_ptr()


def _alert_not_deterministic():
    """The operator backward adds each (Gaussian, tile) sum with float atomics, so its gradients vary run to run: under
    torch.use_deterministic_algorithms(True) it raises (warns with warn_only=True), like PyTorch's own nondeterministic ops.
    The operator's deterministic=True backward and the trainer contexts (GaussianTrainer / DataParallelTrainer with
    deterministic=True) do not alert.
    (PyTorch's Python-level alert; it does nothing while the flag is off.)"""
    from torch._prims_common import alert_not_deterministic
    alert_not_deterministic("psb200 rasterize backward")


def _f32c(t):
    if t is None:
        return None
    if t.dtype != torch.float32:
        raise TypeError("psb200 rasterizer expects float32 tensors")
    return t.contiguous()


def _stream():
    return torch.cuda.current_stream().cuda_stream


class _Scratch:
    """Allocator-callback target: resizes a byte tensor on demand (reference rasterize_points.cu:28-34)."""

    def __init__(self, device):
        self.device = device
        self.tensor = torch.empty(0, dtype=torch.uint8, device=device)
        self.cb = _lib.ALLOC_FN(self._alloc)

    def _alloc(self, nbytes, _user):
        self.tensor = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
        return self.tensor.data_ptr()


def _no_normal_with_cov3d(cov3D_precomp):
    if cov3D_precomp is not None and cov3D_precomp.numel() != 0:
        raise RuntimeError("the normal plane needs scales and rotations, not cov3D_precomp")


def _forward(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix,
             tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, depth, antialiasing=False, alpha=False,
             normal=False, depth2=False):
    """RasterizeGaussiansCUDA, and with depth=True also the [H,W] depth image (psb_rasterize_forward_depth); antialiasing=True:
    psb_rasterize_forward_aa (depth or not). alpha / normal / depth2: also A [H,W], N [3,H,W], M [H,W] (psb_rasterize_forward_planes);
    they come back as the `planes` dict, the last element."""
    if means3D.dim() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")  # AT_ERROR in the reference
    if normal:
        _no_normal_with_cov3d(cov3D_precomp)
    L = _lib.lib()
    dev = means3D.device
    P, H, W = means3D.size(0), int(image_height), int(image_width)
    out_color = torch.zeros((3, H, W), dtype=torch.float32, device=dev)
    out_depth = torch.zeros((H, W), dtype=torch.float32, device=dev) if depth else None
    planes = {}
    if alpha:
        planes["alpha"] = torch.zeros((H, W), dtype=torch.float32, device=dev)
    if normal:
        planes["normal"] = torch.zeros((3, H, W), dtype=torch.float32, device=dev)
    if depth2:
        planes["depth2"] = torch.zeros((H, W), dtype=torch.float32, device=dev)
    radii = torch.zeros((P,), dtype=torch.int32, device=dev)
    geom, binning, img = _Scratch(dev), _Scratch(dev), _Scratch(dev)
    rendered = 0
    if P != 0:
        M = sh.size(1) if (sh is not None and sh.numel() != 0) else 0
        tensors = [_f32c(t) for t in (background, means3D, sh, colors, opacity, scales, rotations, cov3D_precomp,
                                      viewmatrix, projmatrix, campos)]
        bg, m3, shc, col, opa, sca, rot, cov, vm, pm, cp = tensors
        args = [geom.cb, None, binning.cb, None, img.cb, None, P, int(degree), int(M), _ptr(bg), W, H,
                _ptr(m3), _ptr(shc), _ptr(col), _ptr(opa), _ptr(sca), float(scale_modifier), _ptr(rot), _ptr(cov),
                _ptr(vm), _ptr(pm), _ptr(cp), float(tan_fovx), float(tan_fovy), int(bool(prefiltered)),
                out_color.data_ptr(), radii.data_ptr()]
        if planes:
            rec = _lib.RasterPlanes(_ptr(out_depth), _ptr(planes.get("alpha")), _ptr(planes.get("normal")), _ptr(planes.get("depth2")))
            nbytes = L.psb_rasterize_planes_bytes(P, 0) if normal else 0
            scratch = torch.empty((nbytes,), dtype=torch.uint8, device=dev) if normal else None
            rendered = _lib.check(L.psb_rasterize_forward_planes(*args, C.byref(rec), _ptr(scratch), nbytes, int(bool(antialiasing)), _stream()),
                                  "psb_rasterize_forward_planes")
        elif antialiasing:
            rendered = _lib.check(L.psb_rasterize_forward_aa(*args, out_depth.data_ptr() if depth else None, 1, _stream()),
                                  "psb_rasterize_forward_aa")
        elif depth:
            rendered = _lib.check(L.psb_rasterize_forward_depth(*args, out_depth.data_ptr(), _stream()), "psb_rasterize_forward_depth")
        else:
            rendered = _lib.check(L.psb_rasterize_forward(*args, _stream()), "psb_rasterize_forward")
    return rendered, out_color, out_depth, radii, geom.tensor, binning.tensor, img.tensor, planes


def RasterizeGaussiansCUDA(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                           viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos,
                           prefiltered, *, antialiasing=False):
    """-> (num_rendered, out_color [3,H,W], radii [P] int32, geomBuffer, binningBuffer, imgBuffer).
    antialiasing=True: the 2D Mip filter (o' = o h); back-propagate with antialiasing=True as well."""
    rendered, out_color, _, radii, geom, binning, img, _ = _forward(
        background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
        tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, depth=False, antialiasing=antialiasing)
    return rendered, out_color, radii, geom, binning, img


def RasterizeGaussiansDepthCUDA(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                                viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos,
                                prefiltered, *, antialiasing=False):
    """RasterizeGaussiansCUDA plus the depth image -> (num_rendered, out_color [3,H,W], out_depth [H,W], radii [P] int32, geomBuffer,
    binningBuffer, imgBuffer). Colour, radii and buffers are bit-identical to RasterizeGaussiansCUDA's. antialiasing: as there."""
    return _forward(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix,
                    tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, depth=True, antialiasing=antialiasing)[:-1]


def RasterizeGaussiansPlanesCUDA(background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp,
                                 viewmatrix, projmatrix, tan_fovx, tan_fovy, image_height, image_width, sh, degree, campos,
                                 prefiltered, *, depth=False, alpha=False, normal=False, depth2=False, antialiasing=False):
    """RasterizeGaussiansCUDA plus the requested planes -> (num_rendered, out_color [3,H,W], out_depth [H,W], out_alpha [H,W],
    out_normal [3,H,W], out_depth2 [H,W], radii [P] int32, geomBuffer, binningBuffer, imgBuffer); a plane not requested is None.
    Colour, depth, radii and buffers are bit-identical to RasterizeGaussiansDepthCUDA's. normal=True needs scales and rotations.
    antialiasing: as there; back-propagate with the same flag."""
    rendered, out_color, out_depth, radii, geom, binning, img, planes = _forward(
        background, means3D, colors, opacity, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix, tan_fovx,
        tan_fovy, image_height, image_width, sh, degree, campos, prefiltered, depth=depth, antialiasing=antialiasing, alpha=alpha,
        normal=normal, depth2=depth2)
    return (rendered, out_color, out_depth, planes.get("alpha"), planes.get("normal"), planes.get("depth2"), radii, geom, binning, img)


def _backward(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix,
              tan_fovx, tan_fovy, dL_dout_color, dL_dout_depth, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer,
              deterministic=False, antialiasing=False, dL_dout_alpha=None, dL_dout_normal=None, dL_dout_depth2=None):
    """RasterizeGaussiansBackwardCUDA, and with a depth gradient psb_rasterize_backward_depth; deterministic=True calls
    psb_rasterize_backward_deterministic (either gradient set) over a scratch of psb_rasterize_backward_det_bytes(P, R).
    antialiasing=True: psb_rasterize_backward_aa (atomic, or deterministic over that scratch) for an anti-aliased forward.
    dL_dout_alpha / dL_dout_normal / dL_dout_depth2: psb_rasterize_backward_planes (either mode, either flag)."""
    if dL_dout_normal is not None:
        _no_normal_with_cov3d(cov3D_precomp)
    L = _lib.lib()
    P = means3D.size(0)
    H, W = dL_dout_color.size(1), dL_dout_color.size(2)
    M = sh.size(1) if (sh is not None and sh.numel() != 0) else 0
    o = dict(dtype=torch.float32, device=means3D.device)
    dL_dmeans3D = torch.zeros((P, 3), **o)
    dL_dmeans2D = torch.zeros((P, 3), **o)
    dL_dcolors = torch.zeros((P, 3), **o)
    dL_dconic = torch.zeros((P, 2, 2), **o)
    dL_dopacity = torch.zeros((P, 1), **o)
    dL_dcov3D = torch.zeros((P, 6), **o)
    dL_dsh = torch.zeros((P, M, 3), **o)
    dL_dscales = torch.zeros((P, 3), **o)
    dL_drotations = torch.zeros((P, 4), **o)
    if P != 0:
        tensors = [_f32c(t) for t in (background, means3D, sh, colors, scales, rotations, cov3D_precomp, viewmatrix,
                                      projmatrix, campos, dL_dout_color)]
        bg, m3, shc, col, sca, rot, cov, vm, pm, cp, dpix = tensors
        args = [P, int(degree), int(M), int(R), _ptr(bg), W, H, _ptr(m3), _ptr(shc), _ptr(col), _ptr(sca),
                float(scale_modifier), _ptr(rot), _ptr(cov), _ptr(vm), _ptr(pm), _ptr(cp), float(tan_fovx), float(tan_fovy),
                _ptr(radii), _ptr(geomBuffer), _ptr(binningBuffer), _ptr(imageBuffer), _ptr(dpix),
                dL_dmeans2D.data_ptr(), dL_dconic.data_ptr(), dL_dopacity.data_ptr(), dL_dcolors.data_ptr(),
                dL_dmeans3D.data_ptr(), dL_dcov3D.data_ptr(), _ptr(dL_dsh), dL_dscales.data_ptr(), dL_drotations.data_ptr()]
        def plane(g, shape, name):
            if g is None:
                return None
            g = _f32c(g)
            if tuple(g.shape) != shape:
                raise RuntimeError(f"{name} must have dimensions {shape}")
            return g
        ddep = plane(dL_dout_depth, (H, W), "dL_dout_depth")
        dalpha = plane(dL_dout_alpha, (H, W), "dL_dout_alpha")
        dnormal = plane(dL_dout_normal, (3, H, W), "dL_dout_normal")
        ddep2 = plane(dL_dout_depth2, (H, W), "dL_dout_depth2")
        # [P], zero-initialised as the C-ABI requires; folded into dL_dmeans3D there
        dL_dz = torch.zeros((P,), **o) if (ddep is not None or ddep2 is not None) else None
        nbytes, scratch = 0, None
        if deterministic:
            nbytes = L.psb_rasterize_backward_det_bytes(P, int(R))
            scratch = torch.empty((nbytes,), dtype=torch.uint8, device=means3D.device)    # the call zeroes what it reads
        if dalpha is not None or dnormal is not None or ddep2 is not None:
            rec = _lib.RasterPlaneGrads(_ptr(ddep), _ptr(dalpha), _ptr(dnormal), _ptr(ddep2))
            pbytes = L.psb_rasterize_planes_bytes(P, int(R) if deterministic else 0) if dnormal is not None else 0
            pscratch = torch.empty((pbytes,), dtype=torch.uint8, device=means3D.device) if dnormal is not None else None
            _lib.check(L.psb_rasterize_backward_planes(*args, C.byref(rec), _ptr(dL_dz), _ptr(scratch), nbytes, _ptr(pscratch), pbytes,
                                                       int(bool(antialiasing)), int(bool(deterministic)), _stream()),
                       "psb_rasterize_backward_planes")
        elif antialiasing:
            _lib.check(L.psb_rasterize_backward_aa(*args, _ptr(ddep), _ptr(dL_dz), _ptr(scratch), nbytes, 1, _stream()),
                       "psb_rasterize_backward_aa")
        elif deterministic:
            _lib.check(L.psb_rasterize_backward_deterministic(*args, _ptr(ddep), _ptr(dL_dz), scratch.data_ptr(), nbytes, _stream()),
                       "psb_rasterize_backward_deterministic")
        elif ddep is not None:
            _lib.check(L.psb_rasterize_backward_depth(*args, ddep.data_ptr(), dL_dz.data_ptr(), _stream()), "psb_rasterize_backward_depth")
        else:
            _lib.check(L.psb_rasterize_backward(*args, _stream()), "psb_rasterize_backward")
    return dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations


def RasterizeGaussiansBackwardCUDA(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp,
                                   viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, sh, degree, campos,
                                   geomBuffer, R, binningBuffer, imageBuffer, *, deterministic=False, antialiasing=False):
    """-> (dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations).
    deterministic=True: the same gradients, bit-identical from call to call (summed in a fixed order instead of with float atomics).
    antialiasing=True: the backward of an anti-aliased forward (the same flag there); dL_dopacity is then dL/do.
    dL_dmeans2D is in NDC units: dL/dpixel times (W/2, H/2). With scale_modifier != 1, dL_dscales is the gradient with respect to the
    modified scale scale_modifier * scales, not with respect to `scales` (the reference's convention: the factor is not applied); the true
    dL/dscales is dL_dscales * scale_modifier."""
    return _backward(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix,
                     tan_fovx, tan_fovy, dL_dout_color, None, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, deterministic,
                     antialiasing)


def RasterizeGaussiansBackwardDepthCUDA(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp,
                                        viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, dL_dout_depth, sh, degree, campos,
                                        geomBuffer, R, binningBuffer, imageBuffer, *, deterministic=False, antialiasing=False):
    """RasterizeGaussiansBackwardCUDA with the gradient of the depth image as well (dL_dout_depth [H,W]; None = the plain backward).
    dL/dz is folded into dL_dmeans3D, and dL_dmeans2D includes the depth term. Returns the same 8-tuple. deterministic, antialiasing:
    as there."""
    return _backward(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix,
                     tan_fovx, tan_fovy, dL_dout_color, dL_dout_depth, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer,
                     deterministic, antialiasing)


def RasterizeGaussiansBackwardPlanesCUDA(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp,
                                         viewmatrix, projmatrix, tan_fovx, tan_fovy, dL_dout_color, dL_dout_depth, dL_dout_alpha,
                                         dL_dout_normal, dL_dout_depth2, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer, *,
                                         deterministic=False, antialiasing=False):
    """RasterizeGaussiansBackwardCUDA with the gradients of the depth, opacity, normal and second-moment planes as well (None = no
    gradient; all None = RasterizeGaussiansBackwardDepthCUDA's backward). dL/dz (depth and second moment) is folded into dL_dmeans3D,
    dL/dn into dL_drotations. Returns the same 8-tuple. deterministic, antialiasing: as there."""
    return _backward(background, means3D, radii, colors, scales, rotations, scale_modifier, cov3D_precomp, viewmatrix, projmatrix,
                     tan_fovx, tan_fovy, dL_dout_color, dL_dout_depth, sh, degree, campos, geomBuffer, R, binningBuffer, imageBuffer,
                     deterministic, antialiasing, dL_dout_alpha, dL_dout_normal, dL_dout_depth2)


def markVisible(means3D, viewmatrix, projmatrix):
    L = _lib.lib()
    P = means3D.size(0)
    present = torch.zeros((P,), dtype=torch.bool, device=means3D.device)
    if P != 0:
        _lib.check(L.psb_mark_visible(P, _f32c(means3D).data_ptr(), _f32c(viewmatrix).data_ptr(),
                                      _f32c(projmatrix).data_ptr(), present.data_ptr(), _stream()), "psb_mark_visible")
    return present


@dataclass
class GaussianRasterizationSettings:
    """Field for field the reference struct (include/gaussian_rasterizer.h:25-55), without trailing underscores, plus upstream
    diff-gaussian-rasterization's `antialiasing` (the 2D Mip filter; off by default)."""
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool = False
    antialiasing: bool = False


class _RasterizeGaussians(torch.autograd.Function):
    """reference GaussianRasterizerFunction (src/gaussian_rasterizer.cpp:28-180). depth=True: the depth image as a third,
    differentiable output; alpha / normal / depth2: A, N, M as further differentiable outputs, in that order after depth."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings, deterministic=False,
                depth=False, alpha=False, normal=False, depth2=False):
        rs = raster_settings
        num_rendered, color, out_depth, radii, geomBuffer, binningBuffer, imgBuffer, planes = _forward(
            rs.bg, means3D, colors_precomp, opacities, scales, rotations, rs.scale_modifier, cov3Ds_precomp,
            rs.viewmatrix, rs.projmatrix, rs.tanfovx, rs.tanfovy, rs.image_height, rs.image_width, sh, rs.sh_degree,
            rs.campos, rs.prefiltered, depth=bool(depth), antialiasing=bool(rs.antialiasing), alpha=bool(alpha), normal=bool(normal),
            depth2=bool(depth2))
        ctx.raster_settings = rs
        ctx.num_rendered = num_rendered
        ctx.deterministic = bool(deterministic)
        ctx.antialiasing = bool(rs.antialiasing)     # the backward differentiates the forward that ran
        ctx.save_for_backward(colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer,
                              binningBuffer, imgBuffer)
        ctx.mark_non_differentiable(radii)
        ctx.depth = bool(depth)
        ctx.planes = tuple(planes)          # the requested planes of (alpha, normal, depth2), in output order
        if not depth and not planes:
            return color, radii
        ctx.set_materialize_grads(False)    # an output the loss does not use arrives as None, not as a zero image
        return (color, radii) + ((out_depth,) if depth else ()) + tuple(planes.values())

    @staticmethod
    def backward(ctx, grad_out_color, _grad_radii, *grad_planes):
        grad_planes = list(grad_planes)
        grad_out_depth = grad_planes.pop(0) if ctx.depth else None
        g_planes = dict(zip(ctx.planes, grad_planes))
        if not ctx.deterministic:
            _alert_not_deterministic()
        rs = ctx.raster_settings
        colors_precomp, means3D, scales, rotations, cov3Ds_precomp, radii, sh, geomBuffer, binningBuffer, imgBuffer = ctx.saved_tensors
        if grad_out_color is None:      # only with extra planes, which do not materialise the gradients
            grad_out_color = torch.zeros((3, rs.image_height, rs.image_width), dtype=torch.float32, device=means3D.device)
        (grad_means2D, grad_colors_precomp, grad_opacities, grad_means3D, grad_cov3Ds_precomp, grad_sh, grad_scales,
         grad_rotations) = _backward(
            rs.bg, means3D, radii, colors_precomp, scales, rotations, rs.scale_modifier, cov3Ds_precomp, rs.viewmatrix,
            rs.projmatrix, rs.tanfovx, rs.tanfovy, grad_out_color, grad_out_depth, sh, rs.sh_degree, rs.campos, geomBuffer,
            ctx.num_rendered, binningBuffer, imgBuffer, deterministic=ctx.deterministic, antialiasing=ctx.antialiasing,
            dL_dout_alpha=g_planes.get("alpha"), dL_dout_normal=g_planes.get("normal"), dL_dout_depth2=g_planes.get("depth2"))
        # order of reference gaussian_rasterizer.cpp:159-179
        def g(t, ref):
            return t if (ref is not None and ref.numel() != 0) else None
        return (grad_means3D, grad_means2D, g(grad_sh, sh), g(grad_colors_precomp, colors_precomp), grad_opacities,
                g(grad_scales, scales), g(grad_rotations, rotations), g(grad_cov3Ds_precomp, cov3Ds_precomp), None, None, None, None, None, None)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings, *,
                        deterministic=False):
    """reference rasterizeGaussians (include/gaussian_rasterizer.h:77-99). deterministic=True: the backward's gradients are
    bit-identical from run to run (psb_rasterize_backward_deterministic), and it does not alert under
    torch.use_deterministic_algorithms(True)."""
    return _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                                     raster_settings, deterministic)


class GaussianRasterizer:
    """reference GaussianRasterizer (include/gaussian_rasterizer.h:101-127, src/gaussian_rasterizer.cpp:182-234)."""

    def __init__(self, raster_settings: GaussianRasterizationSettings):
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        with torch.no_grad():
            return markVisible(positions, self.raster_settings.viewmatrix, self.raster_settings.projmatrix)

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None, return_depth=False, deterministic=False, return_alpha=False, return_normal=False, return_depth2=False):
        """-> (color, radii), followed by the requested planes in this order: depth [H,W] (return_depth), the accumulated opacity
        A = 1 - T_final [H,W] (return_alpha), the normal plane N [3,H,W] (return_normal; needs scales and rotations) and the second
        depth moment M [H,W] (return_depth2). Every plane is differentiable, as the colour; none has a background term.
        deterministic=True: bit-identical gradients from run to run (see rasterize_gaussians)."""
        has = lambda t: t is not None and t.numel() != 0
        if has(shs) == has(colors_precomp):
            raise RuntimeError("Please provide excatly one of either SHs or precomputed colors!")
        if (has(scales) or has(rotations)) == has(cov3D_precomp) or (has(scales) != has(rotations)):
            raise RuntimeError("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
        if return_normal and not has(scales):
            raise RuntimeError("the normal plane needs scales and rotations, not cov3D_precomp")
        empty = torch.empty(0, dtype=torch.float32, device=means3D.device)
        e = lambda t: t if has(t) else empty
        if return_alpha or return_normal or return_depth2:
            return _RasterizeGaussians.apply(means3D, means2D, e(shs), e(colors_precomp), opacities, e(scales), e(rotations),
                                             e(cov3D_precomp), self.raster_settings, deterministic, bool(return_depth), bool(return_alpha),
                                             bool(return_normal), bool(return_depth2))
        if return_depth:
            return _RasterizeGaussians.apply(means3D, means2D, e(shs), e(colors_precomp), opacities, e(scales), e(rotations),
                                             e(cov3D_precomp), self.raster_settings, deterministic, True)
        return rasterize_gaussians(means3D, means2D, e(shs), e(colors_precomp), opacities, e(scales), e(rotations),
                                   e(cov3D_precomp), self.raster_settings, deterministic=deterministic)

    __call__ = forward
