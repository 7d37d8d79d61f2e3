"""Host-side mirror of the reference's GaussianRenderer::render (include/gaussian_renderer.h, src/gaussian_renderer.cpp:23-149) with
EVERY pipeline branch, on top of the psb200 rasterizer operator (rasterizer.GaussianRasterizer -> C-ABI):

  pipe.compute_cov3D   cov3D_precomp = GaussianModel::getCovarianceActivation(scaling_modifier)   (gaussian_renderer.cpp:83-92, gaussian_model.cpp:73-101)
  use_override_color   colors_precomp = override_color                                           (:103-105)
  pipe.convert_SHs     colors_precomp = clamp_min(eval_sh(active degree, features, dir) + 0.5, 0)  (:106-113, include/sh_utils.h:64-136)
  default              raw SH rows to the rasterizer                                               (:114-117)

and any SH storage size M = (max_sh_degree + 1)^2 (the operator-level path takes M from the tensor). The result tuple is the
reference's: (rendered_image, viewspace_points, visibility_filter, radii), plus the depth image with return_depth=True and the opacity,
normal and second-moment planes with return_alpha / return_normal / return_depth2; gradients
flow through torch autograd into the model tensors, and viewspace_points.grad[:, :2] feeds addDensificationStats like in the reference.

This is the general, differentiable path. The trainer's hot loop does not come through here: psb_trainer_step / psb_trainer_render fuse
the default branch (activations, SH gather, loss, backward, Adam) into the kernels; tests/test_renderer_gpu.py checks that both paths draw
the same picture."""
from dataclasses import dataclass

import torch

from . import sh_utils
from .rasterizer import GaussianRasterizationSettings, GaussianRasterizer


@dataclass
class GaussianPipelineParams:
    """reference include/gaussian_parameters.h:38-47 (all shipped configs: both False), plus `antialiasing`: the rasterizer's 2D Mip
    filter (GaussianRasterizationSettings.antialiasing) in every branch below, and `filter_3d`: the model's 3D smoothing filter
    (GaussianModel.computeFilter3D; scale s' and opacity o' of getScalingWithFilter3D / getOpacityWithFilter3D) in every branch below;
    both off by default"""
    convert_SHs: bool = False
    compute_cov3D: bool = False
    antialiasing: bool = False
    filter_3d: bool = False


def build_rotation(r):
    """include/general_utils.h:31-56 (normalises the quaternion itself)"""
    q = r / torch.sqrt((r * r).sum(dim=1, keepdim=True))
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.zeros((q.size(0), 3, 3), device=r.device, dtype=r.dtype)
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - w * z); R[:, 0, 2] = 2 * (x * z + w * y)
    R[:, 1, 0] = 2 * (x * y + w * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - w * x)
    R[:, 2, 0] = 2 * (x * z - w * y); R[:, 2, 1] = 2 * (y * z + w * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def get_features(model):
    """GaussianModel::getFeatures (gaussian_model.cpp:63-66): [P, M, 3]"""
    return torch.cat((model.features_dc_, model.features_rest_), dim=1)


def get_covariance_activation(model, scaling_modifier=1.0, scales=None):
    """GaussianModel::getCovarianceActivation (gaussian_model.cpp:73-101): L = R diag(s), Sigma = L L^T, upper triangle [P, 6];
    scales: the activated scales to use instead of exp(scaling_) (the 3D filter's s')"""
    R = build_rotation(model.rotation_)
    s = scaling_modifier * (torch.exp(model.scaling_) if scales is None else scales)
    Lm = R * s.unsqueeze(1)                    # R @ diag(s)
    cov = Lm @ Lm.transpose(1, 2)
    return torch.stack((cov[:, 0, 0], cov[:, 0, 1], cov[:, 0, 2], cov[:, 1, 1], cov[:, 1, 2], cov[:, 2, 2]), dim=1)


def render(viewpoint_camera, image_height, image_width, pc, pipe=None, bg_color=None, override_color=None, scaling_modifier=1.0,
           use_override_color=False, return_depth=False, deterministic=False, return_alpha=False, return_normal=False, return_depth2=False):
    """viewpoint_camera: dict(viewmatrix, projmatrix, campos: device tensors; tanfovx, tanfovy) — the fields of GaussianKeyframe the
    reference reads (world_view_transform_, full_proj_transform_, camera_center_, FoVx_/FoVy_ as tangents). pc: trainer.GaussianModel.
    return_depth=True appends the rendered depth [H,W] (include/psb200.h: sum z alpha T, no background term) to the tuple, in every
    branch; gradients flow through it like through the image. return_alpha / return_normal / return_depth2 append, in that order after
    depth, the accumulated opacity A [H,W], the normal plane N [3,H,W] and the second depth moment M [H,W] (include/psb200.h), in every
    branch except N with pipe.compute_cov3D, which is refused (N needs the scales and rotations). deterministic=True: the rasterizer's backward is bit-identical from run to
    run (GaussianRasterizer.forward), so are the gradients it sends into the model tensors and viewspace_points."""
    pipe = pipe or GaussianPipelineParams()
    if return_normal and pipe.compute_cov3D:
        raise RuntimeError("render: return_normal needs scales and rotations; pipe.compute_cov3D passes a covariance instead")
    dev = pc.xyz_.device
    bg_color = bg_color if bg_color is not None else torch.zeros(3, device=dev)
    screenspace_points = torch.zeros_like(pc.xyz_, requires_grad=True)
    settings = GaussianRasterizationSettings(int(image_height), int(image_width), float(viewpoint_camera["tanfovx"]), float(viewpoint_camera["tanfovy"]),
                                             bg_color, float(scaling_modifier), viewpoint_camera["viewmatrix"], viewpoint_camera["projmatrix"],
                                             int(pc.active_sh_degree_), viewpoint_camera["campos"], False, bool(pipe.antialiasing))
    rasterizer = GaussianRasterizer(settings)
    means3D, means2D = pc.xyz_, screenspace_points
    opacity = pc.getOpacityWithFilter3D() if pipe.filter_3d else torch.sigmoid(pc.opacity_)
    activated_scales = pc.getScalingWithFilter3D() if pipe.filter_3d else torch.exp(pc.scaling_)
    scales = rotations = cov3D_precomp = None
    if pipe.compute_cov3D:
        cov3D_precomp = get_covariance_activation(pc, scaling_modifier, activated_scales)
    else:
        scales = activated_scales
        rotations = torch.nn.functional.normalize(pc.rotation_)
    shs = colors_precomp = None
    if use_override_color:
        colors_precomp = override_color
    elif pipe.convert_SHs:
        feats = get_features(pc)
        shs_view = feats.transpose(1, 2).reshape(-1, 3, feats.size(1))
        dir_pp = pc.xyz_ - viewpoint_camera["campos"].reshape(1, 3)
        dir_pp = dir_pp / torch.linalg.vector_norm(dir_pp, dim=1, keepdim=True)
        colors_precomp = torch.clamp_min(sh_utils.eval_sh(pc.active_sh_degree_, shs_view, dir_pp) + 0.5, 0.0)
    else:
        shs = get_features(pc)
    if return_alpha or return_normal or return_depth2:
        rendered_image, radii, *planes = rasterizer(means3D, means2D, opacity, shs=shs, colors_precomp=colors_precomp, scales=scales,
                                                    rotations=rotations, cov3D_precomp=cov3D_precomp, return_depth=return_depth,
                                                    deterministic=deterministic, return_alpha=return_alpha, return_normal=return_normal,
                                                    return_depth2=return_depth2)
        return (rendered_image, screenspace_points, radii > 0, radii, *planes)
    if return_depth:
        rendered_image, radii, depth = rasterizer(means3D, means2D, opacity, shs=shs, colors_precomp=colors_precomp, scales=scales,
                                                  rotations=rotations, cov3D_precomp=cov3D_precomp, return_depth=True,
                                                  deterministic=deterministic)
        return rendered_image, screenspace_points, radii > 0, radii, depth
    rendered_image, radii = rasterizer(means3D, means2D, opacity, shs=shs, colors_precomp=colors_precomp, scales=scales, rotations=rotations,
                                       cov3D_precomp=cov3D_precomp, deterministic=deterministic)
    return rendered_image, screenspace_points, radii > 0, radii
