"""Host-side mirror of the reference's trainer-level surface for the hot path, on the psb200 C-ABI.

  GaussianOptimizationParams   reference include/gaussian_parameters.h:49-96 (values: cfg/gaussian_mapper/RGB-D/Replica/replica_rgbd.yaml:53-74)
  GaussianModel                reference include/gaussian_model.h:59-193 — the tensors, Adam state, learning-rate
                               handling (trainingSetup / updateLearningRate / set*LearningRate / exponLrFunc,
                               src/gaussian_model.cpp:477-554, 1118-1131)
  GaussianTrainer              reference GaussianMapper::trainForOneIteration (src/gaussian_mapper.cpp:614-774) /
                               GaussianTrainer::trainingOnce (src/gaussian_trainer.cpp:31-135): one iteration =
                               render, L1 + DSSIM, backward, densification statistics, Adam step — here ONE call
                               into psb_trainer_step_exposure.
PyTorch provides device memory, streams and (for the data-parallel variant) torch.distributed.
"""
import ctypes as C
import math
from collections import namedtuple
from dataclasses import dataclass

import torch

from . import _lib
from .parallel import SIZES, row_shapes

GROUPS = ("xyz", "features_dc", "features_rest", "opacity", "scaling", "rotation")


class _Model(C.Structure):
    _fields_ = [("param", C.c_void_p * 6), ("exp_avg", C.c_void_p * 6), ("exp_avg_sq", C.c_void_p * 6),
                ("max_radii2D", C.c_void_p), ("xyz_gradient_accum", C.c_void_p), ("denom", C.c_void_p), ("exist_since_iter", C.c_void_p),
                ("adam_live", C.c_void_p)]


def _cmodel_of(p, m=None, v=None, accum=None, denom=None, max_radii=None, exist=None, live=None):
    """psb_model over the given tensors (p, m, v: the six parameter / moment tensors); what is None is passed as NULL."""
    c = _Model()
    ptr = lambda t: None if t is None else t.data_ptr()
    for i in range(6):
        c.param[i] = p[i].data_ptr()
        if m is not None:
            c.exp_avg[i], c.exp_avg_sq[i] = m[i].data_ptr(), v[i].data_ptr()
    c.max_radii2D, c.xyz_gradient_accum, c.denom = ptr(max_radii), ptr(accum), ptr(denom)
    c.exist_since_iter, c.adam_live = ptr(exist), ptr(live)
    return c


class _Camera(C.Structure):
    _fields_ = [("viewmatrix", C.c_void_p), ("projmatrix", C.c_void_p), ("campos", C.c_void_p), ("tan_fovx", C.c_float),
                ("tan_fovy", C.c_float), ("width", C.c_int), ("height", C.c_int)]


class _Step(C.Structure):
    _fields_ = [("lr", C.c_float * 6), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float), ("step", C.c_int),
                ("lambda_dssim", C.c_float), ("sh_degree", C.c_int), ("update_densify_stats", C.c_int)]


class _Depth(C.Structure):
    _fields_ = [("gt_depth", C.c_void_p), ("lambda_depth", C.c_float), ("out_depth", C.c_void_p)]


def _cdepth(gt_depth, lambda_depth, out_depth):
    """psb_depth for a call, or None when it has no depth argument (NULL is passed then)."""
    if gt_depth is None and out_depth is None and not lambda_depth:
        return None
    for t in (gt_depth, out_depth):
        assert t is None or (t.is_contiguous() and t.dtype == torch.float32), "depth planes: contiguous float32 [H,W]"
    return _Depth(gt_depth.data_ptr() if gt_depth is not None else None, float(lambda_depth),
                  out_depth.data_ptr() if out_depth is not None else None)


class _Normal(C.Structure):
    _fields_ = [("gt_normal", C.c_void_p), ("lambda_normal", C.c_float), ("out_normal", C.c_void_p)]


class _Dn(C.Structure):
    _fields_ = [("lambda_dn", C.c_float), ("alpha_min", C.c_float), ("max_rel_jump", C.c_float), ("out_depth_normal", C.c_void_p)]


def _cdn(lambda_dn, alpha_min, max_rel_jump, out_depth_normal, H, W):
    """psb_dn for a call, or None when lambda_dn == 0 and there is no out_depth_normal (the call is then the one without the term); the
    library refuses a lambda_dn, alpha_min or max_rel_jump out of range."""
    if lambda_dn == 0 and out_depth_normal is None:
        return None
    _plane(out_depth_normal, (3, H, W), "out_depth_normal")
    return _Dn(float(lambda_dn), float(alpha_min), float(max_rel_jump), out_depth_normal.data_ptr() if out_depth_normal is not None else None)


class _Dist(C.Structure):
    _fields_ = [("lambda_dist", C.c_float), ("out_depth2", C.c_void_p)]


def _cdist(lambda_dist, out_depth2, H, W):
    """psb_dist for a call, or None when lambda_dist == 0 and there is no out_depth2 (the call is then the one without the term); the
    library refuses a lambda_dist out of range."""
    if lambda_dist == 0 and out_depth2 is None:
        return None
    _plane(out_depth2, (H, W), "out_depth2")
    return _Dist(float(lambda_dist), out_depth2.data_ptr() if out_depth2 is not None else None)


def _cnormal(gt_normal, lambda_normal, out_normal, H, W):
    """psb_normal for a call, or None when it has no normal argument (the call is then the one without the normal term)."""
    if gt_normal is None and out_normal is None and not lambda_normal:
        return None
    _plane(gt_normal, (3, H, W), "gt_normal")
    _plane(out_normal, (3, H, W), "out_normal")
    return _Normal(gt_normal.data_ptr() if gt_normal is not None else None, float(lambda_normal),
                   out_normal.data_ptr() if out_normal is not None else None)


class _Exposure(C.Structure):
    _fields_ = [("param", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p), ("step", C.c_void_p), ("lr", C.c_float)]


class _ExposureTable(C.Structure):
    """psb_exposure_table: the replicated table of the data-parallel steps, this rank's row (-1: none) and the gradient modes' record."""
    _fields_ = [("param", C.c_void_p), ("exp_avg", C.c_void_p), ("exp_avg_sq", C.c_void_p), ("step", C.c_void_p), ("K", C.c_int),
                ("id", C.c_int), ("lr", C.c_float), ("record", C.c_void_p)]


EXPOSURE_RECORD = 16   # floats of one rank's exposure record (PSB_EXPOSURE_RECORD)


class _PixelGrads(C.Structure):
    _fields_ = [("dL_dcolor", C.c_void_p), ("dL_ddepth", C.c_void_p), ("dL_dalpha", C.c_void_p)]


def _plane(t, shape, what):
    """a gradient plane for psb_trainer_backward_pixels: None, or a contiguous float32 tensor of `shape` on the model's device type"""
    if t is None:
        return None
    if not torch.is_tensor(t) or tuple(t.shape) != tuple(shape) or t.dtype != torch.float32 or not t.is_contiguous():
        raise ValueError(f"{what}: want a contiguous float32 tensor of shape {tuple(shape)}, got "
                         f"{tuple(t.shape) if torch.is_tensor(t) else type(t).__name__}")
    return t


# What result() knows of the last enqueuing call when its pass overflowed the binning arena: whether it advanced model.step_ and
# iteration by one, how to enqueue it again (None: it cannot be repeated — backwardPixels on a render the caller computed a loss from),
# and whether its loss is the caller's (result() then reports only that loss's value).
_Call = namedtuple("_Call", "advanced repeat callers_loss")
_NO_CALL = _Call(False, None, False)


class _DensifyCfg(C.Structure):
    _fields_ = [("max_grad", C.c_float), ("min_opacity", C.c_float), ("extent", C.c_float), ("percent_dense", C.c_float), ("max_screen_size", C.c_int),
                ("seed", C.c_ulonglong), ("offset", C.c_ulonglong)]


class _RelocateCfg(C.Structure):
    _fields_ = [("min_opacity", C.c_float), ("iteration", C.c_int), ("seed", C.c_ulonglong), ("offset", C.c_ulonglong)]


class _SeedCfg(C.Structure):
    _fields_ = [("alpha_min", C.c_float), ("depth_rel", C.c_float), ("min_depth", C.c_float), ("max_depth", C.c_float), ("stride", C.c_int),
                ("max_new", C.c_int)]


_INT_MAX = 2 ** 31 - 1


# The unit of the summed contribution score (include/psb200.h, PSB_CONTRIB_SUM_FRAC_BITS = 26).
CONTRIB_SUM_UNIT = 2.0 ** -26


def _check_cams(cams, what):
    """cams: a non-empty list of camera dicts in the form GaussianTrainer takes (ValueError otherwise, before any C call)."""
    if not isinstance(cams, (list, tuple)) or not cams:
        raise ValueError(f"{what}: want a non-empty list of camera dicts")
    for k, cam in enumerate(cams):
        try:
            W, H = cam["W"], cam["H"]
            for key in ("viewmatrix", "projmatrix", "campos", "tanfovx", "tanfovy"):
                cam[key]
        except (KeyError, TypeError) as e:
            raise ValueError(f"{what}: camera {k} is not a camera dict (viewmatrix, projmatrix, campos, tanfovx, tanfovy, W, H): {e}") from None
        if isinstance(W, bool) or isinstance(H, bool) or int(W) != W or int(H) != H or W <= 0 or H <= 0:
            raise ValueError(f"{what}: camera {k}: W and H must be positive integers, got {W}, {H}")
    return list(cams)


def contribution_prune_mask(max_weight, sum_weight, min_weight, keep=None, young=None):
    """bool [P], True = remove: the rows whose max_weight < min_weight and, with keep, every row but the `keep` of highest sum_weight (ties
    go to the lower row index). Rows marked in `young` (bool [P] or None) are never removed."""
    mask = max_weight < min_weight
    if keep is not None and keep < mask.numel():
        order = torch.sort(sum_weight, descending=True, stable=True).indices
        mask[order[keep:]] = True
    if young is not None:
        mask &= ~young
    return mask


def _bind():
    """The library with every trainer, data-parallel, densification and debug entry point declared (include/psb200.h)."""
    L = _lib.lib()
    if getattr(L, "_trainer_bound", False):
        return L
    vp, i, f, u, size_t = C.c_void_p, C.c_int, C.c_float, C.c_uint, C.c_size_t
    P = C.POINTER
    Model, Cam, Step, Depth, Exp, Cfg = P(_Model), P(_Camera), P(_Step), P(_Depth), P(_Exposure), P(_DensifyCfg)
    ull = C.c_ulonglong
    # the arguments every built-in-loss training call starts with: t, P, M, model, camera, background, gt_image, mask, step, out_color, radii
    call = [vp, i, i, Model, Cam, vp, vp, vp, Step, vp, vp]
    render = [vp, i, i, Model, Cam, vp, i, vp, vp]   # t, P, M, model, camera, background, sh_degree, out_color, radii
    sigs = {
        "psb_trainer_create": [P(vp)],
        "psb_trainer_destroy": [vp],
        "psb_trainer_render": render + [vp],
        "psb_trainer_render_depth": render + [vp, vp],
        "psb_trainer_forward": render + [vp, vp, P(u), vp],
        "psb_trainer_forward_normal": render + [vp, vp, vp, P(u), vp],
        "psb_trainer_forward_moment": render + [vp, vp, vp, vp, P(u), vp],
        "psb_trainer_backward_pixels": [vp, u, i, i, Model, Cam, vp, P(_PixelGrads), Step, P(vp), vp],
        "psb_trainer_backward_pixels_normal": [vp, u, i, i, Model, Cam, vp, P(_PixelGrads), vp, Step, P(vp), vp],
        "psb_trainer_backward_pixels_moment": [vp, u, i, i, Model, Cam, vp, P(_PixelGrads), vp, vp, Step, P(vp), vp],
        "psb_trainer_step": call + [vp],
        "psb_trainer_step_depth": call + [Depth, vp],
        "psb_trainer_step_exposure": call + [Depth, Exp, vp],
        "psb_trainer_step_normal": call + [Depth, Exp, P(_Normal), vp],
        "psb_trainer_step_dn": call + [Depth, Exp, P(_Normal), P(_Dn), vp],
        "psb_trainer_step_dist": call + [Depth, Exp, P(_Normal), P(_Dn), P(_Dist), vp],
        "psb_trainer_backward": call + [P(vp), vp],
        "psb_trainer_backward_depth": call + [P(vp), Depth, vp],
        "psb_trainer_backward_exposure": call + [P(vp), Depth, Exp, vp, vp],
        "psb_trainer_backward_dist": call + [P(vp), Depth, Exp, vp, P(_Normal), P(_Dn), P(_Dist), vp],
        "psb_trainer_backward_begin": call + [vp],
        "psb_trainer_backward_begin_depth": call + [Depth, vp],
        "psb_trainer_backward_begin_dist": call + [Depth, P(_Normal), P(_Dn), P(_Dist), vp],
        "psb_trainer_backward_begin_table": call + [Depth, P(_Normal), P(_Dn), P(_Dist), P(_ExposureTable), vp],
        "psb_trainer_backward_table": call + [P(vp), Depth, P(_Normal), P(_Dn), P(_Dist), P(_ExposureTable), vp],
        "psb_exposure_apply": [i, vp, P(_ExposureTable), Step, f, vp],
        "psb_trainer_backward_slab": [vp, i, i, Model, Cam, Step, i, i, P(vp), vp],
        "psb_trainer_result": [vp, P(f), P(i), vp],
        "psb_trainer_result_depth": [vp, P(f), P(i), vp],
        "psb_trainer_result_normal": [vp, P(f), P(i), vp],
        "psb_trainer_result_dn": [vp, P(f), P(i), vp],
        "psb_trainer_result_dist": [vp, P(f), P(i), vp],
        "psb_depth_normals": [Cam, vp, f, vp, vp],
        "psb_dn_loss": [Cam, vp, vp, vp, vp, P(_Dn), vp, vp, vp, P(f), vp],
        "psb_trainer_overflow_info": [vp, P(u), P(u), P(u)],
        "psb_trainer_debug_state": [vp, i, i, vp, vp, P(i), vp],
        "psb_trainer_set_profiling": [vp, i],
        "psb_trainer_stage_times": [vp, P(f), i],
        "psb_trainer_set_deterministic": [vp, i],
        "psb_trainer_set_antialiasing": [vp, i],
        "psb_trainer_set_regularizers": [vp, f, f],
        "psb_trainer_set_filter3d": [vp, vp, i],
        "psb_filter3d": [i, vp, i, vp, vp, P(i), vp],
        "psb_trainer_contribution": [vp, i, i, Model, Cam, vp, i, vp, vp, vp, vp],
        "psb_trainer_inject_noise": [vp, i, Model, f, f, ull, ull, i, vp],
        "psb_adam_update": [i, i, Model, P(vp), Step, f, vp],
        "psb_adam_flat": [size_t, vp, vp, vp, vp, f, Step, f, vp],
        "psb_adam_live_rebuild": [i, Model, vp],
        "psb_loss": [i, i, vp, vp, vp, f, vp, P(f), vp],
        "psb_dp_create": [P(vp), i, i, i],
        "psb_dp_handle_bytes": [],
        "psb_dp_ipc_handle": [vp, vp],
        "psb_dp_connect": [vp, vp],
        "psb_dp_params": [vp, P(vp)],
        "psb_dp_step": [vp] + call + [vp],
        "psb_dp_step_depth": [vp] + call + [Depth, vp],
        "psb_dp_step_dist": [vp] + call + [Depth, P(_Normal), P(_Dn), P(_Dist), vp],
        "psb_dp_step_table": [vp] + call + [Depth, P(_Normal), P(_Dn), P(_Dist), P(_ExposureTable), vp],
        "psb_dp_sync": [vp, vp],
        "psb_dp_status": [vp, vp],
        "psb_dp_destroy": [vp],
        "psb_densify_plan": [i, Model, Cfg, vp, P(i), vp],
        "psb_densify_apply": [i, Model, Model, i, Cfg, vp, vp, vp],
        "psb_prune_plan": [i, vp, vp, P(i), vp],
        "psb_prune_apply": [i, Model, Model, i, vp, i, vp],
        "psb_insert_points": [i, Model, Model, i, vp, vp, vp, i, vp],
        "psb_reset_opacity": [i, vp, vp, vp, vp],
        "psb_relocate": [i, Model, P(_RelocateCfg), vp, vp, P(i), vp],
        "psb_grow": [i, Model, Model, i, P(_RelocateCfg), vp, vp, vp],
        "psb_seed_plan": [Cam, vp, vp, vp, vp, P(_SeedCfg), vp, P(i), vp],
        "psb_seed_apply": [i, Model, Model, i, Cam, vp, vp, P(_SeedCfg), vp, i, vp],
    }
    for name, args in sigs.items():
        fn = getattr(L, name)
        fn.argtypes, fn.restype = args, i
    L.psb_densify_workspace_bytes.argtypes, L.psb_densify_workspace_bytes.restype = [i], size_t
    L.psb_relocate_workspace_bytes.argtypes, L.psb_relocate_workspace_bytes.restype = [i], size_t
    L.psb_seed_workspace_bytes.argtypes, L.psb_seed_workspace_bytes.restype = [i, i, i], size_t
    L._trainer_bound = True
    return L


@dataclass
class GaussianOptimizationParams:
    iterations: int = 30100
    position_lr_init: float = 0.00032
    position_lr_final: float = 0.00032
    position_lr_delay_mult: float = 0.01
    position_lr_max_steps: int = 24
    feature_lr: float = 0.0025
    opacity_lr: float = 0.05
    scaling_lr: float = 0.005
    rotation_lr: float = 0.001
    percent_dense: float = 0.01
    lambda_dssim: float = 0.2
    densification_interval: int = 100
    opacity_reset_interval: int = 0
    densify_from_iter: int = 600
    densify_until_iter: int = 15000
    densify_grad_threshold: float = 0.001
    exposure_lr: float = 0.01     # learning rate of the per-keyframe exposure rows (graphdeco's exposure_lr_init)
    # bounded-budget densification (3DGS-MCMC, Kheradmand et al. 2024; the defaults are the paper's / gsplat MCMCStrategy's). Off by default.
    mcmc: bool = False            # GaussianTrainer: regularisers on the step, position noise behind it, mcmcRefine() instead of densifyAndPrune
    cap_max: int = 1_000_000      # the map never holds more Gaussians than this
    mcmc_noise_lr: float = 5e5    # the noise is Sigma xi * position lr * this * g(opacity)
    mcmc_noise_visible_only: bool = True   # noise only on rows the step's view saw (False: every row, as in offline training)
    opacity_reg: float = 0.01     # lambda of mean sigmoid(opacity)
    scale_reg: float = 0.01       # lambda of mean exp(scaling)
    mcmc_min_opacity: float = 0.005   # a Gaussian at or below is dead and gets relocated
    mcmc_grow_factor: float = 1.05    # growth per mcmcRefine, up to cap_max
    mcmc_seed: int = 0            # key of the relocation draws and of the noise


class GaussianModel:
    """Parameter tensors in the reference's layout + Adam state + learning rates."""

    def __init__(self, sh_degree=3, device="cuda"):
        self.max_sh_degree_ = sh_degree
        self.active_sh_degree_ = 0
        self.device = torch.device(device)
        self.spatial_lr_scale_ = 1.0
        self.lr_ = [0.0] * 6
        self.step_ = 0
        self.lr_delay_steps_ = 0
        self.percent_dense_ = 0.01
        self.exposure_lr_ = GaussianOptimizationParams.exposure_lr
        z = lambda *s, dtype=torch.float32: torch.zeros(s, dtype=dtype, device=self.device)
        # per-keyframe exposure table (ensureExposures): row k = the 3x4 affine of the caller's keyframe id k, its Adam moments and its
        # own Adam step count (advanced on the device by the fused step)
        self.exposure_, self.exposure_exp_avg_, self.exposure_exp_avg_sq_ = z(0, 3, 4), z(0, 3, 4), z(0, 3, 4)
        self.exposure_step_ = z(0, dtype=torch.int32)
        # 3D smoothing filter (computeFilter3D): [P] float32, or None when it has not been computed for the current rows
        self.filter_3D_ = None

    @classmethod
    def from_numpy(cls, scene, device="cuda", sh_degree=3):
        m = cls(sh_degree, device)
        t = lambda a: torch.from_numpy(a).to(m.device).contiguous()
        m.xyz_, m.features_dc_, m.features_rest_ = t(scene["xyz"]), t(scene["features_dc"]), t(scene["features_rest"])
        m.opacity_, m.scaling_, m.rotation_ = t(scene["opacity"]), t(scene["scaling"]), t(scene["rotation"])
        m.active_sh_degree_ = sh_degree
        return m

    def tensors(self):
        return [self.xyz_, self.features_dc_, self.features_rest_, self.opacity_, self.scaling_, self.rotation_]

    def num_points(self):
        return self.xyz_.size(0)

    # --- reference GaussianModel::trainingSetup (gaussian_model.cpp:477-509)
    def trainingSetup(self, args: GaussianOptimizationParams):
        self.percent_dense_ = args.percent_dense
        P = self.num_points()
        z = lambda *s: torch.zeros(s, dtype=torch.float32, device=self.device)
        self.xyz_gradient_accum_, self.denom_, self.max_radii2D_ = z(P, 1), z(P, 1), z(P)
        self.exp_avg_ = [torch.zeros_like(t) for t in self.tensors()]
        self.exp_avg_sq_ = [torch.zeros_like(t) for t in self.tensors()]
        # per row: "its moments may be non-zero" (psb_model.adam_live). The fused step keeps it exact; whatever else replaces or
        # rewrites moments marks it stale and the next fused step rebuilds it from the moments first
        self.adam_live_ = torch.zeros(P, dtype=torch.uint8, device=self.device)
        self.adam_live_valid_ = True
        self.step_ = 0
        self.lr_ = [args.position_lr_init * self.spatial_lr_scale_, args.feature_lr, args.feature_lr / 20.0, args.opacity_lr,
                    args.scaling_lr, args.rotation_lr]
        self.lr_init_ = args.position_lr_init * self.spatial_lr_scale_
        self.lr_final_ = args.position_lr_final * self.spatial_lr_scale_
        self.lr_delay_mult_ = args.position_lr_delay_mult
        self.max_steps_ = args.position_lr_max_steps
        self.exposure_lr_ = args.exposure_lr

    # --- training-state snapshot (parameters, Adam moments, densification statistics, step counter); restore copies in
    #     place so device pointers held elsewhere stay valid. Used by bench.py to time every leg on the same iterations.
    def snapshot(self):
        c = lambda ts: [t.clone() for t in ts]
        live = self._live_tensor()
        return dict(p=c(self.tensors()), m=c(self.exp_avg_), v=c(self.exp_avg_sq_),
                    stats=c([self.xyz_gradient_accum_, self.denom_, self.max_radii2D_]), step=self.step_, lr=list(self.lr_),
                    sh=self.active_sh_degree_, live=live.clone(), live_valid=self.adam_live_valid_,
                    exposure=c(self._exposure_tensors()), exposure_lr=self.exposure_lr_,
                    filter_3D=self.filter_3D_.clone() if self.filter_3D_ is not None else None)

    def restore(self, snap):
        assert snap["p"][0].shape == self.xyz_.shape, "restore: the model was resized since the snapshot"
        for dst, src in zip(self.tensors() + self.exp_avg_ + self.exp_avg_sq_ + [self.xyz_gradient_accum_, self.denom_, self.max_radii2D_],
                            snap["p"] + snap["m"] + snap["v"] + snap["stats"]):
            dst.copy_(src)
        self.step_, self.lr_, self.active_sh_degree_ = snap["step"], list(snap["lr"]), snap["sh"]
        self._live_tensor().copy_(snap["live"])
        self.adam_live_valid_ = snap["live_valid"]
        if snap["exposure"][0].shape == self.exposure_.shape:
            for dst, src in zip(self._exposure_tensors(), snap["exposure"]):
                dst.copy_(src)
        else:   # the table grew since the snapshot
            self.exposure_, self.exposure_exp_avg_, self.exposure_exp_avg_sq_, self.exposure_step_ = [t.clone() for t in snap["exposure"]]
        self.exposure_lr_ = snap["exposure_lr"]
        f = snap["filter_3D"]
        if f is not None and self.filter_3D_ is not None and self.filter_3D_.shape == f.shape:
            self.filter_3D_.copy_(f)
        else:
            self.filter_3D_ = f.clone() if f is not None else None

    def _live_tensor(self):
        """adam_live_, (re)allocated when the row count changed (its content is then stale)."""
        if getattr(self, "adam_live_", None) is None or self.adam_live_.size(0) != self.num_points():
            self.adam_live_ = torch.zeros(self.num_points(), dtype=torch.uint8, device=self.device)
            self.adam_live_valid_ = False
        return self.adam_live_

    # --- per-keyframe exposure compensation: GaussianTrainer.trainForOneIteration(..., exposure_id=k) trains the map against keyframe k's
    #     image through row k, I'(c) = sum_j E[j][c] I(j) + E[c][3] (psb_exposure), and takes one Adam step of that row
    def _exposure_tensors(self):
        return [self.exposure_, self.exposure_exp_avg_, self.exposure_exp_avg_sq_, self.exposure_step_]

    def numExposures(self):
        return self.exposure_.size(0)

    def ensureExposures(self, K):
        """Grows the exposure table to at least K rows. New rows are eye(3, 4) with zero moments and step count; existing rows,
        moments and step counts are kept. Growing reallocates the tensors."""
        n = self.numExposures()
        if K <= n:
            return
        z = torch.zeros((K - n, 3, 4), dtype=torch.float32, device=self.device)
        eye = torch.eye(3, 4, dtype=torch.float32, device=self.device).expand(K - n, 3, 4)
        self.exposure_ = torch.cat([self.exposure_, eye], 0).contiguous()
        self.exposure_exp_avg_ = torch.cat([self.exposure_exp_avg_, z], 0).contiguous()
        self.exposure_exp_avg_sq_ = torch.cat([self.exposure_exp_avg_sq_, z.clone()], 0).contiguous()
        self.exposure_step_ = torch.cat([self.exposure_step_, torch.zeros(K - n, dtype=torch.int32, device=self.device)]).contiguous()

    def applyExposure(self, image, k):
        """image [3,H,W] through exposure row k (graphdeco's form: HWC pixels times E[:3,:3], plus E[:3,3]): the image the fused
        step compares with keyframe k's target. For evaluating against that keyframe and for display."""
        E = self.exposure_[int(k)].to(image.dtype)
        return torch.matmul(image.permute(1, 2, 0), E[:, :3]).permute(2, 0, 1) + E[:, 3, None, None]

    def setExposureLearningRate(self, lr): self.exposure_lr_ = float(lr)

    def saveExposure(self, path):
        """exposure.json: {"<keyframe id>": 3x4 list} for every row of the table."""
        from . import io
        io.save_exposure(path, {k: row for k, row in enumerate(self.exposure_.detach().cpu().numpy())})

    def loadExposure(self, path):
        """Reads exposure.json into the table (grown as needed). The loaded rows restart their Adam state (zero moments and step)."""
        from . import io
        rows = io.load_exposure(path)
        if not rows:
            return
        self.ensureExposures(max(rows) + 1)
        for k, row in rows.items():
            self.exposure_[k] = torch.from_numpy(row).to(self.device)
            self.exposure_exp_avg_[k] = 0.0
            self.exposure_exp_avg_sq_[k] = 0.0
            self.exposure_step_[k] = 0

    def invalidateAdamLive(self):
        """Call after writing moments by any means other than the fused step (the next fused step rebuilds the live bytes)."""
        self.adam_live_valid_ = False

    def adamLive(self):
        """adam_live_, rebuilt from the moments (psb_adam_live_rebuild) if it is stale."""
        live = self._live_tensor()
        if not self.adam_live_valid_:
            m = self._cmodel(live=live)
            _lib.check(_bind().psb_adam_live_rebuild(self.num_points(), C.byref(m), torch.cuda.current_stream().cuda_stream), "psb_adam_live_rebuild")
            self.adam_live_valid_ = True
        return live

    # --- 3D smoothing filter (Mip-Splatting; include/psb200.h, psb_filter3d): every Gaussian is widened to at least the finest sampling
    #     interval at which a keyframe saw it. computeFilter3D computes it; GaussianTrainer(filter3d=True) and
    #     renderer.render(pipe=GaussianPipelineParams(filter_3d=True)) apply it. Every method that changes which row is which, or the map's
    #     spatial scale, drops it (filter_3D_ = None): recompute it after densification, as Mip-Splatting does (and every ~100 iterations).
    def computeFilter3D(self, cams):
        """cams: camera dicts in the form GaussianTrainer takes (viewmatrix: 16 floats; tanfovx, tanfovy, W, H), the full-resolution keyframes.
        Sets filter_3D_ [P] (psb_filter3d) and returns the number of rows at least one camera sees (one host round trip)."""
        rows = []
        for k, cam in enumerate(cams):
            try:
                view = torch.as_tensor(cam["viewmatrix"]).detach().to("cpu", torch.float64).reshape(-1)
                tx, ty, W, H = float(cam["tanfovx"]), float(cam["tanfovy"]), cam["W"], cam["H"]
            except (KeyError, TypeError, ValueError, RuntimeError) as e:
                raise ValueError(f"computeFilter3D: camera {k} is not a camera dict (viewmatrix, tanfovx, tanfovy, W, H): {e}") from None
            if view.numel() != 16 or not bool(torch.isfinite(view).all()):
                raise ValueError(f"computeFilter3D: camera {k}: viewmatrix must hold 16 finite values")
            if int(W) != W or int(H) != H or W <= 0 or H <= 0:
                raise ValueError(f"computeFilter3D: camera {k}: W and H must be positive integers, got {W}, {H}")
            fx, fy = W / (2.0 * tx) if tx else math.inf, H / (2.0 * ty) if ty else math.inf
            if not (math.isfinite(tx) and math.isfinite(ty) and tx > 0 and ty > 0 and math.isfinite(fx) and math.isfinite(fy)):
                raise ValueError(f"computeFilter3D: camera {k}: tanfovx and tanfovy must be finite and positive, got {tx}, {ty}")
            rows.append(torch.cat([view, torch.tensor([fx, fy, float(W), float(H)], dtype=torch.float64)]))
        packed = (torch.stack(rows) if rows else torch.zeros((0, 20), dtype=torch.float64)).to(self.device, torch.float32).contiguous()
        P = self.num_points()
        f = torch.empty(P, dtype=torch.float32, device=self.device)
        seen = C.c_int()
        _lib.check(_bind().psb_filter3d(P, self.xyz_.data_ptr() if P else None, len(rows), packed.data_ptr() if rows else None,
                                        f.data_ptr() if P else None, C.byref(seen), torch.cuda.current_stream().cuda_stream), "psb_filter3d")
        self.filter_3D_ = f
        return seen.value

    def filter3D(self):
        """filter_3D_, checked to belong to the current rows (ValueError otherwise)."""
        f = self.filter_3D_
        if f is None or tuple(f.shape) != (self.num_points(),):
            raise ValueError("the 3D filter is missing or stale (the rows changed since it was computed): call computeFilter3D(cams)")
        return f

    def getScalingWithFilter3D(self):
        """s' = sqrt(s^2 + f^2) per axis (differentiable w.r.t. scaling_)"""
        s = torch.exp(self.scaling_)
        return torch.sqrt(s * s + self.filter3D().square().unsqueeze(1))

    def getOpacityWithFilter3D(self):
        """o' = o sqrt(prod s^2 / prod s'^2) (differentiable w.r.t. opacity_ and scaling_)"""
        s2 = torch.exp(self.scaling_).square()
        c = torch.sqrt((s2 / (s2 + self.filter3D().square().unsqueeze(1))).prod(dim=1, keepdim=True))
        return torch.sigmoid(self.opacity_) * c

    # --- on-disk point cloud (reference GaussianModel::savePly / loadPly / saveSparsePointsPly, gaussian_model.cpp:838-1088)
    def savePly(self, path, fuse_filter3d=False):
        """fuse_filter3d=True writes log s' and logit(o') of the 3D filter instead of the raw scaling and opacity (Mip-Splatting's fused
        export): any standard 3DGS viewer then draws what the trainer draws with the filter on."""
        from . import io
        ts = self.tensors()
        if fuse_filter3d:
            with torch.no_grad():
                ts = list(ts)
                ts[3] = torch.logit(self.getOpacityWithFilter3D())
                ts[4] = torch.log(self.getScalingWithFilter3D())
        io.save_ply(path, *[t.detach().cpu().numpy() for t in ts])

    def loadPly(self, path):
        """Replaces the parameter tensors by the file's content and activates every SH degree (gaussian_model.cpp:951)."""
        from . import io
        a = io.load_ply(path, self.max_sh_degree_)
        t = lambda x: torch.from_numpy(x).to(self.device).contiguous()
        self._set([t(a[k]) for k in ("xyz", "features_dc", "features_rest", "opacity", "scaling", "rotation")])
        self.active_sh_degree_ = self.max_sh_degree_
        self._rows_replaced()

    def setSparsePoints(self, xyz, color):
        """sparse SLAM map points + colours in [0,1] kept for input.ply (reference gaussian_model.cpp: sparse_points_xyz_ / _color_)"""
        self.sparse_points_xyz_, self.sparse_points_color_ = xyz, color

    def saveSparsePointsPly(self, path):
        from . import io
        io.save_sparse_points_ply(path, self.sparse_points_xyz_.cpu().numpy(), self.sparse_points_color_.cpu().numpy())

    def exponLrFunc(self, step):
        if step < 0 or (self.lr_init_ == 0.0 and self.lr_final_ == 0.0):
            return 0.0
        if self.lr_delay_steps_ > 0:
            delay = self.lr_delay_mult_ + (1.0 - self.lr_delay_mult_) * math.sin(0.5 * math.pi * min(max(step / self.lr_delay_steps_, 0.0), 1.0))
        else:
            delay = 1.0
        t = min(max(step / self.max_steps_, 0.0), 1.0)
        return delay * math.exp(math.log(self.lr_init_) * (1 - t) + math.log(self.lr_final_) * t)

    def updateLearningRate(self, step):
        self.lr_[0] = self.exponLrFunc(step)
        return self.lr_[0]

    def setPositionLearningRate(self, lr): self.lr_[0] = lr * self.spatial_lr_scale_
    def setFeatureLearningRate(self, lr): self.lr_[1], self.lr_[2] = lr, lr / 20.0
    def setOpacityLearningRate(self, lr): self.lr_[3] = lr
    def setScalingLearningRate(self, lr): self.lr_[4] = lr
    def setRotationLearningRate(self, lr): self.lr_[5] = lr
    def setShDegree(self, d): self.active_sh_degree_ = min(max(d, 0), self.max_sh_degree_)

    def oneUpShDegree(self):
        if self.active_sh_degree_ < self.max_sh_degree_:
            self.active_sh_degree_ += 1

    # ------------------------------------------------------------------------------------------------------------
    # Densification / pruning / insertion / loop-closure surgery (reference src/gaussian_model.cpp:193-475, 556-815).
    # Every one of them is a fused device pass over the model through the C-ABI (psb_densify_* / psb_prune_* /
    # psb_insert_points / psb_reset_opacity): one read of the surviving rows, one write of the output rows, one host
    # round trip (the new row count). The ATen restatement of the reference code lives in oracle/ref_densify.py (tests only).
    # ------------------------------------------------------------------------------------------------------------
    def getOpacityActivation(self): return torch.sigmoid(self.opacity_)
    def getScalingActivation(self): return torch.exp(self.scaling_)
    def getRotationActivation(self): return torch.nn.functional.normalize(self.rotation_)

    def _set(self, tensors):
        (self.xyz_, self.features_dc_, self.features_rest_, self.opacity_, self.scaling_, self.rotation_) = tensors

    def _exist(self):
        if getattr(self, "exist_since_iter_", None) is None or self.exist_since_iter_.size(0) != self.num_points():
            self.exist_since_iter_ = torch.zeros(self.num_points(), dtype=torch.int32, device=self.device)
        return self.exist_since_iter_

    def _blank(self, P):
        """Uninitialised tensors of a P-row model (parameters, both moments, statistics, exist_since_iter), keyed like _rows()."""
        shapes = row_shapes(P)
        e = lambda sh: torch.empty(sh, dtype=torch.float32, device=self.device)
        return dict(p=[e(sh) for sh in shapes], m=[e(sh) for sh in shapes], v=[e(sh) for sh in shapes], accum=e((P, 1)), denom=e((P, 1)),
                    max_radii=e((P,)), exist=torch.empty(P, dtype=torch.int32, device=self.device))

    def _rows(self):
        """The model's tensors as the row operations take them (_cmodel_of(**rows))."""
        return dict(p=self.tensors(), m=self.exp_avg_, v=self.exp_avg_sq_, accum=self.xyz_gradient_accum_, denom=self.denom_,
                    max_radii=self.max_radii2D_, exist=self._exist())

    def _check_rows(self):
        """The C row operations move 45 features_rest floats per row: any other SH storage is refused before the first C call."""
        want = row_shapes(self.num_points())[2]
        if tuple(self.features_rest_.shape) != want:
            raise ValueError(f"row operations need features_rest of shape {list(want)} (all 16 SH coefficients), got {list(self.features_rest_.shape)}")

    def _out_of_place(self, P_new, call, what):
        """call(src, dst) is a C row operation from the current rows into P_new new ones; the model then adopts the new rows."""
        d = self._blank(P_new)
        _lib.check(call(C.byref(_cmodel_of(**self._rows())), C.byref(_cmodel_of(**d))), what)
        self._adopt(d)

    def _adopt(self, d):
        self._set(d["p"])
        self.exp_avg_, self.exp_avg_sq_ = d["m"], d["v"]
        self.xyz_gradient_accum_, self.denom_, self.max_radii2D_, self.exist_since_iter_ = d["accum"], d["denom"], d["max_radii"], d["exist"]
        self._rows_replaced()

    def _rows_replaced(self):
        """Rows renumbered or replaced: the live bytes are stale (the next fused step rebuilds them) and the 3D filter is dropped."""
        self.invalidateAdamLive()
        self.filter_3D_ = None

    def _geometry_changed(self, fresh_moments=()):
        """Rows moved in place: the 3D filter is dropped; the groups in fresh_moments restart Adam from zero (the live bytes stay valid)."""
        self.filter_3D_ = None
        for i in fresh_moments:
            self.exp_avg_[i] = torch.zeros_like(self.tensors()[i])
            self.exp_avg_sq_[i] = torch.zeros_like(self.tensors()[i])

    def resetOpacity(self):
        """reference gaussian_model.cpp:556-565. NOTE: the reference's misplaced parenthesis makes this
        min(sigmoid(o), 1) — it does NOT clamp to 0.01 (SURVEY §2.2 quirk 9); only the opacity moments are zeroed."""
        L = _bind()
        _lib.check(L.psb_reset_opacity(self.num_points(), self.opacity_.data_ptr(), self.exp_avg_[3].data_ptr(), self.exp_avg_sq_[3].data_ptr(),
                                       torch.cuda.current_stream().cuda_stream), "psb_reset_opacity")

    def prunePoints(self, mask):
        """reference gaussian_model.cpp:588-642 (statistics are compacted, not reset)"""
        self._check_rows()
        L = _bind()
        P = self.num_points()
        stream = torch.cuda.current_stream().cuda_stream
        ws = torch.empty(L.psb_densify_workspace_bytes(P), dtype=torch.uint8, device=self.device)
        counts = (C.c_int * 5)()
        m8 = mask.to(torch.uint8).contiguous()
        _lib.check(L.psb_prune_plan(P, m8.data_ptr(), ws.data_ptr(), counts, stream), "psb_prune_plan")
        self._out_of_place(counts[0], lambda src, dst: L.psb_prune_apply(P, src, dst, counts[0], ws.data_ptr(), 1, stream), "psb_prune_apply")

    def densifyAndPrune(self, max_grad, min_opacity, extent, max_screen_size, seed=0, offset=None, samples=None):
        """reference gaussian_model.cpp:795-815 with densifyAndClone / densifyAndSplit / prunePoints / densificationPostfix folded
        into one plan + one scatter pass. The split draw is Philox(seed, offset) — identical on every data-parallel replica —
        unless `samples` ([2 * n_split, 3] standard normals in the reference's repeat order) is injected (tests).
        Returns (P_new, kept originals, clones, kept split children per copy, split-selected)."""
        self._check_rows()
        L = _bind()
        P = self.num_points()
        stream = torch.cuda.current_stream().cuda_stream
        cfg = _DensifyCfg(float(max_grad), float(min_opacity), float(extent), float(self.percent_dense_), int(max_screen_size or 0), int(seed),
                          int(self.step_ if offset is None else offset))
        ws = torch.empty(L.psb_densify_workspace_bytes(P), dtype=torch.uint8, device=self.device)
        counts = (C.c_int * 5)()
        _lib.check(L.psb_densify_plan(P, C.byref(_cmodel_of(**self._rows())), C.byref(cfg), ws.data_ptr(), counts, stream), "psb_densify_plan")
        if samples is not None:
            samples = samples.to(self.device, torch.float32).contiguous()
            assert samples.shape == (2 * counts[4], 3), (samples.shape, counts[4])
        z = samples.data_ptr() if samples is not None and samples.numel() else None
        self._out_of_place(counts[0], lambda src, dst: L.psb_densify_apply(P, src, dst, counts[0], C.byref(cfg), ws.data_ptr(), z, stream),
                           "psb_densify_apply")
        return tuple(counts)

    # --- bounded-budget densification (3DGS-MCMC; gsplat MCMCStrategy's relocate / sample_add): psb_relocate / psb_grow
    def _uniforms(self, uniforms):
        return None if uniforms is None else uniforms.to(self.device, torch.float32).contiguous()

    def relocateGaussians(self, min_opacity=0.005, seed=0, offset=None, iteration=0, uniforms=None):
        """Every dead row (sigmoid(opacity) <= min_opacity) becomes a copy of an alive row drawn with probability proportional to its
        opacity; the drawn rows and their copies share the corrected opacity and scale that keep the rendered picture (psb_relocate).
        In place, the row count does not change; moments of the rows involved are zeroed. The draw is Philox(seed, offset) — identical
        on every replica — unless `uniforms` (one number in [0, 1) per dead row, at least that many) is injected (tests).
        Returns the number of rows relocated (one host round trip)."""
        self._check_rows()
        L = _bind()
        P = self.num_points()
        cfg = _RelocateCfg(float(min_opacity), int(iteration), int(seed), int(self.step_ if offset is None else offset))
        ws = torch.empty(L.psb_relocate_workspace_bytes(P), dtype=torch.uint8, device=self.device)
        live = self._live_tensor()   # a valid one is kept exact: the bytes of the rows whose moments are zeroed are cleared
        model = _cmodel_of(**self._rows(), live=live if self.adam_live_valid_ else None)
        u = self._uniforms(uniforms)
        counts = (C.c_int * 2)()
        _lib.check(L.psb_relocate(P, C.byref(model), C.byref(cfg), ws.data_ptr(), u.data_ptr() if u is not None and u.numel() else None, counts,
                                  torch.cuda.current_stream().cuda_stream), "psb_relocate")
        if u is not None:
            assert u.numel() >= counts[1], (u.numel(), counts[1])
        self._geometry_changed()
        return counts[0]

    def addNewGaussians(self, cap_max, grow_factor=1.05, min_opacity=0.005, seed=0, offset=None, iteration=0, uniforms=None):
        """Grows the model to min(cap_max, floor(grow_factor * P)) rows: the new rows are copies of rows drawn (over all rows) with
        probability proportional to opacity, corrected together with their sources like relocateGaussians does (psb_grow); they
        start with zero moments and statistics and exist_since_iter = iteration. Returns the number of rows added (0 at the cap)."""
        self._check_rows()
        L = _bind()
        P = self.num_points()
        if not 1.0 < grow_factor <= 2.0:
            raise ValueError(f"grow_factor must be in (1, 2], got {grow_factor}")
        P_new = min(int(cap_max), int(math.floor(grow_factor * P)))
        if P_new <= P:
            return 0
        cfg = _RelocateCfg(float(min_opacity), int(iteration), int(seed), int(self.step_ if offset is None else offset))
        ws = torch.empty(L.psb_relocate_workspace_bytes(P), dtype=torch.uint8, device=self.device)
        u = self._uniforms(uniforms)
        if u is not None:
            assert u.numel() >= P_new - P, (u.numel(), P_new - P)
        self._out_of_place(P_new, lambda src, dst: L.psb_grow(P, src, dst, P_new, C.byref(cfg), ws.data_ptr(), u.data_ptr() if u is not None else None,
                                                              torch.cuda.current_stream().cuda_stream), "psb_grow")
        return P_new - P

    def densifySplitCount(self, max_grad, extent):
        """number of rows densifyAndSplit would select right now (plan only; for tests that inject the normal draw)"""
        L = _bind()
        P = self.num_points()
        cfg = _DensifyCfg(float(max_grad), 0.0, float(extent), float(self.percent_dense_), 0, 0, 0)
        ws = torch.empty(L.psb_densify_workspace_bytes(P), dtype=torch.uint8, device=self.device)
        counts = (C.c_int * 5)()
        _lib.check(L.psb_densify_plan(P, C.byref(_cmodel_of(**self._rows())), C.byref(cfg), ws.data_ptr(), counts, torch.cuda.current_stream().cuda_stream),
                   "psb_densify_plan")
        return counts[4]

    def increasePcd(self, points, colors, iteration=0):
        """reference gaussian_model.cpp:193-377 (both overloads: host vectors / tensors): new Gaussians from sparse points — RGB2SH
        colour, scale from the 3-NN mean distance (distCUDA2 = psb_dist_cuda2), identity rotation, opacity = logit(0.1)."""
        from .points import distCUDA2
        self._check_rows()
        L = _bind()
        points = torch.as_tensor(points, dtype=torch.float32).reshape(-1, 3)
        colors = torch.as_tensor(colors, dtype=torch.float32).reshape(-1, 3)
        n = points.size(0)
        if n == 0:
            return
        pts = points.to(self.device).contiguous()
        cols = colors.to(self.device).contiguous()
        if getattr(self, "sparse_points_xyz_", None) is None or self.sparse_points_xyz_.numel() == 0:
            self.sparse_points_xyz_, self.sparse_points_color_ = pts, cols
        else:
            self.sparse_points_xyz_ = torch.cat((self.sparse_points_xyz_, pts), dim=0)
            self.sparse_points_color_ = torch.cat((self.sparse_points_color_, cols), dim=0)
        dist2 = distCUDA2(pts)
        P = self.num_points()
        if not hasattr(self, "exp_avg_"):
            raise RuntimeError("increasePcd: call trainingSetup() first (the optimizer state is extended together with the parameters)")
        self._out_of_place(P + n, lambda src, dst: L.psb_insert_points(P, src, dst, n, pts.data_ptr(), cols.data_ptr(), dist2.data_ptr(), int(iteration),
                                                                       torch.cuda.current_stream().cuda_stream), "psb_insert_points")

    # --- loop closure / scale refinement (reference gaussian_model.cpp:379-475)
    def scaledTransformationPostfix(self, new_xyz, new_scaling):
        """:403-418: the two tensors replace xyz / scaling in the optimizer with FRESH (zero) moments (replaceTensorToOptimizer :567-586)"""
        self.xyz_, self.scaling_ = new_xyz.contiguous(), new_scaling.contiguous()
        self._geometry_changed(fresh_moments=(0, 4))

    def applyScaledTransformation(self, s, T):
        """:379-401: xyz <- T (s * xyz) through transformPoints; scaling_ (the LOG scale) is multiplied by s like the reference does.
        T: [4,4] row-major world transform (Sophus::SE3f::matrix())."""
        from .points import transformPoints
        T_tensor = torch.as_tensor(T, dtype=torch.float32, device=self.device).reshape(4, 4).transpose(0, 1).contiguous()
        xyz = transformPoints(self.xyz_ * float(s), T_tensor)
        self.scaledTransformationPostfix(xyz, self.scaling_ * float(s))

    def scaledTransformVisiblePointsOfKeyframe(self, point_not_transformed_flags, diff_pose, kf_world_view_transform, kf_full_proj_transform,
                                               kf_creation_iter, stable_num_iter_existence, num_transformed=0, scale=1.0):
        """:420-475: Gaussians younger than `stable_num_iter_existence` relative to the keyframe, not yet transformed and in front of it
        are moved by diff_pose (operate_points.cu:95-143); xyz and rotation (ACTIVATED, as in the reference) re-enter the optimizer with
        zero moments. Returns the updated num_transformed."""
        from .points import scaleAndTransformThenMarkVisiblePoints
        points = self.xyz_.clone()
        rots = self.getRotationActivation()
        unstable = (self._exist() - int(kf_creation_iter)).abs() < int(stable_num_iter_existence)
        num_transformed = scaleAndTransformThenMarkVisiblePoints(points, rots, point_not_transformed_flags, unstable, diff_pose,
                                                                 kf_world_view_transform, kf_full_proj_transform, num_transformed, scale)
        self.xyz_, self.rotation_ = points.contiguous(), rots.contiguous()
        self._geometry_changed(fresh_moments=(0, 5))
        return num_transformed

    def _cmodel(self, with_state=True, live=None):
        """live: adam_live_ (valid) for the fused step; every other caller passes NULL. exist_since_iter is always NULL."""
        for t in self.tensors():
            assert t.is_contiguous() and t.dtype == torch.float32
        if not with_state:
            return _cmodel_of(self.tensors(), live=live)
        return _cmodel_of(self.tensors(), self.exp_avg_, self.exp_avg_sq_, self.xyz_gradient_accum_, self.denom_, self.max_radii2D_, live=live)


def _ccamera(cam):
    c = _Camera()
    c.viewmatrix, c.projmatrix, c.campos = cam["viewmatrix"].data_ptr(), cam["projmatrix"].data_ptr(), cam["campos"].data_ptr()
    c.tan_fovx, c.tan_fovy, c.width, c.height = float(cam["tanfovx"]), float(cam["tanfovy"]), int(cam["W"]), int(cam["H"])
    return c


class GaussianTrainer:
    """One fused training iteration per call. `cam` = dict(viewmatrix, projmatrix, campos: device tensors; tanfovx, tanfovy, W, H).

    deterministic: True makes every training call of this trainer bit-identical from run to run (same inputs, build and GPU model;
    psb_trainer_set_deterministic), False keeps the default (faster) kernels, None follows torch.are_deterministic_algorithms_enabled()
    at each call.

    antialiasing: True renders and trains every pass of this trainer with the 2D Mip filter (psb_trainer_set_antialiasing: each splat
    blends with opacity o * sqrt(max(det0 / det1, 2.5e-5)), det0 / det1 the determinants of its 2D covariance before / after the
    0.3 px^2 dilation), as renderer.render(pipe=GaussianPipelineParams(antialiasing=True)) does on the operator path. Fixed for the
    trainer's lifetime.

    opt.mcmc: bounded-budget densification (3DGS-MCMC). The step's per-Gaussian stage adds the opacity and scale regularisers
    (opt.opacity_reg, opt.scale_reg; psb_trainer_set_regularizers: on the rows the step updates), trainForOneIteration and
    trainWithLoss enqueue the position noise behind the step (psb_trainer_inject_noise, keyed by opt.mcmc_seed and model.step_), and
    mcmcRefine() replaces densifyAndPrune: it relocates the dead Gaussians and grows the map by opt.mcmc_grow_factor up to
    opt.cap_max. With mcmc off nothing of this is launched.

    filter3d: True applies the model's 3D smoothing filter (model.computeFilter3D; psb_trainer_set_filter3d) in every render and training call,
    as renderer.render(pipe=GaussianPipelineParams(filter_3d=True)) does on the operator path. Each call hands over model.filter_3D_ as it is
    then; a missing or stale filter raises ValueError. Recomputing it is the caller's choice (Mip-Splatting: after each densification and
    every 100 iterations). Fixed for the trainer's lifetime."""

    def __init__(self, model: GaussianModel, opt: GaussianOptimizationParams = None, background=None, deterministic=None, antialiasing=False,
                 filter3d=False):
        self.L = _bind()
        self.model = model
        self.opt = opt or GaussianOptimizationParams()
        h = C.c_void_p()
        _lib.check(self.L.psb_trainer_create(C.byref(h)), "psb_trainer_create")
        self.h = h
        self.background = background if background is not None else torch.zeros(3, device=model.device)
        self.iteration = 0
        self._last = _NO_CALL
        self._deterministic = deterministic
        self._det_applied = False      # the mode the context is in (a new context starts with it off)
        self._apply_deterministic()
        self._antialiasing = bool(antialiasing)
        if self._antialiasing:
            _lib.check(self.L.psb_trainer_set_antialiasing(self.h, 1), "psb_trainer_set_antialiasing")
        if self.opt.mcmc:
            _lib.check(self.L.psb_trainer_set_regularizers(self.h, float(self.opt.opacity_reg), float(self.opt.scale_reg)),
                       "psb_trainer_set_regularizers")
        self._filter3d = bool(filter3d)

    def _hand_filter3d(self):
        """filter3d: the context takes model.filter_3D_ as it is now (ValueError when it is missing or stale)."""
        if self._filter3d:
            f = self.model.filter3D()
            _lib.check(self.L.psb_trainer_set_filter3d(self.h, f.data_ptr(), self.model.num_points()), "psb_trainer_set_filter3d")

    @property
    def filter3d(self):
        """Whether this trainer's calls apply the model's 3D filter (set at construction)."""
        return self._filter3d

    def _inject_noise(self):
        """opt.mcmc: the position noise behind the step just enqueued (a no-op on the device if that step's pass overflowed)."""
        if not self.opt.mcmc:
            return
        m, o = self.model, self.opt
        cm = m._cmodel(False)
        _lib.check(self.L.psb_trainer_inject_noise(self.h, m.num_points(), C.byref(cm), float(m.lr_[0]), float(o.mcmc_noise_lr), int(o.mcmc_seed),
                                                   int(m.step_), int(bool(o.mcmc_noise_visible_only)), torch.cuda.current_stream().cuda_stream),
                   "psb_trainer_inject_noise")

    def mcmcRefine(self, iteration=None):
        """The refinement round of 3DGS-MCMC, in place of densifyAndPrune: relocateGaussians, then addNewGaussians up to opt.cap_max, both
        keyed by (opt.mcmc_seed, model.step_) like densifyAndPrune's split draw. Returns (rows relocated, rows added)."""
        m, o = self.model, self.opt
        it = self.iteration if iteration is None else int(iteration)
        n_rel = m.relocateGaussians(o.mcmc_min_opacity, seed=o.mcmc_seed, iteration=it)
        n_add = m.addNewGaussians(o.cap_max, o.mcmc_grow_factor, o.mcmc_min_opacity, seed=o.mcmc_seed, iteration=it)
        return n_rel, n_add

    # --- contribution pruning (include/psb200.h, psb_trainer_contribution): a Gaussian's score is the blending weight alpha T it receives in
    #     the pixels of the keyframes, in this trainer's own forward (tight lists, anti-aliasing, 3D filter). When and on which keyframes to
    #     prune is the caller's choice, as with computeFilter3D.
    def contributionScores(self, cams):
        """cams: a non-empty list of camera dicts (the form trainForOneIteration takes). -> (max_weight [P] float32, sum_weight [P] float64):
        the largest and the summed blending weight of every row over all pixels of all views (0: no view blends it). Bit-identical from run
        to run, in either deterministic mode and in any order of the views. One host round trip for the whole sweep; if a view overflowed the
        binning arena, the sweep is repeated once on the grown arena."""
        cams = _check_cams(cams, "contributionScores")
        m = self.model
        P = m.num_points()
        mx = torch.zeros(P, dtype=torch.int32, device=m.device)
        sm = torch.zeros(P, dtype=torch.int64, device=m.device)
        if P > 0:
            self._hand_filter3d()
            cm = m._cmodel(False)
            stream = torch.cuda.current_stream().cuda_stream
            self._last = _NO_CALL
            for attempt in range(2):
                for cam in cams:
                    cc = _ccamera(cam)
                    _lib.check(self.L.psb_trainer_contribution(self.h, P, 16, C.byref(cm), C.byref(cc), self.background.data_ptr(), m.active_sh_degree_,
                                                               mx.data_ptr(), sm.data_ptr(), None, stream), "psb_trainer_contribution")
                rc = self.L.psb_trainer_result(self.h, None, None, stream)
                if rc != -4:
                    _lib.check(rc, "psb_trainer_result")
                    break
                if attempt:
                    raise _lib.PsbError("contributionScores: a view overflowed the binning arena again after it was grown")
                mx.zero_()
                sm.zero_()
        return mx.view(torch.float32), sm.to(torch.float64) * CONTRIB_SUM_UNIT

    def pruneByContribution(self, cams, min_weight, keep=None, min_age=0):
        """Removes the rows that no view in `cams` shows: max_weight < min_weight (contributionScores) and, with keep, all but the `keep`
        rows of highest sum_weight (ties: the lower row index stays). Rows younger than min_age iterations (iteration - exist_since_iter_ <
        min_age) are never removed. Goes through model.prunePoints (statistics compacted, live bytes and 3D filter dropped). Returns the
        number of rows removed."""
        if isinstance(min_weight, bool) or not isinstance(min_weight, (int, float)) or not math.isfinite(min_weight) or not 0 <= min_weight < 1:
            raise ValueError(f"pruneByContribution: min_weight must be finite and in [0, 1), got {min_weight!r}")
        if keep is not None and (isinstance(keep, bool) or not isinstance(keep, int) or keep <= 0):
            raise ValueError(f"pruneByContribution: keep must be a positive int or None, got {keep!r}")
        if isinstance(min_age, bool) or not isinstance(min_age, int) or min_age < 0:
            raise ValueError(f"pruneByContribution: min_age must be an int >= 0, got {min_age!r}")
        cams = _check_cams(cams, "pruneByContribution")
        m = self.model
        mx, sm = self.contributionScores(cams)
        young = (self.iteration - m._exist()) < min_age if min_age > 0 else None
        mask = contribution_prune_mask(mx, sm, float(min_weight), keep, young)
        n = int(mask.sum())
        if n:
            m.prunePoints(mask)
        return n

    # --- depth-guided seeding (include/psb200.h, psb_seed_*): new rows on the pixels of an RGB-D keyframe where this trainer's render of the
    #     map is nearly transparent (a hole) or lies behind the sensor's surface (in front). ORB keypoints miss textureless surfaces; this
    #     fills them. When to seed is the caller's choice (INTEGRATION §2: once per new RGB-D keyframe, after its pose is set).
    def seedFromDepth(self, cam, gt_image, gt_depth, mask=None, alpha_min=0.5, depth_rel=0.1, min_depth=0.2, max_depth=40.0, stride=1, max_new=None,
                      iteration=None):
        """Adds a Gaussian on every `stride`-th pixel (in u and v) of the keyframe whose depth gt_depth [H,W] (metres, <= 0: none) lies in
        (min_depth, max_depth), that mask[0] (mask [3,H,W] or None, the depth loss's convention) does not exclude, and where this trainer's
        render of the view has accumulated opacity A < alpha_min (hole) or a normalised depth D / A beyond gt_depth / (1 - depth_rel) (in
        front). At most max_new are added, spread evenly over the image. Each new row sits at the pixel's centre at depth gt_depth, takes
        the colour of gt_image [3,H,W] and the scale of one grid cell at that depth, and is otherwise what increasePcd writes (opacity 0.1,
        identity rotation, zero moments, exist_since_iter = iteration, default self.iteration; statistics of all rows reset). Seeded points
        are not SLAM map points: sparse_points_xyz_ is untouched. Like every row operation it drops the live bytes and the 3D filter.
        Defaults: alpha_min = 0.5 is SplaTAM's silhouette threshold; min_depth = 0.2 is the forward's near cull (a seed nearer than that
        is never drawn from this keyframe); max_depth = 40 is RGBD.max_depth in the shipped configs; with opt.mcmc, max_new defaults to
        max(opt.cap_max - P, 0), so seeding never exceeds the budget, and otherwise to no limit.
        Returns (rows added, holes, in front): the counts of selected pixels before the cap."""
        num = lambda x: not isinstance(x, bool) and isinstance(x, (int, float)) and not math.isnan(x)
        if not num(alpha_min) or not 0 < alpha_min <= 1:
            raise ValueError(f"seedFromDepth: alpha_min must be in (0, 1], got {alpha_min!r}")
        if not num(depth_rel) or not 0 <= depth_rel <= 1:
            raise ValueError(f"seedFromDepth: depth_rel must be in [0, 1], got {depth_rel!r}")
        if not num(min_depth) or not num(max_depth) or not 0 <= min_depth < max_depth or math.isinf(min_depth):
            raise ValueError(f"seedFromDepth: want 0 <= min_depth < max_depth, got {min_depth!r}, {max_depth!r}")
        if isinstance(stride, bool) or not isinstance(stride, int) or stride < 1:
            raise ValueError(f"seedFromDepth: stride must be an int >= 1, got {stride!r}")
        if max_new is not None and (isinstance(max_new, bool) or not isinstance(max_new, int) or max_new < 0):
            raise ValueError(f"seedFromDepth: max_new must be an int >= 0 or None, got {max_new!r}")
        if iteration is not None and (isinstance(iteration, bool) or not isinstance(iteration, int)):
            raise ValueError(f"seedFromDepth: iteration must be an int or None, got {iteration!r}")
        cam = _check_cams([cam], "seedFromDepth")[0]
        H, W = int(cam["H"]), int(cam["W"])
        _plane(gt_image, (3, H, W), "seedFromDepth: gt_image")
        _plane(gt_depth, (H, W), "seedFromDepth: gt_depth")
        _plane(mask, (3, H, W), "seedFromDepth: mask")
        if gt_image is None or gt_depth is None:
            raise ValueError("seedFromDepth: gt_image and gt_depth are required")
        m = self.model
        m._check_rows()
        if not hasattr(m, "exp_avg_"):
            raise RuntimeError("seedFromDepth: call trainingSetup() first (the optimizer state is extended together with the parameters)")
        P = m.num_points()
        if max_new is None:
            max_new = max(int(self.opt.cap_max) - P, 0) if self.opt.mcmc else _INT_MAX
        max_new = min(max_new, _INT_MAX)
        it = self.iteration if iteration is None else iteration
        alpha = torch.zeros((H, W), dtype=torch.float32, device=m.device)
        depth = torch.zeros((H, W), dtype=torch.float32, device=m.device)
        if P > 0:     # an empty map is transparent everywhere: A = D = 0 makes every valid grid pixel a hole
            self.render(cam, out_depth=depth, out_alpha=alpha)
        L = self.L
        stream = torch.cuda.current_stream().cuda_stream
        cfg = _SeedCfg(float(alpha_min), float(depth_rel), float(min_depth), float(max_depth), stride, max_new)
        cc = _ccamera(cam)
        ws = torch.empty(L.psb_seed_workspace_bytes(W, H, stride), dtype=torch.uint8, device=m.device)
        counts = (C.c_int * 3)()
        _lib.check(L.psb_seed_plan(C.byref(cc), alpha.data_ptr(), depth.data_ptr(), gt_depth.data_ptr(), mask.data_ptr() if mask is not None else None,
                                   C.byref(cfg), ws.data_ptr(), counts, stream), "psb_seed_plan")
        n = min(counts[0], max_new)
        if n:
            m._out_of_place(P + n, lambda src, dst: L.psb_seed_apply(P, src, dst, n, C.byref(cc), gt_image.data_ptr(), gt_depth.data_ptr(), C.byref(cfg),
                                                                     ws.data_ptr(), int(it), stream), "psb_seed_apply")
        return n, counts[1], counts[2]

    @property
    def antialiasing(self):
        """Whether this trainer's passes use the 2D Mip filter (set at construction)."""
        return self._antialiasing

    @property
    def deterministic(self):
        """Whether the next training call runs in deterministic mode."""
        if self._deterministic is None:
            return torch.are_deterministic_algorithms_enabled()
        return bool(self._deterministic)

    def _apply_deterministic(self):
        want = self.deterministic
        if want != self._det_applied:
            _lib.check(self.L.psb_trainer_set_deterministic(self.h, int(want)), "psb_trainer_set_deterministic")
            self._det_applied = want

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.L.psb_trainer_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def _cstep(self, densify_stats=True):
        m = self.model
        s = _Step()
        for i in range(6):
            s.lr[i] = m.lr_[i]
        s.beta1, s.beta2, s.eps = 0.9, 0.999, 1e-15
        s.step = m.step_ + 1
        s.lambda_dssim = self.opt.lambda_dssim
        s.sh_degree = m.active_sh_degree_
        s.update_densify_stats = int(densify_stats)
        return s

    def render(self, cam, out=None, radii=None, check=True, out_depth=None, out_alpha=None, out_normal=None, out_depth2=None):
        """Forward only. check=True waits for the instance count and renders again if the binning arena had to grow (an
        overflowing render leaves `out` blank); pass check=False to only enqueue (call result() yourself before using `out`).
        out_depth: [H,W] float32 tensor that receives the expected depth sum_i z_i alpha_i T_i; out_alpha: [H,W] float32 tensor that
        receives the accumulated opacity 1 - T_final (psb_trainer_forward); out_normal: [3,H,W] float32 tensor that receives the
        view-space normal plane sum_i n_i alpha_i T_i (psb_trainer_forward_normal; N / |N| is the surface normal); out_depth2: [H,W]
        float32 tensor that receives the second depth moment M = sum_i z_i^2 alpha_i T_i (psb_trainer_forward_moment; with A and D,
        sqrt(max(M / A - (D / A)^2, 0)) is the pixel's depth spread).
        backwardPixels() back-propagates through this render."""
        m = self.model
        H, W = int(cam["H"]), int(cam["W"])
        out = out if out is not None else torch.empty((3, cam["H"], cam["W"]), device=m.device)
        for t in (out_depth, out_alpha):
            assert t is None or (t.is_contiguous() and t.dtype == torch.float32 and t.numel() == cam["H"] * cam["W"])
        _plane(out_normal, (3, H, W), "out_normal")
        _plane(out_depth2, (H, W), "out_depth2")
        self._hand_filter3d()
        cm, cc = m._cmodel(False), _ccamera(cam)
        pass_no = C.c_uint()
        args = (self.h, m.num_points(), 16, C.byref(cm), C.byref(cc), self.background.data_ptr(), m.active_sh_degree_, out.data_ptr(),
                radii.data_ptr() if radii is not None else None, out_depth.data_ptr() if out_depth is not None else None,
                out_alpha.data_ptr() if out_alpha is not None else None)
        if out_depth2 is not None:
            _lib.check(self.L.psb_trainer_forward_moment(*args, out_normal.data_ptr() if out_normal is not None else None, out_depth2.data_ptr(),
                                                         C.byref(pass_no), torch.cuda.current_stream().cuda_stream), "psb_trainer_forward_moment")
        elif out_normal is None:
            _lib.check(self.L.psb_trainer_forward(*args, C.byref(pass_no), torch.cuda.current_stream().cuda_stream), "psb_trainer_forward")
        else:
            _lib.check(self.L.psb_trainer_forward_normal(*args, out_normal.data_ptr(), C.byref(pass_no), torch.cuda.current_stream().cuda_stream),
                       "psb_trainer_forward_normal")
        self._pass = pass_no.value
        self._last_render = (cam, out, radii, out_depth, out_alpha, out_normal, out_depth2)
        self._last = _Call(False, lambda: self.render(cam, out, radii, check=False, out_depth=out_depth, out_alpha=out_alpha, out_normal=out_normal,
                                                      out_depth2=out_depth2), False)
        if check:
            self.result()
        return out

    def backwardPixels(self, dL_dcolor, dL_ddepth=None, dL_dalpha=None, grads=None, densify_stats=None, dL_dnormal=None, dL_ddepth2=None):
        """Back-propagates per-pixel gradients of the caller's loss through the last render() (psb_trainer_backward_pixels).
        dL_dcolor [3,H,W] (required), dL_ddepth / dL_dalpha [H,W] or None: contiguous float32 gradients w.r.t. the image, the depth and
        the accumulated opacity of that render; dL_dnormal [3,H,W] or None: w.r.t. its normal plane (a render with out_normal;
        psb_trainer_backward_pixels_normal); dL_ddepth2 [H,W] or None: w.r.t. its second depth moment (a render with out_depth2;
        psb_trainer_backward_pixels_moment). grads=None: the fused Adam step of trainForOneIteration (advances step_ and iteration);
        grads = six contiguous float32 tensors shaped like the model's parameters: they receive the raw-parameter gradients and the
        parameters stay as they are (for a caller's own optimizer or all-reduce). The model must not change between the render and
        this call. densify_stats as in trainForOneIteration (both modes fold the densification statistics in).
        If the render overflowed the binning arena (render(check=False) not followed by result()), this call is a no-op on the model and
        on `grads`; the next result() then rolls step_ / iteration back and raises: render again, recompute the loss, call again."""
        m = self.model
        if getattr(self, "_last_render", None) is None or getattr(self, "_pass", None) is None:
            raise _lib.PsbError("backwardPixels: no forward pass to back-propagate through; call render() first")
        cam = self._last_render[0]
        H, W = int(cam["H"]), int(cam["W"])
        _plane(dL_dcolor, (3, H, W), "dL_dcolor")
        if dL_dcolor is None:
            raise ValueError("dL_dcolor is required")
        _plane(dL_ddepth, (H, W), "dL_ddepth")
        _plane(dL_dalpha, (H, W), "dL_dalpha")
        _plane(dL_dnormal, (3, H, W), "dL_dnormal")
        if dL_dnormal is not None and (len(self._last_render) < 6 or self._last_render[5] is None):
            raise ValueError("dL_dnormal: the last render() rendered no normal plane (pass out_normal)")
        _plane(dL_ddepth2, (H, W), "dL_ddepth2")
        if dL_ddepth2 is not None and (len(self._last_render) < 7 or self._last_render[6] is None):
            raise ValueError("dL_ddepth2: the last render() rendered no second depth moment (pass out_depth2)")
        if grads is not None:
            grads = list(grads)
            if len(grads) != 6:
                raise ValueError(f"grads: want six tensors (order {GROUPS}), got {len(grads)}")
            for name, g, p in zip(GROUPS, grads, m.tensors()):
                _plane(g, p.shape, "grads[" + name + "]")
        adam = grads is None
        self._hand_filter3d()
        if adam:
            self.iteration += 1
        if densify_stats is None:
            densify_stats = self.iteration < self.opt.densify_until_iter
        cm = m._cmodel(live=m.adamLive()) if adam else m._cmodel()
        cc, cs = _ccamera(cam), self._cstep(densify_stats)
        px = _PixelGrads(dL_dcolor.data_ptr(), dL_ddepth.data_ptr() if dL_ddepth is not None else None,
                         dL_dalpha.data_ptr() if dL_dalpha is not None else None)
        ptrs = None if adam else (C.c_void_p * 6)(*[g.data_ptr() for g in grads])
        head = (self.h, self._pass, m.num_points(), 16, C.byref(cm), C.byref(cc), self.background.data_ptr(), C.byref(px))
        if dL_ddepth2 is not None:
            fn = "psb_trainer_backward_pixels_moment"
            rc = self.L.psb_trainer_backward_pixels_moment(*head, dL_dnormal.data_ptr() if dL_dnormal is not None else None, dL_ddepth2.data_ptr(),
                                                           C.byref(cs), ptrs, torch.cuda.current_stream().cuda_stream)
        elif dL_dnormal is None:
            fn = "psb_trainer_backward_pixels"
            rc = self.L.psb_trainer_backward_pixels(*head, C.byref(cs), ptrs, torch.cuda.current_stream().cuda_stream)
        else:
            fn = "psb_trainer_backward_pixels_normal"
            rc = self.L.psb_trainer_backward_pixels_normal(*head, dL_dnormal.data_ptr(), C.byref(cs), ptrs, torch.cuda.current_stream().cuda_stream)
        if rc < 0 and adam:
            self.iteration -= 1
        _lib.check(rc, fn)
        if adam:
            m.step_ += 1
        self._last = _Call(adam, None, False)     # (trainWithLoss replaces it with its own record)

    def trainWithLoss(self, cam, loss_fn, depth=False, alpha=False, out_color=None, radii=None, densify_stats=None, normal=False, depth2=False):
        """One training iteration against the caller's loss: enqueues the forward (no host synchronisation of its own), calls
        loss = loss_fn(image[, depth][, alpha][, normal][, depth2]) on leaf tensors that require grad (image [3,H,W]; depth [H,W] = sum z
        alpha T with depth=True; alpha [H,W] = 1 - T_final with alpha=True; normal [3,H,W] = sum n alpha T, the view-space normal plane, with
        normal=True; depth2 [H,W] = sum z^2 alpha T, the second depth moment, with depth2=True), takes torch.autograd.grad of the loss w.r.t. those outputs only, and
        back-propagates it through the fused kernels into a fused Adam step (backwardPixels). The model tensors never enter autograd.
        Advances step_ / iteration like trainForOneIteration and returns the (detached) loss tensor; result() repeats the whole call
        if the forward overflowed the binning arena. out_color / radii: optional tensors that receive the image / radii."""
        if not callable(loss_fn):
            raise TypeError("loss_fn must be callable")
        m = self.model
        H, W = int(cam["H"]), int(cam["W"])
        image = out_color if out_color is not None else torch.empty((3, H, W), device=m.device)
        _plane(image, (3, H, W), "out_color")
        D = torch.empty((H, W), device=m.device) if depth else None
        A = torch.empty((H, W), device=m.device) if alpha else None
        N = torch.empty((3, H, W), device=m.device) if normal else None
        M2 = torch.empty((H, W), device=m.device) if depth2 else None
        self._apply_deterministic()
        self.render(cam, image, radii, check=False, out_depth=D, out_alpha=A, out_normal=N, out_depth2=M2)
        outs = [t for t in (image, D, A, N, M2) if t is not None]
        leaves = [t.detach().requires_grad_(True) for t in outs]
        with torch.enable_grad():
            loss = loss_fn(*leaves)
            g = torch.autograd.grad(loss, leaves, allow_unused=True)
        g = iter([None if x is None else x.to(torch.float32).contiguous() for x in g])
        gc = next(g)
        gc = gc if gc is not None else torch.zeros_like(image)
        gd = next(g) if depth else None
        ga = next(g) if alpha else None
        gn = next(g) if normal else None
        gm = next(g) if depth2 else None
        if depth2 and gm is None:
            gm = torch.zeros((H, W), device=m.device)
        self.backwardPixels(gc, gd, ga, densify_stats=densify_stats, dL_dnormal=gn, dL_ddepth2=gm)
        self._inject_noise()
        self._last = _Call(True, lambda: self.trainWithLoss(cam, loss_fn, depth, alpha, out_color, radii, densify_stats, normal, depth2), True)
        self._last_loss = loss.detach()
        return self._last_loss

    def trainForOneIteration(self, cam, gt_image, mask=None, out_color=None, radii=None, densify_stats=None, gt_depth=None, lambda_depth=0.0,
                             out_depth=None, exposure_id=None, gt_normal=None, lambda_normal=0.0, out_normal=None, lambda_dn=0.0, dn_alpha_min=0.5,
                             dn_max_rel_jump=0.05, out_depth_normal=None, lambda_dist=0.0, out_depth2=None):
        """Enqueues render -> loss -> backward -> Adam on the current stream (no host sync).
        gt_depth: [H,W] float32 target depth in metres (<= 0: no measurement) trained with weight lambda_depth (> 0) as an L1 term
        over the valid pixels; out_depth: [H,W] float32 tensor that receives the rendered depth.
        exposure_id: the keyframe id k of gt_image, or None. With an id, the loss compares gt_image with the render through exposure row
        k of the model (applyExposure; the table grows to k + 1 rows if needed) and that row takes one Adam step at
        model.exposure_lr_. out_color stays the raw render; result() reports the compensated loss. One psb_trainer_step_exposure call.
        gt_normal: [3,H,W] float32 view-space unit normals ((0,0,0): no measurement; normals_from_depth) trained with weight lambda_normal
        (> 0) as an L1 term against the rendered normal plane; out_normal: [3,H,W] float32 tensor that receives that plane. With either,
        the call is psb_trainer_step_normal; result_normal() reports the normal L1.
        lambda_dn > 0: the depth-normal consistency term (psb_dn; no sensor needed, so monocular and stereo keyframes can use it) with
        weight lambda_dn: the normal of the rendered depth D / A (where A >= dn_alpha_min; dn_max_rel_jump: the depth-edge rule of
        normals_from_depth) against the rendered normal plane. out_depth_normal: [3,H,W] float32 tensor that receives that depth normal.
        The call is then psb_trainer_step_dn; result_dn() reports the term. lambda_dn = 0 without out_depth_normal makes the call without it.
        lambda_dist > 0: the depth distortion term (psb_dist; no sensor or target needed) with weight lambda_dist: the mean over the (mask's)
        pixels of A M - D^2, which pulls each ray's blending weight onto one depth. out_depth2: [H,W] float32 tensor that receives the second
        depth moment M. The call is then psb_trainer_step_dist; result_dist() reports the term. lambda_dist = 0 without out_depth2 makes
        the call without it."""
        m = self.model
        depth = _cdepth(gt_depth, lambda_depth, out_depth)
        normal = _cnormal(gt_normal, lambda_normal, out_normal, int(cam["H"]), int(cam["W"]))
        dn = _cdn(lambda_dn, dn_alpha_min, dn_max_rel_jump, out_depth_normal, int(cam["H"]), int(cam["W"]))
        dist = _cdist(lambda_dist, out_depth2, int(cam["H"]), int(cam["W"]))
        exposure = None
        if exposure_id is not None:
            k = int(exposure_id)
            if k < 0:
                raise ValueError(f"exposure_id must be >= 0, got {exposure_id}")
            m.ensureExposures(k + 1)
            exposure = _Exposure(m.exposure_[k].data_ptr(), m.exposure_exp_avg_[k].data_ptr(), m.exposure_exp_avg_sq_[k].data_ptr(),
                                 m.exposure_step_[k:].data_ptr(), float(m.exposure_lr_))
        self._hand_filter3d()
        self._apply_deterministic()
        self.iteration += 1
        if densify_stats is None:
            densify_stats = self.iteration < self.opt.densify_until_iter
        cm, cc, cs = m._cmodel(live=m.adamLive()), _ccamera(cam), self._cstep(densify_stats)
        args = (*self._call_args(m, cm, cc, cs, gt_image, mask, out_color, radii), C.byref(depth) if depth is not None else None,
                C.byref(exposure) if exposure is not None else None)
        stream = torch.cuda.current_stream().cuda_stream
        if dist is not None:
            rc = self.L.psb_trainer_step_dist(*args, C.byref(normal) if normal is not None else None, C.byref(dn) if dn is not None else None,
                                              C.byref(dist), stream)
            fn = "psb_trainer_step_dist"
        elif dn is not None:
            rc = self.L.psb_trainer_step_dn(*args, C.byref(normal) if normal is not None else None, C.byref(dn), stream)
            fn = "psb_trainer_step_dn"
        elif normal is not None:
            rc = self.L.psb_trainer_step_normal(*args, C.byref(normal), stream)
            fn = "psb_trainer_step_normal"
        else:
            rc = self.L.psb_trainer_step_exposure(*args, stream)
            fn = "psb_trainer_step_exposure"
        _lib.check(rc, fn)
        m.step_ += 1
        self._inject_noise()
        self._last = _Call(True, lambda: self.trainForOneIteration(cam, gt_image, mask, out_color, radii, densify_stats, gt_depth, lambda_depth,
                                                                   out_depth, exposure_id, gt_normal, lambda_normal, out_normal, lambda_dn,
                                                                   dn_alpha_min, dn_max_rel_jump, out_depth_normal, lambda_dist, out_depth2),
                           False)

    def _call_args(self, m, cm, cc, cs, gt_image, mask, out_color, radii):
        """The leading arguments of a built-in-loss training call (t ... radii)."""
        return (self.h, m.num_points(), 16, C.byref(cm), C.byref(cc), self.background.data_ptr(), gt_image.data_ptr(),
                mask.data_ptr() if mask is not None else None, C.byref(cs), out_color.data_ptr() if out_color is not None else None,
                radii.data_ptr() if radii is not None else None)

    def _overflow_info(self):
        f, n, cur = C.c_uint(), C.c_uint(), C.c_uint()
        self.L.psb_trainer_overflow_info(self.h, C.byref(f), C.byref(n), C.byref(cur))
        return f.value, n.value, cur.value

    def result(self):
        """Blocks; -> (loss, l1, ssim, num_rendered). Transparently repeats the call if the binning arena had to grow for it.
        After trainWithLoss: (the caller's loss, nan, nan, num_rendered).
        The overflow record is sticky on the device: if an EARLIER queued step overflowed (it was a no-op on the model while
        step_ advanced), this raises instead of silently continuing. The loss includes the depth term of a depth step."""
        return self._result(3)

    def result_depth(self):
        """result() with the depth L1 of the last step: -> (loss, l1, ssim, depth_l1, num_rendered); depth_l1 = 0 without a depth target."""
        return self._result(4)

    def result_normal(self):
        """result() with the depth and normal L1 of the last step: -> (loss, l1, ssim, depth_l1, normal_l1, num_rendered); a term the step did
        not have reads 0 (psb_trainer_result_normal)."""
        return self._result(5)

    def result_dn(self):
        """result() with the depth L1, normal L1 and depth-normal consistency of the last step: -> (loss, l1, ssim, depth_l1, normal_l1, dn,
        num_rendered); a term the step did not have reads 0 (psb_trainer_result_dn)."""
        return self._result(6)

    def result_dist(self):
        """result() with the depth L1, normal L1, depth-normal consistency and depth distortion of the last step: -> (loss, l1, ssim,
        depth_l1, normal_l1, dn, dist, num_rendered); a term the step did not have reads 0 (psb_trainer_result_dist)."""
        return self._result(7)

    def _result(self, nterms):
        out, n = (C.c_float * 7)(), C.c_int()
        name = {7: "psb_trainer_result_dist", 6: "psb_trainer_result_dn", 5: "psb_trainer_result_normal"}.get(nterms, "psb_trainer_result_depth")
        result_fn = getattr(self.L, name)
        rc = result_fn(self.h, out, C.byref(n), torch.cuda.current_stream().cuda_stream)
        if rc == -4:
            first, count, cur = self._overflow_info()
            last = self._last
            if not (count == 1 and first == cur):
                if last.advanced:
                    self.model.step_ -= count      # those updates never happened
                    self.iteration -= count
                raise _lib.PsbError(f"{count} queued call(s) (first: pass {first} of {cur}) overflowed the binning arena and were dropped; the arena has "
                                    "been grown. Collect result() after every step, or render() the view once before queueing steps on it.")
            if last.advanced:                      # PSB_ERR_RETRY: the call was a no-op
                self.model.step_ -= 1
                self.iteration -= 1
            if last.repeat is None:
                self._last = _NO_CALL
                raise _lib.PsbError("the render that backwardPixels back-propagated through overflowed the binning arena, so that call was a "
                                    "no-op; the arena has been grown. Render again (with check=True, or collect result() before computing the "
                                    "loss) and repeat the loss and backwardPixels.")
            last.repeat()
            return self._result(nterms)
        _lib.check(rc, name)
        if self._last.callers_loss:
            # the caller's loss: only its value is known (l1, ssim, depth_l1 and normal_l1 are the built-in loss's terms)
            nan = float("nan")
            out = (float(self._last_loss), nan, nan, nan, nan, nan, nan)
        return (*out[:nterms], n.value)

    # ------------------------------------------------------------------------------------------------------------
    # Host-input front end: what the mapper thread does every iteration — `gt_image = original_image_.cuda()`
    # (gaussian_mapper.cpp:637), train, `loss.item()` (:705). The copy of iteration i runs on a side stream while the
    # GPU still works on iteration i-1, and the loss comes back through psb_trainer_result's early read-back event
    # (recorded right behind the loss kernel), so the host enqueues iteration i+1 under the backward half of i.
    # ------------------------------------------------------------------------------------------------------------
    def trainHost(self, host_cam, host_gt, mask=None, host_depth=None, lambda_depth=0.0):
        """host_cam: dict(viewmatrix, projmatrix, campos: pinned CPU tensors; tanfovx, tanfovy, W, H); host_gt: pinned
        [3,H,W] CPU tensor; host_depth: optional pinned [H,W] CPU target depth (metres, <= 0 = none) trained with lambda_depth.
        Enqueues this iteration and returns its loss (the GPU may still be in its backward half; flushHost() waits for it)."""
        dev = self.model.device
        if not hasattr(self, "_hs"):
            self._copy = torch.cuda.Stream()
            mk = lambda t: torch.empty(t.shape, dtype=t.dtype, device=dev)
            self._hs = [dict(gt=mk(host_gt), viewmatrix=mk(host_cam["viewmatrix"]), projmatrix=mk(host_cam["projmatrix"]),
                             campos=mk(host_cam["campos"]), ev=torch.cuda.Event(), done=torch.cuda.Event()) for _ in range(2)]
            self._hslot = 0
        slot = self._hs[self._hslot]
        if host_depth is not None and (slot.get("depth") is None or slot["depth"].shape != host_depth.shape):
            slot["depth"] = torch.empty(host_depth.shape, dtype=host_depth.dtype, device=dev)   # (the slot is free: see "done" below)
        main = torch.cuda.current_stream()
        with torch.cuda.stream(self._copy):
            self._copy.wait_event(slot["done"])           # the iteration that last used this slot has finished reading it
            slot["gt"].copy_(host_gt, non_blocking=True)
            if host_depth is not None:
                slot["depth"].copy_(host_depth, non_blocking=True)
            for k in ("viewmatrix", "projmatrix", "campos"):
                slot[k].copy_(host_cam[k], non_blocking=True)
            slot["ev"].record(self._copy)
        cam = dict(host_cam, viewmatrix=slot["viewmatrix"], projmatrix=slot["projmatrix"], campos=slot["campos"])
        main.wait_event(slot["ev"])
        depth = slot["depth"] if host_depth is not None else None
        self.trainForOneIteration(cam, slot["gt"], mask, gt_depth=depth, lambda_depth=lambda_depth if depth is not None else 0.0)
        loss = self.result()[0]                           # waits for the loss scalars only (repeats the step on RETRY)
        slot["done"].record(main)
        self._hslot ^= 1
        return loss

    def flushHost(self):
        """Waits until every enqueued iteration has finished on the device."""
        torch.cuda.current_stream().synchronize()

    STAGES = ("preprocess", "depth_sort_scan", "binning", "render_fwd", "loss", "render_bwd", "gaussian_backward", "frest_adam")
    DP_STAGES = ("preprocess", "depth_sort_scan", "binning", "render_fwd", "loss", "render_bwd", "push_backward", "wait_grads", "shard_adam", "wait_params",
                 "shard_adam_frest_part")

    def set_profiling(self, enable=True):
        _lib.check(self.L.psb_trainer_set_profiling(self.h, int(enable)), "psb_trainer_set_profiling")

    def stage_times(self):
        """ms per stage of the last profiled step (CUDA events on the step's stream)."""
        ms = (C.c_float * 11)()
        n = _lib.check(self.L.psb_trainer_stage_times(self.h, ms, 11), "psb_trainer_stage_times")
        names = self.DP_STAGES if n >= 10 else self.STAGES
        return dict(zip(names[:n], [float(x) for x in ms][:n]))

    def trainingOnce(self, cam, gt_image, mask=None):
        """Reference-style blocking iteration: returns the loss like loss.item() (gaussian_mapper.cpp:705)."""
        self.trainForOneIteration(cam, gt_image, mask)
        return self.result()[0]


class _DevArray:
    """Zero-copy view of library-owned device memory for torch.as_tensor (CUDA array interface v2)."""

    def __init__(self, ptr, shape):
        self.__cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(ptr), False), "version": 2, "strides": None}


class DataParallelTrainer(GaussianTrainer):
    """Keyframe-sharded data parallelism (SURVEY §8e): replicated Gaussians, rank r renders its own view, K views per
    optimizer step (mean gradient: grad_scale = 1/world keeps the learning-rate scale of one view per step).

    mode="p2p" (default for world > 1): the fused NVLink step of psb_dp_step — the per-Gaussian backward pushes 80-byte
        gradient records straight into the inbox of the rank that owns the Gaussian (chunks of 128, owner = chunk % world),
        the owner applies Adam to its rows only and stores the updated rows into every rank's parameter tensors. No reduced
        gradient in memory, no collective call, optimizer traffic / world. The parameter tensors are re-homed in the
        context's IPC-mapped arena; Adam moments are valid on the owner rank only (gather_moments() before densification
        or a checkpoint).
    mode="nccl": round-1 path kept for A/B — slab-wise backward, one NCCL all-reduce per slab on a side stream, replicated Adam.
    world == 1 and mode=None: backward -> Adam split path on one GPU (tests).
    deterministic: as in GaussianTrainer, kept across rebuild(). "p2p" is then bit-identical run to run at any world size; "nccl"
    gives deterministic per-rank gradients, but the all-reduce's summation order is NCCL's.
    antialiasing: as in GaussianTrainer, in every mode. Every rank must pass the same value.
    geometry_terms=True: trainForOneIteration takes the normal, depth-normal consistency and distortion arguments in every mode
        (psb_dp_step_dist, psb_trainer_backward_begin_dist, psb_trainer_backward_dist); each rank passes its own view's terms or none.
        Off (the default), those arguments raise NotImplementedError, as they always have, and every step makes the calls it made
        before the terms existed.
    exposure=True: trainForOneIteration takes exposure_id in every mode (psb_dp_step_table, psb_trainer_backward_begin_table,
        psb_trainer_backward_table + psb_exposure_apply). Every rank holds a replica of the model's exposure table; each step, every row
        that some rank trained takes one Adam step from the mean of the ranks' gradients (the ranks' own exposure_lr_; the lowest rank's
        where several trained one row), and the replicas stay bit-identical. The table is never grown here: call
        model.ensureExposures(K) on every rank first; K is checked across the ranks when the trainer is built and on rebuild().
        Off (the default), exposure_id raises NotImplementedError as it always has."""

    geometry_terms = False
    exposure = False

    def __init__(self, model, opt=None, background=None, group=None, pipeline=None, nslabs=4, mode=None, deterministic=None,
                 antialiasing=False, filter3d=False, geometry_terms=False, exposure=False):
        if filter3d:
            raise NotImplementedError("DataParallelTrainer: the 3D filter is not wired into the data-parallel steps (the NVLink push backward and "
                                      "the slab pipeline have no filtered variant); train with it on one GPU through GaussianTrainer(filter3d=True)")
        if opt is not None and opt.mcmc:
            raise NotImplementedError("DataParallelTrainer: opt.mcmc is not wired into the data-parallel steps (the owner-side Adam would need the "
                                      "regularisers, every rank the noise, and a refinement gather_moments() first); train with it on one GPU "
                                      "through GaussianTrainer")
        super().__init__(model, opt, background, deterministic=deterministic, antialiasing=antialiasing)
        self.geometry_terms = bool(geometry_terms)
        self.exposure = bool(exposure)
        import os
        import torch.distributed as dist
        self.dist = dist
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.dropped_views = 0
        if mode is None:
            mode = os.environ.get("PSB_DP_MODE") or ("p2p" if self.world > 1 else "nccl")
        self.mode = mode
        self.dp = None
        if self.mode == "p2p":
            try:
                self._setup_p2p()
                ok = 1
            except _lib.PsbError as e:
                self._p2p_error = str(e)
                ok = 0
            if self.world > 1:   # every rank must take the same path
                t = torch.tensor([ok], device=model.device, dtype=torch.int32)
                dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
                ok = int(t.item())
            if not ok:
                import warnings
                warnings.warn("psb200: NVLink peer mapping unavailable (%s); falling back to the NCCL all-reduce path" % getattr(self, "_p2p_error", "a peer failed"))
                self._teardown_p2p()
                self.mode = "nccl"
        if self.mode == "nccl":
            self._setup_nccl(pipeline, nslabs)
        self._check_exposures()

    def _check_exposures(self):
        """exposure=True: every rank's table must have the same number of rows (a row id means the same keyframe on every rank)."""
        if not self.exposure:
            return
        K = self.model.numExposures()
        if self.world > 1:
            t = torch.tensor([K, -K], device=self.model.device, dtype=torch.int64)
            self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX, group=self.group)
            if int(t[0]) != -int(t[1]):
                raise ValueError(f"DataParallelTrainer: the ranks' exposure tables differ in size (from {-int(t[1])} to {int(t[0])} rows): call "
                                 "model.ensureExposures(K) with the same K on every rank")
        self._exp_K = K
        dev = self.model.device
        self._exp_rec = torch.zeros(EXPOSURE_RECORD, device=dev)                       # this rank's record (slab and flat paths)
        self._exp_recs = torch.zeros(self.world, EXPOSURE_RECORD, device=dev)          # every rank's, gathered

    # ---- p2p -----------------------------------------------------------------------------------------------------------
    def _setup_p2p(self):
        m, L = self.model, self.L
        P = m.num_points()
        h = C.c_void_p()
        _lib.check(L.psb_dp_create(C.byref(h), self.rank, self.world, P), "psb_dp_create")
        self.dp = h
        self._dp_P = P
        nb = L.psb_dp_handle_bytes()
        if self.world > 1:
            mine = (C.c_char * nb)()
            _lib.check(L.psb_dp_ipc_handle(h, mine), "psb_dp_ipc_handle")
            blobs = [None] * self.world
            self.dist.all_gather_object(blobs, bytes(mine), group=self.group)
            allb = (C.c_char * (nb * self.world)).from_buffer_copy(b"".join(blobs))
            _lib.check(L.psb_dp_connect(h, allb), "psb_dp_connect")
        else:
            _lib.check(L.psb_dp_connect(h, None), "psb_dp_connect")
        ptrs = (C.c_void_p * 6)()
        _lib.check(L.psb_dp_params(h, ptrs), "psb_dp_params")
        homed = []
        for ptr, shp, src in zip(ptrs, row_shapes(P), m.tensors()):
            t = torch.as_tensor(_DevArray(ptr, shp), device=m.device) if P > 0 else torch.empty(shp, device=m.device)
            t.copy_(src)
            homed.append(t)
        self._homed = homed
        m._set(homed)
        torch.cuda.synchronize()
        if self.world > 1:
            self.dist.barrier(group=self.group)   # nobody pushes into an arena that is still being filled

    def _teardown_p2p(self):
        if self.dp is not None:
            m = self.model
            torch.cuda.synchronize()
            if self.world > 1:
                self.dist.barrier(group=self.group)
            if getattr(self, "_homed", None) is not None and m.tensors()[0] is self._homed[0]:
                m._set([t.clone() for t in m.tensors()])   # the arena is about to disappear
            self._homed = None
            self.L.psb_dp_destroy(self.dp)
            self.dp = None

    def close(self):
        self._teardown_p2p()

    def owner_mask(self):
        """bool [P]: rows whose Adam moments live on this rank (chunks of 128 Gaussians, owner = chunk % world)."""
        from .parallel import owner_of_rows
        return owner_of_rows(self.model.num_points(), self.world, self.model.device) == self.rank

    def sync(self):
        """Device-side wait until every rank's updated rows of the last step have landed in this rank's tensors."""
        if self.mode == "p2p":
            _lib.check(self.L.psb_dp_sync(self.dp, torch.cuda.current_stream().cuda_stream), "psb_dp_sync")

    def status(self):
        return self.L.psb_dp_status(self.dp, torch.cuda.current_stream().cuda_stream) if self.mode == "p2p" else 0

    def render(self, cam, out=None, radii=None, check=True, out_depth=None, out_alpha=None, out_normal=None, out_depth2=None):
        """Forward only, on the complete replica: the peers store their rows of the last step asynchronously, so the render is
        ordered behind every rank's rows (device-side wait)."""
        self.sync()
        return super().render(cam, out, radii, check, out_depth, out_alpha, out_normal, out_depth2)

    def contributionScores(self, cams):
        """As in GaussianTrainer, on the complete replica (ordered behind every rank's rows, like render)."""
        self.sync()
        return super().contributionScores(cams)

    def pruneByContribution(self, cams, min_weight, keep=None, min_age=0):
        raise NotImplementedError("DataParallelTrainer.pruneByContribution: pruning is not wired into the data-parallel steps (in p2p mode the "
                                  "parameters live in the IPC arena, and every rank would need the same mask: an exact all-reduce of the "
                                  "integer scores, then rebuild()); score with contributionScores and prune on one GPU through GaussianTrainer")

    def seedFromDepth(self, *args, **kwargs):
        raise NotImplementedError("DataParallelTrainer.seedFromDepth: each rank trains its own keyframe, so rows seeded from it would exist on "
                                  "one replica only and the replicas would diverge; seed on one GPU through GaussianTrainer, then rebuild()")

    def gather_moments(self):
        """Every rank receives the Adam moments of all rows (they are only maintained on the owner): call before
        densify/prune (which moves rows, hence owners) or before writing a checkpoint."""
        if self.mode != "p2p" or self.world == 1:
            return
        from .parallel import gather_owned_rows
        self.sync()
        m = self.model
        gather_owned_rows(m.exp_avg_ + m.exp_avg_sq_, self.rank, self.world, self.group)
        m.invalidateAdamLive()

    def rebuild(self):
        """After the model was resized (densify / prune / insertion): new arena, new peer mappings."""
        if self.mode == "p2p":
            self._teardown_p2p()
            self._setup_p2p()
        else:
            self._setup_nccl(self.pipeline, len(self.grads.slabs) if self.pipeline else 4)
        self._check_exposures()

    def _exposure_table(self, exposure_id):
        """The psb_exposure_table of this rank's step (id -1 without exposure_id)."""
        m = self.model
        K = m.numExposures()
        if K != self._exp_K:
            raise ValueError(f"DataParallelTrainer: the exposure table has {K} rows, the trainer checked {self._exp_K} across the ranks: after "
                             "model.ensureExposures(K) on every rank, call rebuild()")
        k = -1
        if exposure_id is not None:
            k = int(exposure_id)
            if k < 0 or k >= K:
                raise ValueError(f"exposure_id must lie in [0, {K}), got {exposure_id}: the data-parallel table is not grown on demand; call "
                                 "model.ensureExposures(K) on every rank first")
        return _ExposureTable(m.exposure_.data_ptr(), m.exposure_exp_avg_.data_ptr(), m.exposure_exp_avg_sq_.data_ptr(), m.exposure_step_.data_ptr(),
                              K, k, float(m.exposure_lr_), self._exp_rec.data_ptr())

    def _apply_exposures(self, table, cs, stream):
        """Slab and flat paths: every rank's record (one all-gather of world x 16 floats) -> the same table update on every rank."""
        recs = self._exp_rec
        if self.world > 1:
            self.dist.all_gather_into_tensor(self._exp_recs, self._exp_rec, group=self.group)
            recs = self._exp_recs
        _lib.check(self.L.psb_exposure_apply(self.world, recs.data_ptr(), C.byref(table), C.byref(cs), 1.0 / self.world, stream), "psb_exposure_apply")

    # ---- nccl (round-1 path) -------------------------------------------------------------------------------------------
    def _setup_nccl(self, pipeline, nslabs):
        from .parallel import GradBuffer, SlabGradBuffer
        model = self.model
        self.pipeline = (self.world > 1) if pipeline is None else bool(pipeline)
        P = model.num_points()
        if self.pipeline:
            self.grads = SlabGradBuffer(P, model.device, nslabs)
            self._comm = torch.cuda.Stream()
            n = len(self.grads.slabs)
            self._ev_k = [torch.cuda.Event() for _ in range(n)]
            self._ev_c = [torch.cuda.Event() for _ in range(n)]
        else:
            self.grads = GradBuffer(P, model.device)
            self.segs = self.grads.segments
        self.flat = self.grads.flat

    def trainForOneIteration(self, cam, gt_image, mask=None, out_color=None, radii=None, densify_stats=None, gt_depth=None, lambda_depth=0.0,
                             out_depth=None, exposure_id=None, gt_normal=None, lambda_normal=0.0, out_normal=None, lambda_dn=0.0, dn_alpha_min=0.5,
                             dn_max_rel_jump=0.05, out_depth_normal=None, lambda_dist=0.0, out_depth2=None):
        """Depth arguments as in GaussianTrainer, on every path: "p2p" (psb_dp_step_depth), the slab pipeline
        (psb_trainer_backward_begin_depth) and the flat "nccl" path (psb_trainer_backward_depth). With geometry_terms=True also the normal,
        depth-normal consistency and distortion arguments, on every path: "p2p" (psb_dp_step_dist), the slab pipeline
        (psb_trainer_backward_begin_dist) and the flat "nccl" path (psb_trainer_backward_dist). Each rank passes its own view's terms or
        none: ranks with different terms may train in the same step. exposure_id needs exposure=True (psb_dp_step_table,
        psb_trainer_backward_begin_table, psb_trainer_backward_table): the keyframe id k of gt_image, < model.numExposures(), or None for
        a view without exposure; the row trains as in GaussianTrainer, from the mean of every rank's gradient."""
        if not self.geometry_terms:
            how = "; construct DataParallelTrainer(..., geometry_terms=True) to train it on the data-parallel steps"
            if gt_normal is not None or out_normal is not None or lambda_normal:
                raise NotImplementedError("DataParallelTrainer: the normal term is off on this trainer" + how)
            if lambda_dn or out_depth_normal is not None:
                raise NotImplementedError("DataParallelTrainer: the depth-normal consistency term is off on this trainer" + how)
            if lambda_dist or out_depth2 is not None:
                raise NotImplementedError("DataParallelTrainer: the depth distortion term is off on this trainer" + how)
        if exposure_id is not None and not self.exposure:
            raise NotImplementedError("DataParallelTrainer: exposure compensation is off on this trainer: the per-keyframe exposure table is "
                                      "replicated across the ranks only with DataParallelTrainer(..., exposure=True) (or train with exposure "
                                      "on one GPU through GaussianTrainer)")
        m = self.model
        built = self._dp_P if self.mode == "p2p" else self.grads.P
        if built != m.num_points():
            raise ValueError(f"DataParallelTrainer: the model has {m.num_points()} rows, the trainer was built for {built}: call rebuild() "
                             "after densify, prune or insertion")
        H, W = int(cam["H"]), int(cam["W"])
        depth = _cdepth(gt_depth, lambda_depth, out_depth)
        normal = _cnormal(gt_normal, lambda_normal, out_normal, H, W)
        dn = _cdn(lambda_dn, dn_alpha_min, dn_max_rel_jump, out_depth_normal, H, W)
        dist = _cdist(lambda_dist, out_depth2, H, W)
        table = self._exposure_table(exposure_id) if self.exposure else None
        self._apply_deterministic()
        self.iteration += 1
        if densify_stats is None:
            densify_stats = self.iteration < self.opt.densify_until_iter
        cm, cc, cs = m._cmodel(), _ccamera(cam), self._cstep(densify_stats)
        main = torch.cuda.current_stream()
        stream = main.cuda_stream
        P = m.num_points()
        args = self._call_args(m, cm, cc, cs, gt_image, mask, out_color, radii)
        byref = lambda x: C.byref(x) if x is not None else None
        cdepth = byref(depth)
        terms = (byref(normal), byref(dn), byref(dist))
        geo = self.geometry_terms
        if self.mode == "p2p":
            if table is not None:
                _lib.check(self.L.psb_dp_step_table(self.h, self.dp, *args[1:], cdepth, *terms, C.byref(table), stream), "psb_dp_step_table")
            elif geo:
                _lib.check(self.L.psb_dp_step_dist(self.h, self.dp, *args[1:], cdepth, *terms, stream), "psb_dp_step_dist")
            else:
                _lib.check(self.L.psb_dp_step_depth(self.h, self.dp, *args[1:], cdepth, stream), "psb_dp_step_depth")
        elif not self.pipeline:
            ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in self.segs])
            if table is not None:
                _lib.check(self.L.psb_trainer_backward_table(*args, ptrs, cdepth, *terms, C.byref(table), stream), "psb_trainer_backward_table")
            elif geo:
                _lib.check(self.L.psb_trainer_backward_dist(*args, ptrs, cdepth, None, None, *terms, stream), "psb_trainer_backward_dist")
            else:
                _lib.check(self.L.psb_trainer_backward_depth(*args, ptrs, cdepth, stream), "psb_trainer_backward_depth")
            scale = self.grads.all_reduce(self.group)   # ONE collective per step: 59 floats per Gaussian
            _lib.check(self.L.psb_adam_update(P, 16, C.byref(cm), ptrs, C.byref(cs), scale, stream), "psb_adam_update")
            if table is not None:
                self._apply_exposures(table, cs, stream)
        else:
            if table is not None:
                _lib.check(self.L.psb_trainer_backward_begin_table(*args, cdepth, *terms, C.byref(table), stream), "psb_trainer_backward_begin_table")
            elif geo:
                _lib.check(self.L.psb_trainer_backward_begin_dist(*args, cdepth, *terms, stream), "psb_trainer_backward_begin_dist")
            else:
                _lib.check(self.L.psb_trainer_backward_begin_depth(*args, cdepth, stream), "psb_trainer_backward_begin_depth")
            scale = 1.0 / self.world
            for s, (first, count) in enumerate(self.grads.slabs):
                ptrs = (C.c_void_p * 6)(*self.grads.kernel_pointers(s))
                _lib.check(self.L.psb_trainer_backward_slab(self.h, P, 16, C.byref(cm), C.byref(cc), C.byref(cs), first, count, ptrs, stream),
                           "psb_trainer_backward_slab")
                if self.world > 1:
                    self._ev_k[s].record(main)
                    with torch.cuda.stream(self._comm):
                        self._comm.wait_event(self._ev_k[s])
                        self.dist.all_reduce(self.grads.region(s), op=self.dist.ReduceOp.SUM, group=self.group)
                        self._ev_c[s].record(self._comm)
            for s, (first, count) in enumerate(self.grads.slabs):
                if self.world > 1:
                    main.wait_event(self._ev_c[s])
                for i, (blk, k) in enumerate(zip(self.grads.blocks(s), SIZES)):
                    p, a, b = m.tensors()[i].view(-1), m.exp_avg_[i].view(-1), m.exp_avg_sq_[i].view(-1)
                    o = first * k
                    _lib.check(self.L.psb_adam_flat(count * k, p[o:].data_ptr(), a[o:].data_ptr(), b[o:].data_ptr(), blk.data_ptr(), m.lr_[i],
                                                    C.byref(cs), scale, stream), "psb_adam_flat")
            if table is not None:
                self._apply_exposures(table, cs, stream)
        m.step_ += 1
        m.invalidateAdamLive()   # these steps write moments without maintaining the live bytes (and p2p: only on the owner rank)

    def result(self):
        """-> (loss, l1, ssim, num_rendered) of this rank's view. A view whose binning arena overflowed contributed a zero
        gradient to the step (every rank still stepped, replicas identical); it is counted in `dropped_views`, the arena
        has been grown, and the step is NOT repeated (a one-rank retry would desynchronise the group). result_depth(),
        result_normal(), result_dn() and result_dist() add this rank's terms as GaussianTrainer's do; every term is NaN for a
        dropped view."""
        return self._result(3)

    def _result(self, nterms):
        out, n = (C.c_float * 7)(), C.c_int()
        rc = self.L.psb_trainer_result_dist(self.h, out, C.byref(n), torch.cuda.current_stream().cuda_stream)
        if rc == -4:
            self.dropped_views += 1
            out = (float("nan"),) * 7
        else:
            _lib.check(rc, "psb_trainer_result_dist")
        return (*out[:nterms], n.value)

    def trainWithLoss(self, *args, **kwargs):
        raise NotImplementedError("DataParallelTrainer.trainWithLoss: a caller's loss is not wired into the data-parallel steps (the "
                                  "fused Adam of one rank would desynchronise the replicas); use GaussianTrainer.trainWithLoss on one GPU, or "
                                  "render() + backwardPixels(..., grads=...) + your own all-reduce + psb_adam_update")

    def backwardPixels(self, dL_dcolor, dL_ddepth=None, dL_dalpha=None, grads=None, densify_stats=None, dL_dnormal=None, dL_ddepth2=None):
        """Gradient mode only (grads= required): a one-rank Adam step would desynchronise the replicas."""
        if grads is None:
            raise NotImplementedError("DataParallelTrainer.backwardPixels: pass grads= (the gradient mode); a one-rank Adam step would "
                                      "desynchronise the replicas")
        return super().backwardPixels(dL_dcolor, dL_ddepth, dL_dalpha, grads=grads, densify_stats=densify_stats, dL_dnormal=dL_dnormal,
                                      dL_ddepth2=dL_ddepth2)

    def sync_densify_stats(self):
        """Reduce the rank-local densification statistics (call right before densify/prune)."""
        from .parallel import reduce_densify_stats
        m = self.model
        reduce_densify_stats(m.max_radii2D_, m.xyz_gradient_accum_, m.denom_, self.group)


def normals_from_depth(cam, depth, max_rel_jump=0.05, out=None):
    """View-space unit normals [3,H,W] of a depth image [H,W] (metres; <= 0 or not finite: no measurement) seen by `cam` (psb_depth_normals):
    central differences of the back-projected neighbours, (0,0,0) on the border, at holes and across depth edges (a neighbour more than
    max_rel_jump z away). The target of trainForOneIteration(gt_normal=...): compute it once per keyframe and pyramid level."""
    H, W = int(cam["H"]), int(cam["W"])
    _plane(depth, (H, W), "depth")
    if depth is None:
        raise ValueError("depth is required")
    out = out if out is not None else torch.empty((3, H, W), device=depth.device)
    _plane(out, (3, H, W), "out")
    if not (math.isfinite(max_rel_jump) and max_rel_jump > 0):
        raise ValueError(f"max_rel_jump must be finite and positive, got {max_rel_jump}")
    c = _Camera()
    c.tan_fovx, c.tan_fovy, c.width, c.height = float(cam["tanfovx"]), float(cam["tanfovy"]), W, H
    L = _bind()
    _lib.check(L.psb_depth_normals(C.byref(c), depth.data_ptr(), float(max_rel_jump), out.data_ptr(), torch.cuda.current_stream().cuda_stream),
               "psb_depth_normals")
    return out


def _dn_loss(cam, depth, alpha, normal, mask=None, lambda_dn=1.0, alpha_min=0.5, max_rel_jump=0.05, grads=None, out_depth_normal=None):
    """The depth-normal consistency term on caller planes through psb_dn_loss (synchronises): depth, alpha [H,W], normal [3,H,W] and mask
    [H,W] or None seen by `cam`. grads = (dL_ddepth, dL_dalpha, dL_dnormal) are added into (zeros when None); out_depth_normal [3,H,W]
    receives n_d. -> (dn, N_valid, grads)."""
    H, W = int(cam["H"]), int(cam["W"])
    for t, shape, name in ((depth, (H, W), "depth"), (alpha, (H, W), "alpha"), (normal, (3, H, W), "normal"), (mask, (H, W), "mask"),
                           (out_depth_normal, (3, H, W), "out_depth_normal")):
        _plane(t, shape, name)
    if grads is None:
        grads = (torch.zeros_like(depth), torch.zeros_like(alpha), torch.zeros_like(normal))
    for t, shape, name in zip(grads, ((H, W), (H, W), (3, H, W)), ("dL_ddepth", "dL_dalpha", "dL_dnormal")):
        _plane(t, shape, name)
    c = _Camera()
    c.tan_fovx, c.tan_fovy, c.width, c.height = float(cam["tanfovx"]), float(cam["tanfovy"]), W, H
    dn = _cdn(lambda_dn, alpha_min, max_rel_jump, out_depth_normal, H, W)
    out = (C.c_float * 2)()
    L = _bind()
    _lib.check(L.psb_dn_loss(C.byref(c), depth.data_ptr(), alpha.data_ptr(), normal.data_ptr(), mask.data_ptr() if mask is not None else None,
                             C.byref(dn), *(g.data_ptr() for g in grads), out, torch.cuda.current_stream().cuda_stream), "psb_dn_loss")
    return float(out[0]), int(out[1]), grads


def fused_loss(image, gt, mask=None, lambda_dssim=0.2, want_grad=True):
    """-> (loss, l1, ssim, dL_dimage or None) through psb_loss."""
    L = _bind()
    _, H, W = image.shape
    grad = torch.empty_like(image) if want_grad else None
    out = (C.c_float * 3)()
    _lib.check(L.psb_loss(H, W, image.contiguous().data_ptr(), gt.contiguous().data_ptr(), mask.data_ptr() if mask is not None else None,
                          float(lambda_dssim), grad.data_ptr() if want_grad else None, out, torch.cuda.current_stream().cuda_stream), "psb_loss")
    return out[0], out[1], out[2], grad
