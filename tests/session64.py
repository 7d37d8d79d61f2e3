"""The float64 truth of a training session: step64's step between the row operations of a Photo-SLAM mapper (densify, prune, insert,
seed, relocate, grow, opacity reset, loop-closure transform, 3D filter) and the session facts the mapper changes between steps (the xyz
learning-rate schedule, the learning-rate setters, the SH degree, the 3D filter in force).

A thin composition: the step is step64.step64, and each row operation is its existing restatement (oracle/ref_densify.py, mcmc64, seed64,
filter3d64) or a closed form. Row states are dicts p / m / v (lists of six float64 tensors in step64.GROUPS order), accum [P,1], denom [P,1],
max_radii [P]. `Session` holds the facts the truth decides itself; the rows it steps are read from the kernels' model before every step
(anchored), so errors do not compound.

Conventions the perturbation tests alter live in `SessionConv`."""
import dataclasses
import math

import numpy as np
import torch

import mcmc64
import ref_densify
import seed64
import step64

SH_C0 = 0.28209479177387814


@dataclasses.dataclass(frozen=True)
class SessionConv:
    new_moments_zero: bool = True      # rows a surgery creates start Adam from zero (False: they inherit their parent's moments)
    lr_schedule: bool = True           # updateLearningRate moves the xyz lr along exponLrFunc (False: held at lr_init)
    filter_current: bool = True        # computeFilter3D after a surgery puts the filter of the new rows in force (False: the old one stays)
    sh_raise: bool = True              # setShDegree takes effect (False: the degree stays where it was)


SESSION_CONV = SessionConv()


def expon_lr(step, lr_init, lr_final, delay_mult, max_steps, delay_steps=0):
    """The xyz learning rate at `step` (graphdeco's get_expon_lr_func): log-linear from lr_init to lr_final over max_steps, scaled by
    the delay ramp delay_mult + (1 - delay_mult) sin(pi/2 min(step / delay_steps, 1)) while delay_steps > 0."""
    if step < 0 or (lr_init == 0.0 and lr_final == 0.0):
        return 0.0
    delay = 1.0
    if delay_steps > 0:
        delay = delay_mult + (1.0 - delay_mult) * math.sin(0.5 * math.pi * min(max(step / delay_steps, 0.0), 1.0))
    t = min(max(step / max_steps, 0.0), 1.0)
    return delay * math.exp(math.log(lr_init) * (1.0 - t) + math.log(lr_final) * t)


class Session:
    """The facts of a session the truth keeps: the six learning rates (f_rest at feature_lr / 20), the active SH degree and the 3D filter
    in force. opt: GaussianOptimizationParams (spatial scale 1)."""

    def __init__(self, opt, D, conv=SESSION_CONV):
        self.opt, self.conv, self.D, self.f = opt, conv, D, None
        self.lr = [opt.position_lr_init, opt.feature_lr, opt.feature_lr / 20.0, opt.opacity_lr, opt.scaling_lr, opt.rotation_lr]

    def update_lr(self, step):
        o = self.opt
        self.lr[0] = expon_lr(step, o.position_lr_init, o.position_lr_final, o.position_lr_delay_mult, o.position_lr_max_steps) \
            if self.conv.lr_schedule else o.position_lr_init
        return self.lr[0]

    def set_lr(self, group, lr):
        """group in step64.GROUPS; "features_dc" sets f_rest to lr / 20 as well"""
        i = step64.GROUPS.index(group)
        self.lr[i] = lr
        if group == "features_dc":
            self.lr[2] = lr / 20.0

    def set_sh(self, D):
        if self.conv.sh_raise:
            self.D = D

    def set_filter(self, f):
        """f [P] float64: the filter computeFilter3D made for the current rows; the perturbed truth keeps its old one where it still fits"""
        if self.conv.filter_current or self.f is None or self.f.shape != f.shape:
            self.f = f

    def state(self, st):
        """a state read from the kernels' model, with the facts this session decides"""
        return dict(st, lr=list(self.lr), D=self.D, f=self.f if st.get("f") is not None else None)

    def step(self, st, cam, targets, flags, conv=step64.STEP_CONV):
        return step64.step64(self.state(st), cam, targets, flags, conv)


# ---- row states ---------------------------------------------------------------------------------------------------------------------
def rows_of(st):
    """step64's state -> a row state (float64 copies)"""
    c = lambda d: [d[k].clone() for k in step64.GROUPS]
    return dict(p=c(st["params"]), m=c(st["m"]), v=c(st["v"]), accum=st["accum"].clone(), denom=st["denom"].clone(), max_radii=st["max_radii"].clone())


def _zero_stats(r):
    P, like = r["p"][0].shape[0], r["p"][0]
    r["accum"], r["denom"] = torch.zeros((P, 1), dtype=like.dtype, device=like.device), torch.zeros((P, 1), dtype=like.dtype, device=like.device)
    r["max_radii"] = torch.zeros(P, dtype=like.dtype, device=like.device)


def _inherit(r, new, parents, conv):
    """the perturbed convention: rows `new` take the moments of rows `parents` of the pre-surgery state r0 (m0, v0)"""
    if conv.new_moments_zero:
        return
    for q in range(6):
        r["m"][q][new] = r["m0"][q][parents]
        r["v"][q][new] = r["v0"][q][parents]


def densify(r, samples, max_grad, min_opacity, extent, max_screen_size, percent_dense, conv=SESSION_CONV):
    """densifyAndPrune with the injected normal draw: ref_densify on float64 tensors. -> (row state, parents [P_new] int64: the
    pre-surgery row each output row comes from, K0: the number of kept originals; rows K0: are new)."""
    P = r["p"][0].shape[0]
    g = (r["accum"] / r["denom"]).nan_to_num(0.0).reshape(-1)
    big = torch.exp(r["p"][4]).max(dim=1).values > percent_dense * extent
    clone = torch.nonzero((g >= max_grad) & ~big).reshape(-1)
    split = torch.nonzero((g >= max_grad) & big).reshape(-1)
    st = dict(p=[t.clone() for t in r["p"]], m=[t.clone() for t in r["m"]], v=[t.clone() for t in r["v"]], accum=r["accum"].clone(),
              denom=r["denom"].clone(), max_radii=r["max_radii"].clone())
    ref_densify.densify_and_prune(st, max_grad, min_opacity, extent, max_screen_size, percent_dense, samples)
    keep = torch.ones(P, dtype=torch.bool, device=g.device)
    keep[split] = False
    parents = torch.cat([torch.nonzero(keep).reshape(-1), clone, split, split])
    assert parents.numel() == st["p"][0].shape[0], "densify(): min_opacity / max_screen_size pruned rows; the parent map covers none"
    K0 = int(keep.sum())
    st["m0"], st["v0"] = r["m"], r["v"]
    _inherit(st, torch.arange(K0, parents.numel(), device=g.device), parents[K0:], conv)
    del st["m0"], st["v0"]
    return st, parents, K0


def prune(r, mask):
    """prunePoints: the kept rows in order, statistics compacted (ref_densify.prune_points)"""
    st = dict(p=list(r["p"]), m=list(r["m"]), v=list(r["v"]), accum=r["accum"], denom=r["denom"], max_radii=r["max_radii"])
    ref_densify.prune_points(st, mask)
    return st


def knn_mean_dist2(pts):
    """the mean squared distance of every point to its three nearest other points, by brute force in float64"""
    pts = torch.as_tensor(pts, dtype=torch.float64)
    d2 = ((pts[:, None, :] - pts[None, :, :]) ** 2).sum(-1)
    d2.fill_diagonal_(math.inf)
    return torch.topk(d2, 3, dim=1, largest=False).values.mean(1)


def insert(r, xyz, features_dc, dist2):
    """The insert row recipe (increasePcd, seedFromDepth) appended to r: features_rest 0, opacity logit(0.1), scaling log sqrt(max(dist2,
    1e-7)) on every axis, identity rotation, zero moments; the statistics of every row reset."""
    n, like = xyz.shape[0], r["p"][0]
    f = lambda t: torch.as_tensor(t, dtype=like.dtype).to(like.device)
    scale = torch.log(torch.sqrt(f(dist2).clamp_min(1e-7)))[:, None].repeat(1, 3)
    rot = torch.zeros((n, 4), dtype=like.dtype, device=like.device)
    rot[:, 0] = 1.0
    new = [f(xyz), f(features_dc).reshape(n, 1, 3), torch.zeros((n, 15, 3), dtype=like.dtype, device=like.device),
           torch.full((n, 1), math.log(0.1 / 0.9), dtype=like.dtype, device=like.device), scale, rot]
    out = dict(p=[torch.cat([a, b]) for a, b in zip(r["p"], new)], m=[torch.cat([a, torch.zeros_like(b)]) for a, b in zip(r["m"], new)],
               v=[torch.cat([a, torch.zeros_like(b)]) for a, b in zip(r["v"], new)])
    _zero_stats(out)
    return out


def insert_points(r, points, colors):
    """increasePcd: new rows from sparse points and their colours in [0, 1], scale from the points' own 3-NN"""
    pts = torch.as_tensor(points, dtype=torch.float64)
    return insert(r, pts, (torch.as_tensor(colors, dtype=torch.float64) - 0.5) / SH_C0, knn_mean_dist2(pts))


def seed_rows(r, plan):
    """seedFromDepth: seed64.seed's plan appended with the insert recipe"""
    return insert(r, plan["xyz"], plan["features_dc"], plan["dist2"])


def reset_opacity(r):
    """resetOpacity: logit(min(sigmoid(o), 1)) and fresh opacity moments (ref_densify.reset_opacity)"""
    st = dict(r, p=list(r["p"]), m=list(r["m"]), v=list(r["v"]))
    return ref_densify.reset_opacity(st)


def transform(r, s, T):
    """applyScaledTransformation: xyz <- R (s xyz) + t, log-scales times s, fresh xyz and scaling moments. T: [4,4] row-major."""
    T = torch.as_tensor(np.asarray(T, np.float64)).to(r["p"][0].device)
    p, m, v = list(r["p"]), list(r["m"]), list(r["v"])
    p[0] = (s * p[0]) @ T[:3, :3].T + T[:3, 3]
    p[4] = p[4] * s
    for q in (0, 4):
        m[q], v[q] = torch.zeros_like(p[q]), torch.zeros_like(p[q])
    return dict(r, p=p, m=m, v=v)


def relocate(model, u, min_opacity, iteration, conv=SESSION_CONV):
    """relocateGaussians with injected uniforms: mcmc64.relocate on a host model (mcmc64's format) -> (model, picks, dead)"""
    want, picks, dead, _ = mcmc64.relocate(model, u, min_opacity, iteration)
    _inherit_np(want, model, dead, picks, conv)
    return want, picks, dead


def grow(model, P_new, u, min_opacity, iteration, conv=SESSION_CONV):
    """addNewGaussians with injected uniforms: mcmc64.grow -> (model, picks); the new rows are P: P_new"""
    want, picks, _ = mcmc64.grow(model, P_new, u, min_opacity, iteration)
    _inherit_np(want, model, np.arange(model["p"][0].shape[0], P_new), picks, conv)
    return want, picks


def _inherit_np(want, before, new, parents, conv):
    if conv.new_moments_zero:
        return
    for q in range(6):
        want["m"][q][new] = before["m"][q][parents]
        want["v"][q][new] = before["v"][q][parents]
