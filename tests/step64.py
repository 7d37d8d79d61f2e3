"""A float64 restatement of one whole training iteration of the fused step (include/psb200.h): the forward with the 3D filter, the
anti-aliasing factor and the normal plane, the built-in loss with exposure, depth and normal terms, the 3DGS-MCMC regularisers, the
densification statistics and the Adam update of every parameter, its moments and the exposure row. The arbiter the per-Gaussian stage
(gaussian_backward_kernel<MODE> and frest_stream_kernel) is measured against, in every flag set and base.

Plain torch, differentiable with autograd, on any device. Built on splat64 (render, loss) and normal64 (per-Gaussian normals, normal L1)
without changing their behaviour (normal64.gaussian_normals takes flip=False for the perturbed truth). Decisions this module adds (the normal's axis and flip, the kinks of the depth and normal L1) are constants of the
pass; `margins` reports how far each lies from its threshold, next to splat64.margins'.

Conventions the perturbation tests alter live in `StepConv`.
"""
import dataclasses
import math

import torch

import normal64 as n64
import splat64 as s64

BETA1, BETA2, EPS = 0.9, 0.999, 1e-15     # psb_step beta1 / beta2 / eps as the trainer sets them (trainer._cstep)
GROUPS = s64.RAW


@dataclasses.dataclass(frozen=True)
class StepConv:
    eps: float = EPS                   # Adam's epsilon
    bias_correction: bool = True       # lr / (1 - beta1^t) and sqrt(v) / sqrt(1 - beta2^t)
    mean2d_ndc: bool = True            # xyz_gradient_accum sums |dL/dmean2D| in NDC units: dL/dpixel * (W/2, H/2) (psb_render.cu ddelx_dx)
    reg_reached_only: bool = True      # the regularisers act on the rows the pass reaches, not on all P rows
    f3d_opacity: bool = True           # the 3D filter multiplies the opacity by c
    normal_flip: bool = True           # the normal faces the camera (n = -m when m . t > 0)


STEP_CONV = StepConv()


@dataclasses.dataclass(frozen=True)
class Flags:
    """the per-Gaussian stage's flags (psb_train.cu MODE_DEPTH / _AA / _REG / _F3D / _NORMAL) and the regularisers' lambdas"""
    depth: bool = False
    aa: bool = False
    reg: bool = False
    f3d: bool = False
    normal: bool = False
    lambda_opacity: float = 0.01       # GaussianOptimizationParams.opacity_reg
    lambda_scale: float = 0.01         # GaussianOptimizationParams.scale_reg


ALL_FLAGS = [Flags(depth=bool(k & 1), aa=bool(k & 2), reg=bool(k & 4), f3d=bool(k & 8), normal=bool(k & 16)) for k in range(32)]


def flag_name(fl):
    return "+".join(n for n in ("depth", "aa", "reg", "f3d", "normal") if getattr(fl, n)) or "plain"


# ---- the forward --------------------------------------------------------------------------------------------------------------------
def widen(s, f):
    """(s', c) of activated scales s [P,3] and filters f [P] (include/psb200.h, 3D smoothing filter): s' = sqrt(s^2 + f^2),
    c = sqrt(prod s^2 / prod s'^2). A row with f = 0 keeps s and c = 1 exactly, in value and in gradient (psb_train.cu: f = 0 adds
    nothing)."""
    on = f != 0
    f2 = (f * f)[:, None]
    sp = torch.where(on[:, None], torch.sqrt(s * s + f2), s)
    c = torch.sqrt((s * s).prod(1) / (sp * sp).prod(1))
    return sp, torch.where(on, c, torch.ones_like(c))


def normals(raw, cam, flip=True):
    """normal64.gaussian_normals; flip=False: the shortest axis m = V r without turning it towards the camera"""
    return n64.gaussian_normals(raw, cam, flip)


def splat_inputs(raw, flags, f=None, conv=STEP_CONV):
    """trainer parameters -> the activated splat the forward draws: with the 3D filter, scales s' and opacity o c"""
    g = s64.activate(raw)
    if flags.f3d:
        sp, c = widen(g["scales"], f)
        g["scales"] = sp
        if conv.f3d_opacity:
            g["opacities"] = g["opacities"] * c[:, None]
    return g


def forward(raw, cam, flags, D, bg, f=None, conv=STEP_CONV):
    """-> (s64.composite's dict plus radii and geo, N [3,H,W] or None, n [P,3] or None): the trainer's forward of one pass"""
    g = splat_inputs(raw, flags, f, conv)
    geo = s64.geometry(g, cam, D, flags.aa)
    out = s64.composite(geo, cam["W"], cam["H"], bg)
    out.update(radii=geo["radius"], geo=geo)
    N = n = None
    if flags.normal:
        n = normals(raw, cam, conv.normal_flip)
        N = s64.composite(dict(geo, rgb=n), cam["W"], cam["H"], (0.0, 0.0, 0.0))["color"]
    return out, N, n


def image_loss(out, N, targets, flags, E=None):
    """-> (total, dict of the scalars): loss64 (mask, exposure row E) + lambda_depth depth_l1_64 + lambda_normal normal_l1_64"""
    mask = targets.get("mask")
    L, l1, ssim = s64.loss64(out["color"], targets["gt"], mask, targets.get("lambda_dssim", 0.2), E)
    zero = torch.zeros((), dtype=torch.float64, device=L.device)
    dl1 = s64.depth_l1_64(out["depth"], targets["depth"], mask) if flags.depth else zero
    nl1 = n64.normal_l1_64(N, targets["normal"], mask) if flags.normal else zero
    total = L + targets.get("lambda_depth", 0.0) * dl1 + targets.get("lambda_normal", 0.0) * nl1
    return total, dict(l1=l1, ssim=ssim, depth_l1=dl1, normal_l1=nl1)


def regularizer(raw, rows, flags):
    """(lambda_o / P) sum_rows sigmoid(opacity) + (lambda_s / P) sum_rows sum_c exp(scaling): the 3DGS-MCMC terms on `rows` [P] bool,
    unfiltered activations"""
    P = raw["opacity"].shape[0]
    w = rows.to(raw["opacity"].dtype)
    return (flags.lambda_opacity / P * (torch.sigmoid(raw["opacity"]).reshape(-1) * w).sum()
            + flags.lambda_scale / P * (torch.exp(raw["scaling"]).sum(1) * w).sum())


def adam64(p, g, m, v, lr, t, conv=STEP_CONV):
    """torch.optim.Adam's update at step t (1-based): -> (p', m', v')"""
    m1 = BETA1 * m + (1 - BETA1) * g
    v1 = BETA2 * v + (1 - BETA2) * g * g
    bc1 = 1 - BETA1 ** t if conv.bias_correction else 1.0
    bc2 = 1 - BETA2 ** t if conv.bias_correction else 1.0
    return p - lr / bc1 * m1 / (v1.sqrt() / math.sqrt(bc2) + conv.eps), m1, v1


def _nz_rows(t, P):
    return (t.reshape(P, -1) != 0).any(1)


def grads64(state, cam, targets, flags, conv=STEP_CONV):
    """The gradients of one pass: -> dict(grads {group: dL/dparam, reg included}, E (dL/dE or None), loss scalars, reached [P],
    visible [P], radii [P], mean2D [P,2] (dL/dmean2D in the statistics' units), pixel (dL/dI [3,H,W], dL/dD [H,W], dL/dN [3,H,W] or None:
    the per-pixel gradients of the loss w.r.t. the raw render))"""
    raw = {k: state["params"][k].detach().clone().requires_grad_(True) for k in GROUPS}
    E = state.get("E")
    E = E.detach().clone().requires_grad_(True) if E is not None else None
    out, N, n = forward(raw, cam, flags, state["D"], targets["bg"], state.get("f"), conv)
    geo = out["geo"]
    inter = dict(means2D=geo["means2D"], conic=geo["conic"], o=geo["o"], rgb=geo["rgb"], z=geo["z"])
    if n is not None:
        inter["n"] = n
    pix = dict(color=out["color"], depth=out["depth"])
    if N is not None:
        pix["normal"] = N
    total, scal = image_loss(out, N, targets, flags, E)
    leaves = [raw[k] for k in GROUPS] + ([E] if E is not None else [])
    keys = list(inter) + list(pix)
    res = torch.autograd.grad(total, leaves + [inter[k] for k in inter] + [pix[k] for k in pix], allow_unused=True)
    P = raw["xyz"].shape[0]
    dev = raw["xyz"].device
    grads = {k: (g if g is not None else torch.zeros_like(raw[k])) for k, g in zip(GROUPS, res[:6])}
    gE = res[6] if E is not None else None
    rest = dict(zip(keys, res[len(leaves):]))
    reached = torch.zeros(P, dtype=torch.bool, device=dev)
    for k in inter:
        if rest[k] is not None:
            reached |= _nz_rows(rest[k], P)
    if flags.reg:
        rows = reached if conv.reg_reached_only else torch.ones_like(reached)
        rr = {k: raw[k].detach().clone().requires_grad_(True) for k in ("opacity", "scaling")}
        go, gs = torch.autograd.grad(regularizer(rr, rows, flags), [rr["opacity"], rr["scaling"]])
        grads["opacity"] = grads["opacity"] + go
        grads["scaling"] = grads["scaling"] + gs
    m2 = rest["means2D"] if rest["means2D"] is not None else torch.zeros(P, 2, dtype=torch.float64, device=dev)
    if conv.mean2d_ndc:
        m2 = m2 * torch.tensor([0.5 * cam["W"], 0.5 * cam["H"]], dtype=torch.float64, device=dev)
    z = lambda t, like: t if t is not None else torch.zeros_like(like)
    pixel = dict(color=z(rest["color"], out["color"]), depth=z(rest["depth"], out["depth"]),
                 normal=z(rest["normal"], N) if N is not None else None)
    return dict(grads=grads, E=gE, reached=reached, visible=out["radii"] > 0, radii=out["radii"], mean2D=m2, pixel=pixel,
                loss=dict(loss=float(total.detach()), **{k: float(v.detach()) for k, v in scal.items()}), out=out, N=N)


def step64(state, cam, targets, flags, conv=STEP_CONV, stats=True):
    """One fused training iteration in float64.
    state: dict(params {group: [P,...]}, m, v (same), accum [P,1], denom [P,1], max_radii [P], step (the model's step_: this update is
      Adam step step + 1), lr [6] (the model's lr_, f_rest at lr / 20 already), D (active SH degree), f [P] (the 3D filter, with
      flags.f3d), and optionally the exposure row E [3,4], E_m, E_v, E_step (its step count before this update), E_lr).
    cam: splat64.camera64; targets: dict(gt [3,H,W], mask [3,H,W] or None, depth [H,W], normal [3,H,W], lambda_depth, lambda_normal,
      bg, lambda_dssim).
    -> dict(state = the next state, and grads64's entries: loss scalars, reached and visible masks, gradients)."""
    r = grads64(state, cam, targets, flags, conv)
    t = state["step"] + 1
    nxt = dict(state, params={}, m={}, v={}, step=t)
    for i, k in enumerate(GROUPS):
        nxt["params"][k], nxt["m"][k], nxt["v"][k] = adam64(state["params"][k], r["grads"][k], state["m"][k], state["v"][k], state["lr"][i], t, conv)
    if stats:
        vis = r["visible"]
        nxt["denom"] = state["denom"] + vis.to(torch.float64)[:, None]
        nxt["max_radii"] = torch.where(vis, torch.maximum(state["max_radii"], r["radii"].to(torch.float64)), state["max_radii"])
        nxt["accum"] = state["accum"] + torch.where(vis, r["mean2D"].norm(dim=1), torch.zeros_like(vis, dtype=torch.float64))[:, None]
    if state.get("E") is not None:
        te = state["E_step"] + 1
        nxt["E"], nxt["E_m"], nxt["E_v"] = adam64(state["E"], r["E"], state["E_m"], state["E_v"], state["E_lr"], te, conv)
        nxt["E_step"] = te
    r["state"] = nxt
    return r


# ---- margins ------------------------------------------------------------------------------------------------------------------------
def margins(state, cam, targets, flags, conv=STEP_CONV):
    """splat64.margins of the splat the pass draws (3D filter and anti-aliasing as flagged), plus the decisions this module adds:
    axis (gap between the two smallest raw log-scales of a live row) and flip (|m . t| / (|m| |t|)) with the normal term; depth_kink
    (|D - G| / G) and normal_kink (|N_c - G_c|) at the valid pixels some splat reaches, charged to the pixel's last blended Gaussian."""
    with torch.no_grad():
        raw = {k: state["params"][k] for k in GROUPS}
        g = splat_inputs(raw, flags, state.get("f"), conv)
        res = s64.margins(g, cam, state["D"], flags.aa, targets["bg"])
        if not (flags.normal or flags.depth):
            return res
        out, N, n = forward(raw, cam, flags, state["D"], targets["bg"], state.get("f"), conv)
        alive = out["geo"]["alive"]
        ids = torch.arange(alive.numel(), device=alive.device)
        last = out["last"].reshape(-1)
        mask = targets.get("mask")
        keep = last >= 0
        if mask is not None:
            keep &= mask[0].reshape(-1) != 0
        cover = _covering(out["geo"], cam["W"])
        if flags.depth:
            G = targets["depth"].reshape(-1)
            sel = keep & (G > 0)
            res["depth_kink"] = _charge(((out["depth"].reshape(-1) - G).abs() / G.clamp_min(1e-30))[sel], sel.nonzero().reshape(-1), last, cover)
        if flags.normal:
            sc = torch.sort(raw["scaling"], dim=1).values
            res["axis"] = ((sc[:, 1] - sc[:, 0])[alive], ids[alive])
            V = cam["V"]
            mvec = normals(raw, cam, flip=False)
            tv = raw["xyz"] @ V[:3, :3] + V[3, :3]
            cosang = (mvec * tv).sum(1).abs() / (mvec.norm(dim=1) * tv.norm(dim=1)).clamp_min(1e-300)
            res["flip"] = (cosang[alive], ids[alive])
            G = targets["normal"].reshape(3, -1)
            sel = keep & (G != 0).any(0)
            d = (N.reshape(3, -1) - G).abs()[:, sel].amin(0)
            res["normal_kink"] = _charge(d, sel.nonzero().reshape(-1), last, cover)
    return res


def _covering(geo, W):
    """pixel list -> for each pixel, the alive rows whose 3-sigma square covers it"""
    alive = geo["alive"].nonzero().reshape(-1)
    c = geo["means2D"].detach()[alive]
    r = geo["radius"][alive].to(c.dtype)

    def rows(pix):
        x, y = (pix % W).to(c.dtype), (pix // W).to(c.dtype)
        hit = ((c[None, :, 0] - x[:, None]).abs() <= r[None, :]) & ((c[None, :, 1] - y[:, None]).abs() <= r[None, :])
        return [alive[h] for h in hit]
    return rows


def _charge(vals, pix, last, cover, near=1e-2):
    """a per-pixel kink margin charged to the pixel's last blended Gaussian; a pixel closer than `near` to its kink is charged to every
    row that covers it too (the last one may carry too little weight there to move the pixel)"""
    ids, vs = [last[pix]], [vals]
    close = vals < near
    if close.any():
        for v, rows in zip(vals[close], cover(pix[close])):
            ids.append(rows)
            vs.append(v.expand(rows.numel()))
    return torch.cat(vs), torch.cat(ids)
