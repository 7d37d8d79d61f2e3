"""A float64 restatement of one whole training iteration of the fused step (include/psb200.h): the forward with the 3D filter, the
anti-aliasing factor, the normal plane and the second depth moment, the built-in loss with exposure, depth, normal, depth-normal consistency
and distortion terms, the 3DGS-MCMC regularisers, the densification statistics and the Adam update of every parameter, its moments and the
exposure row. The arbiter the per-Gaussian stage (gaussian_backward_kernel<MODE> and frest_stream_kernel) is measured against, in every
flag set and base.

Plain torch, differentiable with autograd, on any device. Built on splat64 (render, loss), normal64 (per-Gaussian normals, normal L1),
dn64 (consistency) and dist64 (distortion) without changing their behaviour (normal64.gaussian_normals takes flip=False for the perturbed
truth). Decisions this module adds (the normal's axis and flip, the kinks of the depth and normal L1, the consistency term's alpha and
depth-jump tests) are constants of the pass; `margins` reports how far each lies from its threshold, next to splat64.margins'.

Conventions the perturbation tests alter live in `StepConv`.
"""
import dataclasses
import math

import torch

import dist64
import dn64
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
    dist_dz: bool = True               # the second moment's z_i^2 carries its gradient 2 z_i dL/dM into dL/dz_i


STEP_CONV = StepConv()


@dataclasses.dataclass(frozen=True)
class Flags:
    """the per-Gaussian stage's flags (psb_train.cu MODE_DEPTH / _AA / _REG / _F3D / _NORMAL), the optional consistency (dn) and
    distortion (dist) terms of the loss, and the regularisers' lambdas. normal: the normal L1 against targets["normal"]; dn renders the
    normal plane too (the kernels' MODE_NORMAL), dn and dist the depth's dL/dz (MODE_DEPTH) whether or not depth is set."""
    depth: bool = False
    aa: bool = False
    reg: bool = False
    f3d: bool = False
    normal: bool = False
    dn: bool = False
    dist: bool = False
    lambda_opacity: float = 0.01       # GaussianOptimizationParams.opacity_reg
    lambda_scale: float = 0.01         # GaussianOptimizationParams.scale_reg


ALL_FLAGS = [Flags(depth=bool(k & 1), aa=bool(k & 2), reg=bool(k & 4), f3d=bool(k & 8), normal=bool(k & 16)) for k in range(32)]


def flag_name(fl):
    return "+".join(n for n in ("depth", "aa", "reg", "f3d", "normal", "dn", "dist") if getattr(fl, n)) or "plain"


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
    """-> (s64.composite's dict plus radii and geo, N [3,H,W] or None, n [P,3] or None): the trainer's forward of one pass. The dict
    holds the accumulated opacity A = 1 - T_final under "alpha" and, with flags.dist, the second depth moment M = sum_i z_i^2 alpha_i T_i
    under "depth2" (the blend with the colour replaced by (z^2, 0, 0) and no background, as dist64.render_moment)."""
    g = splat_inputs(raw, flags, f, conv)
    geo = s64.geometry(g, cam, D, flags.aa)
    out = s64.composite(geo, cam["W"], cam["H"], bg)
    out.update(radii=geo["radius"], geo=geo)
    N = n = None
    if flags.normal or flags.dn:
        n = normals(raw, cam, conv.normal_flip)
        N = s64.composite(dict(geo, rgb=n), cam["W"], cam["H"], (0.0, 0.0, 0.0))["color"]
    if flags.dist:
        z = geo["z"] if conv.dist_dz else geo["z"].detach()
        zero = torch.zeros_like(z)
        out["depth2"] = s64.composite(dict(geo, rgb=torch.stack([z * z, zero, zero], 1)), cam["W"], cam["H"], (0.0, 0.0, 0.0))["color"][0]
    return out, N, n


def image_loss(out, N, targets, flags, E=None, cam=None):
    """-> (total, dict of the scalars): loss64 (mask, exposure row E) + lambda_depth depth_l1_64 + lambda_normal normal_l1_64, and with
    flags.dn / flags.dist + lambda_dn dn64 (of D, A and N seen by cam; dn_alpha_min, dn_max_rel_jump) + lambda_dist dist64 (of D, A, M),
    both with the mask. targets["colour"] = False drops loss64: the loss of a colour target equal to the render with lambda_dssim = 0,
    whose photometric gradient is exactly zero (l1 reads 0 and ssim 1 then)."""
    mask = targets.get("mask")
    dev = out["depth"].device
    zero = torch.zeros((), dtype=torch.float64, device=dev)
    if targets.get("colour", True):
        L, l1, ssim = s64.loss64(out["color"], targets["gt"], mask, targets.get("lambda_dssim", 0.2), E)
    else:
        L, l1, ssim = zero, zero, torch.ones((), dtype=torch.float64, device=dev)
    dl1 = s64.depth_l1_64(out["depth"], targets["depth"], mask) if flags.depth else zero
    nl1 = n64.normal_l1_64(N, targets["normal"], mask) if flags.normal else zero
    total = L + targets.get("lambda_depth", 0.0) * dl1 + targets.get("lambda_normal", 0.0) * nl1
    dn = dist = zero
    if flags.dn:
        dn = dn64.dn64(out["depth"], out["alpha"], N, cam["W"], cam["H"], cam["tanfovx"], cam["tanfovy"], targets.get("dn_alpha_min", 0.5),
                       targets.get("dn_max_rel_jump", 0.05), mask)[0]
        total = total + targets["lambda_dn"] * dn
    if flags.dist:
        dist = dist64.dist64(out["depth"], out["alpha"], out["depth2"], mask)[0]
        total = total + targets["lambda_dist"] * dist
    return total, dict(l1=l1, ssim=ssim, depth_l1=dl1, normal_l1=nl1, dn=dn, dist=dist)


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
    visible [P], radii [P], mean2D [P,2] (dL/dmean2D in the statistics' units), pixel (dL/dI [3,H,W], dL/dD [H,W], dL/dA [H,W],
    dL/dN [3,H,W] or None, dL/dM [H,W] or None: the per-pixel gradients of the loss w.r.t. the raw render), inter ({means2D, conic, o,
    rgb, z, n}: the per-Gaussian gradients w.r.t. the screen-space record, zeros where the loss does not depend on it; n only with a normal
    plane))"""
    raw = {k: state["params"][k].detach().clone().requires_grad_(True) for k in GROUPS}
    E = state.get("E")
    E = E.detach().clone().requires_grad_(True) if E is not None else None
    out, N, n = forward(raw, cam, flags, state["D"], targets["bg"], state.get("f"), conv)
    geo = out["geo"]
    inter = dict(means2D=geo["means2D"], conic=geo["conic"], o=geo["o"], rgb=geo["rgb"], z=geo["z"])
    if n is not None:
        inter["n"] = n
    pix = dict(color=out["color"], depth=out["depth"], alpha=out["alpha"])
    if N is not None:
        pix["normal"] = N
    if "depth2" in out:
        pix["depth2"] = out["depth2"]
    total, scal = image_loss(out, N, targets, flags, E, cam)
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
    pixel = dict(color=z(rest["color"], out["color"]), depth=z(rest["depth"], out["depth"]), alpha=z(rest["alpha"], out["alpha"]),
                 normal=z(rest["normal"], N) if N is not None else None,
                 depth2=z(rest["depth2"], out["depth2"]) if "depth2" in out else None)
    return dict(grads=grads, E=gE, reached=reached, visible=out["radii"] > 0, radii=out["radii"], mean2D=m2, pixel=pixel,
                inter={k: z(rest[k], inter[k]) for k in inter},
                loss=dict(loss=float(total.detach()), **{k: float(v.detach()) for k, v in scal.items()}), out=out, N=N)


def step64(state, cam, targets, flags, conv=STEP_CONV, stats=True):
    """One fused training iteration in float64.
    state: dict(params {group: [P,...]}, m, v (same), accum [P,1], denom [P,1], max_radii [P], step (the model's step_: this update is
      Adam step step + 1), lr [6] (the model's lr_, f_rest at lr / 20 already), D (active SH degree), f [P] (the 3D filter, with
      flags.f3d), and optionally the exposure row E [3,4], E_m, E_v, E_step (its step count before this update), E_lr).
    cam: splat64.camera64; targets: dict(gt [3,H,W], mask [3,H,W] or None, depth [H,W], normal [3,H,W], lambda_depth, lambda_normal,
      bg, lambda_dssim, and with flags.dn / flags.dist lambda_dn, dn_alpha_min, dn_max_rel_jump / lambda_dist; colour = False drops the
      photometric term).
    -> dict(state = the next state, and grads64's entries: loss scalars, reached and visible masks, gradients)."""
    r = grads64(state, cam, targets, flags, conv)
    t = state["step"] + 1
    nxt = dict(state, params={}, m={}, v={}, step=t)
    for i, k in enumerate(GROUPS):
        nxt["params"][k], nxt["m"][k], nxt["v"][k] = adam64(state["params"][k], r["grads"][k], state["m"][k], state["v"][k], state["lr"][i], t, conv)
    if stats:
        nxt.update(stats64(state, r))
    if state.get("E") is not None:
        te = state["E_step"] + 1
        nxt["E"], nxt["E_m"], nxt["E_v"] = adam64(state["E"], r["E"], state["E_m"], state["E_v"], state["E_lr"], te, conv)
        nxt["E_step"] = te
    r["state"] = nxt
    return r


def stats64(state, r):
    """the densification statistics after the pass r of grads64 -> dict(denom, max_radii, accum): the rows the pass draws count once,
    keep the larger radius and add |dL/dmean2D|"""
    vis = r["visible"]
    return dict(denom=state["denom"] + vis.to(torch.float64)[:, None],
                max_radii=torch.where(vis, torch.maximum(state["max_radii"], r["radii"].to(torch.float64)), state["max_radii"]),
                accum=state["accum"] + torch.where(vis, r["mean2D"].norm(dim=1), torch.zeros_like(vis, dtype=torch.float64))[:, None])


def dp_step64(state, views, world, dropped=(), conv=STEP_CONV, per_view=None, scale=None):
    """One data-parallel optimizer step in float64: every rank r renders views[r] = (cam, targets, flags) of the same replica, and
    g = (1 / world) sum_{r not in dropped} grads64(state, *views[r]) is applied by adam64 once. A dropped view (its binning arena
    overflowed) adds nothing, and still counts in the 1 / world.
    per_view: grads64 results of the views (None for a dropped one), computed once by a caller that also builds perturbed truths from
    them; scale replaces 1 / world. -> dict(state = the next parameters and moments, grads = the g Adam took, views = the per-view results).
    The densification statistics are each rank's own: stats64(state, views[r])."""
    rs = per_view if per_view is not None else [None if i in dropped else grads64(state, *v, conv) for i, v in enumerate(views)]
    s = 1.0 / world if scale is None else scale
    t = state["step"] + 1
    nxt = dict(state, params={}, m={}, v={}, step=t)
    grads = {}
    for i, k in enumerate(GROUPS):
        g = torch.zeros_like(state["params"][k])
        for j, r in enumerate(rs):
            if j not in dropped:
                g = g + r["grads"][k]
        grads[k] = g * s
        nxt["params"][k], nxt["m"][k], nxt["v"][k] = adam64(state["params"][k], grads[k], state["m"][k], state["v"][k], state["lr"][i], t, conv)
    return dict(state=nxt, grads=grads, views=rs)


# ---- margins ------------------------------------------------------------------------------------------------------------------------
def margins(state, cam, targets, flags, conv=STEP_CONV):
    """splat64.margins of the splat the pass draws (3D filter and anti-aliasing as flagged), plus the decisions this module adds:
    axis (gap between the two smallest raw log-scales of a live row) and flip (|m . t| / (|m| |t|)) with a normal plane; depth_kink
    (|D - G| / G) and normal_kink (|N_c - G_c|) at the valid pixels some splat reaches, charged to the pixel's last blended Gaussian.
    With the consistency term: dn_alpha (|A - alpha_min| / alpha_min at every pixel some splat reaches: A >= alpha_min decides whether
    D / A exists there) and dn_jump (| |z_nb - z| - j z | / (j z), j = max_rel_jump, for each stencil pair of a mask-valid interior pixel
    whose normalised depths z, z_nb both exist), charged to the last blended Gaussian of the pixel and, for a pair, of its neighbour too.
    The distortion's validity is the mask alone, a constant of the targets: it adds no decision."""
    with torch.no_grad():
        raw = {k: state["params"][k] for k in GROUPS}
        g = splat_inputs(raw, flags, state.get("f"), conv)
        res = s64.margins(g, cam, state["D"], flags.aa, targets["bg"])
        if not (flags.normal or flags.depth or flags.dn):
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
        if flags.normal or flags.dn:
            sc = torch.sort(raw["scaling"], dim=1).values
            res["axis"] = ((sc[:, 1] - sc[:, 0])[alive], ids[alive])
            V = cam["V"]
            mvec = normals(raw, cam, flip=False)
            tv = raw["xyz"] @ V[:3, :3] + V[3, :3]
            cosang = (mvec * tv).sum(1).abs() / (mvec.norm(dim=1) * tv.norm(dim=1)).clamp_min(1e-300)
            res["flip"] = (cosang[alive], ids[alive])
        if flags.normal:
            G = targets["normal"].reshape(3, -1)
            sel = keep & (G != 0).any(0)
            d = (N.reshape(3, -1) - G).abs()[:, sel].amin(0)
            res["normal_kink"] = _charge(d, sel.nonzero().reshape(-1), last, cover)
        if flags.dn:
            res.update(_dn_margins(out, cam, targets, last, cover))
    return res


def _dn_margins(out, cam, targets, last, cover):
    W, H = cam["W"], cam["H"]
    amin, jump = targets.get("dn_alpha_min", 0.5), targets.get("dn_max_rel_jump", 0.05)
    A = out["alpha"].reshape(-1)
    sel = last >= 0
    res = dict(dn_alpha=_charge(((A - amin).abs() / amin)[sel], sel.nonzero().reshape(-1), last, cover))
    z = dn64.normalised_depth(out["depth"], out["alpha"], amin)
    pix = torch.arange(H * W, device=z.device).reshape(H, W)
    centre = (z > 0)[1:-1, 1:-1]
    mask = targets.get("mask")
    if mask is not None:
        centre &= (mask[0] != 0)[1:-1, 1:-1]
    zc, pc = z[1:-1, 1:-1], pix[1:-1, 1:-1]
    vals, pa, pb = [], [], []
    for zn, pn in ((z[1:-1, :-2], pix[1:-1, :-2]), (z[1:-1, 2:], pix[1:-1, 2:]), (z[:-2, 1:-1], pix[:-2, 1:-1]), (z[2:, 1:-1], pix[2:, 1:-1])):
        both = centre & (zn > 0)
        vals.append((((zn - zc).abs() - jump * zc).abs() / (jump * zc))[both])
        pa.append(pc[both])
        pb.append(pn[both])
    vals, pa, pb = torch.cat(vals), torch.cat(pa), torch.cat(pb)
    ca, cb = _charge(vals, pa, last, cover), _charge(vals, pb, last, cover)
    res["dn_jump"] = (torch.cat([ca[0], cb[0]]), torch.cat([ca[1], cb[1]]))
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
