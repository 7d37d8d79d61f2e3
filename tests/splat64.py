"""A dense float64 restatement of the operation the rasterizer, the fused training step and the loss compute: the ground truth the
kernels are measured against.

Plain torch, differentiable with autograd, on any device. Every (pixel, Gaussian) pair of a tile is evaluated densely: no sort beyond
one global depth order, no tight tile lists and no `pmin` skip, so a test against this truth also checks that those culls never change
a result. Each convention names the kernel line it mirrors. Decisions (culls, skips, termination, clamps) are constants of the pass;
`margins` reports how far every one of them lies from its threshold, so that a scene can assert that float32 takes them the same way.

Conventions the perturbation tests alter live in `Conv`.
"""
import dataclasses
import math

import torch
import torch.nn.functional as F

TILE = 16                     # PSB_TILE_X / PSB_TILE_Y (psb_common.cuh)
NEAR = 0.2                    # psb_forward.cu: alive = p_view.z > 0.2f
FRUSTUM = 1.3                 # psb_geom.cuh cov2d_terms: limx = 1.3f * tan_fovx
MIN_RATIO = 2.5e-5            # psb_geom.cuh kAaMinRatio
ALPHA_MAX = 0.99              # psb_render.cu: alpha = min(0.99f, o * exp(power))
MIN_MARGIN = 1e-4             # the relative distance every decision of a test scene keeps from its threshold
SH_C0 = 0.28209479177387814   # psb_common.cuh kSH_*
SH_C1 = 0.4886025119029199
SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396)
SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658, 1.445305721320277,
         -0.5900435899266435)


@dataclasses.dataclass(frozen=True)
class Conv:
    dilation: float = 0.3              # psb_forward.cu: ct.cov(0, 0) += 0.3f
    alpha_min: float = 1.0 / 255.0     # psb_render.cu: if (alpha < 1.0f / 255.0f) continue
    t_min: float = 1e-4                # psb_render.cu: if (test_T < 0.0001f) { done[p] = true; continue; }
    straight_through: bool = True      # psb_render.cu backward: w = o * dL/dalpha * G, the 0.99 clamp differentiated straight through
    ssim_sigma: float = 1.5            # the 11x11 SSIM window
    depth_weighted: bool = True        # psb_render.cu: Dp = fma(T, z * alpha, Dp)


CONV = Conv()
RAW = ("xyz", "features_dc", "features_rest", "opacity", "scaling", "rotation")   # the trainer's parameter groups, in its order


def _t(x, dev):
    return torch.as_tensor(x).to(device=dev, dtype=torch.float64)


def camera64(cam, dev):
    """cam: dict(viewmatrix[16], projmatrix[16], campos[3], tanfovx, tanfovy, W, H), numpy or torch -> float64 on dev."""
    return dict(V=_t(cam["viewmatrix"], dev).reshape(4, 4), Pm=_t(cam["projmatrix"], dev).reshape(4, 4), campos=_t(cam["campos"], dev).reshape(3),
                tanfovx=float(cam["tanfovx"]), tanfovy=float(cam["tanfovy"]), W=int(cam["W"]), H=int(cam["H"]))


# ---- activations and geometry -------------------------------------------------------------------------------------------------------
def activate(raw):
    """Trainer parameters -> the operator's inputs (psb_forward.cu RAW branch): exp scales, unit (w, x, y, z) quaternion with
    max(norm, 1e-12), sigmoid opacity, SH rows [P, 16, 3] = features_dc ++ features_rest."""
    q = raw["rotation"]
    return dict(means3D=raw["xyz"], shs=torch.cat([raw["features_dc"], raw["features_rest"]], 1),
                opacities=torch.sigmoid(raw["opacity"]), scales=torch.exp(raw["scaling"]),
                rotations=q / q.norm(dim=1, keepdim=True).clamp_min(1e-12))


def quat_cov(scales, rot):
    """cov3D [P,6] = R diag(s)^2 R^T of scale and (w, x, y, z) quaternion (psb_geom.cuh cov3d_from_scale_rot): not normalised here"""
    r, x, y, z = rot.unbind(1)
    R = torch.stack([torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], 1),
                     torch.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], 1),
                     torch.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1)], 1)
    S = R * scales.unsqueeze(1)
    Sig = S @ S.transpose(1, 2)
    return torch.stack([Sig[:, 0, 0], Sig[:, 0, 1], Sig[:, 0, 2], Sig[:, 1, 1], Sig[:, 1, 2], Sig[:, 2, 2]], 1)


def _cov2d(means3D, cov6, V, W, H, tanfovx, tanfovy):
    """-> (a0, b, c0) of the 2D covariance before the dilation, t (view-space mean), tx/tz and ty/tz (psb_geom.cuh cov2d_terms).
    The mean's 1.3 tanfov clamp follows the kernels' backward: a clamped coordinate passes no gradient to the mean, and J's
    dependence on it through t.z is dropped. Gaussians behind the near plane get t = (0, 0, 1) (they are culled)."""
    t = means3D @ V[:3, :3] + V[3, :3]
    front = (t[:, 2] > NEAR).detach()
    t = torch.where(front.unsqueeze(1), t, torch.tensor([0.0, 0.0, 1.0], dtype=t.dtype, device=t.device))
    tz = t[:, 2]
    fx, fy = W / (2.0 * tanfovx), H / (2.0 * tanfovy)
    cols, ratios = [], []
    for k, lim in ((0, FRUSTUM * tanfovx), (1, FRUSTUM * tanfovy)):
        r = t[:, k] / tz
        ratios.append(r.detach())
        out = (r < -lim) | (r > lim)
        cols.append(torch.where(out, (r.clamp(-lim, lim) * tz).detach(), t[:, k]))
    tx, ty = cols
    zero = torch.zeros_like(tz)
    J = torch.stack([torch.stack([fx / tz, zero, -(fx * tx) / (tz * tz)], 1),
                     torch.stack([zero, fy / tz, -(fy * ty) / (tz * tz)], 1)], 1)
    c = cov6
    Sig = torch.stack([torch.stack([c[:, 0], c[:, 1], c[:, 2]], 1), torch.stack([c[:, 1], c[:, 3], c[:, 4]], 1),
                       torch.stack([c[:, 2], c[:, 4], c[:, 5]], 1)], 1)
    T = J @ V[:3, :3].T
    cov2 = T @ Sig @ T.transpose(1, 2)
    return cov2[:, 0, 0], cov2[:, 0, 1], cov2[:, 1, 1], front, ratios


def h_torch(means3D, cov6, viewmatrix, W, H, tanfovx, tanfovy, dilation=CONV.dilation):
    """The anti-aliasing opacity factor h = sqrt(max(det0 / det1, 2.5e-5)) of every Gaussian (psb_geom.cuh aa_factor; 1 where view
    z <= 0.2), differentiable in means3D and cov6, in the dtype of the inputs."""
    V = viewmatrix.reshape(4, 4).to(means3D.dtype)
    a0, b, c0, front, _ = _cov2d(means3D, cov6, V, W, H, tanfovx, tanfovy)
    det0 = a0 * c0 - b * b
    det1 = (a0 + dilation) * (c0 + dilation) - b * b
    h = torch.sqrt(torch.clamp_min(det0 / det1, MIN_RATIO))
    return torch.where(front, h, torch.ones_like(h))


def sh_rgb(D, means3D, campos, shs):
    """Colour before the clamp (psb_geom.cuh sh_to_rgb, result + 0.5), view direction from campos"""
    d = means3D - campos
    d = d / d.norm(dim=1, keepdim=True)
    x, y, z = (d[:, k:k + 1] for k in range(3))
    s = shs
    res = SH_C0 * s[:, 0]
    if D > 0:
        res = res - SH_C1 * y * s[:, 1] + SH_C1 * z * s[:, 2] - SH_C1 * x * s[:, 3]
        if D > 1:
            xx, yy, zz, xy, yz, xz = x * x, y * y, z * z, x * y, y * z, x * z
            res = (res + SH_C2[0] * xy * s[:, 4] + SH_C2[1] * yz * s[:, 5] + SH_C2[2] * (2 * zz - xx - yy) * s[:, 6]
                   + SH_C2[3] * xz * s[:, 7] + SH_C2[4] * (xx - yy) * s[:, 8])
            if D > 2:
                res = (res + SH_C3[0] * y * (3 * xx - yy) * s[:, 9] + SH_C3[1] * xy * z * s[:, 10]
                       + SH_C3[2] * y * (4 * zz - xx - yy) * s[:, 11] + SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * s[:, 12]
                       + SH_C3[4] * x * (4 * zz - xx - yy) * s[:, 13] + SH_C3[5] * z * (xx - yy) * s[:, 14]
                       + SH_C3[6] * x * (xx - 3 * yy) * s[:, 15])
    return res + 0.5


def geometry(g, cam, D=3, aa=False, scale_modifier=1.0, conv=CONV):
    """Per-Gaussian screen-space record (psb_forward.cu preprocess) of activated inputs g = dict(means3D, shs [P,M,3], opacities [P,1],
    scales, rotations) -> dict of float64 tensors; `alive` marks the Gaussians that reach the tile lists."""
    c = cam
    W, H = c["W"], c["H"]
    m = g["means3D"]
    cov6 = quat_cov(g["scales"] * scale_modifier, g["rotations"])
    a0, b, c0, front, (rx, ry) = _cov2d(m, cov6, c["V"], W, H, c["tanfovx"], c["tanfovy"])
    # psb_forward.cu: p_w = 1 / (p_hom.w + 1e-7), ndc_to_pix = ((v + 1) S - 1) / 2
    ph = m @ c["Pm"][:3] + c["Pm"][3]
    pw = 1.0 / (ph[:, 3] + 1e-7)
    means2D = torch.stack([((ph[:, 0] * pw + 1.0) * W - 1.0) * 0.5, ((ph[:, 1] * pw + 1.0) * H - 1.0) * 0.5], 1)
    z = (m @ c["V"][:3, 2] + c["V"][3, 2])
    a, cc = a0 + conv.dilation, c0 + conv.dilation
    det = a * cc - b * b
    det0 = a0 * c0 - b * b
    conic = torch.stack([cc / det, -b / det, a / det], 1)
    o = g["opacities"].reshape(-1)
    ratio = (det0 / det).detach()
    if aa:   # psb_forward.cu: opacity *= aa_h
        o = o * torch.sqrt(torch.clamp_min(det0 / det, MIN_RATIO))
    # radius = ceil(3 sqrt(lambda1)), lambda1 = mid + sqrt(max(0.1, mid^2 - det)) (psb_forward.cu)
    mid = 0.5 * (a + cc).detach()
    disc = (mid * mid - det.detach())
    lam1 = mid + torch.sqrt(torch.clamp_min(disc, 0.1))
    r3 = 3.0 * torch.sqrt(lam1)
    radius = torch.ceil(r3)
    gx, gy = -(-W // TILE), -(-H // TILE)
    px, py = means2D[:, 0].detach(), means2D[:, 1].detach()
    # getRect (psb_geom.cuh tile_rect): truncation toward zero, clamp to [0, grid]
    edges = torch.stack([(px - radius) / TILE, (py - radius) / TILE, (px + radius + TILE - 1) / TILE, (py + radius + TILE - 1) / TILE], 1)
    lims = torch.tensor([gx, gy, gx, gy], dtype=torch.float64, device=m.device)
    rect = torch.minimum(torch.clamp_min(torch.trunc(edges), 0), lims).long()
    area = (rect[:, 2] - rect[:, 0]) * (rect[:, 3] - rect[:, 1])
    alive = front & (det.detach() != 0) & (area != 0)
    rgb_pre = sh_rgb(D, m, c["campos"], g["shs"]) if g.get("colors") is None else g["colors"]
    rgb = torch.clamp_min(rgb_pre, 0.0)        # psb_geom.cuh: fmaxf(result, 0), the clamped channel passes no gradient
    return dict(means2D=means2D, z=z, conic=conic, o=o, rgb=rgb, radius=torch.where(alive, radius, torch.zeros_like(radius)).long(),
                rect=rect, alive=alive, tiles_touched=torch.where(alive, area, torch.zeros_like(area)),
                # for margins
                zd=z.detach(), ratios=(rx, ry), det=det.detach(), detscale=(a * cc).abs().detach() + (b * b).detach(), disc=disc, r3=r3,
                edges=edges, gx=gx, gy=gy, ratio=ratio, rgb_pre=rgb_pre.detach(), front=front)


def _alpha(a_raw, conv):
    if conv.straight_through:
        return a_raw - (a_raw - ALPHA_MAX).clamp_min(0.0).detach()
    return torch.clamp_max(a_raw, ALPHA_MAX)


def composite(geo, W, H, bg, conv=CONV, want_margins=False, tiles=None):
    """Per pixel, over the Gaussians whose rectangle holds the pixel's tile, in depth order (psb_render.cu render_fwd_body).
    -> dict(color [3,H,W], depth [H,W], alpha [H,W] = 1 - T_final, n_contrib [H,W] (1-based list position of the last blended
    splat, 0 = none), last [H,W] (the Gaussian index of that splat, -1 = none), stopped [H,W] (the T test ended the pixel's list), clamped [H,W] (a blended alpha was clamped at 0.99),
    list_len [tiles]) and with want_margins the pair decisions' margins.

    tiles: a list of (tx, ty) composites only those tiles and returns the same keys over their pixels, flattened in the order of the
    list (color [3,N], the others [N]), with pix [N] (y W + x) and, with want_margins, pix_margins: per pixel and decision the smallest
    margin of its pairs (inf for none), T_ulp (the T test's margin over 2^-24 sum 1 / (1 - alpha) of the factors blended up to the
    test) and depth_tie (the relative depth gap of two successive splats of the pixel that pass the alpha test)."""
    dev = geo["z"].device
    bg = _t(bg, dev).reshape(3)
    gx, gy = geo["gx"], geo["gy"]
    live = geo["alive"].nonzero().reshape(-1)
    order = live[torch.argsort(geo["zd"][live], stable=True)]
    rect = geo["rect"][order]
    m2, con, o, rgb, z = geo["means2D"][order], geo["conic"][order], geo["o"][order], geo["rgb"][order], geo["z"][order]
    outs, pix_ids, list_len = [], [], []
    mg = {k: [] for k in ("power", "alpha_min", "alpha_max", "T", "depth_tie")}
    pm = []
    for ty, tx in ([(ty, tx) for ty in range(gy) for tx in range(gx)] if tiles is None else [(ty, tx) for tx, ty in tiles]):
        sel = ((rect[:, 0] <= tx) & (tx < rect[:, 2]) & (rect[:, 1] <= ty) & (ty < rect[:, 3])).nonzero().reshape(-1)
        list_len.append(int(sel.numel()))
        ys, xs = torch.meshgrid(torch.arange(ty * TILE, min(ty * TILE + TILE, H), device=dev),
                                torch.arange(tx * TILE, min(tx * TILE + TILE, W), device=dev), indexing="ij")
        ys, xs = ys.reshape(-1), xs.reshape(-1)
        pix_ids.append(ys * W + xs)
        n = sel.numel()
        if n == 0:
            npx = xs.numel()
            outs.append(torch.cat([bg.expand(npx, 3), torch.zeros(npx, 5, dtype=torch.float64, device=dev),
                                   torch.full((npx, 1), -1.0, dtype=torch.float64, device=dev)], 1))
            if want_margins and tiles is not None:
                pm.append({k: torch.full((npx,), math.inf, dtype=torch.float64, device=dev)
                           for k in ("power", "alpha_min", "alpha_max", "T", "T_ulp", "depth_tie")})
            continue
        dx = m2[sel, 0][None, :] - xs[:, None].double()
        dy = m2[sel, 1][None, :] - ys[:, None].double()
        A, B, C = con[sel, 0][None, :], con[sel, 1][None, :], con[sel, 2][None, :]
        power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy      # psb_geom.cuh splat_power
        pw = power.detach()
        a_raw = o[sel][None, :] * torch.exp(power)
        ad = a_raw.detach()
        valid = (pw <= 0) & (torch.clamp_max(ad, ALPHA_MAX) >= conv.alpha_min)
        alpha = _alpha(a_raw, conv)
        f_all = torch.where(valid, 1.0 - alpha.detach(), torch.ones_like(ad))
        t_after = torch.cumprod(f_all, 1)
        include = valid & (t_after >= conv.t_min)
        fi = torch.where(include, 1.0 - alpha, torch.ones_like(alpha))
        cp = torch.cumprod(fi, 1)
        Tb = torch.cat([torch.ones_like(cp[:, :1]), cp[:, :-1]], 1)
        w = torch.where(include, alpha * Tb, torch.zeros_like(alpha))
        Tf = cp[:, -1:]
        col = w @ rgb[sel] + Tf * bg
        dep = (w @ z[sel]) if conv.depth_weighted else (include.double() @ z[sel])
        pos = torch.arange(1, n + 1, device=dev, dtype=torch.float64)
        nc = (include.double() * pos).amax(1)
        stopped = (valid & ~include).any(1).double()
        clamped = (include & (ad > ALPHA_MAX)).any(1).double()
        last = torch.where(nc > 0, order[sel].double()[(nc.long() - 1).clamp_min(0)], torch.full_like(nc, -1.0))
        outs.append(torch.cat([col, dep[:, None], (1.0 - Tf), nc[:, None], stopped[:, None], clamped[:, None], last[:, None]], 1))
        if want_margins:
            gid = order[sel][None, :].expand_as(pw)
            mag = 0.5 * (A.abs() * dx * dx + C.abs() * dy * dy).detach() + (B * dx * dy).abs().detach()
            nz = mag > 0
            mg["power"].append(((pw.abs() / mag)[nz], gid[nz]))
            tested = pw <= 0
            mg["alpha_min"].append(((ad - conv.alpha_min).abs()[tested] / conv.alpha_min, gid[tested]))
            mg["alpha_max"].append(((ad - ALPHA_MAX).abs()[tested] / ALPHA_MAX, gid[tested]))
            t_before = torch.cat([torch.ones_like(t_after[:, :1]), t_after[:, :-1]], 1)
            ev = valid & (t_before >= conv.t_min)
            mg["T"].append(((t_before * f_all - conv.t_min).abs()[ev] / conv.t_min, gid[ev]))
            zs = geo["zd"][order[sel]]
            if n > 1:
                mg["depth_tie"].append(((zs[1:] - zs[:-1]) / zs[1:], order[sel][1:]))
            if tiles is not None:
                inf = torch.full_like(pw, math.inf)
                t_rel = (t_before * f_all - conv.t_min).abs() / conv.t_min
                ulps = torch.cumsum(torch.where(valid, 1.0 / f_all, torch.zeros_like(f_all)), 1) * 2.0 ** -24
                idx = torch.arange(n, device=dev).expand_as(pw)
                prev = torch.cummax(torch.where(ev, idx, torch.full_like(idx, -1)), 1).values
                prev = torch.cat([torch.full_like(prev[:, :1], -1), prev[:, :-1]], 1)
                gap = (zs[None, :] - zs[prev.clamp_min(0)]) / zs[None, :].abs()
                pm.append(dict(power=torch.where(nz, pw.abs() / mag, inf).amin(1),
                               alpha_min=torch.where(tested, (ad - conv.alpha_min).abs() / conv.alpha_min, inf).amin(1),
                               alpha_max=torch.where(tested, (ad - ALPHA_MAX).abs() / ALPHA_MAX, inf).amin(1),
                               T=torch.where(ev, t_rel, inf).amin(1), T_ulp=torch.where(ev, t_rel / ulps, inf).amin(1),
                               depth_tie=torch.where(ev & (prev >= 0), gap, inf).amin(1)))
    vals = torch.cat(outs, 0)
    if tiles is not None:
        out = dict(pix=torch.cat(pix_ids), color=vals[:, :3].T, depth=vals[:, 3], alpha=vals[:, 4], n_contrib=vals[:, 5].detach().round().long(),
                   stopped=vals[:, 6].detach().bool(), clamped=vals[:, 7].detach().bool(), last=vals[:, 8].detach().round().long(),
                   list_len=torch.tensor(list_len, device=dev))
        if want_margins:
            out["pix_margins"] = {k: torch.cat([d[k] for d in pm]) for k in pm[0]}
        return out
    inv = torch.argsort(torch.cat(pix_ids))
    vals = vals[inv]
    out = dict(color=vals[:, :3].T.reshape(3, H, W), depth=vals[:, 3].reshape(H, W), alpha=vals[:, 4].reshape(H, W),
               n_contrib=vals[:, 5].detach().round().long().reshape(H, W), stopped=vals[:, 6].detach().bool().reshape(H, W),
               clamped=vals[:, 7].detach().bool().reshape(H, W), last=vals[:, 8].detach().round().long().reshape(H, W),
               list_len=torch.tensor(list_len, device=dev))
    if want_margins:
        out["pair_margins"] = {k: (torch.cat([a for a, _ in v]) if v else torch.zeros(0, dtype=torch.float64, device=dev),
                                   torch.cat([i for _, i in v]) if v else torch.zeros(0, dtype=torch.long, device=dev)) for k, v in mg.items()}
    return out


def render(g, cam, bg, D=3, aa=False, scale_modifier=1.0, conv=CONV, raw=False, want_margins=False):
    """The forward of the operator (g activated) or of the trainer (raw=True: g = trainer parameters) in float64.
    cam: camera64(...). -> composite()'s dict plus radii [P], tiles_touched [P] and the geometry record under "geo"."""
    act = activate(g) if raw else g
    geo = geometry(act, cam, D, aa, scale_modifier, conv)
    out = composite(geo, cam["W"], cam["H"], bg, conv, want_margins)
    out.update(radii=geo["radius"], tiles_touched=geo["tiles_touched"], geo=geo)
    return out


def _frac(v):
    """distance of v to the nearest integer, relative to max(|v|, 1)"""
    return (v - torch.round(v)).abs() / v.abs().clamp_min(1.0)


def margins(g, cam, D=3, aa=False, bg=(0.0, 0.0, 0.0), scale_modifier=1.0, conv=CONV, raw=False):
    """Relative distance, in float64, of every discrete decision of one render from its threshold:
    {name: (margins [n], Gaussian index [n])}. Names: near, det, radius, lambda, rect, frustum, colour, aa (with aa), and per
    (pixel, Gaussian) pair power, alpha_min, alpha_max, T, plus depth_tie (relative depth gap of neighbours in a tile list)."""
    with torch.no_grad():
        out = render(g, cam, bg, D, aa, scale_modifier, conv, raw, want_margins=True)
    geo = out["geo"]
    P = geo["zd"].numel()
    ids = torch.arange(P, device=geo["zd"].device)
    al, fr = geo["alive"], geo["front"]
    res = dict(near=((geo["zd"] - NEAR).abs() / NEAR, ids))
    res["det"] = ((geo["det"].abs() / geo["detscale"])[fr], ids[fr])
    res["lambda"] = (((geo["disc"] - 0.1).abs() / 0.1)[fr], ids[fr])
    res["radius"] = ((_frac(geo["r3"].detach()))[fr], ids[fr])
    e = geo["edges"].detach()
    lim = torch.tensor([geo["gx"], geo["gy"], geo["gx"], geo["gy"]], dtype=torch.float64, device=e.device)
    live_edge = fr[:, None] & (e >= 0) & (e <= lim + 1)     # outside [0, grid] the clamp decides, not the truncation
    res["rect"] = (_frac(e)[live_edge], ids[:, None].expand_as(e)[live_edge])
    lims = (FRUSTUM * cam["tanfovx"], FRUSTUM * cam["tanfovy"])
    fm = torch.stack([(r.abs() - l).abs() / l for r, l in zip(geo["ratios"], lims)], 1)
    res["frustum"] = (fm[fr].reshape(-1), ids[fr][:, None].expand(-1, 2).reshape(-1))
    if g.get("colors") is None:
        res["colour"] = (geo["rgb_pre"][al].abs().reshape(-1), ids[al][:, None].expand(-1, 3).reshape(-1))
    if aa:
        res["aa"] = (((geo["ratio"] - MIN_RATIO).abs() / MIN_RATIO)[al], ids[al])
    res.update(out["pair_margins"])
    return res


def min_margins(mg):
    return {k: (float(v.min()) if v.numel() else math.inf) for k, (v, _) in mg.items()}


def offenders(mg, floor=MIN_MARGIN):
    """Gaussians that take part in a decision closer than `floor` to its threshold"""
    bad = [i[v < floor] for v, i in mg.values() if v.numel()]
    return torch.unique(torch.cat(bad)) if bad else torch.zeros(0, dtype=torch.long)


def raw64(scene, dev):
    """trainer parameters (numpy float32, photo_slam_b200.synthetic.make_scene's keys) -> float64 tensors on dev"""
    return {k: _t(v, dev) for k, v in scene.items()}


def settle(scene, cam, D=3, aa=False, bg=(0.0, 0.0, 0.0), seed=0, dev="cpu", tries=80, floor=MIN_MARGIN):
    """Jitter, in place, the position (by ~0.03 px) and opacity of every Gaussian that takes part in a decision closer than `floor`
    to its threshold, until none does (with and without anti-aliasing when aa is None). Returns the minimum margins; raises if the
    scene does not settle. A scene built for an edge asserts that it still reaches it afterwards."""
    import numpy as np
    rng = np.random.default_rng(seed)
    c = camera64(cam, dev)
    fx = c["W"] / (2.0 * c["tanfovx"])
    for _ in range(tries):
        raw = raw64(scene, dev)
        mg = [margins(raw, c, D, a, bg, raw=True) for a in ((False, True) if aa is None else (aa,))]
        bad = torch.unique(torch.cat([offenders(m, floor) for m in mg])).tolist()
        if not bad:
            out = {}
            for m in mg:
                for k, v in min_margins(m).items():
                    out[k] = min(out.get(k, math.inf), v)
            return out
        z =np.linalg.norm(scene["xyz"][bad].astype(np.float64) - np.asarray(cam["campos"], np.float64).reshape(3), axis=1) + 0.1
        scene["xyz"][bad] += (rng.normal(0.0, 0.03, (len(bad), 3)) * (z / fx)[:, None]).astype(np.float32)
        scene["opacity"][bad] += rng.normal(0.0, 0.02, (len(bad), 1)).astype(np.float32)
    raise AssertionError(f"scene did not settle: {min_margins(mg[0])}")


# ---- the loss -------------------------------------------------------------------------------------------------------------------------
def window64(sigma=1.5, device=None):
    g = torch.tensor([math.exp(-(x - 5) ** 2 / (2.0 * sigma * sigma)) for x in range(11)], dtype=torch.float64, device=device)
    g = (g / g.sum()).unsqueeze(1)
    return g.mm(g.t()).unsqueeze(0).unsqueeze(0).expand(3, 1, 11, 11).contiguous()


def ssim64(img1, img2, sigma=1.5):
    """mean SSIM of two [3,H,W] images: 11x11 Gaussian window, zero padding, C1 = 0.01^2, C2 = 0.03^2"""
    window = window64(sigma, img1.device)
    a, b = img1.unsqueeze(0), img2.unsqueeze(0)
    mu1 = F.conv2d(a, window, padding=5, groups=3)
    mu2 = F.conv2d(b, window, padding=5, groups=3)
    mu1_sq, mu2_sq, mu1_mu2 = mu1.pow(2), mu2.pow(2), mu1 * mu2
    sigma1_sq = F.conv2d(a * a, window, padding=5, groups=3) - mu1_sq
    sigma2_sq = F.conv2d(b * b, window, padding=5, groups=3) - mu2_sq
    sigma12 = F.conv2d(a * b, window, padding=5, groups=3) - mu1_mu2
    C1, C2 = 0.01 * 0.01, 0.03 * 0.03
    ssim_map = ((2 * mu1_mu2 + C1) * (2 * sigma12 + C2)) / ((mu1_sq + mu2_sq + C1) * (sigma1_sq + sigma2_sq + C2))
    return ssim_map.mean()


def exposed(I, E):
    """I'(c, p) = sum_k E[k][c] I(k, p) + E[c][3]"""
    return torch.einsum("khw,kc->chw", I, E[:, :3]) + E[:, 3, None, None]


def loss64(I, G, mask=None, lam=0.2, E=None, conv=CONV):
    """-> (L, l1, ssim) with X = mask * I' (I' = exposed(I, E), I without E): L = (1 - lam) mean|X - G| + lam (1 - SSIM(X, G)).
    torch's |x| has the subgradient sign(0) = 0 at a tie, as the kernels."""
    X = exposed(I, E) if E is not None else I
    if mask is not None:
        X = mask * X
    l1 = (X - G).abs().mean()
    s = ssim64(X, G, conv.ssim_sigma)
    return (1.0 - lam) * l1 + lam * (1.0 - s), l1, s


def depth_l1_64(D, Gd, mask=None):
    """sum over valid pixels |D - G| / max(N_valid, 1), valid = G > 0 and mask[0] != 0 (include/psb200.h, depth loss)"""
    valid = Gd > 0
    if mask is not None:
        valid = valid & (mask[0] != 0)
    return torch.where(valid, (D - Gd).abs(), torch.zeros_like(D)).sum() / max(int(valid.sum()), 1)
