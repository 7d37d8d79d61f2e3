"""Float64 restatement of the contribution scores (include/psb200.h, psb_trainer_contribution) on top of tests/splat64.py: per (pixel,
Gaussian) pair the blending weight w = alpha T of splat64.composite's blend, scattered to each Gaussian as a maximum and a sum over the
pixels of one view. `filtered` forms the activated inputs of a pass with the 3D smoothing filter (tests/filter3d64.py), so that
splat64.geometry sees the splat the trainer's preprocess forms."""
import numpy as np
import torch

import filter3d64 as f3d
import splat64 as s64


def weights(geo, W, H, conv=s64.CONV):
    """-> dict(max [P], sum [P], pixels [P] (how many pixels blend the Gaussian), stopped [H,W]) of one view: the pairs that blend are
    those of composite (power <= 0, alpha >= 1/255, T after the splat >= t_min), with w = alpha T, T the transmittance before the splat."""
    dev = geo["z"].device
    P = geo["z"].numel()
    wmax = torch.zeros(P, dtype=torch.float64, device=dev)
    wsum = torch.zeros(P, dtype=torch.float64, device=dev)
    npix = torch.zeros(P, dtype=torch.long, device=dev)
    stopped = torch.zeros(H * W, dtype=torch.bool, device=dev)
    live = geo["alive"].nonzero().reshape(-1)
    order = live[torch.argsort(geo["zd"][live], stable=True)]
    rect = geo["rect"][order]
    m2, con, o = geo["means2D"][order].detach(), geo["conic"][order].detach(), geo["o"][order].detach()
    for ty in range(geo["gy"]):
        for tx in range(geo["gx"]):
            sel = ((rect[:, 0] <= tx) & (tx < rect[:, 2]) & (rect[:, 1] <= ty) & (ty < rect[:, 3])).nonzero().reshape(-1)
            if sel.numel() == 0:
                continue
            ys, xs = torch.meshgrid(torch.arange(ty * s64.TILE, min(ty * s64.TILE + s64.TILE, H), device=dev),
                                    torch.arange(tx * s64.TILE, min(tx * s64.TILE + s64.TILE, W), device=dev), indexing="ij")
            ys, xs = ys.reshape(-1), xs.reshape(-1)
            dx = m2[sel, 0][None, :] - xs[:, None].double()
            dy = m2[sel, 1][None, :] - ys[:, None].double()
            A, B, C = con[sel, 0][None, :], con[sel, 1][None, :], con[sel, 2][None, :]
            power = -0.5 * (A * dx * dx + C * dy * dy) - B * dx * dy
            alpha = torch.clamp_max(o[sel][None, :] * torch.exp(power), s64.ALPHA_MAX)
            valid = (power <= 0) & (alpha >= conv.alpha_min)
            f_all = torch.where(valid, 1.0 - alpha, torch.ones_like(alpha))
            t_after = torch.cumprod(f_all, 1)
            include = valid & (t_after >= conv.t_min)
            fi = torch.where(include, 1.0 - alpha, torch.ones_like(alpha))
            cp = torch.cumprod(fi, 1)
            Tb = torch.cat([torch.ones_like(cp[:, :1]), cp[:, :-1]], 1)
            w = torch.where(include, alpha * Tb, torch.zeros_like(alpha))
            g = order[sel]
            wmax[g] = torch.maximum(wmax[g], w.amax(0))
            wsum.index_add_(0, g, w.sum(0))
            npix.index_add_(0, g, include.sum(0))
            stopped[ys * W + xs] |= (valid & ~include).any(1)
    return dict(max=wmax, sum=wsum, pixels=npix, stopped=stopped.reshape(H, W))


def filtered(raw, f):
    """Activated inputs (splat64.activate) of trainer parameters `raw` (float64 tensors) with the 3D filter f [P] applied: s' = sqrt(s^2 +
    f^2), o' = o c."""
    g = s64.activate(raw)
    sp, c = f3d.widen(g["scales"].cpu().numpy(), np.asarray(f, np.float64))
    dev = g["scales"].device
    g["scales"] = torch.from_numpy(sp).to(dev)
    g["opacities"] = g["opacities"] * torch.from_numpy(c).to(dev).reshape(-1, 1)
    return g


def scores(raw, cams, D=3, aa=False, f=None):
    """Scores of a sweep: raw = trainer parameters (float64 tensors), cams = splat64.camera64 dicts, f = the 3D filter [P] or None.
    -> dict(max [P], sum [P], pixels [P], stopped [views][H,W])."""
    g = filtered(raw, f) if f is not None else s64.activate(raw)
    P = raw["xyz"].shape[0]
    dev = raw["xyz"].device
    out = dict(max=torch.zeros(P, dtype=torch.float64, device=dev), sum=torch.zeros(P, dtype=torch.float64, device=dev),
               pixels=torch.zeros(P, dtype=torch.long, device=dev), stopped=[])
    for c in cams:
        r = weights(s64.geometry(g, c, D, aa), c["W"], c["H"])
        out["max"] = torch.maximum(out["max"], r["max"])
        out["sum"] += r["sum"]
        out["pixels"] += r["pixels"]
        out["stopped"].append(r["stopped"])
    return out


def settle(scene, cams, D=3, aa=False, f_of=None, seed=0, tries=80, floor=s64.MIN_MARGIN):
    """splat64.settle over several cameras and, with f_of (xyz -> filter [P]), on the filtered splats: jitter the rows that take part in a
    decision closer than `floor` to its threshold in any view, until none does."""
    rng = np.random.default_rng(seed)
    for _ in range(tries):
        raw = s64.raw64(scene, "cpu")
        g = filtered(raw, f_of(scene["xyz"])) if f_of is not None else raw
        bad = set()
        for cam in cams:
            c = s64.camera64(cam, "cpu")
            bad.update(s64.offenders(s64.margins(g, c, D, aa, raw=f_of is None), floor).tolist())
        if not bad:
            return
        bad = sorted(bad)
        fx = cams[0]["W"] / (2.0 * float(cams[0]["tanfovx"]))
        z = np.linalg.norm(scene["xyz"][bad].astype(np.float64), axis=1) + 0.1
        scene["xyz"][bad] += (rng.normal(0.0, 0.03, (len(bad), 3)) * (z / fx)[:, None]).astype(np.float32)
        scene["opacity"][bad] += rng.normal(0.0, 0.02, (len(bad), 1)).astype(np.float32)
    raise AssertionError("scene did not settle")
