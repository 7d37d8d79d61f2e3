"""Float64 restatement of the depth distortion term (include/psb200.h, "Depth distortion"), built on splat64 without changing it: the
second depth moment M = sum_i z_i^2 alpha_i T_i (splat64.composite's blend with the colour replaced by z^2 and no background), the
per-pixel distortion A M - D^2, the term sum_valid (A M - D^2) / max(N_valid, 1), its closed-form plane gradients and the depth spread.
Plain torch, differentiable with autograd, on any device."""
import torch

import splat64 as s64


def planes64(w, z):
    """-> (A, D, M) = (sum_i w_i, sum_i w_i z_i, sum_i w_i z_i^2) over the last axis of blending weights w and depths z"""
    return w.sum(-1), (w * z).sum(-1), (w * z * z).sum(-1)


def pairwise64(w, z):
    """2DGS's pairwise distortion in its squared form, a pair counted once: (1/2) sum_i sum_j w_i w_j (z_i - z_j)^2 over the last axis"""
    dz = z[..., :, None] - z[..., None, :]
    return 0.5 * (w[..., :, None] * w[..., None, :] * dz * dz).sum((-1, -2))


def _valid(A, mask):
    if mask is None:
        return torch.ones_like(A, dtype=torch.bool)
    return (mask[0] if mask.dim() == 3 else mask) != 0


def dist64(D, A, M, mask=None):
    """-> (dist, N_valid) for the planes D, A, M [H,W]; mask [H,W] (or [k,H,W], channel 0 read) or None: every pixel is valid"""
    D, A, M = D.to(torch.float64), A.to(torch.float64), M.to(torch.float64)
    valid = _valid(A, mask)
    nv = int(valid.sum())
    return torch.where(valid, A * M - D * D, torch.zeros_like(D)).sum() / max(nv, 1), nv


def grads64(D, A, M, lam, mask=None):
    """the closed-form gradients of lam * dist64 w.r.t. (A, D, M): k M, -2 k D and k A on valid pixels (0 elsewhere), k = lam / max(N_valid, 1)"""
    valid = _valid(A, mask)
    k = lam / max(int(valid.sum()), 1)
    z = torch.zeros_like(D, dtype=torch.float64)
    return (torch.where(valid, k * M.double(), z), torch.where(valid, -2.0 * k * D.double(), z), torch.where(valid, k * A.double(), z))


def spread64(D, A, M):
    """the depth spread sqrt(max(M / A - (D / A)^2, 0)) where A > 0, else 0"""
    D, A, M = D.to(torch.float64), A.to(torch.float64), M.to(torch.float64)
    a = torch.where(A > 0, A, torch.ones_like(A))
    return torch.where(A > 0, torch.sqrt(torch.clamp_min(M / a - (D / a) ** 2, 0.0)), torch.zeros_like(A))


def render_moment(g, cam, D=3, aa=False, raw=True, keep_z_grad=True):
    """-> (s64.render's dict, M [H,W]) for trainer parameters g (raw=True) or activated inputs (raw=False; e.g. contrib64.filtered for a
    3D-filtered pass), cam = splat64.camera64(...). keep_z_grad=False detaches the z^2 of each Gaussian (a truth without dM/dz)."""
    act = s64.activate(g) if raw else g
    out = s64.render(act, cam, (0.0, 0.0, 0.0), D=D, aa=aa)
    geo = s64.geometry(act, cam, D, aa)
    z = geo["z"] if keep_z_grad else geo["z"].detach()
    geo["rgb"] = torch.stack([z * z, torch.zeros_like(z), torch.zeros_like(z)], 1)
    M = s64.composite(geo, cam["W"], cam["H"], (0.0, 0.0, 0.0))["color"][0]
    return out, M
