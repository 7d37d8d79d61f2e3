"""Float64 restatement of the depth-normal consistency term (include/psb200.h, "Depth-normal consistency"), built on normal64 without
changing it: the normalised depth D / A, its depth normal n_d (normal64.depth_normals64), the valid pixels and the term
sum_valid (1 - n_d . N) / max(N_valid, 1). Plain torch, differentiable with autograd in D, A and N, on any device."""
import torch

import normal64


def normalised_depth(D, A, alpha_min):
    """D / A where A >= alpha_min, else 0 (a hole); the division is taken only where it is kept, so autograd sees no 0 / 0"""
    keep = A >= alpha_min
    return torch.where(keep, D / torch.where(keep, A, torch.ones_like(A)), torch.zeros_like(D))


def dn64(D, A, N, W, H, tanfovx, tanfovy, alpha_min=0.5, max_rel_jump=0.05, mask=None):
    """-> (dn, N_valid, n_d [3,H,W]) for D, A [H,W] and N [3,H,W] seen by a camera of W x H pixels; mask [H,W] (or [k,H,W], channel 0
    read) or None. Validity (n_d != 0 and the mask) is a constant of the pass."""
    D, A, N = D.to(torch.float64), A.to(torch.float64), N.to(torch.float64)
    nd = normal64.depth_normals64(normalised_depth(D, A, alpha_min), W, H, tanfovx, tanfovy, max_rel_jump)
    valid = (nd.detach() != 0).any(0)
    if mask is not None:
        valid = valid & ((mask[0] if mask.dim() == 3 else mask) != 0)
    nv = int(valid.sum())
    term = torch.where(valid, 1.0 - (nd * N).sum(0), torch.zeros_like(D))
    return term.sum() / max(nv, 1), nv, nd
