"""Float64 restatement of the rendered normals (include/psb200.h, "Rendered surface normals"), built on splat64 without changing it:
the per-Gaussian normal (argmin of the raw scales, column of R(q), camera-facing flip), the normal plane, the sensor normals of a depth
image and the normal L1 of the built-in loss. Plain torch, differentiable with autograd, on any device."""
import torch

import splat64 as s64


def rotation_columns(q):
    """[P,3,3]: R(q)[:, :, k] = column k of the rotation of the unit (w, x, y, z) quaternions q [P,4] (s64.quat_cov's R)"""
    w, x, y, z = q.unbind(1)
    c0 = torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + w * z), 2 * (x * z - w * y)], 1)
    c1 = torch.stack([2 * (x * y - w * z), 1 - 2 * (x * x + z * z), 2 * (y * z + w * x)], 1)
    c2 = torch.stack([2 * (x * z + w * y), 2 * (y * z - w * x), 1 - 2 * (x * x + y * y)], 1)
    return torch.stack([c0, c1, c2], 2)


def gaussian_normals(raw, cam, flip=True):
    """n_i [P,3] in view space of the trainer parameters raw (dict of s64.RAW) seen by cam (s64.camera64): k = argmin of the raw log-scales
    (the first on ties), r = column k of R(q / max(|q|, 1e-12)), m = V r, n = m if m . t <= 0 else -m (t = the view-space mean). The
    argmin and the flip are constants of the pass. flip=False: m itself, not turned towards the camera."""
    q = raw["rotation"]
    q = q / q.norm(dim=1, keepdim=True).clamp_min(1e-12)
    k = torch.argmin(raw["scaling"].detach(), dim=1)
    r = rotation_columns(q)[torch.arange(q.shape[0], device=q.device), :, k]
    V = cam["V"]                                      # V[c][r] = viewmatrix[4 c + r]: the math V is V.T
    m = r @ V[:3, :3]
    if not flip:
        return m
    t = raw["xyz"] @ V[:3, :3] + V[3, :3]
    sign = torch.where((m * t).sum(1).detach() <= 0, 1.0, -1.0).to(m.dtype)
    return m * sign[:, None]


def render_normal(raw, cam, D=3, aa=False):
    """-> (s64.render's dict of the trainer's forward, N [3,H,W] = sum_i n_i alpha_i T_i): the blend of s64.composite with the colour
    replaced by n_i and no background."""
    out = s64.render(raw, cam, (0.0, 0.0, 0.0), D=D, aa=aa, raw=True)
    geo = s64.geometry(s64.activate(raw), cam, D, aa)
    geo["rgb"] = gaussian_normals(raw, cam)
    N = s64.composite(geo, cam["W"], cam["H"], (0.0, 0.0, 0.0))["color"]
    return out, N


def depth_normals64(depth, W, H, tanfovx, tanfovy, max_rel_jump=0.05):
    """psb_depth_normals in float64: depth [H,W] -> [3,H,W] view-space unit normals, (0,0,0) on the border, at holes (not finite or <= 0),
    across depth edges (|z_nb - z| > max_rel_jump z) and where the cross product vanishes."""
    z = depth.to(torch.float64)
    dev = z.device
    fx, fy = W / (2.0 * tanfovx), H / (2.0 * tanfovy)
    v, u = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float64), torch.arange(W, device=dev, dtype=torch.float64), indexing="ij")
    X = torch.stack([(u + 0.5 - W / 2.0) * z / fx, (v + 0.5 - H / 2.0) * z / fy, z], 0)
    out = torch.zeros((3, H, W), dtype=torch.float64, device=dev)
    if W < 3 or H < 3:
        return out
    c = X[:, 1:-1, 1:-1]
    a = X[:, 1:-1, 2:] - X[:, 1:-1, :-2]
    b = X[:, 2:, 1:-1] - X[:, :-2, 1:-1]
    cr = torch.linalg.cross(a, b, dim=0)
    zc = z[1:-1, 1:-1]
    nbs = (z[1:-1, :-2], z[1:-1, 2:], z[:-2, 1:-1], z[2:, 1:-1])
    ok = torch.isfinite(zc) & (zc > 0)
    for zn in nbs:
        ok &= torch.isfinite(zn) & (zn > 0) & ~((zn - zc).abs() > max_rel_jump * zc)
    length = cr.norm(dim=0)
    ok &= length > 0
    sign = torch.where((cr * c).sum(0) < 0, 1.0, -1.0).to(torch.float64)
    n = cr * (sign / torch.where(ok, length, torch.ones_like(length)))[None]
    out[:, 1:-1, 1:-1] = torch.where(ok[None], n, torch.zeros_like(n))
    return out


def normal_l1_64(N, G, mask=None):
    """sum over valid pixels sum_c |N_c - G_c| / max(N_valid, 1); valid = G != (0,0,0) and mask[0] != 0"""
    valid = (G != 0).any(0)
    if mask is not None:
        valid = valid & (mask[0] != 0)
    return torch.where(valid[None], (N - G).abs(), torch.zeros_like(N)).sum() / max(int(valid.sum()), 1)
