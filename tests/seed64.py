"""Restatement of depth-guided seeding as include/psb200.h defines it (psb_seed_plan / psb_seed_apply): the selection in float32 (the same
rounded products as the kernel), the rank and cap rule in Python integers, and the new rows in float64. Planes are numpy [H,W] (the
image and the mask [3,H,W]); cameras are dicts in the form photo_slam_b200.synthetic.make_camera returns."""
import math

import numpy as np

SH_C0 = 0.28209479177387814
HOLE, FRONT = 1, 2


def select(A, D, G, mask=None, alpha_min=0.5, depth_rel=0.1, min_depth=0.2, max_depth=40.0, stride=1):
    """[H,W] uint8: 0 = not selected (off the grid included), HOLE or FRONT."""
    f32 = np.float32
    A, D, G = (np.asarray(x, f32) for x in (A, D, G))
    am, k = f32(alpha_min), f32(1.0) - f32(depth_rel)   # k formed in float32, as the host does
    with np.errstate(invalid="ignore", over="ignore"):
        valid = np.isfinite(G) & (G > f32(min_depth)) & (G < f32(max_depth))
        if mask is not None:
            valid &= np.asarray(mask, f32)[0] != 0
        hole = A < am
        front = (A >= am) & ((G * A) < (k * D))        # float32 products, each rounded on its own
    out = np.where(valid & hole, HOLE, np.where(valid & front, FRONT, 0)).astype(np.uint8)
    grid = np.zeros_like(out, dtype=bool)
    grid[::stride, ::stride] = True
    return np.where(grid, out, 0).astype(np.uint8)


def keep(c, n):
    """bool [c]: the ranks kept when n of c selected pixels are: floor((k + 1) n / c) > floor(k n / c)."""
    assert 0 <= n <= c
    return np.array([(k + 1) * n // c > k * n // c for k in range(c)], dtype=bool)


def unproject(cam, u, v, z):
    """world points [N,3] (float64) of pixels (u, v) at depth z: p = ((u + 0.5 - W/2) z / fx, (v + 0.5 - H/2) z / fy, z), xyz = R^T (p - t)."""
    W, H = int(cam["W"]), int(cam["H"])
    fx = W / (2.0 * float(np.float32(cam["tanfovx"])))
    fy = H / (2.0 * float(np.float32(cam["tanfovy"])))
    u, v, z = (np.asarray(a, np.float64) for a in (u, v, z))
    p = np.stack([(u + 0.5 - W / 2.0) * z / fx, (v + 0.5 - H / 2.0) * z / fy, z], 1)
    m = np.asarray(cam["viewmatrix"], np.float64).reshape(-1)
    R = np.array([[m[4 * c + r] for c in range(3)] for r in range(3)])
    t = m[12:15]
    return (p - t) @ R        # rows of R^T (p - t)


def project(cam, xyz):
    """(pixel u, pixel v, view depth z) of world points through the forward's formulas (psb_forward.cu): p_hom = projmatrix xyz,
    ndc = p_hom / p_hom.w, pix = ((ndc + 1) S - 1) / 2; z from the view matrix."""
    xyz = np.asarray(xyz, np.float64)
    V = np.asarray(cam["viewmatrix"], np.float64).reshape(4, 4)
    Pm = np.asarray(cam["projmatrix"], np.float64).reshape(4, 4)
    ph = xyz @ Pm[:3] + Pm[3]
    pv = xyz @ V[:3] + V[3]
    W, H = int(cam["W"]), int(cam["H"])
    return ((ph[:, 0] / ph[:, 3] + 1.0) * W - 1.0) * 0.5, ((ph[:, 1] / ph[:, 3] + 1.0) * H - 1.0) * 0.5, pv[:, 2]


def seed(cam, A, D, G, image, mask=None, alpha_min=0.5, depth_rel=0.1, min_depth=0.2, max_depth=40.0, stride=1, max_new=None):
    """The plan and the new rows: dict(flags [H,W], counts (selected, holes, in front), n, u, v (kept pixels in rank order), xyz [n,3],
    color [n,3], dist2 [n], and the row values of the insert rule: features_dc [n,3], scaling [n,3], opacity [n], rotation [n,4])."""
    flags = select(A, D, G, mask, alpha_min, depth_rel, min_depth, max_depth, stride)
    W, H = int(cam["W"]), int(cam["H"])
    v, u = np.nonzero(flags)                      # raster order: row-major nonzero is v W + u ascending
    c = u.size
    n = c if max_new is None else min(c, max_new)
    kept = keep(c, n)
    u, v = u[kept], v[kept]
    z = np.asarray(G, np.float64)[v, u]
    xyz = unproject(cam, u, v, z)
    color = np.asarray(image, np.float64)[:, v, u].T
    fx = W / (2.0 * float(np.float32(cam["tanfovx"])))
    fy = H / (2.0 * float(np.float32(cam["tanfovy"])))
    dist2 = (stride * z / ((fx + fy) / 2.0)) ** 2
    return dict(flags=flags, counts=(c, int((flags == HOLE).sum()), int((flags == FRONT).sum())), n=n, u=u, v=v, xyz=xyz, color=color,
                dist2=dist2, features_dc=(color - 0.5) / SH_C0, scaling=np.repeat(np.log(np.sqrt(np.maximum(dist2, 1e-7)))[:, None], 3, 1),
                opacity=np.full(n, math.log(0.1 / 0.9)), rotation=np.tile([1.0, 0.0, 0.0, 0.0], (n, 1)))
