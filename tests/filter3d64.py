"""Float64 numpy restatement of the 3D smoothing filter (Mip-Splatting) as include/psb200.h defines it: the filter of psb_filter3d, the
widened splat (s', c) and the per-Gaussian backward terms. Cameras are rows of 20 floats: the column-major view matrix (psb_camera.viewmatrix
memory), focal_x, focal_y, W, H."""
import numpy as np

SQRT02 = np.sqrt(0.2)


def view_xyz(xyz, cam):
    """(x, y, z) of the rows in camera `cam`, and the sum of the magnitudes of the terms that form z (the scale of its float32 rounding)"""
    m = np.asarray(cam[:16], np.float64)
    p = np.asarray(xyz, np.float64)
    x = m[0] * p[:, 0] + m[4] * p[:, 1] + m[8] * p[:, 2] + m[12]
    y = m[1] * p[:, 0] + m[5] * p[:, 1] + m[9] * p[:, 2] + m[13]
    z = m[2] * p[:, 0] + m[6] * p[:, 1] + m[10] * p[:, 2] + m[14]
    zs = np.abs(m[2] * p[:, 0]) + np.abs(m[6] * p[:, 1]) + np.abs(m[10] * p[:, 2]) + abs(m[14])
    return x, y, z, zs


def filter3d(xyz, cams, rtol=1e-6):
    """The filter of P rows for K cameras. Returns dict(filter [P], seen [P] bool, d [P] (inf: unseen), F, zs [P] (rounding scale of the
    depth that gave d), near [P] bool: for some camera, a depth or margin test of the row lies within rtol (relative) of its boundary)."""
    xyz = np.asarray(xyz, np.float64).reshape(-1, 3)
    cams = np.asarray(cams, np.float64).reshape(-1, 20)
    P = xyz.shape[0]
    d, zs = np.full(P, np.inf), np.zeros(P)
    near = np.zeros(P, bool)
    for cam in cams:
        fx, fy, W, H = cam[16:20]
        x, y, z, s = view_xyz(xyz, cam)
        with np.errstate(divide="ignore", invalid="ignore"):
            u = x / z * fx + W / 2
            v = y / z * fy + H / 2
        front = z > 0.2
        vis = front & (u >= -0.15 * W) & (u <= 1.15 * W) & (v >= -0.15 * H) & (v <= 1.15 * H)
        near |= np.abs(z - 0.2) <= rtol * 0.2
        for a, lo, hi in ((u, -0.15 * W, 1.15 * W), (v, -0.15 * H, 1.15 * H)):
            scale = np.maximum(np.abs(a), max(abs(lo), abs(hi)))
            near |= (z > 0.2 * (1 - rtol)) & ((np.abs(a - lo) <= rtol * scale) | (np.abs(a - hi) <= rtol * scale))
        better = vis & (z < d)
        d = np.where(better, z, d)
        zs = np.where(better, s, zs)
    seen = np.isfinite(d)
    F = float(cams[:, 16].max()) if len(cams) else 0.0
    if not seen.any():
        return dict(filter=np.zeros(P), seen=seen, d=d, F=F, zs=zs, near=near)
    dmax = d[seen].max()
    zs = np.where(seen, zs, zs[seen][np.argmax(d[seen])])
    return dict(filter=np.where(seen, d, dmax) / F * SQRT02, seen=seen, d=d, F=F, zs=zs, near=near)


def widen(s, f):
    """(s', c) of activated scales s [P,3] and filters f [P]: s' = sqrt(s^2 + f^2), c = sqrt(prod s^2 / prod s'^2)"""
    s = np.asarray(s, np.float64)
    f2 = np.square(np.asarray(f, np.float64))[:, None]
    sp = np.sqrt(s * s + f2)
    return sp, np.sqrt(np.prod(s * s, axis=1) / np.prod(sp * sp, axis=1))


def quat_rot(q):
    q = np.asarray(q, np.float64)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], 1)


def cov3d(s, q):
    """R diag(s)^2 R^T [P,3,3]"""
    R = quat_rot(q)
    return R @ (np.asarray(s, np.float64)[:, :, None] ** 2 * np.transpose(R, (0, 2, 1)))


def backward(s, o, f, dL_dsp, g):
    """dL/ds [P,3] and dL/do [P] of the activated scale s and opacity o, given dL/ds' [P,3] and g = dL/d(o c) [P]:
    dL/ds_c = dL/ds'_c s_c / s'_c + o c g f^2 / (s_c s'_c^2), dL/do = c g"""
    s = np.asarray(s, np.float64)
    sp, c = widen(s, f)
    f2 = np.square(np.asarray(f, np.float64))[:, None]
    k = (np.asarray(o, np.float64) * c * np.asarray(g, np.float64))[:, None]
    return dL_dsp * s / sp + k * f2 / (s * sp * sp), c * g
