"""Synthetic scenes and cameras for tests and bench (SURVEY.md §8(d), BASELINE.md §2.3).

Camera conventions restate reference src/gaussian_keyframe.cpp:119-204 and include/graphics_utils.h:42-50:
  world_view_transform = Rt^T (so the flat memory is column-major Rt: m[4*c + r]),
  projection P: P00 = 1/tan(fovx/2), P11 = 1/tan(fovy/2), P22 = zfar/(zfar-znear),
                P23 = -zfar*znear/(zfar-znear), P32 = 1;   full_proj = (P @ Rt)^T,
  camera_center = inverse(world_view_transform)[3, :3], fov = 2*atan(pixels / (2*focal)).
numpy only at import; device_camera moves a camera to the device.
"""
import math

import numpy as np

C0 = 0.28209479177387814

# name -> (W, H, fx, fy)   intrinsics of the reference's shipped configs (cfg/ORB_SLAM3/...)
CAMERAS = {
    "tum": (640, 480, 520.9, 520.9),        # Monocular/TUM/tum_freiburg2_xyz.yaml:11-14,29-30
    "replica": (1200, 680, 600.0, 600.0),   # RGB-D/Replica/office0.yaml:11-14,29-30
    "euroc": (752, 480, 458.654, 457.296),  # Stereo/EuRoC/EuRoC.yaml:23-26,43-44
}


def make_camera(W, H, fx, fy, R=None, t=None, znear=0.01, zfar=100.0):
    """Returns dict(viewmatrix[16], projmatrix[16], campos[3], tanfovx, tanfovy, W, H) as float32 numpy."""
    R = np.eye(3) if R is None else np.asarray(R, dtype=np.float64)
    t = np.zeros(3) if t is None else np.asarray(t, dtype=np.float64)
    Rt = np.eye(4)
    Rt[:3, :3] = R
    Rt[:3, 3] = t
    fovx = 2.0 * math.atan(W / (2.0 * fx))
    fovy = 2.0 * math.atan(H / (2.0 * fy))
    tanx, tany = math.tan(fovx * 0.5), math.tan(fovy * 0.5)
    Pm = np.zeros((4, 4))
    Pm[0, 0] = 1.0 / tanx
    Pm[1, 1] = 1.0 / tany
    Pm[3, 2] = 1.0
    Pm[2, 2] = zfar / (zfar - znear)
    Pm[2, 3] = -(zfar * znear) / (zfar - znear)
    view_T = Rt.T.astype(np.float32)                       # world_view_transform_ (row-major tensor)
    proj_T = Pm.T.astype(np.float32)                       # projection_matrix_
    full_T = (view_T.astype(np.float64) @ proj_T.astype(np.float64)).astype(np.float32)  # full_proj_transform_
    campos = np.linalg.inv(view_T.astype(np.float64))[3, :3].astype(np.float32)
    return dict(viewmatrix=view_T.reshape(-1).copy(), projmatrix=full_T.reshape(-1).copy(), campos=campos,
                tanfovx=np.float32(tanx), tanfovy=np.float32(tany), W=int(W), H=int(H), Rt=Rt)


def random_pose(rng, max_angle=0.4, max_trans=0.5):
    """Small random rigid world->camera transform (exercises general matrices; bench uses identity)."""
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    ang = rng.uniform(-max_angle, max_angle)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    R = np.eye(3) + math.sin(ang) * K + (1 - math.cos(ang)) * (K @ K)
    t = rng.uniform(-max_trans, max_trans, size=3)
    return R, t


def make_scene(P, cam, seed=0, sh_degree_max=3, culled_frac=0.05, scale_px=2.4):
    """P Gaussians distributed as SURVEY.md §8(d) in front of `cam`. Returns raw trainer parameters
    (xyz, features_dc [P,1,3], features_rest [P,15,3], scaling (log), rotation (unnormalised), opacity (logit))."""
    rng = np.random.default_rng(seed)
    W, H = cam["W"], cam["H"]
    fx = W / (2.0 * float(cam["tanfovx"]))
    fy = H / (2.0 * float(cam["tanfovy"]))
    z = rng.uniform(0.5, 8.0, size=P)
    n_cull = int(P * culled_frac)
    if n_cull:
        z[rng.choice(P, n_cull, replace=False)] = rng.uniform(-1.0, 0.2, size=n_cull)
    u = rng.uniform(-0.1 * W, 1.1 * W, size=P)
    v = rng.uniform(-0.1 * H, 1.1 * H, size=P)
    zc = np.where(np.abs(z) < 0.05, 0.05, z)
    xc = (u - 0.5 * W) / fx * zc
    yc = (v - 0.5 * H) / fy * zc
    pc = np.stack([xc, yc, z], axis=1)
    Rt = cam["Rt"]
    Rinv = Rt[:3, :3].T
    xyz = (pc - Rt[:3, 3]) @ Rinv.T                         # camera -> world
    sigma = (scale_px / fx) * np.maximum(np.abs(z), 0.5)    # ~scale_px pixels at its depth
    scaling = np.log(sigma)[:, None] + rng.normal(0.0, 0.5, size=(P, 3))
    rotation = rng.normal(size=(P, 4))
    opacity = rng.normal(0.0, 1.5, size=(P, 1))
    rgb = rng.uniform(0.0, 1.0, size=(P, 3))
    M = (sh_degree_max + 1) ** 2
    f_dc = ((rgb - 0.5) / C0)[:, None, :]
    f_rest = rng.normal(0.0, 0.05, size=(P, M - 1, 3))
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return dict(xyz=f32(xyz), features_dc=f32(f_dc), features_rest=f32(f_rest), scaling=f32(scaling),
                rotation=f32(rotation), opacity=f32(opacity))


def _quat_of(R):
    """(w, x, y, z) unit quaternion of the rotation matrix R (Shoemake): the inverse of the covariance's R(q)"""
    tr = np.trace(R)
    if tr > 0:
        s = 2.0 * math.sqrt(tr + 1.0)
        return np.array([0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s])
    i = int(np.argmax(np.diag(R)))
    j, k = (i + 1) % 3, (i + 2) % 3
    s = 2.0 * math.sqrt(1.0 + R[i, i] - R[j, j] - R[k, k])
    q = np.zeros(4)
    q[0] = (R[k, j] - R[j, k]) / s
    q[1 + i] = 0.25 * s
    q[1 + j] = (R[j, i] + R[i, j]) / s
    q[1 + k] = (R[k, i] + R[i, k]) / s
    return q


def planar_scene(per_wall=4000, seed=0, in_plane=0.04, thickness=0.004):
    """A room corner seen from near the identity view: a back wall (z = 5), a left wall (x = -1.5) and a floor (y = 1, the image's y axis
    points down), each covered by `per_wall` flat Gaussians (in-plane scale `in_plane`, scale `thickness` along the plane's normal, which
    is the shortest axis, scaling[2]) with a checker texture. -> (scene, normals [P,3]: the world-space unit normal of each row's plane,
    facing the room)."""
    rng = np.random.default_rng(seed)
    planes = [  # (normal facing the room, origin, in-plane axis a, axis b, extent a, extent b)
        (np.array([0.0, 0.0, -1.0]), np.array([-1.5, -1.5, 5.0]), np.array([1.0, 0.0, 0.0]), np.array([0.0, 1.0, 0.0]), 4.0, 2.5),
        (np.array([1.0, 0.0, 0.0]), np.array([-1.5, -1.5, 1.5]), np.array([0.0, 0.0, 1.0]), np.array([0.0, 1.0, 0.0]), 3.5, 2.5),
        (np.array([0.0, -1.0, 0.0]), np.array([-1.5, 1.0, 1.5]), np.array([1.0, 0.0, 0.0]), np.array([0.0, 0.0, 1.0]), 4.0, 3.5)]
    xyz, nrm, rot, rgb = [], [], [], []
    for k, (n, o, a, b, ea, eb) in enumerate(planes):
        u, v = rng.uniform(0, ea, per_wall), rng.uniform(0, eb, per_wall)
        xyz.append(o + u[:, None] * a + v[:, None] * b)
        nrm.append(np.repeat(n[None], per_wall, 0))
        rot.append(np.repeat(_quat_of(np.stack([a, np.cross(n, a), n], 1))[None], per_wall, 0))   # a right-handed frame with n third
        check = ((np.floor(u / 0.5) + np.floor(v / 0.5)) % 2)[:, None]
        base = np.array([[0.8, 0.3, 0.2], [0.2, 0.7, 0.3], [0.3, 0.3, 0.8]])[k]
        rgb.append(np.clip(base * (0.6 + 0.4 * check) + rng.normal(0, 0.03, (per_wall, 3)), 0, 1))
    P = 3 * per_wall
    rgb = np.concatenate(rgb)
    f32 = lambda x: np.ascontiguousarray(x, dtype=np.float32)
    scene = dict(xyz=f32(np.concatenate(xyz)), features_dc=f32(((rgb - 0.5) / C0)[:, None, :]), features_rest=f32(np.zeros((P, 15, 3))),
                 scaling=f32(np.log(np.repeat([[in_plane, in_plane, thickness]], P, 0))), rotation=f32(np.concatenate(rot)),
                 opacity=f32(np.full((P, 1), 3.0)))
    return scene, f32(np.concatenate(nrm))


def activate(scene):
    """The reference's activations (src/gaussian_model.cpp:48-71) in numpy float32: for CPU-side tests."""
    s = scene
    rot = s["rotation"] / np.maximum(np.linalg.norm(s["rotation"], axis=1, keepdims=True), 1e-12)
    return dict(means3D=s["xyz"], shs=np.concatenate([s["features_dc"], s["features_rest"]], axis=1),
                opacities=(1.0 / (1.0 + np.exp(-s["opacity"]))).astype(np.float32),
                scales=np.exp(s["scaling"]).astype(np.float32), rotations=rot.astype(np.float32))


def target_image(H, W, seed=1):
    rng = np.random.default_rng(seed)
    return rng.uniform(0.0, 1.0, size=(3, H, W)).astype(np.float32)


def device_camera(cam, device):
    """The camera dict the trainer and the renderer take (viewmatrix / projmatrix / campos tensors on `device`, tanfovx / tanfovy
    floats, W / H ints), built from a make_camera dict."""
    import torch
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    return dict(viewmatrix=T(cam["viewmatrix"]), projmatrix=T(cam["projmatrix"]), campos=T(cam["campos"]), tanfovx=float(cam["tanfovx"]),
                tanfovy=float(cam["tanfovy"]), W=int(cam["W"]), H=int(cam["H"]))


def quality_scene():
    """The scene of the quality test: 200 k Gaussians laid out in front of the identity view at 640x480 (TUM focal length), seen from six
    small random poses. -> (scene, [six make_camera dicts])."""
    P, W, H, fx = 200_000, 640, 480, 520.9
    scene = make_scene(P, make_camera(W, H, fx, fx), seed=21, scale_px=3.0)
    cams = [make_camera(W, H, fx, fx, *random_pose(np.random.default_rng(50 + k), max_angle=0.06, max_trans=0.12)) for k in range(6)]
    return scene, cams


def thinned_trainee(scene, seed=3):
    """A trainee for `scene`: about 80 % of its rows, positions, colours, opacities and scales perturbed, f_rest zeroed (so training and
    densification have something to do)."""
    rng = np.random.default_rng(seed)
    keep = rng.random(len(scene["xyz"])) < 0.8
    start = {k: v[keep].copy() for k, v in scene.items()}
    start["xyz"] += rng.normal(0, 0.01, start["xyz"].shape).astype(np.float32)
    start["features_dc"] += rng.normal(0, 0.6, start["features_dc"].shape).astype(np.float32)
    start["features_rest"] *= 0
    start["opacity"] += rng.normal(0, 0.7, start["opacity"].shape).astype(np.float32)
    start["scaling"] += np.float32(0.15)
    return start


def distortion_trainee(scene, normals, seed=1, sigma=0.1, opacity=0.3):
    """A trainee for the depth distortion payoff: the rows of planar_scene's (scene, normals) with positions moved along their plane's
    normal by N(0, sigma) metres and every opacity set to `opacity`, so that several half-transparent rows at different depths share each
    pixel."""
    rng = np.random.default_rng(seed)
    start = {k: v.copy() for k, v in scene.items()}
    start["xyz"] += (normals * rng.normal(0.0, sigma, (len(normals), 1))).astype(np.float32)
    start["opacity"][:] = np.float32(math.log(opacity / (1.0 - opacity)))
    return start
