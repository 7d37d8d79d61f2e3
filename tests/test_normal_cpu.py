"""CPU: rendered normals without a device. The float64 restatement (tests/normal64.py) against analytic planes and independent per-pixel
and per-row loops; the C entries' refusals before any CUDA call; the Python front end's checks against a stub library; the
data-parallel refusal; the binding."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

import normal64
import splat64 as s64
from photo_slam_b200 import _lib, trainer
from test_pixel_grads_cpu import _cpu_trainer

ONE = 4096  # fake non-null device pointer; never dereferenced because validation fails first
E = -1      # PSB_ERR_ARG
W, H, TX, TY = 40, 30, 0.6, 0.45


def _plane_depth(n, d, W=W, H=H, tx=TX, ty=TY):
    """depth [H,W] of the plane n . X = d seen through the pixel centres (the seeding rule's rays)"""
    fx, fy = W / (2 * tx), H / (2 * ty)
    v, u = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    ray = np.stack([(u + 0.5 - W / 2) / fx, (v + 0.5 - H / 2) / fy, np.ones_like(u)], 0)
    return d / np.tensordot(n, ray, axes=1)


# (tilt, tan_fov): the view is narrowed as the plane approaches grazing so that every ray still meets it in front of the camera
@pytest.mark.parametrize("tilt_deg,tan_fov", [(0.0, 0.6), (20.0, 0.6), (45.0, 0.4), (70.0, 0.15), (85.0, 0.05)])
def test_sensor_normals_of_tilted_planes(tilt_deg, tan_fov):
    t = math.radians(tilt_deg)
    n = np.array([math.sin(t) * 0.6, math.sin(t) * 0.8, -math.cos(t)])     # faces the camera
    z = _plane_depth(n, -3.0, tx=tan_fov, ty=tan_fov)
    assert (z > 0).all()
    out = normal64.depth_normals64(torch.from_numpy(z), W, H, tan_fov, tan_fov, max_rel_jump=10.0).numpy()
    inner = out[:, 1:-1, 1:-1].reshape(3, -1)
    assert np.abs(inner - n[:, None]).max() < 1e-9
    assert not out[:, 0].any() and not out[:, -1].any() and not out[:, :, 0].any() and not out[:, :, -1].any()


def _loop(z, W, H, tx, ty, jump):
    fx, fy = W / (2 * tx), H / (2 * ty)
    X = lambda u, v: np.array([(u + 0.5 - W / 2) * z[v, u] / fx, (v + 0.5 - H / 2) * z[v, u] / fy, z[v, u]])
    out = np.zeros((3, H, W))
    for v in range(1, H - 1):
        for u in range(1, W - 1):
            zs = [z[v, u], z[v, u - 1], z[v, u + 1], z[v - 1, u], z[v + 1, u]]
            if not all(np.isfinite(q) and q > 0 for q in zs) or any(abs(q - zs[0]) > jump * zs[0] for q in zs[1:]):
                continue
            c = np.cross(X(u + 1, v) - X(u - 1, v), X(u, v + 1) - X(u, v - 1))
            length = np.linalg.norm(c)
            if length == 0:
                continue
            nn = c / length
            out[:, v, u] = nn if nn @ X(u, v) < 0 else -nn
    return out


def test_sensor_normals_equal_a_per_pixel_loop_with_holes_and_edges():
    rng = np.random.default_rng(0)
    z = 2.0 + 0.3 * rng.random((H, W))
    z[:, 25:] += 1.5                                         # a depth edge
    z[rng.random((H, W)) < 0.05] = 0.0
    z[rng.random((H, W)) < 0.03] = np.nan
    z[rng.random((H, W)) < 0.03] = -1.0
    z[rng.random((H, W)) < 0.02] = np.inf
    ref = _loop(z, W, H, TX, TY, 0.05)
    out = normal64.depth_normals64(torch.from_numpy(z), W, H, TX, TY, 0.05).numpy()
    assert np.abs(out - ref).max() < 1e-12
    zero = ~(out != 0).any(0)
    assert zero[:, 24:26].all(), "the depth edge gives zero"
    bad = ~np.isfinite(z) | (z <= 0)
    assert zero[bad].all() and zero[0].all() and zero[-1].all()
    u, v = np.meshgrid(np.arange(W) + 0.5 - W / 2, np.arange(H) + 0.5 - H / 2, indexing="xy")
    ray = np.stack([u * 2 * TX / W, v * 2 * TY / H, np.ones((H, W))], 0)      # X(u, v) / z
    assert ((out * ray).sum(0)[~zero] < 0).all(), "the sensor normal faces the camera"


def _rot(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def test_gaussian_normals_equal_a_per_row_loop():
    import photo_slam_b200.synthetic as syn
    cam = syn.make_camera(64, 48, 50.0, 50.0, *syn.random_pose(np.random.default_rng(3)))
    sc = syn.make_scene(300, cam, seed=4)
    sc["scaling"][:7] = np.float32(-3.0)                  # ties: the lowest index wins
    raw = s64.raw64(sc, "cpu")
    c64 = s64.camera64(cam, "cpu")
    n = normal64.gaussian_normals(raw, c64).numpy()
    Vm = np.asarray(cam["viewmatrix"], np.float64).reshape(4, 4).T       # V[r][c] = viewmatrix[4 c + r]
    for i in range(300):
        q = raw["rotation"][i].numpy()
        q = q / max(np.linalg.norm(q), 1e-12)
        k = int(np.argmin(raw["scaling"][i].numpy()))
        r = _rot(q)[:, k]
        m = Vm[:3, :3] @ r
        t = Vm[:3, :3] @ raw["xyz"][i].numpy() + Vm[:3, 3]
        want = m if m @ t <= 0 else -m
        assert np.abs(n[i] - want).max() < 1e-12, i
        assert n[i] @ t <= 0
    assert (np.argmin(sc["scaling"][:7], 1) == 0).all()
    # the shortest axis is an eigenvector of the covariance with eigenvalue exp(2 s_min)
    cov = s64.quat_cov(torch.exp(raw["scaling"]), raw["rotation"] / raw["rotation"].norm(dim=1, keepdim=True))
    Sig = torch.stack([cov[:, [0, 1, 2]], cov[:, [1, 3, 4]], cov[:, [2, 4, 5]]], 1).numpy()
    Rw = np.linalg.inv(Vm[:3, :3])
    for i in range(20):
        rw = Rw @ n[i]
        lam = math.exp(2 * raw["scaling"][i].min().item())
        assert np.abs(Sig[i] @ rw - lam * rw).max() < 1e-9 * max(1.0, np.abs(Sig[i]).max())


def test_normal_l1_equals_a_loop():
    rng = np.random.default_rng(1)
    N = torch.from_numpy(rng.normal(size=(3, 5, 7)))
    G = torch.from_numpy(rng.normal(size=(3, 5, 7)))
    G[:, 1, 2] = 0.0
    G[:, 3, :] = 0.0
    mask = torch.ones((3, 5, 7), dtype=torch.float64)
    mask[0, 4, 4] = 0.0
    mask[1:, 0, :] = 0.0                                     # only mask[0] is read
    tot, cnt = 0.0, 0
    for v in range(5):
        for u in range(7):
            if (G[:, v, u] != 0).any() and mask[0, v, u] != 0:
                tot += float((N[:, v, u] - G[:, v, u]).abs().sum())
                cnt += 1
    assert abs(float(normal64.normal_l1_64(N, G, mask)) - tot / cnt) < 1e-12
    assert float(normal64.normal_l1_64(N, torch.zeros_like(G))) == 0.0


# ---- the C entries' refusals ---------------------------------------------------------------------------------------------------------
def _cam(W=32, H=24, tanx=0.5, tany=0.5):
    c = trainer._Camera()
    c.viewmatrix, c.projmatrix, c.campos, c.tan_fovx, c.tan_fovy, c.width, c.height = ONE, ONE, ONE, tanx, tany, W, H
    return c


def _rejects(L, name, *args):
    assert getattr(L, name)(*args) == E, (name, args)
    assert name.encode() in L.psb_last_error(), (name, L.psb_last_error())


def test_depth_normals_refuses_bad_arguments_without_a_device():
    L = trainer._bind()
    for cam, d, j, o in ((None, ONE, 0.05, ONE), (_cam(), None, 0.05, ONE), (_cam(), ONE, 0.05, None), (_cam(W=0), ONE, 0.05, ONE),
                         (_cam(H=-1), ONE, 0.05, ONE), (_cam(tanx=0.0), ONE, 0.05, ONE), (_cam(tany=math.inf), ONE, 0.05, ONE),
                         (_cam(tanx=math.nan), ONE, 0.05, ONE), (_cam(), ONE, 0.0, ONE), (_cam(), ONE, -1.0, ONE), (_cam(), ONE, math.nan, ONE),
                         (_cam(), ONE, math.inf, ONE)):
        _rejects(L, "psb_depth_normals", C.byref(cam) if cam is not None else None, d, j, o, None)


def test_step_normal_refuses_bad_terms_without_a_device():
    L = trainer._bind()
    t = C.c_void_p()
    assert L.psb_trainer_create(C.byref(t)) == 0
    try:
        m, cam, step = trainer._Model(), _cam(), trainer._Step()
        for i in range(6):
            m.param[i] = m.exp_avg[i] = m.exp_avg_sq[i] = ONE
        step.step, step.sh_degree = 1, 3
        for gt, lam in ((ONE, 0.0), (None, 0.5), (ONE, -1.0), (ONE, math.nan), (ONE, math.inf), (None, -0.5)):
            nrm = trainer._Normal(gt, lam, None)
            _rejects(L, "psb_trainer_step_normal", t, 10, 16, C.byref(m), C.byref(cam), ONE, ONE, None, C.byref(step), None, None, None, None,
                     C.byref(nrm), None)
        # no forward pass has run: a normal gradient is refused like any other stale pass
        px = trainer._PixelGrads(ONE, None, None)
        assert L.psb_trainer_backward_pixels_normal(t, 1, 10, 16, C.byref(m), C.byref(cam), ONE, C.byref(px), ONE, C.byref(step), None, None) == E
        out = (C.c_float * 5)()
        assert L.psb_trainer_result_normal(t, out, None, None) == E
    finally:
        L.psb_trainer_destroy(t)


def test_header_declares_and_library_exports_the_entries():
    names = _lib.exported_symbols()
    L = _lib.lib()
    for n in ("psb_trainer_forward_normal", "psb_trainer_backward_pixels_normal", "psb_trainer_step_normal", "psb_trainer_result_normal",
              "psb_depth_normals"):
        assert n in names and hasattr(L, n), n


# ---- the Python front end against a stub library -------------------------------------------------------------------------------------
class _StubL:
    """Records the trainer entry points the front end calls; every call succeeds."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("psb_"):
            raise AttributeError(name)
        return lambda *a: self.calls.append(name) or 0


@pytest.fixture
def stubbed(monkeypatch):
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: types.SimpleNamespace(cuda_stream=None))
    tr, m, cam = _cpu_trainer()
    L = _StubL()
    monkeypatch.setattr(trainer, "_bind", lambda: L)
    tr.L = L
    tr.result = lambda: None
    return tr, m, cam, L


def test_the_default_step_stays_the_exposure_call(stubbed):
    tr, m, cam, L = stubbed
    H, W = cam["H"], cam["W"]
    gt = torch.rand(3, H, W)
    tr.trainForOneIteration(cam, gt)
    assert L.calls[-1] == "psb_trainer_step_exposure"
    tr.trainForOneIteration(cam, gt, gt_normal=torch.zeros(3, H, W), lambda_normal=0.1)
    assert L.calls[-1] == "psb_trainer_step_normal"
    tr.trainForOneIteration(cam, gt, out_normal=torch.zeros(3, H, W))
    assert L.calls[-1] == "psb_trainer_step_normal"
    assert m.step_ == 3 and tr.iteration == 3
    # the retry record repeats the call with its normal target
    n = len(L.calls)
    tr._last.repeat()
    assert L.calls[n:] == ["psb_trainer_step_normal"]
    tr.render(cam, check=False)
    assert L.calls[-1] == "psb_trainer_forward"
    tr.render(cam, check=False, out_normal=torch.zeros(3, H, W))
    assert L.calls[-1] == "psb_trainer_forward_normal"
    tr.backwardPixels(torch.zeros(3, H, W), grads=[torch.zeros_like(t) for t in m.tensors()])
    assert L.calls[-1] == "psb_trainer_backward_pixels"
    tr.backwardPixels(torch.zeros(3, H, W), grads=[torch.zeros_like(t) for t in m.tensors()], dL_dnormal=torch.zeros(3, H, W))
    assert L.calls[-1] == "psb_trainer_backward_pixels_normal"


def test_argument_checks_before_any_c_call(stubbed):
    tr, m, cam, L = stubbed
    H, W = cam["H"], cam["W"]
    gt = torch.rand(3, H, W)
    for kw in (dict(gt_normal=torch.zeros(3, W, H), lambda_normal=0.1), dict(gt_normal=torch.zeros(3, H, W, dtype=torch.float64), lambda_normal=0.1),
               dict(gt_normal=torch.zeros(H, W), lambda_normal=0.1), dict(out_normal=torch.zeros(3, H, W)[:, :, ::2]),
               dict(out_normal=torch.zeros(1, H, W))):
        with pytest.raises(ValueError):
            tr.trainForOneIteration(cam, gt, **kw)
    with pytest.raises(ValueError):
        tr.render(cam, check=False, out_normal=torch.zeros(3, W, H))
    assert L.calls == []
    tr.render(cam, check=False)                  # a render without the plane takes no normal gradient
    n = len(L.calls)
    with pytest.raises(ValueError, match="dL_dnormal"):
        tr.backwardPixels(torch.zeros(3, H, W), dL_dnormal=torch.zeros(3, H, W))
    tr.render(cam, check=False, out_normal=torch.zeros(3, H, W))
    with pytest.raises(ValueError):
        tr.backwardPixels(torch.zeros(3, H, W), dL_dnormal=torch.zeros(H, W))
    for bad in (dict(depth=torch.zeros(W, H)), dict(depth=torch.zeros(H, W, dtype=torch.float64)), dict(depth=None),
                dict(depth=torch.zeros(H, W), max_rel_jump=0.0), dict(depth=torch.zeros(H, W), max_rel_jump=math.nan),
                dict(depth=torch.zeros(H, W), out=torch.zeros(3, W, H))):
        with pytest.raises(ValueError):
            trainer.normals_from_depth(cam, **bad)
    assert L.calls[n:] == ["psb_trainer_forward_normal"]
    assert m.step_ == 0 and tr.iteration == 0
    trainer.normals_from_depth(cam, torch.ones(H, W))
    assert L.calls[-1] == "psb_depth_normals"


def test_data_parallel_trainer_refuses_normals():
    dp = object.__new__(trainer.DataParallelTrainer)
    for kw in (dict(gt_normal=torch.zeros(3, 2, 2), lambda_normal=0.1), dict(out_normal=torch.zeros(3, 2, 2)), dict(lambda_normal=0.1)):
        with pytest.raises(NotImplementedError, match="normal term"):
            dp.trainForOneIteration(dict(), None, **kw)
