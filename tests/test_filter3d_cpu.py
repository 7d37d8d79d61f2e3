"""CPU: the 3D smoothing filter. The float64 restatement (tests/filter3d64.py) on constructed rows (near plane, the +-15 % margins, unseen
rows, no row seen, no camera), the widened covariance, the backward terms against central differences, and the Python front end against a
stub library: camera validation and packing, the invalidating methods, the trainer's refusals."""
import types

import numpy as np
import pytest
import torch

import filter3d64 as f64
from photo_slam_b200 import trainer
from test_pixel_grads_cpu import _cpu_trainer


def _cam(fx=128.0, fy=64.0, W=200, H=160):
    """identity view (camera at the origin looking down +z): x, y, z of a row are its coordinates"""
    return np.concatenate([np.eye(4).reshape(-1), [fx, fy, W, H]])


def _at(u, v, z, fx=128.0, fy=64.0, W=200, H=160):
    """the row that projects to pixel (u, v) at depth z in _cam(); with power-of-two focal lengths and depths the projection of a pixel on
    a margin lands exactly on it"""
    return [(u - W / 2) / fx * z, (v - H / 2) / fy * z, z]


def test_filter_rule_on_constructed_rows():
    W, H = 200.0, 160.0
    lo_u, hi_u, lo_v, hi_v = -0.15 * W, 1.15 * W, -0.15 * H, 1.15 * H
    rows = [_at(100, 80, 1.0),                          # 0 centre
            _at(100, 80, 0.1),                          # 1 in front of the near plane
            _at(100, 80, 0.2),                          # 2 exactly on it: z > 0.2 is required
            _at(lo_u, 80, 2.0),                         # 3 exactly on the left margin: seen
            _at(lo_u - 1e-9, 80, 2.0),                  # 4 just outside it
            _at(hi_u, 80, 4.0),                         # 5 exactly on the right margin
            _at(hi_u + 1e-9, 80, 4.0),                  # 6 just outside
            _at(100, lo_v, 0.5),                        # 7 top margin
            _at(100, hi_v, 8.0),                        # 8 bottom margin
            _at(100, hi_v + 1e-9, 8.0),                  # 9 just outside
            [0.0, 0.0, -1.0]]                           # 10 behind the camera
    xyz = np.array(rows)
    r = f64.filter3d(xyz, [_cam()])
    seen = [True, False, False, True, False, True, False, True, True, False, False]
    assert r["seen"].tolist() == seen
    assert r["F"] == 128.0
    d = np.array([1.0, 0, 0, 2.0, 0, 4.0, 0, 0.5, 8.0, 0, 0])
    want = np.where(seen, d, 8.0) / 128.0 * np.sqrt(0.2)     # unseen rows take the largest d of a seen row
    np.testing.assert_allclose(r["filter"], want, rtol=1e-12)
    assert r["near"][[2, 3, 4, 5, 6, 7, 8, 9]].all() and not r["near"][[0, 10]].any()


def test_min_depth_over_cameras_and_max_focal():
    # a second camera 1 m behind the first (view translation +1 in z) with a larger focal length
    c2 = _cam(fx=300.0, fy=300.0, W=640, H=480)
    c2[14] = 1.0
    xyz = np.array([_at(100, 80, 1.0), _at(100, 80, 0.15)])
    r = f64.filter3d(xyz, [_cam(), c2])
    assert r["seen"].tolist() == [True, True] and r["F"] == 300.0
    np.testing.assert_allclose(r["d"], [1.0, 1.15])           # camera 1 sees row 0 nearer; only camera 2 sees row 1 (z 0.15 in camera 1)
    np.testing.assert_allclose(r["filter"], np.array([1.0, 1.15]) / 300.0 * np.sqrt(0.2))


def test_no_row_seen_and_no_camera():
    xyz = np.array([[0.0, 0.0, -1.0], [0.0, 0.0, 0.1]])
    for cams in ([_cam()], np.zeros((0, 20))):
        r = f64.filter3d(xyz, cams)
        assert not r["seen"].any()
        assert (r["filter"] == 0).all()


def test_widened_covariance_is_sigma_plus_f2_identity():
    rng = np.random.default_rng(1)
    s, q, f = np.exp(rng.normal(-3, 1, (50, 3))), rng.normal(size=(50, 4)), np.abs(rng.normal(0, 0.05, 50))
    sp, c = f64.widen(s, f)
    np.testing.assert_allclose(f64.cov3d(sp, q), f64.cov3d(s, q) + f[:, None, None] ** 2 * np.eye(3), rtol=1e-10, atol=1e-16)
    np.testing.assert_allclose(c, np.sqrt(np.linalg.det(f64.cov3d(s, q)) / np.linalg.det(f64.cov3d(sp, q))), rtol=1e-8)
    assert (c <= 1).all() and (c > 0).all()
    sp0, c0 = f64.widen(s, np.zeros(50))
    assert (sp0 == s).all() and (c0 == 1).all()


def test_backward_terms_against_central_differences():
    rng = np.random.default_rng(2)
    n = 20
    s, o, f = np.exp(rng.normal(-3, 0.7, (n, 3))), 1 / (1 + np.exp(-rng.normal(size=n))), np.abs(rng.normal(0, 0.05, n))
    a, b = rng.normal(size=(n, 3)), rng.normal(size=n)

    def loss(s_, o_):   # L = sum a s' + b o c: dL/ds' = a, dL/d(o c) = b
        sp, c = f64.widen(s_, f)
        return (a * sp).sum(1) + b * o_ * c

    gs, go = f64.backward(s, o, f, a, b)
    h = 1e-7
    for ax in range(3):
        e = np.zeros_like(s)
        e[:, ax] = h * s[:, ax]
        fd = (loss(s + e, o) - loss(s - e, o)) / (2 * e[:, ax])
        np.testing.assert_allclose(gs[:, ax], fd, rtol=1e-5, atol=1e-9)
    fd = (loss(s, o + h) - loss(s, o - h)) / (2 * h)
    np.testing.assert_allclose(go, fd, rtol=1e-6, atol=1e-9)


class _StubL:
    """The entry points the model's methods call, doing nothing; psb_filter3d records its arguments."""

    def __init__(self):
        self.filter_calls = []

    def psb_filter3d(self, P, xyz, K, cams, out, seen, stream):
        self.filter_calls.append((P, K, cams))
        seen._obj.value = 3
        return 0

    def psb_densify_plan(self, P, src, cfg, ws, counts, stream):
        counts[0] = P          # (the plans keep every row: the model keeps its size)
        return 0

    def psb_prune_plan(self, P, mask, ws, counts, stream):
        counts[0] = P
        return 0

    def __getattr__(self, name):
        if name.endswith("_bytes"):
            return lambda *a: 16
        return lambda *a: 0


@pytest.fixture
def stub(monkeypatch):
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: types.SimpleNamespace(cuda_stream=None))
    L = _StubL()
    monkeypatch.setattr(trainer, "_bind", lambda: L)
    return L


def _good_cam(**kw):
    c = dict(viewmatrix=torch.eye(4).reshape(-1), projmatrix=torch.zeros(16), campos=torch.zeros(3), tanfovx=0.5, tanfovy=0.25, W=64, H=48)
    c.update(kw)
    return c


def test_compute_filter3d_validates_and_packs_the_cameras(stub, monkeypatch):
    tr, m, _ = _cpu_trainer()
    bad = [dict(tanfovx=0.0), dict(tanfovy=-1.0), dict(tanfovx=float("nan")), dict(tanfovx=float("inf")), dict(W=0), dict(H=-4), dict(W=10.5),
           dict(viewmatrix=torch.zeros(12)), dict(viewmatrix=torch.full((16,), float("nan")))]
    for kw in bad:
        with pytest.raises(ValueError, match="computeFilter3D"):
            m.computeFilter3D([_good_cam(), _good_cam(**kw)])
    with pytest.raises(ValueError, match="not a camera dict"):
        m.computeFilter3D([dict(W=4)])
    assert stub.filter_calls == [] and m.filter_3D_ is None
    packed = {}
    real_stack = torch.stack

    def spy(rows, *a, **k):
        packed["rows"] = real_stack(rows, *a, **k)
        return packed["rows"]
    monkeypatch.setattr(torch, "stack", spy)
    assert m.computeFilter3D([_good_cam(), _good_cam(W=128, tanfovx=0.25)]) == 3
    P, K, _ = stub.filter_calls[-1]
    assert (P, K) == (m.num_points(), 2)
    rows = packed["rows"]
    assert rows.shape == (2, 20)
    assert torch.equal(rows[0, :16], torch.eye(4, dtype=torch.float64).reshape(-1))
    assert rows[0, 16:].tolist() == [64.0, 96.0, 64.0, 48.0] and rows[1, 16:].tolist() == [256.0, 96.0, 128.0, 48.0]
    assert m.filter_3D_.shape == (m.num_points(),)
    monkeypatch.setattr(torch, "stack", real_stack)
    assert m.computeFilter3D([]) == 3 and stub.filter_calls[-1][1:] == (0, None)


def _with_filter(m):
    m.filter_3D_ = torch.zeros(m.num_points())
    return m


def test_every_row_changing_method_drops_the_filter(stub, monkeypatch, tmp_path):
    from photo_slam_b200 import points
    tr, m, _ = _cpu_trainer()
    cases = {
        "densifyAndPrune": lambda: m.densifyAndPrune(0.001, 0.005, 1.0, 0),
        "prunePoints": lambda: m.prunePoints(torch.zeros(m.num_points(), dtype=torch.bool)),
        "relocateGaussians": lambda: m.relocateGaussians(),
        "addNewGaussians": lambda: m.addNewGaussians(10 ** 6, 1.5),
        "increasePcd": lambda: m.increasePcd(torch.zeros((4, 3)), torch.zeros((4, 3))),
        "applyScaledTransformation": lambda: m.applyScaledTransformation(1.1, np.eye(4)),
        "scaledTransformVisiblePointsOfKeyframe": lambda: m.scaledTransformVisiblePointsOfKeyframe(
            torch.zeros(m.num_points(), dtype=torch.uint8), torch.eye(4), torch.eye(4), torch.eye(4), 0, 10),
    }
    monkeypatch.setattr(points, "distCUDA2", lambda p: torch.ones(p.size(0)))
    monkeypatch.setattr(points, "transformPoints", lambda p, T: p.clone())
    monkeypatch.setattr(points, "scaleAndTransformThenMarkVisiblePoints", lambda *a: 0)
    for name, call in cases.items():
        _with_filter(m)
        m.filter3D()
        call()
        assert m.filter_3D_ is None, name
        with pytest.raises(ValueError, match="computeFilter3D"):
            m.filter3D()
    # loadPly
    m.savePly(str(tmp_path / "a.ply"))
    _with_filter(m)
    m.loadPly(str(tmp_path / "a.ply"))
    assert m.filter_3D_ is None
    # a filter of another row count is stale too
    m.filter_3D_ = torch.zeros(m.num_points() + 1)
    with pytest.raises(ValueError, match="stale"):
        m.getOpacityWithFilter3D()


def test_snapshot_restore_carries_the_filter():
    tr, m, _ = _cpu_trainer()
    m.filter_3D_ = torch.arange(m.num_points(), dtype=torch.float32)
    snap = m.snapshot()
    m.filter_3D_.zero_()
    keep = m.filter_3D_
    m.restore(snap)
    assert m.filter_3D_ is keep and torch.equal(keep, torch.arange(m.num_points(), dtype=torch.float32))
    m.filter_3D_ = None
    m.restore(snap)
    assert torch.equal(m.filter_3D_, torch.arange(m.num_points(), dtype=torch.float32))
    m.filter_3D_ = torch.ones(m.num_points())
    m.restore(dict(snap, filter_3D=None))
    assert m.filter_3D_ is None


def test_torch_filtered_activations_and_fused_export(tmp_path):
    from photo_slam_b200 import io
    tr, m, _ = _cpu_trainer()
    m.filter_3D_ = torch.rand(m.num_points()) * 0.05
    sp, c = f64.widen(torch.exp(m.scaling_).double().numpy(), m.filter_3D_.double().numpy())
    np.testing.assert_allclose(m.getScalingWithFilter3D().double().numpy(), sp, rtol=1e-5)
    o = torch.sigmoid(m.opacity_).double().numpy().reshape(-1)
    np.testing.assert_allclose(m.getOpacityWithFilter3D().double().numpy().reshape(-1), o * c, rtol=1e-5)
    plain, fused = str(tmp_path / "plain.ply"), str(tmp_path / "fused.ply")
    m.savePly(plain)
    m.savePly(fused, fuse_filter3d=True)
    a, b = io.load_ply(plain, 3), io.load_ply(fused, 3)
    for k in ("xyz", "features_dc", "features_rest", "rotation"):
        assert np.array_equal(a[k], b[k]), k
    assert np.array_equal(a["scaling"], m.scaling_.detach().numpy()) and np.array_equal(a["opacity"], m.opacity_.detach().numpy())
    np.testing.assert_allclose(np.exp(b["scaling"]), sp, rtol=1e-5)
    np.testing.assert_allclose(1 / (1 + np.exp(-b["opacity"].reshape(-1))), o * c, rtol=1e-5)


def test_trainer_refuses_a_missing_or_stale_filter(monkeypatch):
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: types.SimpleNamespace(cuda_stream=None))
    tr, m, cam = _cpu_trainer()
    ft = trainer.GaussianTrainer(m, background=torch.zeros(3), filter3d=True)
    assert ft.filter3d and not tr.filter3d
    gt = torch.zeros((3, cam["H"], cam["W"]))
    for f in (None, torch.zeros(m.num_points() - 1)):
        m.filter_3D_ = f
        for call in (lambda: ft.render(cam), lambda: ft.trainForOneIteration(cam, gt)):
            with pytest.raises(ValueError, match="computeFilter3D"):
                call()
        ft._last_render, ft._pass = (cam, None, None, None, None), 1
        with pytest.raises(ValueError, match="computeFilter3D"):
            ft.backwardPixels(torch.zeros((3, cam["H"], cam["W"])))
    assert (m.step_, ft.iteration) == (0, 0)
    with pytest.raises(NotImplementedError, match="3D filter"):
        trainer.DataParallelTrainer(m, filter3d=True)
