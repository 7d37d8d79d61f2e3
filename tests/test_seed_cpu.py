"""CPU: depth-guided seeding without a device. The restatement (tests/seed64.py) against a per-pixel loop, the cap rule, the unprojection
against the forward's projection; the C entries' refusals before any CUDA call; the Python front end against a stub library (argument
checks, the empty-model path, the MCMC default of max_new, what the model ends in); the data-parallel refusal; the binding."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn
import seed64
from photo_slam_b200 import _lib, trainer
from test_pixel_grads_cpu import _cpu_trainer

ONE = 4096  # fake non-null device pointer; never dereferenced because validation fails first
E = -1      # PSB_ERR_ARG


# ---- the restatement ----------------------------------------------------------------------------------------------------------------
def _planes(H=23, W=31, seed=0):
    """A, D, G and a mask with exact ties at alpha_min and in the in-front comparison, NaN / inf / <= 0 depths and masked pixels."""
    rng = np.random.default_rng(seed)
    A = rng.uniform(0, 1, (H, W)).astype(np.float32)
    G = rng.uniform(0.1, 8, (H, W)).astype(np.float32)
    D = (A * G * rng.uniform(0.7, 1.3, (H, W))).astype(np.float32)
    A[rng.random((H, W)) < 0.1] = np.float32(0.5)                           # ties at alpha_min
    tie = rng.random((H, W)) < 0.1                                          # G A == k D exactly: not in front
    A[tie] = np.float32(1.0)
    G[tie] = (np.float32(1) - np.float32(0.1)) * D[tie]                     # the float32 product k D: G A == k D exactly
    G[rng.random((H, W)) < 0.05] = np.nan
    G[rng.random((H, W)) < 0.05] = np.inf
    G[rng.random((H, W)) < 0.05] = 0.0
    G[rng.random((H, W)) < 0.05] = -1.0
    G[rng.random((H, W)) < 0.03] = np.float32(0.2)                          # == min_depth: invalid
    mask = np.ones((3, H, W), np.float32)
    mask[0][rng.random((H, W)) < 0.1] = 0.0
    mask[1:] = 0.0                                                          # only mask[0] is read
    return A, D, G, mask


def _loop(A, D, G, mask, alpha_min, depth_rel, min_depth, max_depth, stride):
    H, W = A.shape
    k = np.float32(1) - np.float32(depth_rel)
    out = np.zeros((H, W), np.uint8)
    for v in range(H):
        for u in range(W):
            if u % stride or v % stride:
                continue
            g, a, d = G[v, u], A[v, u], D[v, u]
            if not (math.isfinite(g) and min_depth < g < max_depth) or (mask is not None and mask[0, v, u] == 0):
                continue
            if a < np.float32(alpha_min):
                out[v, u] = seed64.HOLE
            elif np.float32(g * a) < np.float32(k * d):
                out[v, u] = seed64.FRONT
    return out


@pytest.mark.parametrize("stride", [1, 2, 3])
def test_selection_equals_a_per_pixel_loop(stride):
    A, D, G, mask = _planes()
    for m in (mask, None):
        for cfg in (dict(alpha_min=0.5, depth_rel=0.1, min_depth=0.2, max_depth=40.0), dict(alpha_min=1.0, depth_rel=0.0, min_depth=0.0, max_depth=5.0),
                    dict(alpha_min=0.25, depth_rel=1.0, min_depth=0.2, max_depth=np.inf)):
            got = seed64.select(A, D, G, m, stride=stride, **cfg)
            want = _loop(A, D, G, m, stride=stride, **cfg)
            assert np.array_equal(got, want), (stride, cfg)
    got = seed64.select(A, D, G, mask, stride=stride)
    assert (got == seed64.HOLE).sum() > 5 and (got == seed64.FRONT).sum() > 5
    k = np.float32(1) - np.float32(0.1)
    with np.errstate(invalid="ignore"):
        ties = (G * A == k * D) & (A >= np.float32(0.5)) & (G > np.float32(0.2)) & (G < np.float32(40)) & (mask[0] != 0)
        assert ties[::stride, ::stride].sum() > 0 and not got[ties].any()      # an exact tie is not in front
        assert ((A == np.float32(0.5)) & (got != 0))[::stride, ::stride].any()  # A == alpha_min is not a hole, but may be in front
    assert not got[np.isnan(G) | (G <= 0.2) | (mask[0] == 0)].any()
    # depth_rel = 1 turns the in-front test off
    assert not (seed64.select(A, D, G, mask, depth_rel=1.0, stride=stride) == seed64.FRONT).any()


def test_the_cap_keeps_exactly_n_spread_evenly():
    for c in (1, 2, 7, 100, 1013):
        for n in sorted({0, 1, 2, c // 3, c - 1, c}):
            if not 0 <= n <= c:
                continue
            k = seed64.keep(c, n)
            assert k.sum() == n, (c, n)
            if n:
                idx = np.nonzero(k)[0]
                gaps = np.diff(np.concatenate([[-1], idx]))
                assert gaps.max() - gaps.min() <= 1, (c, n)      # every gap is floor or ceil of c / n
    assert seed64.keep(5, 5).all() and not seed64.keep(5, 0).any() and seed64.keep(0, 0).size == 0


def test_seed_rows_follow_the_insert_rule():
    W, H = 31, 23
    cam = syn.make_camera(W, H, 25.0, 27.0, *syn.random_pose(np.random.default_rng(4)))
    A, D, G, mask = _planes(H, W)
    img = np.random.default_rng(1).uniform(0, 1, (3, H, W)).astype(np.float32)
    s = seed64.seed(cam, A, D, G, img, mask, stride=2, max_new=17)
    c = s["counts"][0]
    assert c > 17 and s["n"] == 17 and s["counts"][1] + s["counts"][2] == c
    assert np.all(np.diff(s["v"] * W + s["u"]) > 0) and np.all(s["u"] % 2 == 0) and np.all(s["v"] % 2 == 0)
    np.testing.assert_allclose(s["color"], img[:, s["v"], s["u"]].T)
    np.testing.assert_allclose(np.exp(s["scaling"][:, 0]), 2 * G[s["v"], s["u"]] / 26.0, rtol=1e-6)   # one grid cell at depth z
    assert np.allclose(1 / (1 + np.exp(-s["opacity"])), 0.1)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_unprojected_points_land_on_pixel_centres(seed):
    rng = np.random.default_rng(seed)
    W, H = 64, 48
    R, t = syn.random_pose(rng, max_angle=1.0, max_trans=3.0)
    cam = syn.make_camera(W, H, 50.0, 47.0, R, t)
    u, v = rng.integers(0, W, 200), rng.integers(0, H, 200)
    z = rng.uniform(0.2, 40.0, 200)
    xyz = seed64.unproject(cam, u, v, z)
    pu, pv, pz = seed64.project(cam, xyz)
    assert np.abs(pu - u).max() < 1e-3 and np.abs(pv - v).max() < 1e-3
    np.testing.assert_allclose(pz, z, rtol=1e-6)


# ---- the C entries ------------------------------------------------------------------------------------------------------------------
def _cmodel(**kw):
    m = trainer._Model()
    for i in range(6):
        m.param[i] = ONE
        m.exp_avg[i], m.exp_avg_sq[i] = ONE, ONE
    return m


def _cam(W=32, H=24, view=ONE, tanx=0.5, tany=0.5):
    c = trainer._Camera()
    c.viewmatrix, c.projmatrix, c.campos, c.tan_fovx, c.tan_fovy, c.width, c.height = view, ONE, ONE, tanx, tany, W, H
    return c


def _cfg(**kw):
    d = dict(alpha_min=0.5, depth_rel=0.1, min_depth=0.2, max_depth=40.0, stride=1, max_new=1000)
    d.update(kw)
    return trainer._SeedCfg(d["alpha_min"], d["depth_rel"], d["min_depth"], d["max_depth"], d["stride"], d["max_new"])


BAD_CFGS = [dict(alpha_min=0.0), dict(alpha_min=-0.1), dict(alpha_min=1.5), dict(alpha_min=math.nan), dict(depth_rel=-0.01), dict(depth_rel=1.01),
            dict(depth_rel=math.nan), dict(min_depth=-1.0), dict(min_depth=math.nan), dict(max_depth=math.nan), dict(min_depth=5.0, max_depth=5.0),
            dict(min_depth=6.0, max_depth=5.0), dict(stride=0), dict(stride=-2), dict(max_new=-1)]


def _rejects(L, name, *args):
    assert getattr(L, name)(*args) == E, (name, args)
    assert name.encode() in L.psb_last_error(), (name, L.psb_last_error())


def test_plan_refuses_bad_arguments_without_a_device():
    L = trainer._bind()
    counts = (C.c_int * 3)()
    plan = lambda cam, a, d, g, cfg, ws, cnt: _rejects(L, "psb_seed_plan", cam, a, d, g, None, cfg, ws, cnt, None)
    cam, cfg = _cam(), _cfg()
    plan(None, ONE, ONE, ONE, C.byref(cfg), ONE, counts)
    for k in range(3):
        planes = [ONE, ONE, ONE]
        planes[k] = None
        plan(C.byref(cam), *planes, C.byref(cfg), ONE, counts)
    plan(C.byref(cam), ONE, ONE, ONE, None, ONE, counts)
    plan(C.byref(cam), ONE, ONE, ONE, C.byref(cfg), None, counts)
    plan(C.byref(cam), ONE, ONE, ONE, C.byref(cfg), ONE, None)
    for bad in (_cam(W=0), _cam(H=-3), _cam(W=70000, H=70000)):
        plan(C.byref(bad), ONE, ONE, ONE, C.byref(cfg), ONE, counts)
    for kw in BAD_CFGS:
        plan(C.byref(cam), ONE, ONE, ONE, C.byref(_cfg(**kw)), ONE, counts)


def test_apply_refuses_bad_arguments_without_a_device():
    L = trainer._bind()
    src, dst, cam, cfg = _cmodel(), _cmodel(), _cam(), _cfg(max_new=10)
    apply = lambda P, s, d, n, c, img, g, cf, ws: _rejects(L, "psb_seed_apply", P, s, d, n, c, img, g, cf, ws, 0, None)
    apply(10, C.byref(src), C.byref(dst), 5, None, ONE, ONE, C.byref(cfg), ONE)
    apply(10, C.byref(src), C.byref(dst), 5, C.byref(_cam(view=None)), ONE, ONE, C.byref(cfg), ONE)
    for bad in (_cam(tanx=0.0), _cam(tany=-1.0), _cam(tanx=math.nan), _cam(tany=math.inf), _cam(W=0)):
        apply(10, C.byref(src), C.byref(dst), 5, C.byref(bad), ONE, ONE, C.byref(cfg), ONE)
    apply(10, C.byref(src), C.byref(dst), 5, C.byref(cam), None, ONE, C.byref(cfg), ONE)
    apply(10, C.byref(src), C.byref(dst), 5, C.byref(cam), ONE, None, C.byref(cfg), ONE)
    apply(10, C.byref(src), C.byref(dst), 5, C.byref(cam), ONE, ONE, None, ONE)
    apply(10, C.byref(src), C.byref(dst), 5, C.byref(cam), ONE, ONE, C.byref(cfg), None)
    apply(10, C.byref(src), C.byref(dst), -1, C.byref(cam), ONE, ONE, C.byref(cfg), ONE)
    apply(10, C.byref(src), C.byref(dst), 11, C.byref(cam), ONE, ONE, C.byref(cfg), ONE)      # n > max_new
    for kw in BAD_CFGS:
        apply(10, C.byref(src), C.byref(dst), 0, C.byref(cam), ONE, ONE, C.byref(_cfg(**kw)), ONE)
    # a workspace no plan has filled (n > selected cannot be known)
    apply(10, C.byref(src), C.byref(dst), 5, C.byref(cam), ONE, ONE, C.byref(cfg), ONE)
    assert b"no psb_seed_plan" in L.psb_last_error()
    apply(10, C.byref(src), C.byref(dst), 0, C.byref(cam), ONE, ONE, C.byref(cfg), ONE + 256)


def test_workspace_bytes():
    L = trainer._bind()
    assert L.psb_seed_workspace_bytes(0, 10, 1) == 0 and L.psb_seed_workspace_bytes(10, 10, 0) == 0
    assert L.psb_seed_workspace_bytes(70000, 70000, 1) == 0
    full, half = L.psb_seed_workspace_bytes(1200, 680, 1), L.psb_seed_workspace_bytes(1200, 680, 2)
    assert full >= 1200 * 680 * (1 + 7 * 4) and half >= 600 * 340 * 29 and half < full


def test_header_declares_and_library_exports_the_entries():
    names = ("psb_seed_workspace_bytes", "psb_seed_plan", "psb_seed_apply")
    exported = _lib.exported_symbols()
    L = trainer._bind()
    for n in names:
        assert n in exported and hasattr(L, n)
    assert len(L.psb_seed_plan.argtypes) == 9 and len(L.psb_seed_apply.argtypes) == 11
    assert L.psb_seed_workspace_bytes.restype is C.c_size_t
    assert [f for f, _ in trainer._SeedCfg._fields_] == ["alpha_min", "depth_rel", "min_depth", "max_depth", "stride", "max_new"]
    hdr = open(__import__("test_bindings_cpu").HEADER).read()
    assert "typedef struct psb_seed_cfg" in hdr


# ---- the Python front end against a stub library -------------------------------------------------------------------------------------
class _StubL:
    """psb_seed_plan reports fixed counts; psb_seed_apply records its arguments."""

    def __init__(self, counts=(40, 30, 10)):
        self.counts, self.plans, self.applies = counts, [], []

    def psb_seed_workspace_bytes(self, W, H, stride):
        return 64

    def psb_seed_plan(self, cam, alpha, depth, gt, mask, cfg, ws, counts, stream):
        c = cfg._obj
        self.plans.append(dict(alpha=alpha, depth=depth, mask=mask, alpha_min=c.alpha_min, depth_rel=c.depth_rel, min_depth=c.min_depth,
                               max_depth=c.max_depth, stride=c.stride, max_new=c.max_new))
        for k in range(3):
            counts[k] = self.counts[k]
        return 0

    def psb_seed_apply(self, P, src, dst, n, cam, img, gt, cfg, ws, iteration, stream):
        self.applies.append(dict(P=P, n=n, iteration=iteration, max_new=cfg._obj.max_new))
        return 0

    def __getattr__(self, name):
        return lambda *a: 0


@pytest.fixture
def stubbed(monkeypatch):
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: types.SimpleNamespace(cuda_stream=None))

    def make(counts=(40, 30, 10), mcmc=False, cap_max=1000):
        tr, m, cam = _cpu_trainer()
        tr.opt = trainer.GaussianOptimizationParams(mcmc=mcmc, cap_max=cap_max)
        L = _StubL(counts)
        monkeypatch.setattr(trainer, "_bind", lambda: L)
        tr.L = L
        renders = []

        def render(c, out=None, radii=None, check=True, out_depth=None, out_alpha=None):
            renders.append((out_depth, out_alpha))
            out_alpha.fill_(0.75)
        tr.render = render
        H, W = cam["H"], cam["W"]
        planes = (torch.rand(3, H, W), torch.rand(H, W) + 1)
        return tr, m, cam, L, renders, planes
    return make


def test_seed_plans_renders_and_applies(stubbed):
    tr, m, cam, L, renders, (img, gt) = stubbed()
    P = m.num_points()
    m.filter_3D_ = torch.zeros(P)
    sparse = m.sparse_points_xyz_ = torch.zeros((5, 3))
    tr.iteration = 77
    assert tr.seedFromDepth(cam, img, gt) == (40, 30, 10)
    assert len(renders) == 1 and L.plans[0]["alpha"] == renders[0][1].data_ptr() and L.plans[0]["mask"] is None
    p = L.plans[0]
    assert (p["alpha_min"], round(p["depth_rel"], 6), round(p["min_depth"], 6), p["max_depth"], p["stride"]) == (0.5, 0.1, 0.2, 40.0, 1)
    assert p["max_new"] == 2 ** 31 - 1
    assert L.applies == [dict(P=P, n=40, iteration=77, max_new=2 ** 31 - 1)]
    assert m.num_points() == P + 40 and m.exp_avg_[2].shape == (P + 40, 15, 3) and m._exist().shape == (P + 40,)
    assert m.filter_3D_ is None and not m.adam_live_valid_ and m.sparse_points_xyz_ is sparse
    # the cap, an explicit iteration, a mask
    mask = torch.ones(3, cam["H"], cam["W"])
    assert tr.seedFromDepth(cam, img, gt, mask=mask, max_new=7, stride=3, iteration=5) == (7, 30, 10)
    assert L.applies[-1]["n"] == 7 and L.applies[-1]["iteration"] == 5 and L.plans[-1]["mask"] == mask.data_ptr() and L.plans[-1]["stride"] == 3
    # nothing selected (or max_new = 0): the model is not touched
    m.filter_3D_ = torch.zeros(m.num_points())
    k = len(L.applies)
    assert tr.seedFromDepth(cam, img, gt, max_new=0) == (0, 30, 10) and len(L.applies) == k and m.filter_3D_ is not None


def test_an_empty_model_is_not_rendered(stubbed):
    tr, m, cam, L, renders, (img, gt) = stubbed()
    keep = torch.zeros(m.num_points(), dtype=torch.bool)
    m._set([t[keep].contiguous() for t in m.tensors()])
    m.exp_avg_ = [t[keep].contiguous() for t in m.exp_avg_]
    m.exp_avg_sq_ = [t[keep].contiguous() for t in m.exp_avg_sq_]
    assert m.num_points() == 0
    assert tr.seedFromDepth(cam, img, gt)[0] == 40
    assert renders == [] and L.applies[-1]["P"] == 0 and m.num_points() == 40


def test_mcmc_default_of_max_new_is_the_budget(stubbed):
    tr, m, cam, L, renders, (img, gt) = stubbed(mcmc=True, cap_max=55)
    P = m.num_points()
    assert tr.seedFromDepth(cam, img, gt) == (55 - P, 30, 10)
    assert L.plans[-1]["max_new"] == 55 - P
    assert tr.seedFromDepth(cam, img, gt) == (0, 30, 10)           # at the cap: nothing more
    assert L.plans[-1]["max_new"] == 0 and len(L.applies) == 1
    assert tr.seedFromDepth(cam, img, gt, max_new=3)[0] == 3        # an explicit max_new wins


def test_argument_checks_before_any_c_call(stubbed):
    tr, m, cam, L, renders, (img, gt) = stubbed()
    H, W = cam["H"], cam["W"]
    bad = [dict(alpha_min=0), dict(alpha_min=1.1), dict(alpha_min=math.nan), dict(alpha_min=True), dict(alpha_min="0.5"),
           dict(depth_rel=-0.1), dict(depth_rel=1.5), dict(depth_rel=math.nan), dict(min_depth=-1), dict(min_depth=5, max_depth=5),
           dict(min_depth=math.inf, max_depth=math.inf), dict(max_depth=math.nan), dict(stride=0), dict(stride=2.0), dict(stride=True),
           dict(max_new=-1), dict(max_new=3.0), dict(max_new=False), dict(iteration=1.5), dict(iteration=True)]
    for kw in bad:
        with pytest.raises(ValueError, match="seedFromDepth"):
            tr.seedFromDepth(cam, img, gt, **kw)
    for args in ((cam, None, gt), (cam, img, None), (cam, img[:, :, :-1], gt), (cam, img, gt.t()), (cam, img.double(), gt),
                 (cam, img, gt[None]), (dict(W=W), img, gt), (None, img, gt)):
        with pytest.raises(ValueError):
            tr.seedFromDepth(*args)
    with pytest.raises(ValueError, match="mask"):
        tr.seedFromDepth(cam, img, gt, mask=torch.ones(1, H, W))
    m.features_rest_ = m.features_rest_[:, :8].contiguous()
    with pytest.raises(ValueError, match="features_rest"):
        tr.seedFromDepth(cam, img, gt)
    assert L.plans == [] and L.applies == [] and renders == []


def test_data_parallel_trainer_refuses_seeding():
    dp = object.__new__(trainer.DataParallelTrainer)
    with pytest.raises(NotImplementedError, match="diverge"):
        dp.seedFromDepth(dict(), None, None)
