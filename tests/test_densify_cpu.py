"""CPU: the row operations (psb_densify_*, psb_prune_*, psb_insert_points, psb_reset_opacity, and GaussianModel's row-changing methods).

  * every entry point rejects bad arguments with PSB_ERR_ARG before its first CUDA call (no device here: a call that reached the
    device would return -2), and psb_last_error() names it;
  * the Python methods against a stub library: which C call each makes (P, P_new, keep_stats, the NULL fields of its models), and the
    state the model ends in (shapes, adam_live_valid_, filter_3D_, exist_since_iter_);
  * a model whose features_rest is not [P, 15, 3] is refused before any C call (the row kernels move 45 floats per row).
"""
import ctypes as C
import types

import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn
from photo_slam_b200 import points, trainer

ONE = 4096  # fake non-null device pointer; never dereferenced because validation fails first
E = -1      # PSB_ERR_ARG


def _cmodel(moments=True, stats=False, exist=False):
    m = trainer._Model()
    for i in range(6):
        m.param[i] = ONE
        if moments:
            m.exp_avg[i], m.exp_avg_sq[i] = ONE, ONE
    if stats:
        m.max_radii2D = m.xyz_gradient_accum = m.denom = ONE
    if exist:
        m.exist_since_iter = ONE
    return m


def _without(field, i=None, **kw):
    m = _cmodel(**kw)
    if i is None:
        setattr(m, field, None)
    else:
        getattr(m, field)[i] = None
    return m


def _misaligned_rotation(**kw):
    m = _cmodel(**kw)
    m.param[5] = ONE + 4
    return m


def _rejects(L, name, *args):
    assert getattr(L, name)(*args) == E, (name, args)
    assert name.encode() in L.psb_last_error(), (name, L.psb_last_error())


def test_densify_plan_and_apply_reject_bad_arguments_without_a_device():
    L = trainer._bind()
    cfg = trainer._DensifyCfg(0.001, 0.005, 1.0, 0.01, 0, 0, 0)
    m, counts = _cmodel(stats=True), (C.c_int * 5)()
    plan = lambda P, src, c, ws, cnt: _rejects(L, "psb_densify_plan", P, src, c, ws, cnt, None)
    plan(-1, C.byref(m), C.byref(cfg), ONE, counts)
    plan(10, C.byref(m), None, ONE, counts)
    plan(10, C.byref(m), C.byref(cfg), ONE, None)
    plan(10, None, C.byref(cfg), ONE, counts)
    plan(10, C.byref(m), C.byref(cfg), None, counts)
    for f, i in (("param", 3), ("param", 4), ("xyz_gradient_accum", None), ("denom", None)):
        plan(10, C.byref(_without(f, i, stats=True)), C.byref(cfg), ONE, counts)
    counts[0] = 7
    assert L.psb_densify_plan(0, None, C.byref(cfg), None, counts, None) == 0 and list(counts) == [0] * 5

    src, dst = _cmodel(), _cmodel()
    apply = lambda P, s, d, P_new, c, ws: _rejects(L, "psb_densify_apply", P, s, d, P_new, c, ws, None, None)
    apply(-1, C.byref(src), C.byref(dst), 10, C.byref(cfg), ONE)
    apply(10, C.byref(src), C.byref(dst), -1, C.byref(cfg), ONE)
    apply(10, C.byref(src), C.byref(dst), 10, None, ONE)
    apply(10, None, C.byref(dst), 10, C.byref(cfg), ONE)
    apply(10, C.byref(src), C.byref(dst), 10, C.byref(cfg), None)
    apply(10, C.byref(src), None, 10, C.byref(cfg), ONE)
    for f in ("param", "exp_avg", "exp_avg_sq"):
        for i in (0, 2, 5):
            apply(10, C.byref(_without(f, i)), C.byref(dst), 12, C.byref(cfg), ONE)
            apply(10, C.byref(src), C.byref(_without(f, i)), 12, C.byref(cfg), ONE)
    apply(10, C.byref(_misaligned_rotation()), C.byref(dst), 12, C.byref(cfg), ONE)
    # dst has statistics to zero: every argument is still checked before the first of those memsets
    apply(10, C.byref(src), C.byref(_without("exp_avg", 4, stats=True)), 12, C.byref(cfg), ONE)
    assert L.psb_densify_apply(0, None, None, 0, C.byref(cfg), None, None, None) == 0
    assert L.psb_densify_workspace_bytes(0) == 256 and L.psb_densify_workspace_bytes(1000) >= 1000


def test_prune_plan_and_apply_reject_bad_arguments_without_a_device():
    L = trainer._bind()
    counts = (C.c_int * 5)()
    plan = lambda P, mask, ws, cnt: _rejects(L, "psb_prune_plan", P, mask, ws, cnt, None)
    plan(-1, ONE, ONE, counts)
    plan(10, ONE, ONE, None)
    plan(10, None, ONE, counts)
    plan(10, ONE, None, counts)
    counts[0] = 7
    assert L.psb_prune_plan(0, None, None, counts, None) == 0 and list(counts) == [0] * 5

    src, dst = _cmodel(stats=True), _cmodel()
    for keep in (0, 1):
        apply = lambda P, s, d, P_new, ws: _rejects(L, "psb_prune_apply", P, s, d, P_new, ws, keep, None)
        apply(-1, C.byref(src), C.byref(dst), 5, ONE)
        apply(10, C.byref(src), C.byref(dst), -1, ONE)
        apply(10, None, C.byref(dst), 5, ONE)
        apply(10, C.byref(src), C.byref(dst), 5, None)
        apply(10, C.byref(src), None, 5, ONE)
        for f in ("param", "exp_avg", "exp_avg_sq"):
            for i in (1, 3, 5):
                apply(10, C.byref(_without(f, i, stats=True)), C.byref(dst), 5, ONE)
                apply(10, C.byref(src), C.byref(_without(f, i)), 5, ONE)
        apply(10, C.byref(_misaligned_rotation(stats=True)), C.byref(dst), 5, ONE)
        assert L.psb_prune_apply(0, None, None, 0, None, keep, None) == 0


def test_insert_points_and_reset_opacity_reject_bad_arguments_without_a_device():
    L = trainer._bind()
    src, dst = _cmodel(exist=True), _cmodel(stats=True, exist=True)
    ins = lambda P, s, d, n, pts, cols, d2: _rejects(L, "psb_insert_points", P, s, d, n, pts, cols, d2, 0, None)
    ins(-1, C.byref(src), C.byref(dst), 4, ONE, ONE, ONE)
    ins(10, C.byref(src), C.byref(dst), -1, ONE, ONE, ONE)
    ins(10, C.byref(src), None, 4, ONE, ONE, ONE)
    ins(10, None, C.byref(dst), 4, ONE, ONE, ONE)
    ins(10, C.byref(src), C.byref(dst), 4, None, ONE, ONE)
    ins(10, C.byref(src), C.byref(dst), 4, ONE, None, ONE)
    ins(10, C.byref(src), C.byref(dst), 4, ONE, ONE, None)
    for f in ("param", "exp_avg", "exp_avg_sq"):
        ins(10, C.byref(src), C.byref(_without(f, 0, stats=True)), 4, ONE, ONE, ONE)
        ins(0, None, C.byref(_without(f, 0, stats=True)), 4, ONE, ONE, ONE)
    # the rotation tensor the new rows are written to: checked before the old rows are copied
    ins(10, C.byref(src), C.byref(_misaligned_rotation(stats=True, exist=True)), 4, ONE, ONE, ONE)
    assert L.psb_insert_points(0, None, C.byref(_cmodel(False)), 0, None, None, None, 0, None) == 0

    reset = lambda P, o, m, v: _rejects(L, "psb_reset_opacity", P, o, m, v, None)
    reset(-1, ONE, ONE, ONE)
    reset(10, None, ONE, ONE)
    reset(10, ONE, None, ONE)
    reset(10, ONE, ONE, None)
    assert L.psb_reset_opacity(0, None, None, None, None) == 0


# ---- the Python methods against a stub library -------------------------------------------------------------------------------------
_FIELDS = ("max_radii2D", "xyz_gradient_accum", "denom", "exist_since_iter", "adam_live")


def _nulls(ref):
    m = ref._obj
    out = [f for f in _FIELDS if not getattr(m, f)]
    return tuple(out + [f"{g}[{i}]" for g in ("param", "exp_avg", "exp_avg_sq") for i in range(6) if not getattr(m, g)[i]])


class _RecL:
    """The row entry points, recording (function, P, P_new, keep_stats, NULL fields of each model); the plans change the row count."""

    def __init__(self):
        self.calls = []

    def psb_densify_plan(self, P, src, cfg, ws, counts, stream):
        self.calls.append(("psb_densify_plan", P, None, None, _nulls(src)))
        counts[0], counts[4] = P + 2, 1
        return 0

    def psb_densify_apply(self, P, src, dst, P_new, cfg, ws, samples, stream):
        self.calls.append(("psb_densify_apply", P, P_new, None, _nulls(src), _nulls(dst)))
        return 0

    def psb_prune_plan(self, P, mask, ws, counts, stream):
        self.calls.append(("psb_prune_plan", P, None, None))
        counts[0] = P - 3
        return 0

    def psb_prune_apply(self, P, src, dst, P_new, ws, keep_stats, stream):
        self.calls.append(("psb_prune_apply", P, P_new, keep_stats, _nulls(src), _nulls(dst)))
        return 0

    def psb_insert_points(self, P, src, dst, n, pts, cols, dist2, iteration, stream):
        self.calls.append(("psb_insert_points", P, P + n, None, _nulls(src), _nulls(dst)))
        return 0

    def psb_reset_opacity(self, P, o, m, v, stream):
        self.calls.append(("psb_reset_opacity", P, None, None))
        return 0

    def psb_relocate(self, P, model, cfg, ws, u, counts, stream):
        self.calls.append(("psb_relocate", P, None, None, _nulls(model)))
        counts[0], counts[1] = 2, 3
        return 0

    def psb_grow(self, P, src, dst, P_new, cfg, ws, u, stream):
        self.calls.append(("psb_grow", P, P_new, None, _nulls(src), _nulls(dst)))
        return 0

    def __getattr__(self, name):
        if name.endswith("_bytes"):
            return lambda *a: 16
        raise AttributeError(name)


@pytest.fixture
def rec(monkeypatch):
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: types.SimpleNamespace(cuda_stream=None))
    monkeypatch.setattr(points, "distCUDA2", lambda p: torch.ones(p.size(0)))
    monkeypatch.setattr(points, "transformPoints", lambda p, T: p.clone())
    monkeypatch.setattr(points, "scaleAndTransformThenMarkVisiblePoints", lambda *a: 0)
    L = _RecL()
    monkeypatch.setattr(trainer, "_bind", lambda: L)
    return L


def _shapes_ok(m, P):
    want = [(P, 3), (P, 1, 3), (P, 15, 3), (P, 1), (P, 3), (P, 4)]
    for ts in (m.tensors(), m.exp_avg_, m.exp_avg_sq_):
        assert [tuple(t.shape) for t in ts] == want
    assert m.xyz_gradient_accum_.shape == (P, 1) and m.denom_.shape == (P, 1) and m.max_radii2D_.shape == (P,)


NOLIVE = ("adam_live",)


def _model(sh_degree=3):
    sc = syn.make_scene(40, syn.make_camera(32, 24, 30.0, 30.0), seed=1, sh_degree_max=sh_degree)
    m = trainer.GaussianModel.from_numpy(sc, "cpu", sh_degree=sh_degree)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    return m


def test_row_changing_methods_make_one_c_call_each_and_end_in_the_documented_state(rec, tmp_path):
    m = _model()
    P = m.num_points()

    def run(name, call, calls, P_after, valid, filt, exist):
        m.filter_3D_ = torch.zeros(m.num_points())
        m.adam_live_, m.adam_live_valid_ = torch.zeros(m.num_points(), dtype=torch.uint8), True
        rec.calls.clear()
        call()
        assert rec.calls == calls, name
        _shapes_ok(m, P_after)
        assert m.adam_live_valid_ is valid, name
        assert (m.filter_3D_ is not None) is filt, name
        ex = getattr(m, "exist_since_iter_", None)
        assert (None if ex is None else tuple(ex.shape)) == exist, name

    run("densifySplitCount", lambda: m.densifySplitCount(0.001, 1.0),
        [("psb_densify_plan", P, None, None, NOLIVE)], P, True, True, (P,))
    run("resetOpacity", m.resetOpacity, [("psb_reset_opacity", P, None, None)], P, True, True, (P,))
    run("prunePoints", lambda: m.prunePoints(torch.zeros(P, dtype=torch.bool)),
        [("psb_prune_plan", P, None, None), ("psb_prune_apply", P, P - 3, 1, NOLIVE, NOLIVE)], P - 3, False, False, (P - 3,))
    P -= 3
    run("densifyAndPrune", lambda: m.densifyAndPrune(0.001, 0.005, 1.0, 0),
        [("psb_densify_plan", P, None, None, NOLIVE), ("psb_densify_apply", P, P + 2, None, NOLIVE, NOLIVE)], P + 2, False, False, (P + 2,))
    P += 2
    run("relocateGaussians", m.relocateGaussians, [("psb_relocate", P, None, None, ())], P, True, False, (P,))
    m.invalidateAdamLive()
    rec.calls.clear()
    m.relocateGaussians()
    assert rec.calls == [("psb_relocate", P, None, None, NOLIVE)] and not m.adam_live_valid_
    run("addNewGaussians", lambda: m.addNewGaussians(10 ** 6, 1.5),
        [("psb_grow", P, int(1.5 * P), None, NOLIVE, NOLIVE)], int(1.5 * P), False, False, (int(1.5 * P),))
    P = int(1.5 * P)
    run("addNewGaussians at the cap", lambda: m.addNewGaussians(P, 1.5), [], P, True, True, (P,))
    run("increasePcd", lambda: m.increasePcd(torch.zeros((4, 3)), torch.zeros((4, 3)), iteration=3),
        [("psb_insert_points", P, P + 4, None, NOLIVE, NOLIVE)], P + 4, False, False, (P + 4,))
    P += 4
    m.exp_avg_[0].fill_(1.0)
    m.exp_avg_sq_[5].fill_(1.0)
    run("applyScaledTransformation", lambda: m.applyScaledTransformation(1.1, np.eye(4)), [], P, True, False, (P,))
    assert not m.exp_avg_[0].any() and not m.exp_avg_sq_[4].any() and m.exp_avg_sq_[5].all()
    m.exp_avg_[4].fill_(1.0)
    run("scaledTransformVisiblePointsOfKeyframe", lambda: m.scaledTransformVisiblePointsOfKeyframe(
        torch.zeros(P, dtype=torch.uint8), torch.eye(4), torch.eye(4), torch.eye(4), 0, 10), [], P, True, False, (P,))
    assert not m.exp_avg_[0].any() and not m.exp_avg_sq_[5].any() and m.exp_avg_[4].all()
    m.savePly(str(tmp_path / "a.ply"))
    run("loadPly", lambda: m.loadPly(str(tmp_path / "a.ply")), [], P, False, False, (P,))


def test_row_operations_refuse_a_model_without_all_sixteen_sh_coefficients(rec):
    m = _model(sh_degree=2)
    P = m.num_points()
    assert m.features_rest_.shape == (P, 8, 3)
    for call in (lambda: m.prunePoints(torch.zeros(P, dtype=torch.bool)), lambda: m.densifyAndPrune(0.001, 0.005, 1.0, 0),
                 m.relocateGaussians, lambda: m.addNewGaussians(10 ** 6, 1.5),
                 lambda: m.increasePcd(torch.zeros((4, 3)), torch.zeros((4, 3)))):
        with pytest.raises(ValueError, match="features_rest"):
            call()
    assert rec.calls == [] and m.num_points() == P and m.features_rest_.shape == (P, 8, 3)
