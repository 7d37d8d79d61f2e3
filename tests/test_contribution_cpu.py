"""CPU: contribution pruning without a device. The float64 restatement (tests/contrib64.py) against an independent per-pixel loop; the C
entry's refusals before any CUDA call; the Python front end against a stub library (argument checks, the sweep and its one retry, the unit of
the sum); the prune mask rule (threshold, keep with ties, min_age); the data-parallel refusal; the ctypes declaration."""
import ctypes as C
import math
import types

import numpy as np
import pytest
import torch

import contrib64
import splat64 as s64
from photo_slam_b200 import _lib, trainer
from test_pixel_grads_cpu import _cpu_trainer


# ---- the restatement ----------------------------------------------------------------------------------------------------------------
def _tiny():
    import photo_slam_b200.synthetic as syn
    cam = syn.make_camera(40, 24, 36.0, 36.0)
    sc = syn.make_scene(30, cam, seed=3, scale_px=3.0)
    sc["opacity"][:] = np.abs(sc["opacity"]) + 1.0     # opaque enough that some pixels end at the T test
    return cam, sc


def _loop_scores(geo, W, H):
    """per pixel, walk the Gaussians whose rectangle holds the pixel's tile in depth order and blend one by one"""
    P = geo["z"].numel()
    wmax, wsum = np.zeros(P), np.zeros(P)
    live = [i for i in range(P) if bool(geo["alive"][i])]
    live.sort(key=lambda i: float(geo["zd"][i]))
    for y in range(H):
        for x in range(W):
            tx, ty = x // s64.TILE, y // s64.TILE
            T = 1.0
            for i in live:
                r = geo["rect"][i].tolist()
                if not (r[0] <= tx < r[2] and r[1] <= ty < r[3]):
                    continue
                dx, dy = float(geo["means2D"][i, 0]) - x, float(geo["means2D"][i, 1]) - y
                A, B, Cc = (float(v) for v in geo["conic"][i])
                power = -0.5 * (A * dx * dx + Cc * dy * dy) - B * dx * dy
                if power > 0:
                    continue
                alpha = min(0.99, float(geo["o"][i]) * math.exp(power))
                if alpha < 1 / 255:
                    continue
                if T * (1 - alpha) < 1e-4:
                    break
                w = alpha * T
                wmax[i] = max(wmax[i], w)
                wsum[i] += w
                T *= 1 - alpha
    return wmax, wsum


def test_restatement_equals_a_per_pixel_loop():
    cam, sc = _tiny()
    c = s64.camera64(cam, "cpu")
    geo = s64.geometry(s64.activate(s64.raw64(sc, "cpu")), c, D=3)
    got = contrib64.weights(geo, c["W"], c["H"])
    wmax, wsum = _loop_scores(geo, c["W"], c["H"])
    assert (wmax > 0).sum() > 5 and (wmax == 0).any()
    np.testing.assert_allclose(got["max"].numpy(), wmax, rtol=1e-12, atol=0)
    np.testing.assert_allclose(got["sum"].numpy(), wsum, rtol=1e-12, atol=1e-15)
    assert torch.equal(got["max"] > 0, got["pixels"] > 0)
    # a second view: the sweep's max is the larger, the sum adds
    two = contrib64.scores(s64.raw64(sc, "cpu"), [c, c])
    np.testing.assert_allclose(two["max"].numpy(), wmax, rtol=1e-12)
    np.testing.assert_allclose(two["sum"].numpy(), 2 * wsum, rtol=1e-12, atol=1e-15)


def test_restatement_agrees_with_composite():
    """sum_i w_i c_i + T_final bg is composite's colour: the weights are the blend's"""
    cam, sc = _tiny()
    c = s64.camera64(cam, "cpu")
    raw = s64.raw64(sc, "cpu")
    geo = s64.geometry(s64.activate(raw), c, D=3)
    out = s64.composite(geo, c["W"], c["H"], (0.0, 0.0, 0.0))
    got = contrib64.weights(geo, c["W"], c["H"])
    assert torch.equal(got["stopped"], out["stopped"])
    # every pixel's alpha is the sum of its weights; summed over the image, the weights are the total alpha
    np.testing.assert_allclose(float(got["sum"].sum()), float(out["alpha"].sum()), rtol=1e-12)


# ---- the C entry --------------------------------------------------------------------------------------------------------------------
def test_c_entry_refuses_before_any_cuda_call():
    L = trainer._bind()
    one = 4096   # fake non-null pointer: never dereferenced, validation fails first
    cam, model = trainer._Camera(), trainer._Model()
    cases = [((None, 10, 16, model, cam, one, 3, one, one, None, None), b"null argument"),
             ((one, 10, 16, model, None, one, 3, one, one, None, None), b"null argument"),
             ((one, 10, 16, model, cam, None, 3, one, one, None, None), b"null argument"),
             ((one, 10, 16, model, cam, one, 3, None, one, None, None), b"null argument"),
             ((one, 10, 16, model, cam, one, 3, one, None, None, None), b"null argument"),
             ((one, -1, 16, model, cam, one, 3, one, one, None, None), b"P >= 0")]
    for args, msg in cases:
        a = list(args)
        for k in (3, 4):
            a[k] = C.byref(a[k]) if a[k] is not None else None
        assert L.psb_trainer_contribution(*a) == -1
        assert msg in L.psb_last_error(), (args, L.psb_last_error())


def test_header_declares_and_library_exports_the_entry():
    assert "psb_trainer_contribution" in _lib.exported_symbols()
    L = trainer._bind()
    assert len(L.psb_trainer_contribution.argtypes) == 11 and L.psb_trainer_contribution.restype is C.c_int
    hdr = open(__import__("test_bindings_cpu").HEADER).read()
    assert "#define PSB_CONTRIB_SUM_FRAC_BITS 26" in hdr and trainer.CONTRIB_SUM_UNIT == 2.0 ** -26


# ---- the Python front end against a stub library -------------------------------------------------------------------------------------
class _StubL:
    """psb_trainer_contribution adds fixed per-view scores; psb_trainer_result reports an overflow on the first `overflows` collections."""

    def __init__(self, P, overflows=0):
        self.P, self.overflows, self.calls, self.results, self.prune_masks = P, overflows, [], 0, []

    def psb_trainer_contribution(self, t, P, M, cm, cc, bg, D, mx, sm, out, stream):
        k = len(self.calls)
        self.calls.append(P)
        amx = (C.c_uint32 * P).from_address(mx)
        asm = (C.c_uint64 * P).from_address(sm)
        for i in range(P):
            w = np.float32((i % 7) / 8.0)     # rows 0, 7, 14, ... never blend
            amx[i] = max(amx[i], int(np.array(w).view(np.uint32)))
            asm[i] += int(w * 2 ** 26) * (1 + k % 2)
        return 0

    def psb_trainer_result(self, t, out, n, stream):
        self.results += 1
        if self.overflows:
            self.overflows -= 1
            return -4
        return 0

    def psb_prune_plan(self, P, mask, ws, counts, stream):
        m = np.ctypeslib.as_array((C.c_uint8 * P).from_address(mask)).copy()
        self.prune_masks.append(m)
        counts[0] = int(P - m.sum())
        return 0

    def __getattr__(self, name):
        if name.endswith("_bytes"):
            return lambda *a: 16
        return lambda *a: 0


@pytest.fixture
def stubbed(monkeypatch):
    monkeypatch.setattr(torch.cuda, "current_stream", lambda: types.SimpleNamespace(cuda_stream=None))

    def make(overflows=0):
        tr, m, cam = _cpu_trainer()
        L = _StubL(m.num_points(), overflows)
        monkeypatch.setattr(trainer, "_bind", lambda: L)
        tr.L = L
        return tr, m, cam, L
    return make


def test_scores_sweep_and_units(stubbed):
    tr, m, cam, L = stubbed()
    P = m.num_points()
    mx, sm = tr.contributionScores([cam, cam, cam])
    assert L.calls == [P] * 3 and L.results == 1            # one collection for the whole sweep
    assert mx.dtype == torch.float32 and sm.dtype == torch.float64 and mx.shape == sm.shape == (P,)
    w = torch.tensor([(i % 7) / 8.0 for i in range(P)])
    assert torch.equal(mx, w.float())
    assert torch.equal(sm, w.double() * 4)                  # views weighted 1, 2, 1


def test_an_overflowing_sweep_is_repeated_once_from_zero(stubbed):
    tr, m, cam, L = stubbed(overflows=1)
    mx, sm = tr.contributionScores([cam, cam])
    assert len(L.calls) == 4 and L.results == 2
    w = torch.tensor([(i % 7) / 8.0 for i in range(m.num_points())], dtype=torch.float64)
    assert torch.equal(sm, w * 3)                           # the arrays were zeroed before the repeat
    tr, m, cam, L = stubbed(overflows=2)
    with pytest.raises(_lib.PsbError, match="again"):
        tr.contributionScores([cam])


def test_argument_checks_before_any_c_call(stubbed):
    tr, m, cam, L = stubbed()
    bad_cams = [[], None, cam, [dict(W=4)], [dict(cam, W=0)], [dict(cam, H=2.5)], [cam, "x"]]
    for cams in bad_cams:
        with pytest.raises(ValueError):
            tr.contributionScores(cams)
        with pytest.raises(ValueError):
            tr.pruneByContribution(cams, 0.01)
    for kw in (dict(min_weight=-0.1), dict(min_weight=1.0), dict(min_weight=float("nan")), dict(min_weight=float("inf")), dict(min_weight=None),
               dict(min_weight=True), dict(min_weight=0.1, keep=0), dict(min_weight=0.1, keep=-3), dict(min_weight=0.1, keep=2.0),
               dict(min_weight=0.1, keep=True), dict(min_weight=0.1, min_age=-1), dict(min_weight=0.1, min_age=1.5)):
        with pytest.raises(ValueError, match="pruneByContribution"):
            tr.pruneByContribution([cam], **kw)
    assert L.calls == [] and L.results == 0


def test_prune_goes_through_prune_points(stubbed):
    tr, m, cam, L = stubbed()
    P = m.num_points()
    m.filter_3D_ = torch.zeros(P)
    n = tr.pruneByContribution([cam], 0.1)                 # removes the rows that never blend (max 0)
    want = np.array([(i % 7) == 0 for i in range(P)])
    assert n == int(want.sum()) and np.array_equal(L.prune_masks[-1].astype(bool), want)
    assert m.filter_3D_ is None and not m.adam_live_valid_
    # nothing to remove: no prune call
    k = len(L.prune_masks)
    tr2, m2, cam2, L2 = stubbed()
    assert tr2.pruneByContribution([cam2], 0.0) == 0 and L2.prune_masks == [] and k == 1


# ---- the mask rule ------------------------------------------------------------------------------------------------------------------
def test_mask_threshold_keep_ties_and_age():
    mx = torch.tensor([0.0, 0.5, 0.02, 0.3, 0.3, 0.009, 0.9, 0.3])
    sm = torch.tensor([0.0, 5.0, 1.0, 2.0, 2.0, 0.5, 9.0, 2.0], dtype=torch.float64)
    f = trainer.contribution_prune_mask
    assert f(mx, sm, 0.01).tolist() == [True, False, False, False, False, True, False, False]
    assert not f(mx, sm, 0.0).any()
    # keep 4 by the sum: 9.0 (6), 5.0 (1), then the tie at 2.0 goes to the lower indices 3 and 4; row 7 is removed
    assert f(mx, sm, 0.0, keep=4).tolist() == [True, False, True, False, False, True, False, True]
    assert f(mx, sm, 0.0, keep=8).sum() == 0 and f(mx, sm, 0.0, keep=100).sum() == 0
    # threshold and keep together: the union
    assert f(mx, sm, 0.01, keep=6).tolist() == [True, False, False, False, False, True, False, False]
    assert f(mx, sm, 0.01, keep=5).tolist() == [True, False, True, False, False, True, False, False]
    young = torch.tensor([True, False, False, False, False, False, False, True])
    assert f(mx, sm, 0.01, keep=4, young=young).tolist() == [False, False, True, False, False, True, False, False]


def test_min_age_uses_exist_since_iter(stubbed):
    tr, m, cam, L = stubbed()
    P = m.num_points()
    tr.iteration = 100
    m.exist_since_iter_ = torch.tensor([95 if i < 14 else 10 for i in range(P)], dtype=torch.int32)
    n = tr.pruneByContribution([cam], 0.1, min_age=10)     # rows 0 and 7 are 5 iterations old: kept
    want = np.array([(i % 7) == 0 and i >= 14 for i in range(P)])
    assert n == int(want.sum()) and np.array_equal(L.prune_masks[-1].astype(bool), want)


def test_data_parallel_trainer_refuses_the_prune():
    dp = object.__new__(trainer.DataParallelTrainer)
    with pytest.raises(NotImplementedError, match="IPC arena"):
        dp.pruneByContribution([dict()], 0.01)
