"""CPU: per-keyframe exposure compensation in the fused step's loss.

  * a float64 restatement of the definition (I'(c) = sum_k E[k][c] I(k) + E[c][3], X = mask * I', L1 + D-SSIM on X) and of the
    gradients the kernels compute from g = dL/dI' (dL/dI = E[:3,:3] g, dL/dE[k][c] = sum_p g(c) I(k), dL/dE[c][3] = sum_p g(c)), checked
    against autograd and central finite differences, with a non-identity E, a mask and a non-black background in the image;
  * psb_trainer_step_exposure / psb_trainer_backward_exposure reject bad arguments before any CUDA call, and NULL is the _depth call;
  * the symbols are declared and exported;
  * the Python exposure table: identity rows, growth, applyExposure, snapshot / restore and the exposure.json round trip.
"""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from photo_slam_b200 import _lib, io, trainer
from splat64 import exposed, loss64

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "psb200.h")
ONE = 4096  # fake non-null device pointer; never dereferenced because validation fails first


# ---- the spec ----------------------------------------------------------------------------------------------------------------------
def loss_of_prime(Ip, G, mask, lam):
    return loss64(Ip, G, mask, lam)[0]


def loss(I, E, G, mask, lam):
    return loss_of_prime(exposed(I, E), G, mask, lam)


def spec_gradients(I, E, G, mask, lam):
    """What the kernels compute: g = dL/dI' (the loss backward at x = X, mask factor applied), then the mix and the 12 sums."""
    Ip = exposed(I, E).detach().requires_grad_(True)
    g, = torch.autograd.grad(loss_of_prime(Ip, G, mask, lam), Ip)
    dI = torch.einsum("kc,chw->khw", E[:, :3], g)
    dE = torch.zeros(3, 4, dtype=torch.float64)
    dE[:, :3] = torch.einsum("chw,khw->kc", g, I)
    dE[:, 3] = g.sum((1, 2))
    return dI, dE


def _case(seed=0, H=23, W=29):
    gen = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(s, generator=gen, dtype=torch.float64)
    bg = torch.tensor([0.3, 0.5, 0.7], dtype=torch.float64)
    T = r(1, H, W)
    I = r(3, H, W) * (1 - T) + T * bg[:, None, None]          # a render: colour plus the background's share
    G = r(3, H, W)
    mask = (r(1, H, W) > 0.2).double().expand(3, H, W).contiguous()
    E = torch.tensor([[1.2, 0.05, -0.03, 0.04], [0.02, 0.8, 0.06, -0.05], [-0.04, 0.03, 1.1, 0.02]], dtype=torch.float64)
    return I, E, G, mask, 0.2


def test_spec_gradients_match_autograd():
    I, E, G, mask, lam = _case()
    Ia, Ea = I.clone().requires_grad_(True), E.clone().requires_grad_(True)
    dI_ref, dE_ref = torch.autograd.grad(loss(Ia, Ea, G, mask, lam), (Ia, Ea))
    dI, dE = spec_gradients(I, E, G, mask, lam)
    assert torch.allclose(dI, dI_ref, rtol=1e-12, atol=1e-16)
    assert torch.allclose(dE, dE_ref, rtol=1e-12, atol=1e-16)


def test_spec_gradients_match_finite_differences():
    I, E, G, mask, lam = _case(seed=1)
    dI, dE = spec_gradients(I, E, G, mask, lam)
    h = 1e-6
    for j in range(12):
        Ep, Em = E.clone(), E.clone()
        Ep.view(-1)[j] += h
        Em.view(-1)[j] -= h
        fd = (loss(I, Ep, G, mask, lam) - loss(I, Em, G, mask, lam)).item() / (2 * h)
        assert abs(fd - dE.view(-1)[j].item()) <= 1e-6 * max(1.0, abs(fd)), (j, fd, dE.view(-1)[j].item())
    rng = np.random.default_rng(0)
    for idx in rng.integers(0, I.numel(), 40):
        Ip, Im = I.clone(), I.clone()
        Ip.view(-1)[idx] += h
        Im.view(-1)[idx] -= h
        fd = (loss(Ip, E, G, mask, lam) - loss(Im, E, G, mask, lam)).item() / (2 * h)
        assert abs(fd - dI.view(-1)[idx].item()) <= 1e-7 + 1e-5 * abs(fd), (idx, fd, dI.view(-1)[idx].item())


def test_identity_row_is_the_plain_loss():
    I, _, G, mask, lam = _case(seed=2)
    E = torch.eye(3, 4, dtype=torch.float64)
    assert torch.equal(exposed(I, E), I)
    dI, _ = spec_gradients(I, E, G, mask, lam)
    Ia = I.clone().requires_grad_(True)
    g, = torch.autograd.grad(loss_of_prime(Ia, G, mask, lam), Ia)
    assert torch.equal(dI, g)


# ---- host-side validation ----------------------------------------------------------------------------------------------------------
def _step_call(L, h, exposure, depth=None):
    return L.psb_trainer_step_exposure(h, 10, 16, None, None, None, None, None, None, None, None, depth, exposure, None)


def _bwd_call(L, h, exposure, grad, depth=None):
    return L.psb_trainer_backward_exposure(h, 10, 16, None, None, None, None, None, None, None, None, (C.c_void_p * 6)(*[ONE] * 6), depth,
                                           exposure, grad, None)


BAD_STEP = [("param", dict(param=None)), ("exp_avg", dict(exp_avg=None)), ("exp_avg_sq", dict(exp_avg_sq=None)), ("step", dict(step=None)),
            ("lr nan", dict(lr=float("nan"))), ("lr inf", dict(lr=float("inf"))), ("lr negative", dict(lr=-1e-3))]


def _exposure(**kw):
    f = dict(param=ONE, exp_avg=ONE, exp_avg_sq=ONE, step=ONE, lr=0.01)
    f.update(kw)
    return trainer._Exposure(f["param"], f["exp_avg"], f["exp_avg_sq"], f["step"], f["lr"])


@pytest.mark.parametrize("what,fields", BAD_STEP, ids=[b[0] for b in BAD_STEP])
def test_step_exposure_rejects_bad_rows(what, fields):
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        assert _step_call(L, h, C.byref(_exposure(**fields))) == -1
        assert b"psb_trainer_step_exposure" in L.psb_last_error() and b"exposure" in L.psb_last_error()
    finally:
        L.psb_trainer_destroy(h)


BAD_BWD = [("param", dict(param=None), ONE), ("lr nan", dict(lr=float("nan")), ONE), ("lr negative", dict(lr=-1.0), ONE),
           ("no exposure_grad", {}, None)]


@pytest.mark.parametrize("what,fields,grad", BAD_BWD, ids=[b[0] for b in BAD_BWD])
def test_backward_exposure_rejects_bad_rows(what, fields, grad):
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        # the moments and the step count are not needed in gradient mode
        assert _bwd_call(L, h, C.byref(_exposure(exp_avg=None, exp_avg_sq=None, step=None, **fields)), grad) == -1
        assert b"psb_trainer_backward_exposure" in L.psb_last_error()
    finally:
        L.psb_trainer_destroy(h)


def test_null_exposure_is_the_depth_call():
    """exposure == NULL: the _depth call's validation and messages (here: a bad depth term, and then a null camera)."""
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        bad = trainer._Depth(None, -1.0, None)
        assert _step_call(L, h, None, C.byref(bad)) == -1 and b"psb_trainer_step_depth: lambda_depth" in L.psb_last_error()
        assert _bwd_call(L, h, None, None, C.byref(bad)) == -1 and b"psb_trainer_backward_depth: lambda_depth" in L.psb_last_error()
        assert _step_call(L, h, None) == -1 and b"null argument" in L.psb_last_error()
        # a valid row still passes its own checks and stops at the same null argument
        assert _step_call(L, h, C.byref(_exposure())) == -1 and b"null argument" in L.psb_last_error()
        assert _bwd_call(L, h, C.byref(_exposure()), ONE) == -1 and b"null argument" in L.psb_last_error()
    finally:
        L.psb_trainer_destroy(h)


def test_symbols_declared_and_exported():
    L = _lib.lib()
    txt = open(HEADER).read()
    for n in ("psb_trainer_step_exposure", "psb_trainer_backward_exposure"):
        assert n in _lib.exported_symbols() and hasattr(L, n)
    assert "typedef struct psb_exposure {" in txt
    assert [f[0] for f in trainer._Exposure._fields_] == ["param", "exp_avg", "exp_avg_sq", "step", "lr"]


# ---- the Python table --------------------------------------------------------------------------------------------------------------
def _model():
    import photo_slam_b200.synthetic as syn
    sc = syn.make_scene(64, syn.make_camera(32, 24, 30.0, 30.0), seed=0)
    m = trainer.GaussianModel.from_numpy(sc, "cpu")
    m.trainingSetup(trainer.GaussianOptimizationParams())
    return m


def test_table_starts_empty_and_grows_with_identity_rows():
    m = trainer.GaussianModel(device="cpu")
    assert m.numExposures() == 0 and m.exposure_lr_ == 0.01 == trainer.GaussianOptimizationParams().exposure_lr
    m.ensureExposures(3)
    assert m.exposure_.shape == (3, 3, 4) and m.exposure_.dtype == torch.float32
    assert torch.equal(m.exposure_, torch.eye(3, 4).expand(3, 3, 4))
    assert not m.exposure_exp_avg_.any() and not m.exposure_exp_avg_sq_.any()
    assert m.exposure_step_.dtype == torch.int32 and m.exposure_step_.tolist() == [0, 0, 0]
    m.setExposureLearningRate(0.002)
    assert m.exposure_lr_ == 0.002


def test_growth_keeps_rows_moments_and_steps():
    m = trainer.GaussianModel(device="cpu")
    m.ensureExposures(2)
    gen = torch.Generator().manual_seed(0)
    for t in (m.exposure_, m.exposure_exp_avg_, m.exposure_exp_avg_sq_):
        t.copy_(torch.rand(t.shape, generator=gen))
    m.exposure_step_.copy_(torch.tensor([5, 7], dtype=torch.int32))
    old = [t.clone() for t in (m.exposure_, m.exposure_exp_avg_, m.exposure_exp_avg_sq_, m.exposure_step_)]
    m.ensureExposures(1)                      # never shrinks
    assert m.numExposures() == 2
    m.ensureExposures(5)
    assert m.numExposures() == 5
    for t, o in zip((m.exposure_, m.exposure_exp_avg_, m.exposure_exp_avg_sq_, m.exposure_step_), old):
        assert torch.equal(t[:2], o) and t.is_contiguous()
    assert torch.equal(m.exposure_[2:], torch.eye(3, 4).expand(3, 3, 4))
    assert not m.exposure_exp_avg_[2:].any() and m.exposure_step_[2:].tolist() == [0, 0, 0]


def test_apply_exposure_matches_einsum():
    m = trainer.GaussianModel(device="cpu")
    m.ensureExposures(2)
    m.exposure_[1] = torch.tensor([[1.3, 0.1, -0.05, 0.02], [0.04, 0.7, 0.03, -0.01], [-0.02, 0.05, 1.1, 0.03]])
    img = torch.rand(3, 7, 9)
    ref = torch.einsum("khw,kc->chw", img.double(), m.exposure_[1, :, :3].double()) + m.exposure_[1, :, 3, None, None].double()
    assert torch.allclose(m.applyExposure(img, 1).double(), ref, rtol=1e-6, atol=1e-6)
    assert torch.equal(m.applyExposure(img, 0), img)


def test_snapshot_restores_the_table():
    m = _model()
    m.ensureExposures(2)
    snap = m.snapshot()
    m.exposure_[1] += 0.5
    m.exposure_step_[1] = 3
    m.setExposureLearningRate(0.5)
    m.restore(snap)
    assert torch.equal(m.exposure_, torch.eye(3, 4).expand(2, 3, 4)) and m.exposure_step_.tolist() == [0, 0] and m.exposure_lr_ == 0.01
    m.ensureExposures(4)                      # grown since the snapshot: the snapshot's table comes back
    m.restore(snap)
    assert m.numExposures() == 2


def test_exposure_json_round_trip(tmp_path):
    m = trainer.GaussianModel(device="cpu")
    m.ensureExposures(3)
    m.exposure_[2] = torch.tensor([[1.25, 0.5, -0.125, 0.0625], [0.0, 0.75, 0.0, -0.25], [0.375, 0.0, 1.5, 0.125]])
    path = str(tmp_path / "exposure.json")
    m.saveExposure(path)
    raw = json.load(open(path))
    assert sorted(raw) == ["0", "1", "2"] and raw["2"][0] == [1.25, 0.5, -0.125, 0.0625]
    n = trainer.GaussianModel(device="cpu")
    n.ensureExposures(1)
    n.exposure_step_[0] = 4
    n.loadExposure(path)
    assert n.numExposures() == 3 and torch.equal(n.exposure_, m.exposure_)
    assert n.exposure_step_.tolist() == [0, 0, 0]
    assert set(io.load_exposure(path)) == {0, 1, 2}


def test_exposure_json_rejects_malformed_entries(tmp_path):
    with pytest.raises(ValueError):
        io.save_exposure(str(tmp_path / "a.json"), {0: np.eye(3)})
    p = tmp_path / "b.json"
    p.write_text(json.dumps({"frame_0001.png": np.eye(3, 4).tolist()}))
    with pytest.raises(ValueError):
        io.load_exposure(str(p))
    p.write_text(json.dumps({"0": [[1, 0, 0], [0, 1, 0], [0, 0, 1]]}))
    with pytest.raises(ValueError):
        io.load_exposure(str(p))


def test_data_parallel_trainer_refuses_an_exposure():
    dp = object.__new__(trainer.DataParallelTrainer)
    with pytest.raises(NotImplementedError, match="replicated"):
        dp.trainForOneIteration(None, None, exposure_id=0)
