"""Depth-normal consistency (include/psb200.h, "Depth-normal consistency") without a device: the float64 restatement tests/dn64.py against a
per-pixel loop, on analytic tilted planes and under gradcheck; the psb_dn layout, the refusals of the C entries, and the Python front end
against a stub library."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import dn64
from photo_slam_b200 import _lib, trainer
from test_normal_cpu import ONE, E, _StubL, _cam, _loop, _plane_depth, _rejects, stubbed  # noqa: F401  (stubbed: a fixture)

W, H, TX, TY = 12, 9, 0.6, 0.45


def _dn_loop(D, A, N, mask, W, H, tx, ty, alpha_min, jump):
    """the definition pixel by pixel: D-bar, n_d by normal64's per-pixel loop of psb_depth_normals, then the valid sum"""
    Db = np.where(A >= alpha_min, D / np.where(A >= alpha_min, A, 1.0), 0.0)
    nd = _loop(Db, W, H, tx, ty, jump)
    tot, nv = 0.0, 0
    for v in range(H):
        for u in range(W):
            if nd[:, v, u].any() and (mask is None or mask[v, u] != 0):
                tot += 1.0 - nd[:, v, u] @ N[:, v, u]
                nv += 1
    return tot / max(nv, 1), nv, nd


def _random_planes(seed, W=W, H=H, holes=True):
    rng = np.random.default_rng(seed)
    z = 2.0 + 0.02 * rng.standard_normal((H, W))     # D-bar: a bumpy surface, within max_rel_jump of its neighbours
    A = rng.uniform(0.55, 1.0, (H, W))
    if holes:
        A[rng.random((H, W)) < 0.1] = 0.2          # below alpha_min: holes of D-bar
        z[rng.random((H, W)) < 0.05] *= 1.5        # depth edges
    D = z * A
    N = rng.standard_normal((3, H, W))
    N *= (A / np.linalg.norm(N, axis=0))[None] * rng.uniform(0.3, 1.0, (H, W))[None]   # |N| <= A
    return D, A, N


@pytest.mark.parametrize("with_mask", [False, True])
def test_dn64_equals_a_per_pixel_loop(with_mask):
    D, A, N = _random_planes(1)
    mask = (np.random.default_rng(2).random((H, W)) > 0.3).astype(np.float64) if with_mask else None
    ref, nv_ref, nd_ref = _dn_loop(D, A, N, mask, W, H, TX, TY, 0.5, 0.05)
    T = torch.from_numpy
    dn, nv, nd = dn64.dn64(T(D), T(A), T(N), W, H, TX, TY, 0.5, 0.05, T(mask) if mask is not None else None)
    assert nv == nv_ref and nv > 10 and (nd_ref == 0).all(0).sum() > 10
    assert np.abs(nd.numpy() - nd_ref).max() < 1e-12
    assert abs(float(dn) - ref) < 1e-12


# (tilt, tan_fov) as tests/test_normal_cpu.py: the view narrows as the plane approaches grazing
@pytest.mark.parametrize("tilt_deg,tan_fov", [(0.0, 0.6), (30.0, 0.6), (60.0, 0.3), (85.0, 0.05)])
def test_tilted_planes_give_the_plane_normal_and_one_minus_n_dot_N(tilt_deg, tan_fov):
    Wp, Hp = 40, 30
    t = math.radians(tilt_deg)
    n = np.array([math.sin(t) * 0.6, math.sin(t) * 0.8, -math.cos(t)])     # faces the camera
    z = _plane_depth(n, -3.0, W=Wp, H=Hp, tx=tan_fov, ty=tan_fov)
    A = np.full((Hp, Wp), 0.8)
    rng = np.random.default_rng(3)
    N = rng.standard_normal((3, Hp, Wp)) * 0.4
    T = torch.from_numpy
    # the rendered depth is D = z A: the normalisation by A recovers the plane (the scale of the depth does not matter)
    for scale in (1.0, 0.01):
        dn, nv, nd = dn64.dn64(T(scale * z * A), T(A), T(N), Wp, Hp, tan_fov, tan_fov, 0.5, 10.0)
        inner = nd[:, 1:-1, 1:-1].reshape(3, -1).numpy()
        assert nv == (Wp - 2) * (Hp - 2)
        assert np.abs(inner - n[:, None]).max() < 1e-9
        want = (1.0 - np.einsum("c,chw->hw", n, N[:, 1:-1, 1:-1])).mean()
        assert abs(float(dn) - want) < 1e-9


@pytest.mark.parametrize("with_mask", [False, True])
def test_gradcheck_in_depth_alpha_and_normal(with_mask):
    Wg, Hg = 6, 5
    D, A, N = _random_planes(4, Wg, Hg, holes=False)
    A[1, 2] = 0.3                                  # one hole of D-bar inside the image
    mask = torch.from_numpy((np.random.default_rng(5).random((Hg, Wg)) > 0.3).astype(np.float64)) if with_mask else None
    Dt, At, Nt = (torch.from_numpy(x).requires_grad_(True) for x in (D, A, N))
    f = lambda d, a, nn: dn64.dn64(d, a, nn, Wg, Hg, TX, TY, 0.5, 1.0, mask)[0]
    assert dn64.dn64(Dt, At, Nt, Wg, Hg, TX, TY, 0.5, 1.0, mask)[1] > 3
    assert torch.autograd.gradcheck(f, (Dt, At, Nt), eps=1e-6, atol=1e-7)
    # the gradient reaches D and A only where A >= alpha_min
    gD, gA, _ = torch.autograd.grad(f(Dt, At, Nt), (Dt, At, Nt))
    assert gD[1, 2] == 0 and gA[1, 2] == 0 and gD.abs().sum() > 0 and gA.abs().sum() > 0


# ---- the C entries ---------------------------------------------------------------------------------------------------------------
def test_psb_dn_layout():
    assert [f[0] for f in trainer._Dn._fields_] == ["lambda_dn", "alpha_min", "max_rel_jump", "out_depth_normal"]
    assert trainer._Dn.lambda_dn.offset == 0 and trainer._Dn.alpha_min.offset == 4 and trainer._Dn.max_rel_jump.offset == 8
    assert trainer._Dn.out_depth_normal.offset == 16 and C.sizeof(trainer._Dn) == 24


def test_header_declares_and_library_exports_the_entries():
    names = _lib.exported_symbols()
    L = _lib.lib()
    for n in ("psb_trainer_step_dn", "psb_trainer_result_dn", "psb_dn_loss"):
        assert n in names and hasattr(L, n), n


_BAD_DN = ((0.0, 0.5, 0.05), (-1.0, 0.5, 0.05), (math.nan, 0.5, 0.05), (math.inf, 0.5, 0.05), (0.05, 0.0, 0.05), (0.05, -0.1, 0.05),
           (0.05, 1.5, 0.05), (0.05, math.nan, 0.05), (0.05, 0.5, 0.0), (0.05, 0.5, -1.0), (0.05, 0.5, math.nan), (0.05, 0.5, math.inf))


def test_dn_loss_refuses_bad_arguments_without_a_device():
    L = trainer._bind()
    ok = trainer._Dn(0.05, 0.5, 0.05, None)
    planes = [ONE] * 3
    for i in range(3):                             # a NULL input plane
        p = list(planes)
        p[i] = None
        _rejects(L, "psb_dn_loss", C.byref(_cam()), *p, None, C.byref(ok), ONE, ONE, ONE, None, None)
    for i in range(3):                             # a NULL gradient plane
        g = [ONE] * 3
        g[i] = None
        _rejects(L, "psb_dn_loss", C.byref(_cam()), *planes, None, C.byref(ok), *g, None, None)
    _rejects(L, "psb_dn_loss", None, *planes, None, C.byref(ok), ONE, ONE, ONE, None, None)
    _rejects(L, "psb_dn_loss", C.byref(_cam()), *planes, None, None, ONE, ONE, ONE, None, None)
    for cam in (_cam(W=0), _cam(H=-1), _cam(tanx=0.0), _cam(tany=math.inf), _cam(tanx=math.nan)):
        _rejects(L, "psb_dn_loss", C.byref(cam), *planes, None, C.byref(ok), ONE, ONE, ONE, None, None)
    for lam, amin, jump in _BAD_DN:
        d = trainer._Dn(lam, amin, jump, None)
        _rejects(L, "psb_dn_loss", C.byref(_cam()), *planes, ONE, C.byref(d), ONE, ONE, ONE, None, None)


def test_step_dn_refuses_bad_terms_without_a_device():
    L = trainer._bind()
    t = C.c_void_p()
    assert L.psb_trainer_create(C.byref(t)) == 0
    try:
        m, cam, step = trainer._Model(), _cam(), trainer._Step()
        for i in range(6):
            m.param[i] = m.exp_avg[i] = m.exp_avg_sq[i] = ONE
        step.step, step.sh_degree = 1, 3
        for lam, amin, jump in _BAD_DN:
            d = trainer._Dn(lam, amin, jump, None)
            _rejects(L, "psb_trainer_step_dn", t, 10, 16, C.byref(m), C.byref(cam), ONE, ONE, None, C.byref(step), None, None, None, None, None,
                     C.byref(d), None)
        # what psb_trainer_step_normal refuses, psb_trainer_step_dn refuses with a valid term
        ok = trainer._Dn(0.05, 0.5, 0.05, None)
        nrm = trainer._Normal(None, 0.5, None)
        _rejects(L, "psb_trainer_step_dn", t, 10, 16, C.byref(m), C.byref(cam), ONE, ONE, None, C.byref(step), None, None, None, None, C.byref(nrm),
                 C.byref(ok), None)
        step.step = 0
        assert L.psb_trainer_step_dn(t, 10, 16, C.byref(m), C.byref(cam), ONE, ONE, None, C.byref(step), None, None, None, None, None, C.byref(ok),
                                     None) == E
        out = (C.c_float * 6)()
        assert L.psb_trainer_result_dn(t, out, None, None) == E
    finally:
        L.psb_trainer_destroy(t)


# ---- the Python front end against a stub library -------------------------------------------------------------------------------------
def test_lambda_dn_zero_is_todays_call(stubbed):
    tr, m, cam, L = stubbed
    Hc, Wc = cam["H"], cam["W"]
    gt = torch.rand(3, Hc, Wc)
    tr.trainForOneIteration(cam, gt, lambda_dn=0.0)
    assert L.calls[-1] == "psb_trainer_step_exposure"
    tr.trainForOneIteration(cam, gt, gt_normal=torch.zeros(3, Hc, Wc), lambda_normal=0.1, lambda_dn=0.0)
    assert L.calls[-1] == "psb_trainer_step_normal"
    tr.trainForOneIteration(cam, gt, lambda_dn=0.05)
    assert L.calls[-1] == "psb_trainer_step_dn"
    tr.trainForOneIteration(cam, gt, lambda_dn=0.05, out_depth_normal=torch.zeros(3, Hc, Wc), gt_normal=torch.zeros(3, Hc, Wc), lambda_normal=0.1)
    assert L.calls[-1] == "psb_trainer_step_dn"
    assert m.step_ == 4 and tr.iteration == 4
    n = len(L.calls)
    tr._last.repeat()                              # the retry record repeats the call with its term
    assert L.calls[n:] == ["psb_trainer_step_dn"]
    with pytest.raises(ValueError):
        tr.trainForOneIteration(cam, gt, lambda_dn=0.05, out_depth_normal=torch.zeros(3, Wc, Hc))
    assert L.calls[n + 1:] == []


def test_data_parallel_trainer_refuses_the_term():
    dp = object.__new__(trainer.DataParallelTrainer)
    for kw in (dict(lambda_dn=0.05), dict(out_depth_normal=torch.zeros(3, 2, 2))):
        with pytest.raises(NotImplementedError, match="consistency"):
            dp.trainForOneIteration(dict(), None, **kw)
