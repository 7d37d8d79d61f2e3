"""Depth distortion (include/psb200.h, "Depth distortion") without a device: the float64 restatement tests/dist64.py against a per-pixel
pairwise loop, its closed-form gradients under gradcheck, the moment plane of a small scene against a per-pixel loop over splat64's
weights, the psb_dist layout, the refusals of the C entries, and the Python front end against a stub library."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import dist64
import splat64 as s64
from photo_slam_b200 import _lib, trainer
from test_normal_cpu import ONE, E, _StubL, _cam, _rejects, stubbed  # noqa: F401  (stubbed: a fixture)


def _pixels(seed, npix=40, n=6):
    rng = np.random.default_rng(seed)
    alpha = rng.uniform(0.05, 0.9, (npix, n))
    T = np.cumprod(np.concatenate([np.ones((npix, 1)), 1.0 - alpha[:, :-1]], 1), 1)
    return torch.from_numpy(alpha * T), torch.from_numpy(rng.uniform(1.0, 6.0, (npix, n)))


def test_distortion_equals_the_pairwise_sum_pixel_by_pixel():
    w, z = _pixels(1)
    A, D, M = dist64.planes64(w, z)
    for p in range(w.shape[0]):
        pair = 0.0
        for i in range(w.shape[1]):
            for j in range(w.shape[1]):
                pair += 0.5 * float(w[p, i] * w[p, j]) * float(z[p, i] - z[p, j]) ** 2
        assert abs(float(A[p] * M[p] - D[p] ** 2) - pair) <= 1e-12 * max(pair, 1.0)
        assert abs(float(dist64.pairwise64(w[p], z[p])) - pair) <= 1e-12 * max(pair, 1.0)
    # one depth per ray: no distortion, and no depth spread
    A1, D1, M1 = dist64.planes64(w, torch.full_like(z, 3.0))
    assert float((A1 * M1 - D1 * D1).abs().max()) < 1e-12
    assert float(dist64.spread64(D1, A1, M1).max()) < 1e-6
    # the spread is the weighted standard deviation of the depths
    sd = torch.sqrt((w * (z - (D / A)[:, None]) ** 2).sum(1) / A)
    assert float((dist64.spread64(D, A, M) - sd).abs().max()) < 1e-12


@pytest.mark.parametrize("with_mask", [False, True])
def test_dist64_is_the_valid_mean(with_mask):
    w, z = _pixels(2, npix=48)
    A, D, M = (x.reshape(6, 8) for x in dist64.planes64(w, z))
    mask = torch.from_numpy((np.random.default_rng(3).random((6, 8)) > 0.4).astype(np.float64)) if with_mask else None
    dist, nv = dist64.dist64(D, A, M, mask)
    per = dist64.pairwise64(w, z).reshape(6, 8)
    keep = mask != 0 if with_mask else torch.ones_like(per, dtype=torch.bool)
    assert nv == int(keep.sum()) and nv > 10
    assert abs(float(dist) - float(per[keep].sum()) / nv) < 1e-12
    # a [k,H,W] mask reads channel 0
    if with_mask:
        assert float(dist64.dist64(D, A, M, mask[None].expand(3, 6, 8))[0]) == float(dist)


@pytest.mark.parametrize("with_mask", [False, True])
def test_closed_form_gradients_against_gradcheck(with_mask):
    w, z = _pixels(4, npix=20)
    A, D, M = (x.reshape(4, 5).clone().requires_grad_(True) for x in dist64.planes64(w, z))
    mask = torch.from_numpy((np.random.default_rng(5).random((4, 5)) > 0.3).astype(np.float64)) if with_mask else None
    lam = 0.7
    f = lambda d, a, m: lam * dist64.dist64(d, a, m, mask)[0]
    assert torch.autograd.gradcheck(f, (D, A, M), eps=1e-6, atol=1e-8)
    gD, gA, gM = torch.autograd.grad(f(D, A, M), (D, A, M))
    cA, cD, cM = dist64.grads64(D.detach(), A.detach(), M.detach(), lam, mask)
    for a, b in ((gA, cA), (gD, cD), (gM, cM)):
        assert float((a - b).abs().max()) < 1e-15
    # per Gaussian, dL/dz_i = 2k w_i (A z_i - D) (2DGS's gradient) through M = sum w z^2 and D = sum w z
    zz = z.clone().requires_grad_(True)
    A2, D2, M2 = dist64.planes64(w, zz)
    (gz,) = torch.autograd.grad(lam * dist64.dist64(D2, A2, M2)[0], zz)
    k = lam / w.shape[0]
    assert float((gz - 2 * k * w * (A2.detach()[:, None] * z - D2.detach()[:, None])).abs().max()) < 1e-14


def test_moment_plane_of_a_small_scene_is_the_blend_of_z_squared():
    """render_moment's M equals sum w z^2 over the per-pixel weights of splat64's blend, recomputed here pixel by pixel"""
    import photo_slam_b200.synthetic as syn
    W, H = 24, 16
    cam = syn.make_camera(W, H, 20.0, 20.0, *syn.random_pose(np.random.default_rng(0)))
    sc = syn.make_scene(60, cam, seed=2, scale_px=3.0)
    c = s64.camera64(cam, "cpu")
    raw = s64.raw64(sc, "cpu")
    out, M = dist64.render_moment(raw, c, D=1)
    geo = s64.geometry(s64.activate(raw), c, 1)
    live = geo["alive"].nonzero().reshape(-1)
    order = live[torch.argsort(geo["zd"][live], stable=True)]
    ref = torch.zeros(H, W, dtype=torch.float64)
    for y in range(H):
        for x in range(W):
            T, acc = 1.0, 0.0
            for g in order.tolist():
                r = geo["rect"][g]
                if not (r[0] <= x // s64.TILE < r[2] and r[1] <= y // s64.TILE < r[3]):
                    continue
                dx, dy = float(geo["means2D"][g, 0]) - x, float(geo["means2D"][g, 1]) - y
                a, b, cc = (float(v) for v in geo["conic"][g])
                power = -0.5 * (a * dx * dx + cc * dy * dy) - b * dx * dy
                alpha = min(s64.ALPHA_MAX, float(geo["o"][g]) * math.exp(power))
                if power > 0 or alpha < s64.CONV.alpha_min:
                    continue
                if T * (1.0 - alpha) < s64.CONV.t_min:
                    break
                acc += alpha * T * float(geo["z"][g]) ** 2
                T *= 1.0 - alpha
            ref[y, x] = acc
    assert float(M.max()) > 1.0
    assert float((M.detach() - ref).abs().max()) < 1e-9 * float(ref.max())
    assert float((dist64.spread64(out["depth"], out["alpha"], M)).min()) >= 0.0


# ---- the C entries ---------------------------------------------------------------------------------------------------------------
def test_psb_dist_layout():
    assert [f[0] for f in trainer._Dist._fields_] == ["lambda_dist", "out_depth2"]
    assert trainer._Dist.lambda_dist.offset == 0 and trainer._Dist.out_depth2.offset == 8 and C.sizeof(trainer._Dist) == 16


def test_header_declares_and_library_exports_the_entries():
    names = _lib.exported_symbols()
    L = _lib.lib()
    for n in ("psb_trainer_forward_moment", "psb_trainer_backward_pixels_moment", "psb_trainer_step_dist", "psb_trainer_result_dist"):
        assert n in names and hasattr(L, n), n


def test_step_dist_refuses_bad_terms_without_a_device():
    L = trainer._bind()
    t = C.c_void_p()
    assert L.psb_trainer_create(C.byref(t)) == 0
    try:
        m, cam, step = trainer._Model(), _cam(), trainer._Step()
        for i in range(6):
            m.param[i] = m.exp_avg[i] = m.exp_avg_sq[i] = ONE
        step.step, step.sh_degree = 1, 3
        for lam in (-1.0, -1e-30, math.nan, math.inf, -math.inf):
            d = trainer._Dist(lam, None)
            _rejects(L, "psb_trainer_step_dist", t, 10, 16, C.byref(m), C.byref(cam), ONE, ONE, None, C.byref(step), None, None, None, None, None, None,
                     C.byref(d), None)
        # what psb_trainer_step_dn refuses, psb_trainer_step_dist refuses with a valid term
        ok = trainer._Dist(1.0, None)
        bad_dn = trainer._Dn(-1.0, 0.5, 0.05, None)
        _rejects(L, "psb_trainer_step_dist", t, 10, 16, C.byref(m), C.byref(cam), ONE, ONE, None, C.byref(step), None, None, None, None, None,
                 C.byref(bad_dn), C.byref(ok), None)
        nrm = trainer._Normal(None, 0.5, None)
        _rejects(L, "psb_trainer_step_dist", t, 10, 16, C.byref(m), C.byref(cam), ONE, ONE, None, C.byref(step), None, None, None, None, C.byref(nrm),
                 None, C.byref(ok), None)
        step.step = 0
        assert L.psb_trainer_step_dist(t, 10, 16, C.byref(m), C.byref(cam), ONE, ONE, None, C.byref(step), None, None, None, None, None, None,
                                       C.byref(ok), None) == E
        # no forward pass has run: a moment gradient is refused like any other stale pass
        step.step = 1
        px = trainer._PixelGrads(ONE, None, None)
        assert L.psb_trainer_backward_pixels_moment(t, 1, 10, 16, C.byref(m), C.byref(cam), ONE, C.byref(px), None, ONE, C.byref(step), None,
                                                    None) == E
        out = (C.c_float * 7)()
        assert L.psb_trainer_result_dist(t, out, None, None) == E
    finally:
        L.psb_trainer_destroy(t)


# ---- the Python front end against a stub library -------------------------------------------------------------------------------------
def test_lambda_dist_zero_is_todays_call(stubbed):
    tr, m, cam, L = stubbed
    Hc, Wc = cam["H"], cam["W"]
    gt = torch.rand(3, Hc, Wc)
    tr.trainForOneIteration(cam, gt, lambda_dist=0.0)
    assert L.calls[-1] == "psb_trainer_step_exposure"
    tr.trainForOneIteration(cam, gt, lambda_dn=0.05, lambda_dist=0.0)
    assert L.calls[-1] == "psb_trainer_step_dn"
    tr.trainForOneIteration(cam, gt, lambda_dist=1.0)
    assert L.calls[-1] == "psb_trainer_step_dist"
    tr.trainForOneIteration(cam, gt, out_depth2=torch.zeros(Hc, Wc))
    assert L.calls[-1] == "psb_trainer_step_dist"
    tr.trainForOneIteration(cam, gt, lambda_dist=1.0, lambda_dn=0.05, gt_normal=torch.zeros(3, Hc, Wc), lambda_normal=0.1)
    assert L.calls[-1] == "psb_trainer_step_dist"
    assert m.step_ == 5 and tr.iteration == 5
    n = len(L.calls)
    tr._last.repeat()                              # the retry record repeats the call with its term
    assert L.calls[n:] == ["psb_trainer_step_dist"]
    with pytest.raises(ValueError):
        tr.trainForOneIteration(cam, gt, lambda_dist=1.0, out_depth2=torch.zeros(Wc, Hc))
    assert L.calls[n + 1:] == []


def test_render_and_backward_pixels_take_the_moment_plane(stubbed):
    tr, m, cam, L = stubbed
    H, W = cam["H"], cam["W"]
    grads = [torch.zeros_like(t) for t in m.tensors()]
    tr.render(cam, check=False, out_depth2=torch.zeros(H, W))
    assert L.calls[-1] == "psb_trainer_forward_moment"
    tr.backwardPixels(torch.zeros(3, H, W), grads=grads, dL_ddepth2=torch.zeros(H, W))
    assert L.calls[-1] == "psb_trainer_backward_pixels_moment"
    tr.backwardPixels(torch.zeros(3, H, W), grads=grads)
    assert L.calls[-1] == "psb_trainer_backward_pixels"
    tr.render(cam, check=False, out_normal=torch.zeros(3, H, W))
    assert L.calls[-1] == "psb_trainer_forward_normal"
    n = len(L.calls)
    with pytest.raises(ValueError, match="dL_ddepth2"):     # a render without the plane takes no moment gradient
        tr.backwardPixels(torch.zeros(3, H, W), grads=grads, dL_ddepth2=torch.zeros(H, W))
    with pytest.raises(ValueError):
        tr.render(cam, check=False, out_depth2=torch.zeros(W, H))
    assert L.calls[n:] == []
    tr.render(cam, check=False, out_depth2=torch.zeros(H, W))
    with pytest.raises(ValueError):
        tr.backwardPixels(torch.zeros(3, H, W), grads=grads, dL_ddepth2=torch.zeros(3, H, W))
    # trainWithLoss hands M to the loss as an autograd leaf, after image, depth, alpha and normal
    seen = []

    def loss_fn(img, D, M):
        seen.append((tuple(img.shape), tuple(D.shape), tuple(M.shape), M.requires_grad))
        return img.sum() + (D * M).sum()
    tr.trainWithLoss(cam, loss_fn, depth=True, depth2=True)
    assert seen == [((3, H, W), (H, W), (H, W), True)]
    assert L.calls[-2:] == ["psb_trainer_forward_moment", "psb_trainer_backward_pixels_moment"]
    assert m.step_ == 1 and tr.iteration == 1


def test_data_parallel_trainer_refuses_the_term():
    dp = object.__new__(trainer.DataParallelTrainer)
    for kw in (dict(lambda_dist=1.0), dict(out_depth2=torch.zeros(2, 2))):
        with pytest.raises(NotImplementedError, match="distortion"):
            dp.trainForOneIteration(dict(), None, **kw)
