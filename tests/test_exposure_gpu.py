"""-m gpu: per-keyframe exposure compensation in the fused step (psb_trainer_step_exposure / psb_trainer_backward_exposure,
GaussianTrainer.trainForOneIteration(..., exposure_id=k)).

  * an identity row with lr 0 is the plain step bit for bit (deterministic mode, mask, depth, SH-degree change);
  * the gradient mode's raw-parameter and exposure gradients match float64 autograd of the definition, back-propagated through
    render() + backwardPixels(grads=...) on the same model state (configs A, B and a 300x170 level; depth and anti-aliasing on / off);
  * the row's Adam matches torch.optim.Adam fed the fused gradients, its device step count advances by one per step, and every other
    row is untouched;
  * rows are bit-identical run to run in deterministic mode, and the exposure gradient is bit-identical call to call in default mode;
  * an overflowing pass leaves the row alone and the internal retry updates it exactly once;
  * on a scene whose targets went through known affines, compensation recovers them and the raw render's PSNR.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from helpers import scene_tensors
from splat64 import ssim64

pytestmark = pytest.mark.gpu
LAMBDA_DSSIM = 0.2
LAMBDA_DEPTH = 0.1
CONFIGS = {"A": (50_000, "tum", (640, 480)), "B": (500_000, "replica", (1200, 680)), "B300": (500_000, "replica", (300, 170))}
E_TEST = [[1.2, 0.05, -0.03, 0.04], [0.02, 0.8, 0.06, -0.05], [-0.04, 0.03, 1.1, 0.02]]


def _inputs(cuda, P, camname, wh, seed=3):
    cam, sc, act, g, c = scene_tensors(P, camname, seed=seed, pose_seed=seed + 1, dev=cuda, wh=wh, scale_px=2.4)
    W, H = wh
    gen = torch.Generator().manual_seed(seed + 2)
    gt = torch.rand((3, H, W), generator=gen).to(cuda)
    mask = torch.ones((3, H, W))
    mask[:, H // 8: H // 3, W // 6: W // 2] = 0.0
    depth = 0.5 + 7.5 * torch.rand((H, W), generator=gen)
    depth[torch.rand((H, W), generator=gen) < 0.1] = 0.0
    return sc, c, gt, mask.to(cuda), depth.to(cuda)


def _model(sc, cuda, sh=1):
    from photo_slam_b200 import trainer
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    m.setShDegree(sh)
    return m


def _trainer(m, **kw):
    from photo_slam_b200 import trainer
    tr = trainer.GaussianTrainer(m, background=torch.tensor([0.2, 0.3, 0.4], device=m.device), **kw)
    tr.opt.lambda_dssim = LAMBDA_DSSIM
    return tr


def _state(m):
    return [t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + [m.xyz_gradient_accum_, m.denom_, m.max_radii2D_]]


def _exposure_state(m):
    return [t.clone() for t in (m.exposure_, m.exposure_exp_avg_, m.exposure_exp_avg_sq_, m.exposure_step_)]


def _same(a, b):
    return len(a) == len(b) and all(x.shape == y.shape and torch.equal(x, y) for x, y in zip(a, b))


def _exposure_grads(tr, c, gt, mask, gd, E, segs):
    """psb_trainer_backward_exposure on the model's current state: raw-parameter gradients into segs, dL/dE returned ([3,4])"""
    from photo_slam_b200 import _lib, trainer
    m = tr.model
    cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)
    ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in segs])
    E = E.contiguous()
    egrad = torch.full((3, 4), float("nan"), device=m.device)
    ex = trainer._Exposure(E.data_ptr(), None, None, None, 0.01)
    d = trainer._Depth(gd.data_ptr(), LAMBDA_DEPTH, None) if gd is not None else None
    _lib.check(tr.L.psb_trainer_backward_exposure(tr.h, m.num_points(), 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(),
                                                  mask.data_ptr() if mask is not None else None, C.byref(cs), None, None, ptrs,
                                                  C.byref(d) if d is not None else None, C.byref(ex), egrad.data_ptr(),
                                                  torch.cuda.current_stream().cuda_stream), "psb_trainer_backward_exposure")
    tr.result()
    return egrad


def _reference_grads(tr, c, gt, mask, gd, E, grads):
    """float64 autograd of the definition on render(), then dL/dI through backwardPixels(grads=...): -> dL/dE [3,4] float64"""
    m = tr.model
    H, W = c["H"], c["W"]
    img = torch.empty((3, H, W), device=m.device)
    D = torch.empty((H, W), device=m.device) if gd is not None else None
    tr.render(c, img, out_depth=D)
    I = img.double().requires_grad_(True)
    E64 = E.double().requires_grad_(True)
    X = mask.double() * (torch.einsum("khw,kc->chw", I, E64[:, :3]) + E64[:, 3, None, None])
    G = gt.double()
    L = (1 - LAMBDA_DSSIM) * (X - G).abs().mean() + LAMBDA_DSSIM * (1 - ssim64(X, G))
    dI, dE = torch.autograd.grad(L, (I, E64))
    dD = None
    if gd is not None:   # the built-in depth L1: lambda * sign(D - G) / max(N_valid, 1) on the valid pixels
        valid = (gd > 0) & (mask[0] != 0)
        scale = np.float32(LAMBDA_DEPTH) / np.float32(max(int(valid.sum().item()), 1))
        dD = torch.where(valid, torch.sign(D - gd) * float(scale), torch.zeros_like(D)).contiguous()
    tr.backwardPixels(dI.float().contiguous(), dD, grads=grads)
    tr.result()
    return dE


def _relnorm(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize("aa", [False, True], ids=["plain", "aa"])
@pytest.mark.parametrize("with_depth", [False, True], ids=["colour", "depth"])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_gradients_match_autograd(cuda, config, with_depth, aa):
    from photo_slam_b200.parallel import GradBuffer
    P, camname, wh = CONFIGS[config]
    sc, c, gt, mask, gd = _inputs(cuda, P, camname, wh)
    m = _model(sc, cuda, sh=2)
    tr = _trainer(m, deterministic=True, antialiasing=aa)
    tr.render(c)      # grows the binning arena
    E = torch.tensor(E_TEST, device=cuda)
    P = m.num_points()
    fused, ref = GradBuffer(P, cuda), GradBuffer(P, cuda)
    egrad = _exposure_grads(tr, c, gt, mask, gd if with_depth else None, E, fused.segments)
    dE = _reference_grads(tr, c, gt, mask, gd if with_depth else None, E, ref.views())
    torch.cuda.synchronize()
    assert torch.isfinite(egrad).all() and fused.flat.abs().sum() > 0
    assert _relnorm(fused.flat, ref.flat) <= 1e-5, _relnorm(fused.flat, ref.flat)
    assert _relnorm(egrad, dE) <= 1e-5, (egrad, dE)


def test_identity_row_is_the_plain_step(cuda):
    P, camname, wh = CONFIGS["B300"]
    sc, c, gt, mask, gd = _inputs(cuda, P, camname, wh, seed=5)
    H, W = c["H"], c["W"]
    runs = []
    for use in (False, True):
        m = _model(sc, cuda)
        m.setExposureLearningRate(0.0)
        tr = _trainer(m, deterministic=True)
        tr.render(c)
        images, losses = [], []
        for it in range(8):
            if it == 4:
                m.oneUpShDegree()
            msk = mask if it % 2 == 0 else None
            kw = dict(gt_depth=gd, lambda_depth=LAMBDA_DEPTH) if it % 3 == 1 else {}
            img = torch.empty((3, H, W), device=cuda)
            tr.trainForOneIteration(c, gt, msk, out_color=img, exposure_id=0 if use else None, **kw)
            losses.append(tr.result_depth()[:4])
            images.append(img)
        torch.cuda.synchronize()
        runs.append((images, losses, _state(m), m))
    (ia, la, sa, _), (ib, lb, sb, mb) = runs
    assert _same(ia, ib) and la == lb
    assert _same(sa, sb)
    assert torch.equal(mb.exposure_[0], torch.eye(3, 4, device=cuda)) and mb.exposure_step_.tolist() == [8]


def test_adam_matches_torch_and_touches_one_row(cuda):
    from photo_slam_b200.parallel import GradBuffer
    P, camname, wh = CONFIGS["B300"]
    sc, c, gt, mask, gd = _inputs(cuda, P, camname, wh, seed=6)
    m = _model(sc, cuda)
    m.ensureExposures(5)
    gen = torch.Generator(device=cuda).manual_seed(0)
    m.exposure_ += 0.05 * torch.randn(m.exposure_.shape, device=cuda, generator=gen)   # every row non-identity
    m.exposure_exp_avg_ += 1e-3 * torch.randn(m.exposure_.shape, device=cuda, generator=gen)
    m.exposure_exp_avg_sq_ += 1e-6
    m.exposure_step_ += 2
    lr = m.exposure_lr_
    tr = _trainer(m, deterministic=True)
    tr.render(c)
    k = 3
    leaf = m.exposure_[k].clone().requires_grad_(True)
    opt = torch.optim.Adam([leaf], lr=lr, eps=1e-15, foreach=False, fused=False)
    opt.state[leaf] = dict(step=torch.tensor(2.0), exp_avg=m.exposure_exp_avg_[k].clone(), exp_avg_sq=m.exposure_exp_avg_sq_[k].clone())
    others = [i for i in range(5) if i != k]
    before = [t[others].clone() for t in _exposure_state(m)]
    buf = GradBuffer(m.num_points(), cuda)
    for it in range(5):
        g = _exposure_grads(tr, c, gt, mask, None, m.exposure_[k], buf.segments)   # the gradient the step below computes
        tr.trainForOneIteration(c, gt, mask, exposure_id=k)
        tr.result()
        leaf.grad = g.clone()
        opt.step()
        torch.cuda.synchronize()
        assert m.exposure_step_[k].item() == 3 + it
        d = (m.exposure_[k] - leaf.detach()).abs().max().item()
        assert d <= 2e-5 * lr + 1e-6 * leaf.detach().abs().max().item(), (it, d)
        assert torch.allclose(m.exposure_exp_avg_[k], opt.state[leaf]["exp_avg"], rtol=1e-5, atol=1e-9)
        assert torch.allclose(m.exposure_exp_avg_sq_[k], opt.state[leaf]["exp_avg_sq"], rtol=1e-5, atol=1e-12)
    assert _same([t[others] for t in _exposure_state(m)], before)


def test_deterministic_rows_repeat_and_gradient_repeats_in_default_mode(cuda):
    from photo_slam_b200.parallel import GradBuffer
    P, camname, wh = CONFIGS["A"]
    sc, c, gt, mask, gd = _inputs(cuda, P, camname, wh, seed=8)
    runs = []
    for _ in range(2):
        m = _model(sc, cuda)
        tr = _trainer(m, deterministic=True)
        tr.render(c)
        for it in range(6):
            tr.trainForOneIteration(c, gt, mask if it % 2 else None, exposure_id=1 + it % 2,
                                    **(dict(gt_depth=gd, lambda_depth=LAMBDA_DEPTH) if it == 3 else {}))
            tr.result()
        torch.cuda.synchronize()
        runs.append(_exposure_state(m) + _state(m))
    assert _same(runs[0], runs[1])
    assert not torch.equal(runs[0][0][1], torch.eye(3, 4, device=cuda))
    # default mode: the exposure gradient has no atomics behind it
    m = _model(sc, cuda)
    tr = _trainer(m, deterministic=False)
    tr.render(c)
    E = torch.tensor(E_TEST, device=cuda)
    buf = GradBuffer(m.num_points(), cuda)
    a = _exposure_grads(tr, c, gt, mask, gd, E, buf.segments).clone()
    b = _exposure_grads(tr, c, gt, mask, gd, E, buf.segments).clone()
    torch.cuda.synchronize()
    assert torch.equal(a, b) and a.abs().sum() > 0


def test_overflowing_pass_leaves_the_row_and_the_retry_updates_it_once(cuda):
    from photo_slam_b200 import trainer
    P, wh = 2_000, (640, 480)
    cam, sc, act, g, c = scene_tensors(P, "tum", seed=2, pose_seed=None, dev=cuda, wh=wh, scale_px=150.0)  # overflows the initial arena
    gt = torch.rand((3, wh[1], wh[0]), device=cuda)
    a = trainer.GaussianModel.from_numpy(sc, cuda)
    a.trainingSetup(trainer.GaussianOptimizationParams())
    a.ensureExposures(1)
    ta = trainer.GaussianTrainer(a)
    ta.trainForOneIteration(c, gt, exposure_id=0)
    torch.cuda.synchronize()
    assert _same(_exposure_state(a), [torch.eye(3, 4, device=cuda)[None], torch.zeros(1, 3, 4, device=cuda), torch.zeros(1, 3, 4, device=cuda),
                                      torch.zeros(1, dtype=torch.int32, device=cuda)]), "the overflowing attempt moved the row"
    n = ta.result()[3]        # repeated internally
    assert n > 6 * P + 65536, "test scene must overflow the initial arena"
    torch.cuda.synchronize()
    assert a.step_ == 1 and a.exposure_step_.tolist() == [1]
    # the same step on an arena grown beforehand
    b = trainer.GaussianModel.from_numpy(sc, cuda)
    b.trainingSetup(trainer.GaussianOptimizationParams())
    tb = trainer.GaussianTrainer(b)
    tb.render(c)
    tb.render(c)
    tb.trainForOneIteration(c, gt, exposure_id=0)
    tb.result()
    torch.cuda.synchronize()
    assert _same(_exposure_state(a), _exposure_state(b))
    assert not torch.equal(a.exposure_[0], torch.eye(3, 4, device=cuda))


def _recovery(cuda, compensate, steps, W=300, H=170, views=8):
    """Targets: renders of a target scene from `views` poses, view k through a known affine E*_k (view 0: identity). A model from another
    seed trains on them with or without compensation (view 0 at lr 0). -> (mean PSNR of the raw render against the untransformed
    renders, ||E - E*|| over views 1.., the true rows)"""
    import photo_slam_b200.synthetic as syn
    from photo_slam_b200 import trainer
    rng = np.random.default_rng(1)
    cams = []
    for _ in range(views):
        cam = syn.make_camera(W, H, 150.0, 150.0, *syn.random_pose(rng, max_angle=0.1, max_trans=0.1))
        cams.append((cam, syn.device_camera(cam, cuda)))
    tm = trainer.GaussianModel.from_numpy(syn.make_scene(20_000, cams[0][0], seed=11, scale_px=2.0), cuda)
    raw = [trainer.GaussianTrainer(tm).render(c) for _, c in cams]
    Es = torch.zeros(views, 3, 4)
    Es[:, :, :3] = torch.eye(3)
    for k in range(1, views):
        Es[k, :, :3] = torch.diag(torch.from_numpy(rng.uniform(0.6, 1.4, 3)).float()) + torch.from_numpy(rng.uniform(-0.05, 0.05, (3, 3))).float() * (1 - torch.eye(3))
        Es[k, :, 3] = torch.from_numpy(rng.uniform(-0.05, 0.05, 3)).float()
    Es = Es.to(cuda)
    em = trainer.GaussianModel(device=cuda)
    em.ensureExposures(views)
    em.exposure_.copy_(Es)
    targets = [em.applyExposure(img, k).contiguous() for k, img in enumerate(raw)]
    m = trainer.GaussianModel.from_numpy(syn.make_scene(20_000, cams[0][0], seed=12, scale_px=2.0), cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    m.ensureExposures(views)
    tr = trainer.GaussianTrainer(m)
    lr = m.exposure_lr_
    for it in range(steps):
        k = it % views
        m.setExposureLearningRate(0.0 if k == 0 else lr)
        tr.trainForOneIteration(cams[k][1], targets[k], densify_stats=False, exposure_id=k if compensate else None)
        tr.result()
    psnr = []
    for (_, c), ref in zip(cams, raw):
        mse = ((tr.render(c) - ref) ** 2).mean().item()
        psnr.append(10 * math.log10(1.0 / max(mse, 1e-12)))
    return float(np.mean(psnr)), (m.exposure_[1:] - Es[1:]).norm().item(), (torch.eye(3, 4, device=cuda) - Es[1:]).norm().item()


def test_compensation_recovers_the_exposures(cuda):
    # measured on an H100 80GB HBM3 (700 W): PSNR 24.85 dB compensated, 21.39 dB uncompensated (+3.46 dB); |E - E*| 0.454 against 0.994
    # for the identity rows. The gates keep about half of each margin as headroom.
    p_on, err_on, err_eye = _recovery(cuda, True, 400)
    p_off, _, _ = _recovery(cuda, False, 400)
    print(f"recovery: PSNR compensated {p_on:.3f} dB, uncompensated {p_off:.3f} dB; |E - E*| {err_on:.4f} (identity: {err_eye:.4f})")
    assert p_on > p_off + 1.5
    assert err_on < 0.75 * err_eye
