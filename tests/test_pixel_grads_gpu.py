"""-m gpu: training the fused step against a caller's loss (psb_trainer_forward / psb_trainer_backward_pixels; GaussianTrainer.render
with out_alpha, backwardPixels, trainWithLoss).

  * the forward's colour, depth and radii equal psb_trainer_render_depth's, and its accumulated opacity is 1 - final_T;
  * the built-in loss fed through the pixel-gradient path reproduces trainForOneIteration bit for bit in deterministic mode (Adam and
    gradient modes), over steps with a mask, an SH-degree change and a depth target on some steps;
  * the gradients of a linear loss on image, depth and opacity match autograd through the operator path (renderer.render);
  * trainWithLoss is bit-identical run to run in deterministic mode, and an overflowing forward is repeated by result();
  * a stale pass, a size or SH-degree mismatch and a missing colour gradient raise and leave the model untouched.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from helpers import scene_tensors

pytestmark = pytest.mark.gpu
WH = (600, 340)
LAMBDA_DSSIM = 0.2
LAMBDA_DEPTH = 0.1


def _inputs(cuda, P=60_000, scale_px=6.0, seed=3, wh=WH):
    cam, sc, act, g, c = scene_tensors(P, "replica", seed=seed, pose_seed=seed + 1, dev=cuda, wh=wh, scale_px=scale_px)
    W, H = wh
    gen = torch.Generator().manual_seed(seed + 2)
    gt = torch.rand((3, H, W), generator=gen).to(cuda)
    mask = torch.ones((3, H, W))
    mask[:, 40:120, 100:260] = 0.0
    depth = 0.5 + 7.5 * torch.rand((H, W), generator=gen)
    depth[torch.rand((H, W), generator=gen) < 0.1] = 0.0
    return sc, c, gt, mask.to(cuda), depth.to(cuda)


def _model(sc, cuda, sh=1):
    from photo_slam_b200 import trainer
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    m.setShDegree(sh)
    return m


def _state(m):
    return [t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + [m.xyz_gradient_accum_, m.denom_, m.max_radii2D_]]


def _assert_same_state(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and torch.equal(x, y), f"model state tensor {i} differs"


def _debug_final_T(tr, W, H, dev):
    from photo_slam_b200 import _lib
    last = torch.empty(W * H, dtype=torch.int32, device=dev)
    fT = torch.empty(W * H, dtype=torch.float32, device=dev)
    _lib.check(tr.L.psb_trainer_debug_state(tr.h, W, H, last.data_ptr(), fT.data_ptr(), None, torch.cuda.current_stream().cuda_stream), "debug_state")
    return last.reshape(H, W), fT.reshape(H, W)


def _builtin_dL_ddepth(D, G, mask):
    """dL/dD of the built-in depth term, with the float expression of depth_grad_scale_kernel: sign(D - G) * (lambda / max(N_valid, 1))"""
    valid = G > 0
    if mask is not None:
        valid &= mask[0] != 0
    scale = np.float32(LAMBDA_DEPTH) / np.float32(max(int(valid.sum().item()), 1))
    return torch.where(valid, torch.sign(D - G) * float(scale), torch.zeros_like(D)).contiguous()


def test_forward_outputs_and_opacity(cuda):
    from photo_slam_b200 import trainer
    sc, c, gt, mask, gd = _inputs(cuda)
    P, H, W = sc["xyz"].shape[0], c["H"], c["W"]
    tr = trainer.GaussianTrainer(_model(sc, cuda))
    tr.render(c)      # grows the binning arena: the direct call below fits
    img0, rad0, dep0 = torch.empty((3, H, W), device=cuda), torch.zeros(P, dtype=torch.int32, device=cuda), torch.empty((H, W), device=cuda)
    from photo_slam_b200 import _lib
    m = tr.model
    cm, cc = m._cmodel(False), trainer._ccamera(c)
    _lib.check(tr.L.psb_trainer_render_depth(tr.h, P, 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), m.active_sh_degree_, img0.data_ptr(),
                                             rad0.data_ptr(), dep0.data_ptr(), torch.cuda.current_stream().cuda_stream), "psb_trainer_render_depth")
    tr.result()
    img1, rad1 = torch.empty((3, H, W), device=cuda), torch.zeros(P, dtype=torch.int32, device=cuda)
    dep1, alpha = torch.full((H, W), -7.0, device=cuda), torch.full((H, W), -7.0, device=cuda)
    tr.render(c, img1, rad1, out_depth=dep1, out_alpha=alpha)
    last, fT = _debug_final_T(tr, W, H, cuda)
    torch.cuda.synchronize()
    assert torch.equal(img0, img1) and torch.equal(rad0, rad1) and torch.equal(dep0, dep1)
    assert torch.equal(alpha, 1.0 - fT)
    assert ((alpha > 0) == (last >= 0)).all() and (alpha <= 1).all()
    # A is 0 where no splat lands: 200 of the Gaussians leave most pixels empty
    sparse = trainer.GaussianTrainer(_model({k: v[:200].copy() for k, v in sc.items()}, cuda))
    a_sparse = torch.full((H, W), -7.0, device=cuda)
    sparse.render(c, out_alpha=a_sparse)
    last_s, fT_s = _debug_final_T(sparse, W, H, cuda)
    torch.cuda.synchronize()
    empty = last_s < 0
    assert empty.any() and (~empty).any(), "want pixels with and without splats"
    assert torch.equal(a_sparse, 1.0 - fT_s)
    assert (a_sparse[empty] == 0).all() and (a_sparse[~empty] > 0).all()
    # opacity alone (no depth plane): the same A
    alpha2 = torch.empty((H, W), device=cuda)
    tr.render(c, torch.empty((3, H, W), device=cuda), out_alpha=alpha2)
    torch.cuda.synchronize()
    assert torch.equal(alpha, alpha2)


def _pixel_step(tr, c, gt, mask, gd, img, rad, grads=None):
    """One built-in-loss iteration through the pixel-gradient path: render, psb_loss and the depth term in torch, backwardPixels."""
    from photo_slam_b200 import trainer
    H, W = c["H"], c["W"]
    D = torch.empty((H, W), device=img.device) if gd is not None else None
    tr.render(c, img, rad, check=False, out_depth=D)
    _, _, _, gc = trainer.fused_loss(img, gt, mask, LAMBDA_DSSIM)
    tr.backwardPixels(gc, _builtin_dL_ddepth(D, gd, mask) if gd is not None else None, grads=grads)


def test_builtin_step_reproduced_bit_for_bit(cuda):
    from photo_slam_b200 import trainer
    sc, c, gt, mask, gd = _inputs(cuda)
    P, H, W = sc["xyz"].shape[0], c["H"], c["W"]
    runs = []
    for path in ("builtin", "pixels"):
        m = _model(sc, cuda)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        tr.opt.lambda_dssim = LAMBDA_DSSIM
        tr.render(c)      # grows the binning arena: no step overflows
        radii, images = [], []
        for it in range(8):
            if it == 4:
                m.oneUpShDegree()
            msk = mask if it % 2 == 0 else None
            depth = gd if it % 3 == 1 else None
            img, rad = torch.empty((3, H, W), device=cuda), torch.empty(P, dtype=torch.int32, device=cuda)
            if path == "builtin":
                kw = dict(gt_depth=depth, lambda_depth=LAMBDA_DEPTH) if depth is not None else {}
                tr.trainForOneIteration(c, gt, msk, out_color=img, radii=rad, **kw)
            else:
                _pixel_step(tr, c, gt, msk, depth, img, rad)
            tr.result()
            radii.append(rad)
            images.append(img)
        torch.cuda.synchronize()
        assert m.step_ == 8 and tr.iteration == 8
        runs.append((radii, images, _state(m), m.adam_live_.clone()))
    (ra, ia, sa, la), (rb, ib, sb, lb) = runs
    assert all(torch.equal(x, y) for x, y in zip(ra, rb)), "radii differ"
    assert all(torch.equal(x, y) for x, y in zip(ia, ib)), "images differ"
    _assert_same_state(sa, sb)
    assert torch.equal(la, lb)


def _builtin_grads(tr, m, c, gt, mask, gd, segs):
    from photo_slam_b200 import _lib, trainer
    cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)
    ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in segs])
    args = (tr.h, m.num_points(), 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), mask.data_ptr() if mask is not None else None,
            C.byref(cs), None, None, ptrs)
    stream = torch.cuda.current_stream().cuda_stream
    if gd is None:
        _lib.check(tr.L.psb_trainer_backward(*args, stream), "psb_trainer_backward")
    else:
        d = trainer._Depth(gd.data_ptr(), LAMBDA_DEPTH, None)
        _lib.check(tr.L.psb_trainer_backward_depth(*args, C.byref(d), stream), "psb_trainer_backward_depth")
    tr.result()


@pytest.mark.parametrize("case", ["mask", "depth"])
def test_gradient_mode_equals_psb_trainer_backward(cuda, case):
    from photo_slam_b200 import trainer
    from photo_slam_b200.parallel import GradBuffer
    sc, c, gt, mask, gd = _inputs(cuda, seed=7)
    P, H, W = sc["xyz"].shape[0], c["H"], c["W"]
    msk, depth = (mask, None) if case == "mask" else (None, gd)
    outs = []
    for path in ("builtin", "pixels"):
        m = _model(sc, cuda, sh=2)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        tr.opt.lambda_dssim = LAMBDA_DSSIM
        tr.render(c)
        buf = GradBuffer(P, cuda)
        if path == "builtin":
            _builtin_grads(tr, m, c, gt, msk, depth, buf.segments)
        else:
            _pixel_step(tr, c, gt, msk, depth, torch.empty((3, H, W), device=cuda), None, grads=buf.views())
            tr.result()
        torch.cuda.synchronize()
        assert m.step_ == 0, "the gradient mode is not an optimizer step"
        outs.append((buf.flat.clone(), _state(m)))
    (ga, sa), (gb, sb) = outs
    assert ga.abs().sum() > 0
    assert torch.equal(ga, gb)
    _assert_same_state(sa, sb)   # parameters and moments untouched by both, statistics equal


def _operator_grads(sc, c, cuda, bg, wc, wd, wa, sh):
    """autograd of sum wc*image + sum wd*depth + sum wa*A through the operator path; A = channel 0 of a second render with
    colors_precomp = (1, 0, 0) and a black background"""
    from photo_slam_b200 import renderer, trainer
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.setShDegree(sh)
    for t in m.tensors():
        t.requires_grad_(True)
    H, W = c["H"], c["W"]
    img, _, vis, radii, depth = renderer.render(c, H, W, m, bg_color=bg, return_depth=True)
    loss = (wc * img).sum()
    if wd is not None:
        loss = loss + (wd * depth).sum()
    P = m.num_points()
    red = torch.zeros((P, 3), device=cuda)
    red[:, 0] = 1.0
    A = renderer.render(c, H, W, m, bg_color=torch.zeros(3, device=cuda), override_color=red, use_override_color=True)[0][0]
    loss = loss + (wa * A).sum()
    loss.backward()
    return [t.grad.detach().clone() for t in m.tensors()], img.detach(), A.detach(), radii


@pytest.mark.parametrize("terms,background", [("alpha", "black"), ("alpha", "colour"), ("all", "black"), ("all", "colour")])
def test_gradients_match_the_operator_path(cuda, terms, background):
    """black: the tile backward's fast path for a black background must still carry the opacity gradient"""
    from photo_slam_b200 import trainer
    sc, c, gt, mask, gd = _inputs(cuda, P=30_000, seed=11, wh=(320, 240))
    sc = {k: v.copy() for k, v in sc.items()}
    # some Gaussians behind the camera: culled by both paths
    V = c["viewmatrix"].reshape(-1).cpu().numpy()
    zrow = V[[2, 6, 10]].astype(np.float64)
    z = sc["xyz"].astype(np.float64) @ zrow + V[14]
    sc["xyz"][:500] = (sc["xyz"][:500] - 2.0 * np.outer(z[:500], zrow) / (zrow @ zrow)).astype(np.float32)
    P, H, W = sc["xyz"].shape[0], c["H"], c["W"]
    bg = torch.tensor([0.3, 0.5, 0.7] if background == "colour" else [0.0, 0.0, 0.0], device=cuda)
    gen = torch.Generator().manual_seed(12)
    wc = (torch.rand((3, H, W), generator=gen) - 0.5).to(cuda) if terms == "all" else torch.zeros((3, H, W), device=cuda)
    wd = (0.1 * (torch.rand((H, W), generator=gen) - 0.5)).to(cuda) if terms == "all" else None
    wa = (torch.rand((H, W), generator=gen) - 0.5).to(cuda)
    ref, ref_img, ref_A, ref_radii = _operator_grads(sc, c, cuda, bg, wc, wd, wa, sh=2)
    m = _model(sc, cuda, sh=2)
    tr = trainer.GaussianTrainer(m, background=bg)
    img, A, rad = torch.empty((3, H, W), device=cuda), torch.empty((H, W), device=cuda), torch.empty(P, dtype=torch.int32, device=cuda)
    tr.render(c, img, rad, out_depth=torch.empty((H, W), device=cuda), out_alpha=A)
    grads = [torch.zeros_like(t) for t in m.tensors()]
    tr.backwardPixels(wc, wd, wa, grads=grads)
    tr.result()
    torch.cuda.synchronize()
    assert (rad == 0).sum() >= 500 and ((rad > 0) != (ref_radii > 0)).double().mean().item() < 1e-3
    assert (img - ref_img).abs().max().item() < 1e-4
    assert (A - ref_A).abs().max().item() < 1e-4
    for name, a, b in zip(trainer.GROUPS, grads, ref):
        rn = ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()
        print(f"{terms}, {background} background: grad {name}: rel-norm error vs the operator path {rn:.2e}")
        if b.abs().max() == 0:    # the colour groups of an opacity-only loss
            assert terms == "alpha" and name in ("features_dc", "features_rest") and not a.any(), name
            continue
        assert rn < 2e-4, f"grad {name}: {rn}"
    assert not grads[0][rad == 0].any()


def _custom_loss(gt, mask, gd):
    def loss_fn(image, depth, alpha):
        l1 = ((image - gt).abs() * mask).mean()
        valid = (gd > 0) & (alpha.detach() > 0.05)
        dn = depth / alpha.clamp_min(1e-3)
        return l1 + LAMBDA_DEPTH * ((dn - gd).abs() * valid).sum() / valid.sum().clamp_min(1)
    return loss_fn


def _loss_run(cuda, inputs, steps=6, pregrow=True):
    from photo_slam_b200 import trainer
    sc, c, gt, mask, gd = inputs
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m, deterministic=True)
    if pregrow:
        tr.render(c)
    losses, radii = [], []
    for it in range(steps):
        if it == 3:
            m.oneUpShDegree()
        rad = torch.empty(m.num_points(), dtype=torch.int32, device=cuda)
        tr.trainWithLoss(c, _custom_loss(gt, mask, gd), depth=True, alpha=True, radii=rad)
        losses.append(tr.result())
        radii.append(rad)
    torch.cuda.synchronize()
    return m, tr, losses, radii


def test_train_with_loss_is_bit_identical_run_to_run(cuda):
    inputs = _inputs(cuda)
    ma, ta, la, ra = _loss_run(cuda, inputs)
    mb, tb, lb, rb = _loss_run(cuda, inputs)
    assert ma.step_ == 6 and ta.iteration == 6
    assert repr(la) == repr(lb) and all(x[0] > 0 for x in la)
    assert all(torch.equal(x, y) for x, y in zip(ra, rb))
    _assert_same_state(_state(ma), _state(mb))
    before = _model(inputs[0], cuda)
    assert not torch.equal(before.xyz_, ma.xyz_), "the steps must move the parameters"


def test_overflowing_forward_is_repeated_by_result(cuda):
    """A: the first trainWithLoss overflows the initial arena, result() repeats it; B: the arena is grown by a render first."""
    from photo_slam_b200 import trainer
    wh = (640, 480)
    cam, sc, act, g, c = scene_tensors(2_000, "tum", seed=2, pose_seed=None, dev=cuda, wh=wh, scale_px=150.0)  # ~100s of tiles per Gaussian
    gen = torch.Generator().manual_seed(4)
    gt = torch.rand((3, wh[1], wh[0]), generator=gen).to(cuda)
    gd = (torch.rand((wh[1], wh[0]), generator=gen) * 4.0).to(cuda)
    mask = torch.ones((3, wh[1], wh[0]), device=cuda)
    runs = []
    for pregrow in (False, True):
        m = _model(sc, cuda)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        if pregrow:
            tr.render(c)
        tr.trainWithLoss(c, _custom_loss(gt, mask, gd), depth=True, alpha=True)
        res = tr.result()
        ov = tr._overflow_info()
        torch.cuda.synchronize()
        assert res[3] > 6 * 2_000 + 65536, "the view must overflow the initial arena"
        assert m.step_ == 1 and tr.iteration == 1
        assert ov[1] == 1 and ov[0] == 1, ov
        runs.append((res, _state(m)))
    (ra, sa), (rb, sb) = runs
    assert repr(ra) == repr(rb)
    _assert_same_state(sa, sb)


def test_backward_pixels_after_an_unchecked_overflowing_render_raises_and_rolls_back(cuda):
    """render(check=False) overflows, backwardPixels is a no-op on the model: result() undoes its step count and raises; the caller
    renders again and repeats."""
    from photo_slam_b200 import _lib, trainer
    wh = (640, 480)
    cam, sc, act, g, c = scene_tensors(2_000, "tum", seed=2, pose_seed=None, dev=cuda, wh=wh, scale_px=150.0)
    m = _model(sc, cuda)
    before = _state(m)
    gc = torch.full((3, wh[1], wh[0]), 1e-3, device=cuda)
    for grads in ([torch.zeros_like(t) for t in m.tensors()], None):
        tr = trainer.GaussianTrainer(m)     # a fresh context: its first render overflows
        tr.render(c, check=False)
        tr.backwardPixels(gc, grads=grads)
        assert m.step_ == (1 if grads is None else 0)
        with pytest.raises(_lib.PsbError, match="overflowed"):
            tr.result()
        torch.cuda.synchronize()
        assert m.step_ == 0 and tr.iteration == 0
        _assert_same_state(before, _state(m))
        if grads is not None:
            assert not any(x.any() for x in grads), "an overflowing pass leaves the gradients zero"
    tr.render(c)                  # checked: grown and rendered again
    tr.backwardPixels(gc)
    tr.result()
    torch.cuda.synchronize()
    assert m.step_ == 1 and not torch.equal(before[0], m.xyz_)


def test_stale_pass_and_mismatches_raise_and_leave_the_model_untouched(cuda):
    from photo_slam_b200 import _lib, trainer
    sc, c, gt, mask, gd = _inputs(cuda, P=20_000)
    P, H, W = sc["xyz"].shape[0], c["H"], c["W"]
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m)
    tr.render(c)
    stale = tr._pass
    tr.render(c)
    latest = tr._pass
    torch.cuda.synchronize()
    before = _state(m)
    gc = torch.full((3, H, W), 1e-3, device=cuda)
    tr._pass = stale
    with pytest.raises(_lib.PsbError, match="latest forward pass"):
        tr.backwardPixels(gc)
    tr._pass = latest
    cm, cc, cs = m._cmodel(live=m.adamLive()), trainer._ccamera(c), tr._cstep(True)
    px = trainer._PixelGrads(gc.data_ptr(), None, None)
    stream = torch.cuda.current_stream().cuda_stream
    call = lambda p, cam, step, pg: tr.L.psb_trainer_backward_pixels(tr.h, tr._pass, p, 16, C.byref(cm), C.byref(cam), tr.background.data_ptr(),
                                                                     C.byref(pg), C.byref(step), None, stream)
    assert call(P - 1, cc, cs, px) == -1 and b"must be those of the forward pass" in tr.L.psb_last_error()
    small = trainer._ccamera(dict(c, W=W - 16))
    assert call(P, small, cs, px) == -1 and b"must be those of the forward pass" in tr.L.psb_last_error()
    other = tr._cstep(True)
    other.sh_degree = 3
    assert call(P, cc, other, px) == -1 and b"must be those of the forward pass" in tr.L.psb_last_error()
    assert call(P, cc, cs, trainer._PixelGrads(None, None, None)) == -1 and b"dL_dcolor is required" in tr.L.psb_last_error()
    torch.cuda.synchronize()
    _assert_same_state(before, _state(m))
    assert m.step_ == 0 and tr.iteration == 0
    # the matching call still goes through, and the stage timing keeps its names ("loss" = the time between the two calls)
    tr.set_profiling(True)
    tr.render(c, check=False)
    tr.backwardPixels(gc)
    tr.result()
    st = tr.stage_times()
    assert tuple(st) == trainer.GaussianTrainer.STAGES and all(v >= 0 for v in st.values())
    torch.cuda.synchronize()
    assert m.step_ == 1 and not torch.equal(before[0], m.xyz_)
    # a training call's pass had its own backward: it cannot be back-propagated again
    tr.trainForOneIteration(c, gt)
    tr.result()
    torch.cuda.synchronize()
    after = _state(m)
    current = tr._overflow_info()[2]
    cm, cs = m._cmodel(live=m.adamLive()), tr._cstep(True)
    rc = tr.L.psb_trainer_backward_pixels(tr.h, current, P, 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), C.byref(px), C.byref(cs), None,
                                          stream)
    assert rc == -1 and b"latest forward pass" in tr.L.psb_last_error()
    torch.cuda.synchronize()
    _assert_same_state(after, _state(m))
