"""-m gpu: the 3D smoothing filter (Mip-Splatting) on the fused training path.

  1. psb_filter3d against the float64 restatement (tests/filter3d64.py) at P = 200 k, K in {1, 37, 300} (chunks of 64 cameras: none of these
     is a multiple), rows within 1e-6 of a depth or margin boundary excluded and counted; bit-identical on a second run;
  2. a filter of zeros: step, gradient mode, caller's loss, depth, AA, deterministic mode bit-identical to the filter being off, and within
     float32 tolerances with the regularisers on;
  3. a non-zero filter: psb_trainer_backward and backwardPixels against autograd through renderer.render(filter_3d=True), AA on and off,
     with and without depth;
  4. the fused Adam step with the filter equals the gradient mode + psb_adam_update;
  5. refusals: stale or missing filter, P mismatch, a switched filter behind backward_pixels, the data-parallel entry points;
  6. the fused PLY export draws what the trainer draws with the filter;
  7. a short trained run with the filter recomputed after densification stays close to the unfiltered run at the training resolution.
"""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import filter3d64 as f64  # noqa: E402
from helpers import scene_tensors  # noqa: E402

pytestmark = pytest.mark.gpu
LRS = [0.00032, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
# PSNR (dB) the filtered run may lose against the unfiltered one at the training resolution (section 7; DESIGN.md §5 gives the measurement)
QUALITY_MARGIN_DB = 0.3


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "the -m gpu tests need a CUDA device"
    return torch.device("cuda:0")


def _rn(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def _cams(dev, K, seed, W=640, H=480, f=500.0):
    """K camera dicts around the synthetic scene's camera (small random poses, focal lengths that differ per camera)"""
    import photo_slam_b200.synthetic as syn
    rng = np.random.default_rng(seed)
    out = []
    for k in range(K):
        R, t = syn.random_pose(rng, max_angle=0.3, max_trans=0.5)
        fk = f * (0.7 + 0.6 * rng.random())
        cam = syn.make_camera(W, H, fk, fk * (0.9 + 0.2 * rng.random()), R, t)
        out.append(syn.device_camera(cam, dev))
    return out


def _packed(cams):
    return np.stack([np.concatenate([c["viewmatrix"].double().cpu().numpy().reshape(-1),
                                     [c["W"] / (2 * c["tanfovx"]), c["H"] / (2 * c["tanfovy"]), c["W"], c["H"]]]) for c in cams])


@pytest.mark.parametrize("K", [1, 37, 300])
def test_filter_kernel_against_the_restatement(dev, K):
    from photo_slam_b200 import trainer
    cam, sc, act, g, c = scene_tensors(200_000, "tum", seed=4, pose_seed=5, dev=dev)
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.xyz_[-2000:, 2] *= -1.0          # mirrored behind every camera: rows no camera sees
    cams = _cams(dev, K, seed=K)
    seen = m.computeFilter3D(cams)
    first = m.filter_3D_.clone()
    assert m.computeFilter3D(cams) == seen
    torch.cuda.synchronize()
    assert torch.equal(first, m.filter_3D_), "two runs differ"
    ref = f64.filter3d(m.xyz_.double().cpu().numpy(), np.float32(_packed(cams)).astype(np.float64))
    got = first.double().cpu().numpy()
    keep = ~ref["near"]
    print(f"K={K}: {int(ref['seen'].sum())} of {len(got)} rows seen, {int((~keep).sum())} rows within 1e-6 of a boundary excluded")
    assert abs(seen - int(ref["seen"].sum())) <= int((~keep).sum())
    assert 0 < ref["seen"].sum() < len(got)
    # 1 ulp of d / F plus the float32 rounding of the view transform that forms z (sum of |terms| times a few float32 epsilons)
    want = ref["filter"]
    ulp = np.spacing(np.float32(want)).astype(np.float64)
    bound = ulp + 4 * 2.0 ** -24 * ref["zs"] / ref["F"] * f64.SQRT02
    err = np.abs(got - want)
    print(f"K={K}: max |gpu - restatement| / bound {float((err / bound)[keep].max()):.3f}, in ulps of the result {float((err / ulp)[keep].max()):.2f}")
    assert (err <= bound)[keep].all()


def _train_inputs(dev, P=60_000, wh=(600, 340), seed=3):
    cam, sc, act, g, c = scene_tensors(P, "replica", seed=seed, pose_seed=seed + 1, dev=dev, wh=wh, scale_px=3.0)
    gen = torch.Generator().manual_seed(seed + 2)
    gt = torch.rand((3, wh[1], wh[0]), generator=gen).to(dev)
    gd = (0.5 + 7.5 * torch.rand((wh[1], wh[0]), generator=gen)).to(dev)
    return sc, c, gt, gd


def _model(sc, dev, sh=2):
    from photo_slam_b200 import trainer
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    m.setShDegree(sh)
    return m


def _filter(m, c, dev, boost=4.0):
    """the model's filter from its own camera and a few around it, made `boost` times wider so that it changes most splats"""
    m.computeFilter3D([c] + _cams(dev, 5, seed=21, W=c["W"], H=c["H"], f=c["W"] / (2 * c["tanfovx"])))
    m.filter_3D_.mul_(boost)
    return m.filter_3D_


def _state(m):
    return [t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + [m.xyz_gradient_accum_, m.denom_, m.max_radii2D_]]


@pytest.mark.parametrize("reg", [0.0, 0.01], ids=["noreg", "reg"])
@pytest.mark.parametrize("aa", [False, True], ids=["plain", "aa"])
def test_zero_filter_is_bit_identical_to_no_filter(dev, aa, reg):
    """bit for bit without the regularisers; with them, the compiler may contract the regulariser's add into the opacity gradient the
    other way round in a filtered variant (one rounding of g_opacity), so that case is compared within float32 tolerances"""
    from photo_slam_b200 import _lib, trainer
    from photo_slam_b200.parallel import GradBuffer
    sc, c, gt, gd = _train_inputs(dev, P=30_000, wh=(320, 240), seed=7)
    P = sc["xyz"].shape[0]
    res = {}
    for filt in (False, True):
        m = _model(sc, dev, sh=1)
        tr = trainer.GaussianTrainer(m, deterministic=True, antialiasing=aa, filter3d=filt)
        if filt:
            m.filter_3D_ = torch.zeros(P, device=dev)
        _lib.check(tr.L.psb_trainer_set_regularizers(tr.h, reg, reg), "psb_trainer_set_regularizers")
        tr.render(c)
        outs = []
        for it in range(4):
            kw = dict(gt_depth=gd, lambda_depth=0.1) if it % 2 else {}
            img = torch.empty((3, c["H"], c["W"]), device=dev)
            tr.trainForOneIteration(c, gt, out_color=img, **kw)
            outs.append(tr.result())
            outs.append(img)
        # gradient mode (psb_trainer_backward_depth) and a caller's loss through backwardPixels
        buf = GradBuffer(P, dev)
        cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)
        tr._hand_filter3d()
        ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in buf.segments])
        d = trainer._Depth(gd.data_ptr(), 0.1, None)
        _lib.check(tr.L.psb_trainer_backward_depth(tr.h, P, 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), None, C.byref(cs),
                                                   None, None, ptrs, C.byref(d), torch.cuda.current_stream().cuda_stream), "psb_trainer_backward_depth")
        tr.result()
        outs.append(buf.flat.clone())
        tr.trainWithLoss(c, lambda i, dd: (i * gt).sum() + 0.01 * dd.sum(), depth=True)
        tr.result()
        torch.cuda.synchronize()
        res[filt] = outs + _state(m) + [m.adamLive().clone()]
    differ = 0
    for i, (x, y) in enumerate(zip(res[False], res[True])):
        if torch.is_tensor(x):
            differ += int((x != y).sum())
            if not reg:
                assert torch.equal(x, y), i
            else:   # (Adam turns the one-rounding difference into up to lr on elements whose gradient is near zero)
                assert _rn(x.float(), y.float()) < 1e-4 and ((x.float() - y.float()).abs() > 5e-4).float().mean().item() < 2e-3, i
        else:
            assert x == y if not reg else max(abs(a - b) for a, b in zip(x, y)) < 1e-5, i
    print(f"aa={aa} reg={reg}: {differ} values differ from the run without the filter")


def _operator_grads(sc, c, dev, filt, wc, wd, wa, sh, aa):
    """autograd through renderer.render(filter_3d=True) of sum wc*image + sum wd*depth + sum wa*A"""
    from photo_slam_b200 import renderer, trainer
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.setShDegree(sh)
    m.filter_3D_ = filt
    for t in m.tensors():
        t.requires_grad_(True)
    pipe = renderer.GaussianPipelineParams(antialiasing=aa, filter_3d=True)
    H, W = c["H"], c["W"]
    img, _, _, radii, depth = renderer.render(c, H, W, m, pipe=pipe, return_depth=True)
    loss = (wc * img).sum()
    if wd is not None:
        loss = loss + (wd * depth).sum()
    if wa is not None:
        red = torch.zeros((m.num_points(), 3), device=dev)
        red[:, 0] = 1.0
        A = renderer.render(c, H, W, m, pipe=pipe, override_color=red, use_override_color=True)[0][0]
        loss = loss + (wa * A).sum()
    loss.backward()
    return [t.grad.detach().clone() for t in m.tensors()], img.detach(), radii


@pytest.mark.parametrize("aa", [False, True], ids=["plain", "aa"])
def test_trainer_backward_matches_the_operator_path(dev, aa):
    from photo_slam_b200 import _lib, trainer
    from photo_slam_b200.parallel import GradBuffer
    sc, c, gt, gd = _train_inputs(dev)
    P = sc["xyz"].shape[0]
    m = _model(sc, dev)
    filt = _filter(m, c, dev)
    assert (filt > 0).all()
    tr = trainer.GaussianTrainer(m, antialiasing=aa, filter3d=True)
    radii = torch.zeros(P, dtype=torch.int32, device=dev)
    img = tr.render(c, radii=radii)
    buf = GradBuffer(P, dev)
    cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)
    ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in buf.segments])
    _lib.check(tr.L.psb_trainer_backward(tr.h, P, 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), None, C.byref(cs), None, None,
                                         ptrs, torch.cuda.current_stream().cuda_stream), "psb_trainer_backward")
    tr.result()
    _, _, _, gcol = trainer.fused_loss(img, gt, None, tr.opt.lambda_dssim)
    ref, ref_img, ref_radii = _operator_grads(sc, c, dev, filt, gcol, None, None, m.active_sh_degree_, aa)
    torch.cuda.synchronize()
    plain = trainer.GaussianTrainer(_model(sc, dev), antialiasing=aa).render(c)
    print(f"aa={aa}: filtered vs plain image max diff {(img - plain).abs().max().item():.3e}, vs operator {(img - ref_img).abs().max().item():.2e}")
    _image_close(img, ref_img, aa, f"aa={aa}: trainer render vs operator")
    assert (img - plain).abs().max().item() > 1e-2
    assert (radii != ref_radii).sum().item() <= 4
    for name, a, b in zip(trainer.GROUPS, buf.views(), ref):
        rn = _rn(a, b)
        print(f"aa={aa} psb_trainer_backward with the 3D filter, {name}: rel-norm vs operator {rn:.2e}")
        assert rn < 2e-4, (name, rn)


@pytest.mark.parametrize("aa", [False, True], ids=["plain", "aa"])
@pytest.mark.parametrize("depth", [False, True], ids=["colour", "depth"])
def test_pixel_gradients_match_the_operator_path(dev, aa, depth):
    from photo_slam_b200 import trainer
    sc, c, gt, gd = _train_inputs(dev, P=30_000, wh=(320, 240), seed=11)
    H, W = c["H"], c["W"]
    gen = torch.Generator().manual_seed(12)
    wc = (torch.rand((3, H, W), generator=gen) - 0.5).to(dev)
    wd = (0.1 * (torch.rand((H, W), generator=gen) - 0.5)).to(dev) if depth else None
    wa = (torch.rand((H, W), generator=gen) - 0.5).to(dev)
    m = _model(sc, dev)
    filt = _filter(m, c, dev)
    ref, ref_img, _ = _operator_grads(sc, c, dev, filt, wc, wd, wa, 2, aa)
    tr = trainer.GaussianTrainer(m, antialiasing=aa, filter3d=True)
    img, A = torch.empty((3, H, W), device=dev), torch.empty((H, W), device=dev)
    tr.render(c, img, out_depth=torch.empty((H, W), device=dev), out_alpha=A)
    grads = [torch.zeros_like(t) for t in m.tensors()]
    tr.backwardPixels(wc, wd, wa, grads=grads)
    tr.result()
    torch.cuda.synchronize()
    _image_close(img, ref_img, aa, f"aa={aa} depth={depth}: trainer render vs operator")
    for name, a, b in zip(trainer.GROUPS, grads, ref):
        rn = _rn(a, b)
        print(f"aa={aa} depth={depth} backwardPixels with the 3D filter, {name}: rel-norm vs operator {rn:.2e}")
        assert rn < 2e-4, (name, rn)


def test_fused_step_equals_gradients_plus_adam_update(dev):
    from photo_slam_b200 import _lib, trainer
    from photo_slam_b200.parallel import GradBuffer
    sc, c, gt, gd = _train_inputs(dev)
    P = sc["xyz"].shape[0]
    a, b = _model(sc, dev, sh=0), _model(sc, dev, sh=0)
    filt = _filter(a, c, dev)
    b.filter_3D_ = filt.clone()
    ta = trainer.GaussianTrainer(a, deterministic=True, antialiasing=True, filter3d=True)
    tb = trainer.GaussianTrainer(b, deterministic=True, antialiasing=True, filter3d=True)
    for t in (ta, tb):
        t.render(c)
    buf = GradBuffer(P, dev)
    for it in range(5):
        if it == 2:
            a.oneUpShDegree()
            b.oneUpShDegree()
        depth = gd if it % 2 == 1 else None
        kw = dict(gt_depth=depth, lambda_depth=0.1) if depth is not None else {}
        ta.trainForOneIteration(c, gt, densify_stats=False, **kw)
        ta.result()
        buf.flat.zero_()
        tb._hand_filter3d()
        cm, cc, cs = b._cmodel(), trainer._ccamera(c), tb._cstep(False)
        ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in buf.segments])
        d = trainer._Depth(depth.data_ptr(), 0.1, None) if depth is not None else None
        _lib.check(tb.L.psb_trainer_backward_depth(tb.h, P, 16, C.byref(cm), C.byref(cc), tb.background.data_ptr(), gt.data_ptr(), None, C.byref(cs),
                                                   None, None, ptrs, C.byref(d) if d is not None else None, torch.cuda.current_stream().cuda_stream),
                   "psb_trainer_backward_depth")
        tb.result()
        cm2 = b._cmodel()
        _lib.check(tb.L.psb_adam_update(P, 16, C.byref(cm2), ptrs, C.byref(cs), 1.0, None), "psb_adam_update")
        b.step_ += 1
    torch.cuda.synchronize()
    for name, x, y, lr in zip(trainer.GROUPS, a.tensors(), b.tensors(), LRS):
        frac = ((x - y).abs() > 0.5 * lr).float().mean().item()
        rn = _rn(x, y)
        print(f"fused step with the 3D filter vs gradients + Adam: {name} rel-norm {rn:.2e}, entries apart by > lr/2: {frac:.2e}")
        assert frac < 2e-3 and rn < 1e-4, (name, frac, rn)


def test_refusals(dev):
    from photo_slam_b200 import _lib, trainer
    from photo_slam_b200.parallel import GradBuffer
    sc, c, gt, gd = _train_inputs(dev, P=20_000, wh=(320, 240), seed=13)
    P = sc["xyz"].shape[0]
    m = _model(sc, dev)
    tr = trainer.GaussianTrainer(m, filter3d=True)
    with pytest.raises(ValueError, match="computeFilter3D"):
        tr.render(c)
    _filter(m, c, dev, boost=1.0)
    tr.render(c)
    tr.trainForOneIteration(c, gt)
    tr.result()
    # every invalidating method leaves a stale filter behind
    m.densifyAndPrune(0.0002, 0.005, 1.0, 0)
    with pytest.raises(ValueError, match="computeFilter3D"):
        tr.trainForOneIteration(c, gt)
    _filter(m, c, dev, boost=1.0)
    m.relocateGaussians()
    with pytest.raises(ValueError, match="computeFilter3D"):
        tr.render(c)
    _filter(m, c, dev, boost=1.0)
    m.prunePoints(torch.zeros(m.num_points(), dtype=torch.bool, device=dev))
    with pytest.raises(ValueError, match="computeFilter3D"):
        tr.render(c)
    P = m.num_points()
    filt = _filter(m, c, dev, boost=1.0)
    # the C-ABI: a pass over another row count
    cm, cc, cs = m._cmodel(live=m.adamLive()), trainer._ccamera(c), tr._cstep(True)
    _lib.check(tr.L.psb_trainer_set_filter3d(tr.h, filt.data_ptr(), P + 1), "psb_trainer_set_filter3d")
    s = torch.cuda.current_stream().cuda_stream
    rc = tr.L.psb_trainer_step(tr.h, P, 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), None, C.byref(cs), None, None, s)
    assert rc == -1 and b"row count" in tr.L.psb_last_error()
    out = torch.empty((3, c["H"], c["W"]), device=dev)
    assert tr.L.psb_trainer_render(tr.h, P, 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), 2, out.data_ptr(), None, s) == -1
    assert tr.L.psb_trainer_set_filter3d(tr.h, filt.data_ptr(), -1) == -1
    # the data-parallel entry points refuse while a filter is set
    _lib.check(tr.L.psb_trainer_set_filter3d(tr.h, filt.data_ptr(), P), "psb_trainer_set_filter3d")
    buf = GradBuffer(P, dev)
    ptrs = (C.c_void_p * 6)(*[x.data_ptr() for x in buf.segments])
    cm0 = m._cmodel()
    assert tr.L.psb_trainer_backward_begin(tr.h, P, 16, C.byref(cm0), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), None, C.byref(cs),
                                           None, None, s) == -1
    assert tr.L.psb_trainer_backward_slab(tr.h, P, 16, C.byref(cm0), C.byref(cc), C.byref(cs), 0, 128, ptrs, s) == -1
    assert tr.L.psb_dp_step(tr.h, None, P, 16, C.byref(cm0), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), None, C.byref(cs), None, None,
                            s) == -1
    assert b"data-parallel" in tr.L.psb_last_error()
    with pytest.raises(NotImplementedError, match="3D filter"):
        trainer.DataParallelTrainer(m, filter3d=True)
    # backward_pixels after the filter was replaced by another array
    tr.render(c, out)
    m.filter_3D_ = filt.clone()
    with pytest.raises(_lib.PsbError, match="3D filter changed"):
        tr.backwardPixels(torch.zeros_like(out), grads=[torch.zeros_like(t) for t in m.tensors()])
    # ... or switched off
    plain = trainer.GaussianTrainer(m)
    plain.render(c, out)
    _lib.check(plain.L.psb_trainer_set_filter3d(plain.h, filt.data_ptr(), P), "psb_trainer_set_filter3d")
    with pytest.raises(_lib.PsbError, match="3D filter changed"):
        plain.backwardPixels(torch.zeros_like(out), grads=[torch.zeros_like(t) for t in m.tensors()])
    # psb_filter3d's argument checks
    assert tr.L.psb_filter3d(-1, None, 0, None, None, None, s) == -1
    assert tr.L.psb_filter3d(P, m.xyz_.data_ptr(), -1, None, filt.data_ptr(), None, s) == -1
    assert tr.L.psb_filter3d(P, m.xyz_.data_ptr(), 2, None, filt.data_ptr(), None, s) == -1
    assert tr.L.psb_filter3d(P, None, 0, None, filt.data_ptr(), None, s) == -1
    # no camera: zeros, nothing seen
    assert m.computeFilter3D([]) == 0 and (m.filter_3D_ == 0).all()


def test_fused_ply_renders_what_the_trainer_draws(dev, tmp_path):
    from photo_slam_b200 import trainer
    sc, c, gt, gd = _train_inputs(dev, P=30_000, wh=(320, 240), seed=15)
    m = _model(sc, dev, sh=3)
    _filter(m, c, dev)
    for aa in (False, True):
        img = trainer.GaussianTrainer(m, antialiasing=aa, filter3d=True).render(c)
        path = str(tmp_path / "fused.ply")
        m.savePly(path, fuse_filter3d=True)
        n = trainer.GaussianModel(3, dev)
        n.loadPly(path)
        again = trainer.GaussianTrainer(n, antialiasing=aa).render(c)
        torch.cuda.synchronize()
        _image_close(again, img, aa, f"aa={aa}: fused PLY render vs filtered render")


def _image_close(a, b, aa, what):
    """within 1e-4 everywhere; with anti-aliasing, a few values may lie further apart (see DESIGN.md §5, 3D smoothing filter)"""
    d = (a - b).abs()
    share = (d > 1e-4).double().mean().item()
    print(f"{what}: max diff {d.max().item():.2e}, share of values beyond 1e-4 {share:.2e}")
    if aa:
        assert share < 1e-4 and d.max().item() < 2e-3
    else:
        assert d.max().item() < 1e-4


def _psnr(a, b):
    return 10 * np.log10(1.0 / max(((a - b) ** 2).mean().item(), 1e-12))


def test_trained_run_with_the_filter(dev):
    """8 views of a target scene at 320x240; 400 steps from a perturbed copy with densification at 150 and 300, with and without the filter
    (recomputed from the 8 cameras after each densification and every 100 steps); mean PSNR over the views at the training resolution"""
    import photo_slam_b200.synthetic as syn
    from photo_slam_b200 import trainer
    W, H, f = 320, 240, 260.0
    rng = np.random.default_rng(3)
    poses = [syn.random_pose(rng, max_angle=0.1, max_trans=0.1) for _ in range(8)]
    cams = []
    for p in poses:
        cm = syn.make_camera(W, H, f, f, *p)
        cams.append((cm, syn.device_camera(cm, dev)))
    target = trainer.GaussianModel.from_numpy(syn.make_scene(20_000, cams[0][0], seed=31, scale_px=2.0), dev)
    gts = [trainer.GaussianTrainer(target).render(c) for _, c in cams]
    res = {}
    for filt in (False, True):
        m = trainer.GaussianModel.from_numpy(syn.make_scene(20_000, cams[0][0], seed=32, scale_px=2.0), dev)
        opt = trainer.GaussianOptimizationParams()
        m.trainingSetup(opt)
        tr = trainer.GaussianTrainer(m, opt, antialiasing=True, filter3d=filt)
        if filt:
            m.computeFilter3D([c for _, c in cams])
        for it in range(1, 401):
            k = it % len(cams)
            tr.trainForOneIteration(cams[k][1], gts[k])
            tr.result()
            if it in (150, 300):
                m.densifyAndPrune(opt.densify_grad_threshold, 0.005, 2.0, 0)
            if filt and (it in (150, 300) or it % 100 == 0):
                m.computeFilter3D([c for _, c in cams])
        res[filt] = float(np.mean([_psnr(tr.render(c), gt) for (_, c), gt in zip(cams, gts)]))
    print(f"trained 400 steps at 320x240: PSNR without the filter {res[False]:.3f} dB, with it {res[True]:.3f} dB")
    assert res[True] >= res[False] - QUALITY_MARGIN_DB
