"""-m gpu: rendered depth and the RGB-D depth term of the fused step (psb_trainer_*_depth).

The reference renders no depth, but depth blends exactly like a colour channel whose per-Gaussian value is the view-space
depth z. Its chain is therefore the reference's own rasterizer called a second time with colors_precomp = (z, 0, 0), z computed
in torch from xyz and the view matrix, and a black background; autograd of that chain is what the fused kernels must give.
The reference outputs are stored in tests/golden/test_depth_gpu.npz, written by `python tests/golden/make_ref_golden.py test_depth_gpu`
(which runs reference_cases() below)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn
from helpers import SAMPLE, Gold, scene_tensors

pytestmark = pytest.mark.gpu

LRS = [0.00032, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
MODULE = "test_depth_gpu"
LAMBDA_DEPTH = 0.1
CASES = ("holes", "holes_mask")


def _inputs(cuda, case):
    """The inputs of test_trainer_gpu.py's backward test (30 k Gaussians, 320x240) plus a target depth with ~10 % holes and some
    negative (invalid) values, and for "holes_mask" an undistortion mask."""
    P, wh = 30_000, (320, 240)
    cam, sc, act, g, c = scene_tensors(P, "tum", seed=3, pose_seed=4, dev=cuda, wh=wh, scale_px=5.0)
    gt = torch.rand((3, wh[1], wh[0]), generator=torch.Generator().manual_seed(7)).to(cuda)
    V = cam["viewmatrix"].reshape(-1)
    z = sc["xyz"] @ V[[2, 6, 10]] + V[14]
    zs = np.quantile(z[z > 0.2], [0.1, 0.9])
    gen = torch.Generator().manual_seed(11)
    depth = zs[0] + (zs[1] - zs[0]) * torch.rand((wh[1], wh[0]), generator=gen)
    r = torch.rand((wh[1], wh[0]), generator=gen)
    depth[r < 0.1] = 0.0
    depth[(r >= 0.1) & (r < 0.12)] = -1.0
    mask = None
    if case == "holes_mask":
        m = (torch.rand((wh[1], wh[0]), generator=gen) > 0.15).float()
        mask = m.expand(3, -1, -1).contiguous().to(cuda)
    return P, sc, c, gt, depth.float().contiguous().to(cuda), mask


def _torch_depth_l1(D, G, mask):
    valid = G > 0
    if mask is not None:
        valid &= mask[0] != 0
    n = int(valid.sum().item())
    return ((D - G).abs() * valid).sum().item() / max(n, 1)


class _RefRasterizeColors(torch.autograd.Function):
    """The reference's rasterizer with colors_precomp as a differentiable input (its dL_dcolors)."""

    @staticmethod
    def forward(ctx, means3D, means2D, colors, opacities, scales, rotations, rs):
        import ref_gpu
        e = torch.empty(0, device=means3D.device)
        R, img, radii, gb, bb, ib = ref_gpu.rasterize_forward(rs["bg"], means3D, colors, opacities, scales, rotations, 1.0, e, rs["viewmatrix"],
                                                              rs["projmatrix"], rs["tanfovx"], rs["tanfovy"], rs["H"], rs["W"], e, 0, rs["campos"])
        ctx.rs, ctx.R = rs, R
        ctx.save_for_backward(colors, means3D, scales, rotations, radii, gb, bb, ib)
        return img

    @staticmethod
    def backward(ctx, grad_out):
        import ref_gpu
        rs = ctx.rs
        colors, means3D, scales, rotations, radii, gb, bb, ib = ctx.saved_tensors
        e = torch.empty(0, device=means3D.device)
        g = ref_gpu.rasterize_backward(rs["bg"], means3D, radii, colors, scales, rotations, 1.0, e, rs["viewmatrix"], rs["projmatrix"],
                                       rs["tanfovx"], rs["tanfovy"], grad_out.contiguous(), e, 0, rs["campos"], gb, ctx.R, bb, ib)
        dm2, dcol, dop, dm3, dcov, dsh, dsc, drot, _ = g
        return dm3, dm2, dcol, dop, dsc, drot, None


def _reference_depth(cuda, case):
    import ref_trainer
    import torch.nn.functional as F
    from photo_slam_b200 import trainer
    P, sc, c, gt, gd, mask = _inputs(cuda, case)
    ref = ref_trainer.RefTrainer(sc, cuda, LRS)
    image, viewspace, vis, radii = ref.render(c)
    V = c["viewmatrix"].reshape(-1)   # column-major: the view-space z row is V[2], V[6], V[10], V[14]
    z = ref.xyz @ V[[2, 6, 10]] + V[14]
    cols = torch.stack([z, torch.zeros_like(z), torch.zeros_like(z)], dim=1).contiguous()
    rs = dict(bg=torch.zeros(3, device=cuda), viewmatrix=c["viewmatrix"], projmatrix=c["projmatrix"], campos=c["campos"], tanfovx=c["tanfovx"],
              tanfovy=c["tanfovy"], H=c["H"], W=c["W"])
    dimg = _RefRasterizeColors.apply(ref.xyz, viewspace, cols, torch.sigmoid(ref.opacity), torch.exp(ref.scaling), F.normalize(ref.rotation), rs)
    D = dimg[0]
    masked = image * mask if mask is not None else image
    valid = gd > 0
    if mask is not None:
        valid &= mask[0] != 0
    dl1 = ((D - gd).abs() * valid).sum() / max(int(valid.sum().item()), 1)
    loss = 0.8 * (masked - gt).abs().mean() + 0.2 * (1 - ref_trainer.ssim(masked, gt)) + LAMBDA_DEPTH * dl1
    loss.backward()
    d = dict(loss=loss.item(), depth_l1=dl1.item(), radii=radii, image=image.detach(), depth=D.detach(),
             acc=torch.norm(viewspace.grad[:, :2], dim=-1) * vis)
    for name, t in zip(trainer.GROUPS, ref.tensors()):
        d["grad_" + name] = t.grad
    return d


def _model(sc, cuda):
    from photo_slam_b200 import trainer
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    return m


def _debug_state(tr, W, H, dev):
    last = torch.empty(W * H, dtype=torch.int32, device=dev)
    fT = torch.empty(W * H, dtype=torch.float32, device=dev)
    from photo_slam_b200 import _lib
    _lib.check(tr.L.psb_trainer_debug_state(tr.h, W, H, last.data_ptr(), fT.data_ptr(), None, torch.cuda.current_stream().cuda_stream), "debug_state")
    return last, fT


def test_forward_depth_matches_reference_and_leaves_colour_bit_identical(cuda):
    from photo_slam_b200 import trainer
    r = Gold(MODULE, "holes")
    P, sc, c, gt, gd, mask = _inputs(cuda, "holes")
    tr = trainer.GaussianTrainer(_model(sc, cuda))
    H, W = c["H"], c["W"]
    img0, rad0 = torch.empty((3, H, W), device=cuda), torch.zeros(P, dtype=torch.int32, device=cuda)
    tr.render(c, img0, rad0)
    last0, T0 = _debug_state(tr, W, H, cuda)
    img1, rad1, dep = torch.empty((3, H, W), device=cuda), torch.zeros(P, dtype=torch.int32, device=cuda), torch.full((H, W), -7.0, device=cuda)
    tr.render(c, img1, rad1, out_depth=dep)
    last1, T1 = _debug_state(tr, W, H, cuda)
    torch.cuda.synchronize()
    assert torch.equal(img0, img1) and torch.equal(rad0, rad1) and torch.equal(last0, last1) and torch.equal(T0, T1)
    assert (dep >= 0).all()
    bad = r.frac("depth", dep, rtol=1e-4, atol=1e-4)
    print(f"depth: fraction of sampled pixels off by more than 1e-4: {bad:.2e}")
    assert bad <= 2 / SAMPLE
    # a training step writes the same plane to the caller's out_depth
    out_d = torch.empty((H, W), device=cuda)
    tr.trainForOneIteration(c, gt, gt_depth=gd, lambda_depth=LAMBDA_DEPTH, out_depth=out_d)
    tr.result()
    torch.cuda.synchronize()
    assert torch.equal(out_d, dep)


@pytest.mark.parametrize("case", CASES)
def test_backward_depth_gradients_match_reference_chain(cuda, case):
    """psb_trainer_backward_depth: raw-parameter gradients and densification statistics == autograd of the reference chain."""
    from photo_slam_b200 import trainer
    r = Gold(MODULE, case)
    P, sc, c, gt, gd, mask = _inputs(cuda, case)
    few = max(P // 5000 / P, 2 / SAMPLE)
    model = _model(sc, cuda)
    dp = trainer.DataParallelTrainer(model)  # world == 1: backward -> (no all-reduce) -> Adam
    my_radii = torch.zeros(P, dtype=torch.int32, device=cuda)
    my_depth = torch.zeros((c["H"], c["W"]), device=cuda)
    dp.trainForOneIteration(c, gt, mask, radii=my_radii, gt_depth=gd, lambda_depth=LAMBDA_DEPTH, out_depth=my_depth)
    l, l1, ss, dl1, n = dp.result_depth()
    print(f"{case}: loss {l:.6f} (reference {r['loss']:.6f}), depth_l1 {dl1:.6f} (reference {r['depth_l1']:.6f})")
    assert abs(l - r["loss"]) < 1e-5 * max(1.0, abs(r["loss"]))
    assert abs(dl1 - r["depth_l1"]) < 1e-5 * max(1.0, abs(r["depth_l1"]))
    a, radii = r.pair("radii", my_radii)
    assert (a != radii).double().mean().item() <= few
    assert r.frac("depth", my_depth, rtol=1e-4, atol=1e-4) <= 2 / SAMPLE
    for name, seg in zip(trainer.GROUPS, dp.segs):
        rn = r.relnorm("grad_" + name, seg)
        print(f"{case}: grad {name}: rel-norm error {rn:.2e}")
        assert rn < 2e-4, f"grad {name}: {rn}"
    assert (r.pair("radii", model.max_radii2D_)[0] != radii).double().mean().item() <= few
    assert (r.pair("radii", model.denom_)[0] != (radii > 0).double()).double().mean().item() <= few
    assert r.relnorm("acc", model.xyz_gradient_accum_) < 2e-4


def test_depth_loss_value_and_all_invalid_target(cuda):
    from photo_slam_b200 import trainer
    P, sc, c, gt, gd, mask = _inputs(cuda, "holes_mask")
    H, W = c["H"], c["W"]
    tr = trainer.GaussianTrainer(_model(sc, cuda))
    D = torch.empty((H, W), device=cuda)
    tr.trainForOneIteration(c, gt, mask, gt_depth=gd, lambda_depth=LAMBDA_DEPTH, out_depth=D)
    l, l1, ss, dl1, n = tr.result_depth()
    want = _torch_depth_l1(D, gd, mask)
    assert abs(dl1 - want) <= 1e-6 * max(1.0, want), (dl1, want)
    assert abs(l - (0.8 * l1 + 0.2 * (1 - ss) + LAMBDA_DEPTH * dl1)) < 1e-6 * max(1.0, l)
    assert tr.result()[0] == l
    # an all-invalid target: no depth term, the gradients of the plain path
    grads = []
    for depth_args in (dict(), dict(gt_depth=torch.zeros((H, W), device=cuda), lambda_depth=LAMBDA_DEPTH)):
        dp = trainer.DataParallelTrainer(_model(sc, cuda))
        dp.trainForOneIteration(c, gt, mask, **depth_args)
        res = dp.result_depth()
        if depth_args:
            assert res[3] == 0.0
        grads.append(([s.clone() for s in dp.segs], res[0]))
    assert abs(grads[0][1] - grads[1][1]) < 1e-6 * max(1.0, grads[0][1])
    for name, a, b in zip(trainer.GROUPS, grads[0][0], grads[1][0]):
        rn = ((a.double() - b.double()).norm() / (a.double().norm() + 1e-30)).item()
        assert rn < 1e-5, (name, rn)


def _step_c(tr, m, c, gt, gd, live):
    """one psb_trainer_step_depth through the C-ABI, with or without the adam_live bytes"""
    from photo_slam_b200 import _lib, trainer
    cm, cc, cs = m._cmodel(live=m.adamLive() if live else None), trainer._ccamera(c), tr._cstep(True)
    d = trainer._Depth(gd.data_ptr(), LAMBDA_DEPTH, None)
    _lib.check(tr.L.psb_trainer_step_depth(tr.h, m.num_points(), 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), None,
                                           C.byref(cs), None, None, C.byref(d), torch.cuda.current_stream().cuda_stream), "psb_trainer_step_depth")
    m.step_ += 1
    tr.result()


@pytest.mark.parametrize("live", [True, False])
def test_fused_depth_step_equals_split_path(cuda, live):
    """psb_trainer_step_depth == psb_trainer_backward_depth -> psb_adam_update, with and without adam_live; after depth steps every row
    whose parameters moved has its live byte set."""
    from photo_slam_b200 import trainer
    P, sc, c, gt, gd, mask = _inputs(cuda, "holes")
    fm, sm = _model(sc, cuda), _model(sc, cuda)
    fused, split = trainer.GaussianTrainer(fm), trainer.DataParallelTrainer(sm, pipeline=False)
    before = [t.clone() for t in fm.tensors()]
    for it in range(3):
        _step_c(fused, fm, c, gt, gd, live)
        split.trainForOneIteration(c, gt, gt_depth=gd, lambda_depth=LAMBDA_DEPTH)
        split.result()
    torch.cuda.synchronize()
    for a, b, lrate, name in zip(fm.tensors(), sm.tensors(), LRS, trainer.GROUPS):
        frac = ((a - b).abs() > 0.5 * lrate).float().mean().item()
        assert frac < 2e-3, f"{name}: {frac} of entries differ by more than half a step"
    if live:
        moved = torch.zeros(P, dtype=torch.bool, device=cuda)
        for a, b in zip(fm.tensors(), before):
            moved |= (a != b).reshape(P, -1).any(dim=1)
        assert moved.any()
        assert not (moved & (fm.adam_live_ == 0)).any(), "a row moved by a depth step has adam_live == 0"


def test_depth_only_rows_are_updated(cuda):
    """A row whose only gradient is dL/dz (every colour target equals the render) still moves and gets its live byte."""
    from photo_slam_b200 import trainer
    P, sc, c, gt, gd, mask = _inputs(cuda, "holes")
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m)
    img = tr.render(c)
    torch.cuda.synchronize()
    before = m.xyz_.clone()
    # lambda_dssim = 0 and gt == render: the photometric gradient is exactly zero, only the depth term drives the step
    tr.opt.lambda_dssim = 0.0
    tr.trainForOneIteration(c, img.clone(), gt_depth=gd, lambda_depth=LAMBDA_DEPTH)
    l, l1, ss, dl1, n = tr.result_depth()
    torch.cuda.synchronize()
    assert l1 == 0.0 and dl1 > 0.0
    moved = (m.xyz_ != before).any(dim=1)
    assert moved.sum().item() > 100
    assert not (moved & (m.adam_live_ == 0)).any()


def test_depth_step_overflow_is_retried_with_its_target(cuda):
    from photo_slam_b200 import trainer
    P, wh = 2_000, (640, 480)
    cam, sc, act, g, c = scene_tensors(P, "tum", seed=2, pose_seed=None, dev=cuda, wh=wh, scale_px=150.0)  # ~100s of tiles per Gaussian
    gt = torch.rand((3, wh[1], wh[0]), device=cuda)
    gd = torch.rand((wh[1], wh[0]), device=cuda) * 4.0
    a = _model(sc, cuda)
    ta = trainer.GaussianTrainer(a)
    da = torch.zeros((wh[1], wh[0]), device=cuda)
    ta.trainForOneIteration(c, gt, gt_depth=gd, lambda_depth=LAMBDA_DEPTH, out_depth=da)
    la, _, _, dla, n = ta.result_depth()     # first attempt overflows 6*P + 65536 instances, is repeated internally with its target
    assert n > 6 * P + 65536, "test scene must overflow the initial arena"
    assert a.step_ == 1 and dla > 0.0
    b = _model(sc, cuda)
    tb = trainer.GaussianTrainer(b)
    db = torch.zeros((wh[1], wh[0]), device=cuda)
    tb.render(c, out_depth=db)                # same view: grows the arena before the training step (the render is retried too)
    tb.trainForOneIteration(c, gt, gt_depth=gd, lambda_depth=LAMBDA_DEPTH, out_depth=db)
    lb, _, _, dlb, _ = tb.result_depth()
    torch.cuda.synchronize()
    assert abs(la - lb) < 1e-6 and abs(dla - dlb) < 1e-6 * max(1.0, dlb)
    assert torch.equal(da, db)
    for x, y, lrate in zip(a.tensors(), b.tensors(), LRS):
        assert ((x - y).abs() > 0.5 * lrate).float().mean().item() < 2e-3


CONV_ITERS = 300
# On one H100 (400 W): depth_l1 0.311 -> 0.288 and PSNR 55.46 -> 55.24 dB at this weight (0.005: 0.261, -0.42 dB; 0.05: 0.138, -4.9 dB)
CONV_LAMBDA = 0.002


def _psnr(img, gt):
    return 10.0 * math.log10(1.0 / ((img - gt) ** 2).mean().item())


def test_depth_term_converges_towards_the_target_depth(cuda):
    """300 iterations against the render of a displaced copy of the scene: with lambda_depth > 0 the final depth L1 is lower than
    without (by more than 3 %), at a PSNR cost of at most 0.5 dB."""
    from photo_slam_b200 import trainer
    P, W, H = 20_000, 200, 150
    cam = syn.make_camera(W, H, 170.0, 170.0, *syn.random_pose(np.random.default_rng(3)))
    sc = syn.make_scene(P, cam, seed=4, scale_px=4.0)
    c = syn.device_camera(cam, cuda)
    rng = np.random.default_rng(5)
    sc2 = {k: v.copy() for k, v in sc.items()}
    V = cam["viewmatrix"].reshape(-1)
    zrow = V[[2, 6, 10]] / np.linalg.norm(V[[2, 6, 10]])
    sc2["xyz"] = (sc2["xyz"] + np.outer(rng.normal(0.0, 0.15, P), zrow)).astype(np.float32)   # pushed along the viewing axis
    sc2["features_dc"] = (sc2["features_dc"] + rng.normal(0, 0.3, sc2["features_dc"].shape)).astype(np.float32)
    tgt = trainer.GaussianTrainer(_model(sc2, cuda))
    gt_img, gt_depth = torch.empty((3, H, W), device=cuda), torch.empty((H, W), device=cuda)
    tgt.render(c, gt_img, out_depth=gt_depth)
    gt_img.clamp_(0.0, 1.0)
    holes = torch.rand((H, W), generator=torch.Generator().manual_seed(6)) < 0.1
    gt_depth[holes.to(cuda)] = 0.0
    res = {}
    for lam in (0.0, CONV_LAMBDA):
        tr = trainer.GaussianTrainer(_model(sc, cuda))
        for _ in range(CONV_ITERS):
            if lam > 0:
                tr.trainForOneIteration(c, gt_img, gt_depth=gt_depth, lambda_depth=lam)
            else:
                tr.trainForOneIteration(c, gt_img)
            tr.result()
        img, D = torch.empty((3, H, W), device=cuda), torch.empty((H, W), device=cuda)
        tr.render(c, img, out_depth=D)
        res[lam] = (_torch_depth_l1(D, gt_depth, None), _psnr(img, gt_img))
    (d0, p0), (d1, p1) = res[0.0], res[CONV_LAMBDA]
    print(f"after {CONV_ITERS} iterations: lambda_depth 0: depth_l1 {d0:.4f}, PSNR {p0:.2f} dB; lambda_depth {CONV_LAMBDA}: depth_l1 {d1:.4f}, PSNR {p1:.2f} dB")
    assert d1 < 0.97 * d0
    assert p1 > p0 - 0.5


def reference_cases(cuda):
    """(case, {name: array | scalar}) of the reference chain for the comparisons above (python tests/golden/make_ref_golden.py test_depth_gpu)."""
    for case in CASES:
        yield case, _reference_depth(cuda, case)
