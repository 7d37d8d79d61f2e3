"""-m gpu: anti-aliasing (the 2D Mip filter, o' = o h) on the operator, the fused step and the NVLink step.

  1. operator forward: the tile structures (radii, tiles_touched, num_rendered, sorted keys / values, ranges) equal the plain forward's bit
     for bit; the exported o' / o is the torch h; the plain forward fed o' reproduces the AA image, depth, final_T and n_contrib bit for bit;
     antialiasing = 0 on the new calls is the existing calls bit for bit;
  2. operator backward: every B1 gradient equals autograd through the plain operator with opacities = o h_torch (colour only and with a
     depth gradient, atomic and deterministic); the deterministic AA backward repeats bit for bit;
  3. trainer: psb_trainer_backward and backwardPixels match autograd through renderer.render with AA; the fused AA step equals AA gradients
     + psb_adam_update; backwardPixels refuses a pass whose AA mode was switched;
  4. deterministic mode: the fused and NVLink AA steps repeat bit for bit; DataParallelTrainer(mode="p2p") at world 1 equals the fused AA
     step; several ranks where the machine has them.
Run as a script (python tests/test_antialias_gpu.py <steps>) under torch.distributed.run it is the multi-rank worker of section 4.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from helpers import scene_tensors  # noqa: E402
from splat64 import h_torch, quat_cov as _quat_cov  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(HERE)
CONFIGS = {"A": (50_000, "tum", (640, 480)), "B": (500_000, "replica", (1200, 680)),
           "B600": (500_000, "replica", (600, 340)), "B300": (500_000, "replica", (300, 170))}
LRS = [0.00032, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "the -m gpu tests need a CUDA device"
    return torch.device("cuda:0")


def _rn(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def _scene(dev, config, D, cov_input, seed=5):
    P, camname, wh = CONFIGS[config]
    cam, sc, act, g, c = scene_tensors(P, camname, seed=seed, pose_seed=seed + 1, dev=dev, wh=wh, scale_px=2.4)
    x = dict(means3D=g["means3D"], opacities=g["opacities"], shs=g["shs"][:, : (D + 1) ** 2].contiguous(), scales=g["scales"],
             rotations=g["rotations"], cov3D=None)
    if cov_input:
        x["cov3D"] = _quat_cov(g["scales"].double(), g["rotations"].double()).float().contiguous()
    return c, x


def _settings(c, D, aa, bg):
    from photo_slam_b200 import rasterizer
    return rasterizer.GaussianRasterizationSettings(c["H"], c["W"], c["tanfovx"], c["tanfovy"], bg, 1.0, c["viewmatrix"], c["projmatrix"], D,
                                                    c["campos"], False, aa)


class _Buf:
    def __init__(self, dev):
        self.t, self.dev = torch.empty(0, dtype=torch.uint8, device=dev), dev
        from photo_slam_b200 import _lib
        self.cb = _lib.ALLOC_FN(self._alloc)

    def _alloc(self, n, _u):
        self.t = torch.empty(int(n), dtype=torch.uint8, device=self.dev)
        return self.t.data_ptr()


def _fwd(c, x, opac, D, bg, entry, aa=0):
    """one operator forward through the named C entry point ('plain', 'depth' or 'aa'); everything it leaves behind"""
    from photo_slam_b200 import _lib
    L = _lib.lib()
    dev = x["means3D"].device
    P, H, W = x["means3D"].size(0), c["H"], c["W"]
    color, depth = torch.zeros((3, H, W), device=dev), torch.zeros((H, W), device=dev)
    radii = torch.zeros(P, dtype=torch.int32, device=dev)
    gb, bb, ib = _Buf(dev), _Buf(dev), _Buf(dev)
    cov = x["cov3D"]
    sc, rot = (None, None) if cov is not None else (x["scales"].data_ptr(), x["rotations"].data_ptr())
    args = [gb.cb, None, bb.cb, None, ib.cb, None, P, D, x["shs"].size(1), bg.data_ptr(), W, H, x["means3D"].data_ptr(), x["shs"].data_ptr(), None,
            opac.data_ptr(), sc, 1.0, rot, cov.data_ptr() if cov is not None else None, c["viewmatrix"].data_ptr(), c["projmatrix"].data_ptr(),
            c["campos"].data_ptr(), c["tanfovx"], c["tanfovy"], 0, color.data_ptr(), radii.data_ptr()]
    s = torch.cuda.current_stream().cuda_stream
    if entry == "plain":
        R = _lib.check(L.psb_rasterize_forward(*args, s), "fwd")
        depth = None
    elif entry == "depth":
        R = _lib.check(L.psb_rasterize_forward_depth(*args, depth.data_ptr(), s), "fwd_depth")
    else:
        R = _lib.check(L.psb_rasterize_forward_aa(*args, depth.data_ptr(), aa, s), "fwd_aa")
    # intermediates
    tt = torch.zeros(P, dtype=torch.int32, device=dev)
    co = torch.zeros((P, 4), device=dev)
    keys, vals = torch.zeros(max(R, 1), dtype=torch.int64, device=dev), torch.zeros(max(R, 1), dtype=torch.int32, device=dev)
    ntiles = ((W + 15) // 16) * ((H + 15) // 16)
    ranges = torch.zeros((ntiles, 2), dtype=torch.int32, device=dev)
    nc, fT = torch.zeros(H * W, dtype=torch.int32, device=dev), torch.zeros(H * W, device=dev)
    _lib.check(L.psb_debug_export(P, R, W, H, gb.t.data_ptr(), bb.t.data_ptr() if R else None, ib.t.data_ptr(), None, None, co.data_ptr(), None, None,
                                  tt.data_ptr(), keys.data_ptr(), vals.data_ptr(), ranges.data_ptr(), nc.data_ptr(), fT.data_ptr(), s), "export")
    torch.cuda.synchronize()
    return dict(R=R, color=color, depth=depth, radii=radii, tt=tt, o=co[:, 3].clone(), keys=keys[:R], vals=vals[:R], ranges=ranges, nc=nc, fT=fT,
                bufs=(gb, bb, ib))


def _h(c, x):
    cov = x["cov3D"].double() if x["cov3D"] is not None else _quat_cov(x["scales"].double(), x["rotations"].double())
    return h_torch(x["means3D"].double(), cov, c["viewmatrix"].double(), c["W"], c["H"], c["tanfovx"], c["tanfovy"])


@pytest.mark.parametrize("cov_input", [False, True], ids=["scale-rot", "cov3D"])
@pytest.mark.parametrize("D", [0, 3])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_operator_forward(dev, config, D, cov_input):
    c, x = _scene(dev, config, D, cov_input)
    bg = torch.tensor([0.2, 0.3, 0.4], device=dev)
    plain = _fwd(c, x, x["opacities"], D, bg, "depth")
    aa = _fwd(c, x, x["opacities"], D, bg, "aa", 1)
    assert aa["R"] == plain["R"] > 0
    for k in ("radii", "tt", "keys", "vals", "ranges"):
        assert torch.equal(aa[k], plain[k]), k
    vis = aa["tt"] > 0
    # o' / o against the torch h; beyond 1e-5 only where the float32 det0 = a0 c0 - b^2 loses digits to cancellation
    o = x["opacities"].reshape(-1).double()
    ratio = aa["o"].double()[vis] / o[vis]
    h = _h(c, x)[vis]
    err = (ratio - h).abs() / h
    assert (h < 0.999).float().mean() > 0.5
    frac = (err > 1e-5).double().mean().item()
    print(f"{config} D={D} cov={cov_input}: {int(vis.sum())} visible, max rel err of o'/o vs h {err.max().item():.2e}, share > 1e-5: {frac:.2e}, "
          f"mean h {h.mean().item():.4f}")
    assert frac < 1e-3 and err.max().item() < 1e-3
    # the plain forward fed o' reproduces the AA pass bit for bit
    o_prime = torch.where(vis, aa["o"], x["opacities"].reshape(-1)).reshape(-1, 1).contiguous()
    again = _fwd(c, x, o_prime, D, bg, "depth")
    for k in ("color", "depth", "fT", "nc", "radii", "keys", "vals", "ranges"):
        assert torch.equal(again[k], aa[k]), k
    # antialiasing = 0 on the new call is the existing call
    off = _fwd(c, x, x["opacities"], D, bg, "aa", 0)
    for k in ("color", "depth", "fT", "nc", "radii", "tt", "o", "keys", "vals", "ranges"):
        assert torch.equal(off[k], plain[k]), k
    assert not torch.equal(aa["color"], plain["color"])


def _grad_pair(c, x, D, bg, wc, wd, deterministic):
    """(AA operator gradients, oracle gradients) of sum wc*color [+ sum wd*depth] w.r.t. the B1 leaves"""
    from photo_slam_b200 import rasterizer
    names = ["means3D", "opacities", "shs"] + (["cov3D"] if x["cov3D"] is not None else ["scales", "rotations"])
    out = []
    for mode in ("aa", "oracle"):
        leaves = {k: x[k].detach().clone().requires_grad_(True) for k in names}
        means2D = torch.zeros_like(x["means3D"], requires_grad=True)
        opac = leaves["opacities"]
        if mode == "oracle":
            cov = leaves["cov3D"].double() if "cov3D" in leaves else _quat_cov(leaves["scales"].double(), leaves["rotations"].double())
            h = h_torch(leaves["means3D"].double(), cov, c["viewmatrix"].double(), c["W"], c["H"], c["tanfovx"], c["tanfovy"])
            opac = (opac.double() * h.unsqueeze(1)).float()
        r = rasterizer.GaussianRasterizer(_settings(c, D, mode == "aa", bg))
        color, radii, depth = r(leaves["means3D"], means2D, opac, shs=leaves["shs"], scales=leaves.get("scales"), rotations=leaves.get("rotations"),
                                cov3D_precomp=leaves.get("cov3D"), return_depth=True, deterministic=deterministic)
        loss = (wc * color).sum() + ((wd * depth).sum() if wd is not None else 0.0)
        loss.backward()
        out.append({k: v.grad.detach().clone() for k, v in leaves.items()} | {"means2D": means2D.grad.detach().clone()})
    return out


@pytest.mark.parametrize("cov_input", [False, True], ids=["scale-rot", "cov3D"])
@pytest.mark.parametrize("D", [0, 3])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_operator_backward_matches_autograd_through_h(dev, config, D, cov_input):
    c, x = _scene(dev, config, D, cov_input)
    bg = torch.tensor([0.2, 0.3, 0.4], device=dev)
    gen = torch.Generator().manual_seed(3)
    wc = ((torch.rand((3, c["H"], c["W"]), generator=gen) - 0.5) / (c["H"] * c["W"])).to(dev)
    wd = ((torch.rand((c["H"], c["W"]), generator=gen) - 0.5) / (c["H"] * c["W"])).to(dev)
    for depth in (False, True):
        for det in (False, True):
            mine, ref = _grad_pair(c, x, D, bg, wc, wd if depth else None, det)
            for k in ref:
                rn = _rn(mine[k], ref[k])
                print(f"{config} D={D} cov={cov_input} depth={depth} det={det}: {k} rel-norm {rn:.2e}")
                assert ref[k].abs().sum() > 0, k
                assert rn <= 1e-4, (k, rn)
    # the deterministic AA backward repeats bit for bit
    a, _ = _grad_pair(c, x, D, bg, wc, wd, True)
    b, _ = _grad_pair(c, x, D, bg, wc, wd, True)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_libtorch_ops_equal_the_python_path(dev):
    import photo_slam_b200  # noqa: F401  (loads the LibTorch ops)
    from photo_slam_b200 import rasterizer
    torch.ops.load_library(os.path.join(ROOT, "photo-slam_b200", "lib", "libcuda_rasterizer.so"))
    c, x = _scene(dev, "A", 3, False)
    bg = torch.tensor([0.1, 0.2, 0.3], device=dev)
    e = torch.empty(0, device=dev)
    args = (bg, x["means3D"], e, x["opacities"], x["scales"], x["rotations"], 1.0, e, c["viewmatrix"], c["projmatrix"], c["tanfovx"], c["tanfovy"],
            c["H"], c["W"], x["shs"], 3, c["campos"], False)
    py = rasterizer.RasterizeGaussiansDepthCUDA(*args, antialiasing=True)
    op = torch.ops.psb200.rasterize_gaussians_antialiased(*args)
    assert py[0] == op[0]
    for a, b in zip(py[1:4], op[1:4]):
        assert torch.equal(a, b)
    dpix = torch.randn((3, c["H"], c["W"]), device=dev) / 1e4
    ddep = torch.randn((c["H"], c["W"]), device=dev) / 1e4
    gpy = rasterizer.RasterizeGaussiansBackwardDepthCUDA(bg, x["means3D"], py[3], e, x["scales"], x["rotations"], 1.0, e, c["viewmatrix"], c["projmatrix"],
                                                         c["tanfovx"], c["tanfovy"], dpix, ddep, x["shs"], 3, c["campos"], py[4], py[0], py[5], py[6],
                                                         deterministic=True, antialiasing=True)
    gop = torch.ops.psb200.rasterize_gaussians_backward_antialiased(bg, x["means3D"], op[3], e, x["scales"], x["rotations"], 1.0, e, c["viewmatrix"],
                                                                    c["projmatrix"], c["tanfovx"], c["tanfovy"], dpix, ddep, x["shs"], 3, c["campos"],
                                                                    op[4], op[0], op[5], op[6], True)
    for a, b in zip(gpy, gop):
        assert torch.equal(a, b)


# ---- trainer -----------------------------------------------------------------------------------------------------------------------
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


def _operator_grads(sc, c, dev, wc, wd, wa, sh):
    """autograd through renderer.render with AA of sum wc*image + sum wd*depth + sum wa*A (A = the red channel of a black-background
    render with colour (1, 0, 0))"""
    from photo_slam_b200 import renderer, trainer
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.setShDegree(sh)
    for t in m.tensors():
        t.requires_grad_(True)
    pipe = renderer.GaussianPipelineParams(antialiasing=True)
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
    return [t.grad.detach().clone() for t in m.tensors()], img.detach()


def test_trainer_backward_matches_the_operator_path(dev):
    """psb_trainer_backward (built-in L1 + D-SSIM) with AA == autograd through renderer.render(AA) of the loss's pixel gradient"""
    from photo_slam_b200 import trainer
    from photo_slam_b200.parallel import GradBuffer
    sc, c, gt, gd = _train_inputs(dev)
    P, H, W = sc["xyz"].shape[0], c["H"], c["W"]
    m = _model(sc, dev)
    tr = trainer.GaussianTrainer(m, antialiasing=True)
    assert tr.antialiasing
    img = tr.render(c)
    buf = GradBuffer(P, dev)
    cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)
    ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in buf.segments])
    from photo_slam_b200 import _lib
    _lib.check(tr.L.psb_trainer_backward(tr.h, P, 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), None, C.byref(cs), None, None,
                                         ptrs, torch.cuda.current_stream().cuda_stream), "psb_trainer_backward")
    tr.result()
    _, _, _, gc = trainer.fused_loss(img, gt, None, tr.opt.lambda_dssim)
    ref, ref_img = _operator_grads(sc, c, dev, gc, None, None, m.active_sh_degree_)
    torch.cuda.synchronize()
    assert (img - ref_img).abs().max().item() < 1e-4
    for name, a, b in zip(trainer.GROUPS, buf.views(), ref):
        rn = _rn(a, b)
        print(f"psb_trainer_backward AA grad {name}: rel-norm vs operator {rn:.2e}")
        assert rn < 2e-4, (name, rn)


def test_pixel_gradients_match_the_operator_path_and_refuse_a_switched_mode(dev):
    from photo_slam_b200 import _lib, trainer
    sc, c, gt, gd = _train_inputs(dev, P=30_000, wh=(320, 240), seed=11)
    P, H, W = sc["xyz"].shape[0], c["H"], c["W"]
    gen = torch.Generator().manual_seed(12)
    wc = (torch.rand((3, H, W), generator=gen) - 0.5).to(dev)
    wd = (0.1 * (torch.rand((H, W), generator=gen) - 0.5)).to(dev)
    wa = (torch.rand((H, W), generator=gen) - 0.5).to(dev)
    ref, ref_img = _operator_grads(sc, c, dev, wc, wd, wa, 2)
    m = _model(sc, dev)
    tr = trainer.GaussianTrainer(m, antialiasing=True)
    img, A = torch.empty((3, H, W), device=dev), torch.empty((H, W), device=dev)
    tr.render(c, img, out_depth=torch.empty((H, W), device=dev), out_alpha=A)
    grads = [torch.zeros_like(t) for t in m.tensors()]
    tr.backwardPixels(wc, wd, wa, grads=grads)
    tr.result()
    torch.cuda.synchronize()
    assert (img - ref_img).abs().max().item() < 1e-4
    for name, a, b in zip(trainer.GROUPS, grads, ref):
        rn = _rn(a, b)
        print(f"backwardPixels AA grad {name}: rel-norm vs operator {rn:.2e}")
        assert rn < 2e-4, (name, rn)
    # trainWithLoss with the same linear loss takes one fused Adam step from those gradients
    m2 = _model(sc, dev)
    tr2 = trainer.GaussianTrainer(m2, antialiasing=True)
    tr2.render(c)
    before = [t.clone() for t in m2.tensors()]
    tr2.trainWithLoss(c, lambda i, d, a: (wc * i).sum() + (wd * d).sum() + (wa * a).sum(), depth=True, alpha=True)
    tr2.result()
    torch.cuda.synchronize()
    for name, p0, p1, g, lr in zip(trainer.GROUPS, before, m2.tensors(), ref, LRS):
        moved = (p1 - p0).abs() > 0.5 * lr                    # the first Adam step moves every element with a gradient by ~lr
        has = g.abs() > 1e-3 * g.abs().max()
        assert (moved == has)[has].double().mean() > 0.99, name
        assert (torch.sign(p0 - p1)[has & moved] == torch.sign(g)[has & moved]).double().mean() > 0.99, name
    # a pass rendered with AA cannot be back-propagated after the mode was switched off
    tr.render(c, img)
    _lib.check(tr.L.psb_trainer_set_antialiasing(tr.h, 0), "psb_trainer_set_antialiasing")
    with pytest.raises(_lib.PsbError, match="anti-aliasing mode changed"):
        tr.backwardPixels(wc, grads=grads)
    _lib.check(tr.L.psb_trainer_set_antialiasing(tr.h, 1), "psb_trainer_set_antialiasing")


def _state(m):
    return [t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + [m.xyz_gradient_accum_, m.denom_, m.max_radii2D_]]


def test_fused_step_equals_gradients_plus_adam_update(dev):
    """the fused AA step (adam_live on) == psb_trainer_backward_depth with AA + psb_adam_update, over steps with an SH-degree change and a
    depth target"""
    from photo_slam_b200 import _lib, trainer
    from photo_slam_b200.parallel import GradBuffer
    sc, c, gt, gd = _train_inputs(dev)
    P = sc["xyz"].shape[0]
    a, b = _model(sc, dev, sh=0), _model(sc, dev, sh=0)
    ta = trainer.GaussianTrainer(a, deterministic=True, antialiasing=True)
    tb = trainer.GaussianTrainer(b, deterministic=True, antialiasing=True)
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
        print(f"fused AA vs gradients + Adam: {name} rel-norm {rn:.2e}, entries apart by > lr/2: {frac:.2e}")
        assert frac < 2e-3 and rn < 1e-4, (name, frac, rn)


def _aa_run(sc, c, gt, gd, dev, cls, **kw):
    from photo_slam_b200 import trainer
    m = _model(sc, dev, sh=1)
    tr = getattr(trainer, cls)(m, deterministic=True, antialiasing=True, **kw)
    tr.render(c)
    for it in range(4):
        extra = dict(gt_depth=gd, lambda_depth=0.1) if it % 2 else {}
        tr.trainForOneIteration(c, gt, **extra)
        tr.result()
    if cls == "DataParallelTrainer":
        tr.sync()
    torch.cuda.synchronize()
    out = _state(m)
    if cls == "DataParallelTrainer":
        tr.close()
    return out


def test_deterministic_fused_and_nvlink_steps_repeat_and_agree_at_world_1(dev):
    sc, c, gt, gd = _train_inputs(dev, P=20_000, wh=(320, 240), seed=5)
    f1 = _aa_run(sc, c, gt, gd, dev, "GaussianTrainer")
    f2 = _aa_run(sc, c, gt, gd, dev, "GaussianTrainer")
    for i, (x, y) in enumerate(zip(f1, f2)):
        assert torch.equal(x, y), i
    p1 = _aa_run(sc, c, gt, gd, dev, "DataParallelTrainer", mode="p2p")
    p2 = _aa_run(sc, c, gt, gd, dev, "DataParallelTrainer", mode="p2p")
    for i, (x, y) in enumerate(zip(p1, p2)):
        assert torch.equal(x, y), i
    # world 1: the NVLink step's parameters are the fused step's (as test_dp_gpu.py checks for the plain step)
    for x, y, lr in zip(f1[:6], p1[:6], LRS):
        assert ((x - y).abs() > 0.5 * lr).float().mean().item() < 2e-3
    # and AA changes the result
    from photo_slam_b200 import trainer
    m = _model(sc, dev, sh=1)
    tr = trainer.GaussianTrainer(m, deterministic=True)
    tr.render(c)
    tr.trainForOneIteration(c, gt)
    tr.result()
    assert not torch.equal(m.xyz_, f1[0])


def test_multi_rank_aa_replicas_identical(dev):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    world = 2 if n < 4 else (4 if n < 8 else 8)
    port = 29500 + (os.getpid() % 400) + 7
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1", "--master-port",
           str(port), os.path.abspath(__file__), "3"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=420, env=dict(os.environ, PSB_DP_TIMEOUT_MS="15000"))
    assert r.returncode == 0 and "AA_WORKER_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])


def _worker(steps):
    """one rank of the multi-rank test: AA p2p steps on this rank's own view; every replica must end bit-identical"""
    import torch.distributed as dist
    sys.path.insert(0, ROOT)
    import photo_slam_b200.synthetic as syn
    from photo_slam_b200 import trainer
    dist.init_process_group("nccl")
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)
    sc, c0, gt, gd = _train_inputs(dev, P=30_001, wh=(320, 240), seed=9)
    cam = syn.make_camera(320, 240, 600.0 * 320 / 1200, 600.0 * 240 / 680, *syn.random_pose(np.random.default_rng(100 + rank)))
    c = syn.device_camera(cam, dev)
    m = _model(sc, dev, sh=1)
    tr = trainer.DataParallelTrainer(m, mode="p2p", deterministic=True, antialiasing=True)
    assert tr.mode == "p2p"
    for _ in range(steps):
        tr.trainForOneIteration(c, gt)
        tr.result()
    tr.sync()
    torch.cuda.synchronize()
    flat = torch.cat([t.reshape(-1) for t in m.tensors()])
    allv = [torch.empty_like(flat) for _ in range(world)]
    dist.all_gather(allv, flat)
    assert all(torch.equal(allv[0], v) for v in allv), "replicas differ"
    assert tr.status() == 0
    tr.close()
    dist.barrier()
    if rank == 0:
        print("AA_WORKER_OK", world)
    dist.destroy_process_group()


if __name__ == "__main__":
    _worker(int(sys.argv[1]) if len(sys.argv) > 1 else 3)
