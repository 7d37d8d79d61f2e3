"""-m gpu: rendered normals (include/psb200.h, "Rendered surface normals").

  1. the normal plane of psb_trainer_forward_normal matches tests/normal64.py on settled scenes, plain, anti-aliased and with the 3D
     filter's other outputs untouched: colour, depth, A, radii, final T and the last blended Gaussian equal psb_trainer_forward's;
  2. backwardPixels(grads=...) with colour, depth, A and normal gradients matches autograd on normal64 per parameter group, and a normal
     pass back-propagated without a normal gradient is the plain backward bit for bit (deterministic mode);
  3. psb_trainer_step_normal equals forward_normal + psb_loss + the depth and normal gradients in torch + backward_pixels_normal bit for
     bit over 8 deterministic steps with a mask and depth; normal == NULL is psb_trainer_step_exposure bit for bit (with an exposure row);
     normal_l1 matches float64;
  4. psb_depth_normals matches normal64 on a rendered depth with holes and edges;
  5. 20 deterministic steps with the normal term are bit-identical run to run, plain, AA and 3D-filtered;
  6. an overflowing normal step is repeated with its target;
  7. the refusals leave the model untouched;
  8. on the planar scene the normal term lowers the angle error well below the depth-only run's without lowering PSNR materially.
"""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

import normal64
import photo_slam_b200.synthetic as syn
import splat64 as s64

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
pytestmark = pytest.mark.gpu
LAMBDA_DSSIM, LAMBDA_DEPTH, LAMBDA_NORMAL = 0.2, 0.1, 0.05
GATE_NORMAL = 1e-5        # max |N - N64| (|N_c| <= 1): measured 1.3e-6 (scene b, plain)
GATE_GRAD = 2e-5          # rel-norm per raw parameter group, as tests/test_splat64_gpu.py: measured 1.2e-6 (xyz, scene a)
GATE_SENSOR = 2e-5        # max |n - n64| of the sensor normals on valid pixels: measured 1.8e-6
GATE_L1 = 1e-4            # normal_l1, relative to float64 on the kernel's own plane
# planar payoff (300 steps, 3 x 3000 Gaussians): angle error measured 45.0 deg (depth only) -> 8.8 deg (depth + normals), PSNR 36.29 ->
# 35.67 dB on the held-out views
GATE_ANGLE_RATIO = 0.6
GATE_PSNR_DROP = 1.0


def _model(sc, dev, sh=1):
    from photo_slam_b200 import trainer
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    m.setShDegree(sh)
    return m


def _state(m):
    return [t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + [m.xyz_gradient_accum_, m.denom_, m.max_radii2D_]]


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


_SCENES = {}


def _settled(name):
    """small dense scenes (splat64.settle: every decision at least 1e-4 from its threshold), as tests/test_splat64_gpu.py builds them"""
    if name not in _SCENES:
        seed, P, W, H = {"a": (5, 700, 64, 48), "b": (6, 1500, 80, 56)}[name]
        cam = syn.make_camera(W, H, 0.9 * W, 0.9 * W, *syn.random_pose(np.random.default_rng(seed)))
        sc = syn.make_scene(P, cam, seed=seed, scale_px=3.0)
        s64.settle(sc, cam, D=1, aa=None, bg=(0.0, 0.0, 0.0), seed=1, dev="cuda")
        _SCENES[name] = (cam, sc)
    return _SCENES[name]


def _debug(tr, W, H, dev):
    last = torch.empty(W * H, dtype=torch.int32, device=dev)
    fT = torch.empty(W * H, dtype=torch.float32, device=dev)
    from photo_slam_b200 import _lib
    _lib.check(tr.L.psb_trainer_debug_state(tr.h, W, H, last.data_ptr(), fT.data_ptr(), None, torch.cuda.current_stream().cuda_stream), "debug")
    return last, fT


def _filter(m, c):
    m.computeFilter3D([c])


@pytest.mark.parametrize("name,mode", [(n, md) for n in ("a", "b") for md in ("plain", "aa", "f3d")])
def test_normal_plane_against_truth(cuda, name, mode):
    from photo_slam_b200 import trainer
    cam, sc = _settled(name)
    c = syn.device_camera(cam, cuda)
    W, H, P = c["W"], c["H"], sc["xyz"].shape[0]
    m = _model(sc, cuda)
    if mode == "f3d":
        _filter(m, c)
    tr = trainer.GaussianTrainer(m, antialiasing=mode == "aa", filter3d=mode == "f3d")
    tr.render(c)
    outs = []
    for with_normal in (False, True):
        img, rad = torch.empty((3, H, W), device=cuda), torch.zeros(P, dtype=torch.int32, device=cuda)
        D, A = torch.full((H, W), -7.0, device=cuda), torch.full((H, W), -7.0, device=cuda)
        N = torch.full((3, H, W), -7.0, device=cuda) if with_normal else None
        tr.render(c, img, rad, out_depth=D, out_alpha=A, out_normal=N)
        outs.append((img, rad, D, A, *_debug(tr, W, H, cuda), N))
    torch.cuda.synchronize()
    for x, y in zip(outs[0][:6], outs[1][:6]):
        assert torch.equal(x, y)
    N = outs[1][6]
    if mode == "f3d":
        return     # normal64 has no 3D filter; n_i does not depend on it (the widening keeps the axes) and the blend is checked bit for bit above
    raw = s64.raw64(sc, cuda)
    _, N64 = normal64.render_normal(raw, s64.camera64(cam, cuda), D=1, aa=mode == "aa")
    err = float((N.double() - N64).abs().max())
    print(f"MEASURED normal plane {name} {mode}: max err {err:.3g}, |N| max {float(N64.abs().max()):.3g}")
    assert (N64.abs() > 0.1).any() and err < GATE_NORMAL


def _relnorm(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).norm() / b.norm()) if b.norm() > 0 else float(a.norm())


@pytest.mark.parametrize("name,aa", [("a", False), ("b", True)])
def test_pixel_gradients_against_autograd(cuda, name, aa):
    from photo_slam_b200 import trainer
    from photo_slam_b200.parallel import GradBuffer
    cam, sc = _settled(name)
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    gen = torch.Generator().manual_seed(7)
    wc, wd, wa, wn = (torch.rand((3, H, W), generator=gen) - 0.5, 0.2 * (torch.rand((H, W), generator=gen) - 0.5),
                      torch.rand((H, W), generator=gen) - 0.5, torch.rand((3, H, W), generator=gen) - 0.5)
    wc, wd, wa, wn = (x.to(cuda).contiguous() for x in (wc, wd, wa, wn))
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m, antialiasing=aa, deterministic=True)
    tr._apply_deterministic()
    tr.render(c)
    D, A, N = torch.empty((H, W), device=cuda), torch.empty((H, W), device=cuda), torch.empty((3, H, W), device=cuda)
    tr.render(c, out_depth=D, out_alpha=A, out_normal=N)
    buf = GradBuffer(m.num_points(), cuda)
    tr.backwardPixels(wc, wd, wa, grads=buf.views(), dL_dnormal=wn)
    torch.cuda.synchronize()
    kern = [g.clone() for g in buf.views()]
    raw = {k: v.requires_grad_(True) for k, v in s64.raw64(sc, cuda).items()}
    out, N64 = normal64.render_normal(raw, s64.camera64(cam, cuda), D=1, aa=aa)
    L = (out["color"] * wc.double()).sum() + (out["depth"] * wd.double()).sum() + (out["alpha"] * wa.double()).sum() + (N64 * wn.double()).sum()
    L.backward()
    errs = {}
    for k, g in zip(s64.RAW, kern):
        ref = raw[k].grad
        if k == "features_rest":
            ref = ref[:, :3]
            g = g.reshape(ref.shape[0], 15, 3)[:, :3]
        errs[k] = _relnorm(g.reshape(ref.shape), ref)
    print(f"MEASURED pixel gradients {name} aa={aa}: {errs}")
    assert all(v < GATE_GRAD for v in errs.values()), errs
    # the rotation gradient carries the normal term: without it the gate fails
    raw2 = {k: v.detach().clone().requires_grad_(True) for k, v in raw.items()}
    out2 = s64.render(raw2, s64.camera64(cam, cuda), (0.0, 0.0, 0.0), D=1, aa=aa, raw=True)
    ((out2["color"] * wc.double()).sum() + (out2["depth"] * wd.double()).sum() + (out2["alpha"] * wa.double()).sum()).backward()
    assert _relnorm(kern[5].reshape(raw2["rotation"].shape), raw2["rotation"].grad) > 10 * GATE_GRAD
    # a normal pass back-propagated without a normal gradient is the plain backward, bit for bit
    res = []
    for with_plane in (False, True):
        buf2 = GradBuffer(m.num_points(), cuda)
        tr.render(c, out_depth=D, out_alpha=A, out_normal=N if with_plane else None)
        tr.backwardPixels(wc, wd, wa, grads=buf2.views())
        torch.cuda.synchronize()
        res.append([g.clone() for g in buf2.views()])
    assert _same(res[0], res[1])


def _targets(H, W, dev, seed=3):
    gen = torch.Generator().manual_seed(seed)
    gt = torch.rand((3, H, W), generator=gen).to(dev)
    mask = (torch.rand((1, H, W), generator=gen) > 0.2).float().expand(3, H, W).contiguous().to(dev)
    gd = (0.5 + 6 * torch.rand((H, W), generator=gen)).to(dev)
    gd[(torch.rand((H, W), generator=gen) < 0.2).to(dev)] = 0.0
    gn = torch.nn.functional.normalize(torch.randn((3, H, W), generator=gen), dim=0).to(dev)
    gn[:, (torch.rand((H, W), generator=gen) < 0.2).to(dev)] = 0.0
    return gt, mask, gd, gn.contiguous()


def _grad_of_l1(X, G, valid, lam):
    """the built-in L1 gradient with the kernels' float expression: sign(X - G) * (lambda / max(N_valid, 1)) on valid pixels; valid [H,W]
    (X, G: [H,W] or [3,H,W])"""
    scale = np.float32(lam) / np.float32(max(int(valid.sum().item()), 1))
    return torch.where(valid.expand_as(X), torch.sign(X - G) * float(scale), torch.zeros_like(X)).contiguous()


def test_builtin_step_reproduced_bit_for_bit(cuda):
    from photo_slam_b200 import trainer
    cam, sc = _settled("b")
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    gt, mask, gd, gn = _targets(H, W, cuda)
    runs, l1s = [], []
    for path in ("builtin", "pixels"):
        m = _model(sc, cuda)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        tr.opt.lambda_dssim = LAMBDA_DSSIM
        tr.render(c)
        imgs = []
        for it in range(8):
            msk = mask if it % 2 == 0 else None
            img = torch.empty((3, H, W), device=cuda)
            if path == "builtin":
                N = torch.empty((3, H, W), device=cuda)
                tr.trainForOneIteration(c, gt, msk, out_color=img, gt_depth=gd, lambda_depth=LAMBDA_DEPTH, gt_normal=gn, lambda_normal=LAMBDA_NORMAL,
                                        out_normal=N)
                res = tr.result_normal()
                vmask = msk if msk is not None else None
                l1s.append((res[4], float(normal64.normal_l1_64(N.double(), gn.double(), vmask))))
            else:
                D, N = torch.empty((H, W), device=cuda), torch.empty((3, H, W), device=cuda)
                tr.render(c, img, check=False, out_depth=D, out_normal=N)
                _, _, _, g = trainer.fused_loss(img, gt, msk, LAMBDA_DSSIM)
                vd = gd > 0
                vn = (gn != 0).any(0)
                if msk is not None:
                    vd, vn = vd & (msk[0] != 0), vn & (msk[0] != 0)
                tr.backwardPixels(g, _grad_of_l1(D, gd, vd, LAMBDA_DEPTH), dL_dnormal=_grad_of_l1(N, gn, vn, LAMBDA_NORMAL))
                tr.result()
            imgs.append(img)
        torch.cuda.synchronize()
        runs.append((imgs, _state(m)))
    assert all(torch.equal(x, y) for x, y in zip(runs[0][0], runs[1][0]))
    assert _same(runs[0][1], runs[1][1])
    for k, t in l1s:
        assert abs(k - t) <= GATE_L1 * t, (k, t)
    print(f"MEASURED normal_l1 kernel vs float64: {l1s[:2]}")


def test_null_normal_is_the_exposure_step(cuda):
    from photo_slam_b200 import _lib, trainer
    cam, sc = _settled("a")
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    gt, mask, gd, _ = _targets(H, W, cuda)
    states = []
    for fn in ("psb_trainer_step_exposure", "psb_trainer_step_normal"):
        m = _model(sc, cuda)
        m.ensureExposures(1)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        tr._apply_deterministic()
        tr.render(c)
        for it in range(3):
            cm, cc, cs = m._cmodel(live=m.adamLive()), trainer._ccamera(c), tr._cstep(True)
            d = trainer._Depth(gd.data_ptr(), LAMBDA_DEPTH, None)
            ex = trainer._Exposure(m.exposure_[0].data_ptr(), m.exposure_exp_avg_[0].data_ptr(), m.exposure_exp_avg_sq_[0].data_ptr(),
                                   m.exposure_step_.data_ptr(), 0.01)
            args = (*tr._call_args(m, cm, cc, cs, gt, mask, None, None), C.byref(d), C.byref(ex))
            stream = torch.cuda.current_stream().cuda_stream
            rc = getattr(tr.L, fn)(*args, stream) if fn.endswith("exposure") else tr.L.psb_trainer_step_normal(*args, None, stream)
            _lib.check(rc, fn)
            m.step_ += 1
            tr.result()
        torch.cuda.synchronize()
        states.append(_state(m) + [m.exposure_.clone()])
    assert _same(states[0], states[1])


def test_sensor_normals_against_truth(cuda):
    from photo_slam_b200 import trainer
    cam, sc = _settled("b")
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    tr = trainer.GaussianTrainer(_model(sc, cuda))
    D, A = torch.empty((H, W), device=cuda), torch.empty((H, W), device=cuda)
    tr.render(c, out_depth=D, out_alpha=A)
    z = torch.where(A > 0.3, D / A.clamp_min(1e-6), torch.zeros_like(D))
    z[5:9, 10:14] = float("nan")
    z[20:22, :] = -1.0
    out = trainer.normals_from_depth(c, z.contiguous(), 0.05)
    out2 = trainer.normals_from_depth(c, z.contiguous(), 0.05)
    torch.cuda.synchronize()
    assert torch.equal(out, out2)
    ref = normal64.depth_normals64(z, W, H, float(c["tanfovx"]), float(c["tanfovy"]), 0.05)
    # the validity pattern is exact away from the jump threshold
    zz = z.double()
    nb = [zz[1:-1, :-2], zz[1:-1, 2:], zz[:-2, 1:-1], zz[2:, 1:-1]]
    ratio = torch.stack([(n - zz[1:-1, 1:-1]).abs() / zz[1:-1, 1:-1].abs().clamp_min(1e-12) for n in nb]).nan_to_num(0.0)
    near = torch.zeros((H, W), dtype=torch.bool, device=cuda)
    near[1:-1, 1:-1] = ((ratio - 0.05).abs() < 1e-4).any(0)
    vk, vr = (out != 0).any(0), (ref != 0).any(0)
    assert torch.equal(vk[~near], vr[~near])
    both = vk & vr
    err = float((out.double() - ref).abs()[:, both].max())
    print(f"MEASURED sensor normals: {int(both.sum())} valid pixels, max err {err:.3g}")
    assert both.sum() > 100 and err < GATE_SENSOR


@pytest.mark.parametrize("mode", ["plain", "aa", "f3d"])
def test_normal_steps_bit_identical_run_to_run(cuda, mode):
    from photo_slam_b200 import trainer
    cam, sc = _settled("b")
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    gt, mask, gd, gn = _targets(H, W, cuda)
    runs = []
    for _ in range(2):
        m = _model(sc, cuda)
        if mode == "f3d":
            _filter(m, c)
        tr = trainer.GaussianTrainer(m, deterministic=True, antialiasing=mode == "aa", filter3d=mode == "f3d")
        for it in range(20):
            tr.trainForOneIteration(c, gt, mask if it % 2 else None, gt_depth=gd, lambda_depth=LAMBDA_DEPTH, gt_normal=gn, lambda_normal=LAMBDA_NORMAL)
            tr.result()
        torch.cuda.synchronize()
        runs.append(_state(m))
    assert _same(runs[0], runs[1])


def test_overflowing_normal_step_is_repeated_with_its_target(cuda):
    """A: the first normal step overflows the initial binning arena and result_normal() repeats it with its target; B: a render grows the
    arena first. Same model state and normal_l1 either way."""
    from helpers import scene_tensors
    from photo_slam_b200 import trainer
    wh = (640, 480)
    cam, sc, act, g, c = scene_tensors(2_000, "tum", seed=2, pose_seed=None, dev=cuda, wh=wh, scale_px=150.0)  # ~100s of tiles per Gaussian
    gt, _, gd, gn = _targets(wh[1], wh[0], cuda)
    runs = []
    for pregrow in (False, True):
        m = _model(sc, cuda)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        if pregrow:
            tr.render(c)
        tr.trainForOneIteration(c, gt, gt_depth=gd, lambda_depth=LAMBDA_DEPTH, gt_normal=gn, lambda_normal=LAMBDA_NORMAL)
        res = tr.result_normal()
        ov = tr._overflow_info()
        torch.cuda.synchronize()
        assert res[5] > 6 * 2_000 + 65536, "the view must overflow the initial arena"
        assert m.step_ == 1 and tr.iteration == 1 and ov[1] == 1 and res[4] > 0
        runs.append((res, _state(m)))
    assert repr(runs[0][0]) == repr(runs[1][0])
    assert _same(runs[0][1], runs[1][1])


def test_refusals_leave_the_model_untouched(cuda):
    from photo_slam_b200 import _lib, trainer
    cam, sc = _settled("a")
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    gt, _, gd, gn = _targets(H, W, cuda)
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m)
    tr.trainForOneIteration(c, gt, gt_normal=gn, lambda_normal=LAMBDA_NORMAL)
    tr.result()
    before = _state(m)
    for gt_n, lam in ((gn, 0.0), (None, 0.1), (gn, -1.0), (gn, math.nan)):
        with pytest.raises(_lib.PsbError, match="psb_trainer_step_normal"):
            tr.trainForOneIteration(c, gt, gt_normal=gt_n, lambda_normal=lam)
    tr.render(c)    # no normal plane: a normal gradient is refused by the library too
    px = trainer._PixelGrads(torch.zeros((3, H, W), device=cuda).data_ptr(), None, None)
    cm, cc, cs = m._cmodel(live=m.adamLive()), trainer._ccamera(c), tr._cstep(True)
    rc = tr.L.psb_trainer_backward_pixels_normal(tr.h, tr._pass, m.num_points(), 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), C.byref(px),
                                                 torch.zeros((3, H, W), device=cuda).data_ptr(), C.byref(cs), None, torch.cuda.current_stream().cuda_stream)
    assert rc == -1 and b"dL_dnormal" in tr.L.psb_last_error()
    torch.cuda.synchronize()
    assert _same(before, _state(m))


def test_planar_scene_payoff(cuda):
    from normal_bench import planar_payoff
    res = planar_payoff(cuda, per_wall=3000, steps=300, lambda_normal=LAMBDA_NORMAL, lambda_depth=LAMBDA_DEPTH)
    print(f"MEASURED planar payoff: {res}")
    d, n = res["depth"], res["depth+normal"]
    assert n["angle"] < GATE_ANGLE_RATIO * d["angle"], res
    assert n["psnr"] > d["psnr"] - GATE_PSNR_DROP, res
