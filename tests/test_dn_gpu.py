"""-m gpu: depth-normal consistency (include/psb200.h, "Depth-normal consistency").

  1. n_d (out_depth_normal) equals normals_from_depth of where(A >= alpha_min, D / A, 0) bit for bit: both run one device function;
  2. psb_dn_loss's dn and its dL/dD, dL/dA and dL/dN match autograd on tests/dn64.py on settled scenes, with and without a mask;
  3. psb_trainer_forward_normal + psb_dn_loss + backwardPixels match autograd through normal64.render_normal + dn64 per raw parameter
     group, plain and anti-aliased; without the D-bar path the position gradient misses the gate;
  4. the built-in step with depth + normal + consistency terms equals forward_normal + psb_loss + the depth and normal L1 gradients +
     psb_dn_loss (adding) + backwardPixels bit for bit over 8 deterministic steps;
  5. dn == NULL is psb_trainer_step_normal bit for bit;
  6. 20 deterministic steps with the term are bit-identical run to run, plain, anti-aliased and 3D-filtered;
  7. an overflowing step is repeated with its term; the refusals leave the model untouched;
  8. on the planar scene without depth or normal targets the term lowers the angle error well below the colour-only run's, with PSNR
     within 1 dB.
"""
import ctypes as C
import math
import os
import sys

import pytest
import torch

import dn64
import normal64
import photo_slam_b200.synthetic as syn
import splat64 as s64
from test_normal_gpu import _filter, _grad_of_l1, _model, _relnorm, _same, _settled, _state, _targets

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
pytestmark = pytest.mark.gpu
LAMBDA_DSSIM, LAMBDA_DEPTH, LAMBDA_NORMAL, LAMBDA_DN = 0.2, 0.1, 0.05, 0.05
ALPHA_MIN, JUMP = 0.5, 0.05
# Measured on an H100 80GB HBM3 (700 W). The planes' error is float32's rounding of D / A, amplified by the central differences where
# neighbouring depths are close; weighted through the blend into the raw parameters it is far smaller.
GATE_PLANES = 5e-4        # rel-norm of dL/dD, dL/dA, dL/dN of psb_dn_loss against float64 on the kernel's own planes: measured 1.4e-4 (dL/dN, b)
GATE_DN = 1e-5            # dn, relative: measured 1.3e-8
GATE_GRAD = 2e-5          # rel-norm per raw parameter group: measured 7.2e-6 (xyz, b, anti-aliased); 3.9 without the D-bar path
# planar payoff (300 steps, 3 x 3000 Gaussians, no depth or normal target): angle error measured 46.5 deg (colour only) -> 12.8 deg
# (colour + dn), PSNR 36.96 -> 36.41 dB on the held-out views
GATE_ANGLE_RATIO = 0.5
GATE_PSNR_DROP = 1.0


def _planes(tr, c, dev):
    H, W = c["H"], c["W"]
    D, A, N = torch.empty((H, W), device=dev), torch.empty((H, W), device=dev), torch.empty((3, H, W), device=dev)
    img = torch.empty((3, H, W), device=dev)
    tr.render(c, img, out_depth=D, out_alpha=A, out_normal=N)
    return img, D, A, N


def _mask(H, W, dev, seed=11):
    gen = torch.Generator().manual_seed(seed)
    return (torch.rand((H, W), generator=gen) > 0.25).float().to(dev).contiguous()


@pytest.mark.parametrize("name", ["a", "b"])
def test_depth_normal_equals_normals_from_depth(cuda, name):
    from photo_slam_b200 import trainer
    cam, sc = _settled(name)
    c = syn.device_camera(cam, cuda)
    tr = trainer.GaussianTrainer(_model(sc, cuda))
    tr.render(c)
    _, D, A, N = _planes(tr, c, cuda)
    nd = torch.full((3, c["H"], c["W"]), -7.0, device=cuda)
    trainer._dn_loss(c, D, A, N, lambda_dn=LAMBDA_DN, alpha_min=ALPHA_MIN, max_rel_jump=JUMP, out_depth_normal=nd)
    ref = trainer.normals_from_depth(c, torch.where(A >= ALPHA_MIN, D / A, torch.zeros_like(D)).contiguous(), JUMP)
    torch.cuda.synchronize()
    valid = int((nd != 0).any(0).sum())
    print(f"MEASURED depth normal {name}: {valid} valid pixels of {c['W'] * c['H']}, bit-identical {torch.equal(nd, ref)}")
    assert valid > 100 and torch.equal(nd, ref)


@pytest.mark.parametrize("name,with_mask", [("a", False), ("b", False), ("b", True)])
def test_loss_planes_against_float64(cuda, name, with_mask):
    from photo_slam_b200 import trainer
    cam, sc = _settled(name)
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    tr = trainer.GaussianTrainer(_model(sc, cuda))
    tr.render(c)
    _, D, A, N = _planes(tr, c, cuda)
    mask = _mask(H, W, cuda) if with_mask else None
    # the planes are added into: start from a known offset
    base = [torch.full_like(D, 0.25), torch.full_like(A, -0.5), torch.full_like(N, 0.125)]
    nd = torch.empty_like(N)
    dn, nv, grads = trainer._dn_loss(c, D, A, N, mask, LAMBDA_DN, ALPHA_MIN, JUMP, grads=[b.clone() for b in base], out_depth_normal=nd)
    torch.cuda.synchronize()
    Dt, At, Nt = (x.double().requires_grad_(True) for x in (D, A, N))
    dn_ref, nv_ref, nd_ref = dn64.dn64(Dt, At, Nt, W, H, float(c["tanfovx"]), float(c["tanfovy"]), ALPHA_MIN, JUMP, mask)
    assert torch.equal((nd != 0).any(0), (nd_ref != 0).any(0)), "the valid pixels differ from float64's"
    (LAMBDA_DN * dn_ref).backward()
    errs = {k: _relnorm(g - b, r.grad) for k, g, b, r in zip(("D", "A", "N"), grads, base, (Dt, At, Nt))}
    rel_dn = abs(dn - float(dn_ref.detach())) / float(dn_ref.detach())
    print(f"MEASURED loss planes {name} mask={with_mask}: N_valid {nv}, dn rel {rel_dn:.3g}, {errs}")
    assert nv == nv_ref > 100 and rel_dn < GATE_DN
    assert all(v < GATE_PLANES for v in errs.values()), errs


@pytest.mark.parametrize("name,aa", [("a", False), ("b", True)])
def test_raw_gradients_against_autograd(cuda, name, aa):
    from photo_slam_b200 import trainer
    from photo_slam_b200.parallel import GradBuffer
    cam, sc = _settled(name)
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m, antialiasing=aa, deterministic=True)
    tr._apply_deterministic()
    tr.render(c)
    _, D, A, N = _planes(tr, c, cuda)
    _, nv, (gd, ga, gn) = trainer._dn_loss(c, D, A, N, None, 1.0, ALPHA_MIN, JUMP)
    buf = GradBuffer(m.num_points(), cuda)
    tr.backwardPixels(torch.zeros((3, H, W), device=cuda), gd, ga, grads=buf.views(), dL_dnormal=gn)
    torch.cuda.synchronize()
    kern = [g.clone() for g in buf.views()]

    def truth(detach_dbar):
        raw = {k: v.requires_grad_(True) for k, v in s64.raw64(sc, cuda).items()}
        out, N64 = normal64.render_normal(raw, s64.camera64(cam, cuda), D=1, aa=aa)
        D64, A64 = out["depth"], out["alpha"]
        if detach_dbar:
            D64, A64 = D64.detach(), A64.detach()
        dn, _, _ = dn64.dn64(D64, A64, N64, W, H, float(c["tanfovx"]), float(c["tanfovy"]), ALPHA_MIN, JUMP)
        dn.backward()
        errs = {}
        for k, g in zip(s64.RAW, kern):
            ref = raw[k].grad if raw[k].grad is not None else torch.zeros_like(raw[k])
            if k == "features_rest":
                ref = ref[:, :3]
                g = g.reshape(ref.shape[0], 15, 3)[:, :3]
            errs[k] = _relnorm(g.reshape(ref.shape), ref)
        return errs

    errs = truth(False)
    print(f"MEASURED raw gradients {name} aa={aa}: N_valid {nv}, {errs}")
    assert all(v < GATE_GRAD for v in errs.values()), errs
    # without the D-bar path (only N carries the term) the position gradient misses the gate
    errs2 = truth(True)
    print(f"MEASURED raw gradients without the D-bar path {name} aa={aa}: {errs2}")
    assert errs2["xyz"] > 10 * GATE_GRAD


def test_builtin_step_equals_the_split_path_bit_for_bit(cuda):
    from photo_slam_b200 import trainer
    cam, sc = _settled("b")
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    gt, mask, gd_t, gn_t = _targets(H, W, cuda)
    runs, vals = [], []
    for path in ("builtin", "pixels"):
        m = _model(sc, cuda)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        tr.opt.lambda_dssim = LAMBDA_DSSIM
        tr.render(c)
        imgs = []
        for it in range(8):
            msk = mask if it % 2 == 0 else None
            img, nd = torch.empty((3, H, W), device=cuda), torch.empty((3, H, W), device=cuda)
            if path == "builtin":
                tr.trainForOneIteration(c, gt, msk, out_color=img, gt_depth=gd_t, lambda_depth=LAMBDA_DEPTH, gt_normal=gn_t,
                                        lambda_normal=LAMBDA_NORMAL, lambda_dn=LAMBDA_DN, dn_alpha_min=ALPHA_MIN, dn_max_rel_jump=JUMP,
                                        out_depth_normal=nd)
                vals.append(tr.result_dn()[5])
            else:
                D, A, N = torch.empty((H, W), device=cuda), torch.empty((H, W), device=cuda), torch.empty((3, H, W), device=cuda)
                tr.render(c, img, check=False, out_depth=D, out_alpha=A, out_normal=N)
                _, _, _, g = trainer.fused_loss(img, gt, msk, LAMBDA_DSSIM)
                vd, vn = gd_t > 0, (gn_t != 0).any(0)
                if msk is not None:
                    vd, vn = vd & (msk[0] != 0), vn & (msk[0] != 0)
                grads = (_grad_of_l1(D, gd_t, vd, LAMBDA_DEPTH), torch.zeros_like(A), _grad_of_l1(N, gn_t, vn, LAMBDA_NORMAL))
                dn, _, grads = trainer._dn_loss(c, D, A, N, msk[0].contiguous() if msk is not None else None, LAMBDA_DN, ALPHA_MIN, JUMP,
                                                grads=grads, out_depth_normal=nd)
                vals.append(dn)
                tr.backwardPixels(g, grads[0], grads[1], dL_dnormal=grads[2])
                tr.result()
            imgs.append((img, nd))
        torch.cuda.synchronize()
        runs.append((imgs, _state(m)))
    for (a, na), (b, nb) in zip(runs[0][0], runs[1][0]):
        assert torch.equal(a, b) and torch.equal(na, nb)
    assert _same(runs[0][1], runs[1][1])
    for k, s in zip(vals[:8], vals[8:]):
        assert abs(k - s) <= 1e-6 * abs(s), (k, s)
    print(f"MEASURED dn built-in vs psb_dn_loss: {list(zip(vals[:2], vals[8:10]))}")


def test_null_dn_is_the_normal_step(cuda):
    from photo_slam_b200 import _lib, trainer
    cam, sc = _settled("a")
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    gt, mask, gd, gn = _targets(H, W, cuda)
    states = []
    for fn in ("psb_trainer_step_normal", "psb_trainer_step_dn"):
        m = _model(sc, cuda)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        tr._apply_deterministic()
        tr.render(c)
        for it in range(3):
            cm, cc, cs = m._cmodel(live=m.adamLive()), trainer._ccamera(c), tr._cstep(True)
            d = trainer._Depth(gd.data_ptr(), LAMBDA_DEPTH, None)
            nrm = trainer._Normal(gn.data_ptr(), LAMBDA_NORMAL, None)
            args = (*tr._call_args(m, cm, cc, cs, gt, mask, None, None), C.byref(d), None, C.byref(nrm))
            stream = torch.cuda.current_stream().cuda_stream
            rc = tr.L.psb_trainer_step_normal(*args, stream) if fn.endswith("normal") else tr.L.psb_trainer_step_dn(*args, None, stream)
            _lib.check(rc, fn)
            m.step_ += 1
            tr.result()
        torch.cuda.synchronize()
        states.append(_state(m))
    assert _same(states[0], states[1])


@pytest.mark.parametrize("mode", ["plain", "aa", "f3d"])
def test_dn_steps_bit_identical_run_to_run(cuda, mode):
    from photo_slam_b200 import trainer
    cam, sc = _settled("b")
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    gt, mask, _, _ = _targets(H, W, cuda)
    runs = []
    for _ in range(2):
        m = _model(sc, cuda)
        if mode == "f3d":
            _filter(m, c)
        tr = trainer.GaussianTrainer(m, deterministic=True, antialiasing=mode == "aa", filter3d=mode == "f3d")
        res = []
        for it in range(20):
            tr.trainForOneIteration(c, gt, mask if it % 2 else None, lambda_dn=LAMBDA_DN)
            res.append(tr.result_dn())
        torch.cuda.synchronize()
        runs.append((repr(res), _state(m)))
    assert runs[0][0] == runs[1][0]
    assert _same(runs[0][1], runs[1][1])


def test_overflowing_dn_step_is_repeated_with_its_term(cuda):
    """A: the first step overflows the initial binning arena and result_dn() repeats it with its term; B: a render grows the arena first.
    Same model state and dn either way."""
    from helpers import scene_tensors
    from photo_slam_b200 import trainer
    wh = (640, 480)
    cam, sc, act, g, c = scene_tensors(2_000, "tum", seed=2, pose_seed=None, dev=cuda, wh=wh, scale_px=150.0)  # ~100s of tiles per Gaussian
    gt, _, _, _ = _targets(wh[1], wh[0], cuda)
    runs = []
    for pregrow in (False, True):
        m = _model(sc, cuda)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        if pregrow:
            tr.render(c)
        tr.trainForOneIteration(c, gt, lambda_dn=LAMBDA_DN)
        res = tr.result_dn()
        ov = tr._overflow_info()
        torch.cuda.synchronize()
        assert res[6] > 6 * 2_000 + 65536, "the view must overflow the initial arena"
        assert m.step_ == 1 and tr.iteration == 1 and ov[1] == 1 and res[5] > 0
        runs.append((res, _state(m)))
    assert repr(runs[0][0]) == repr(runs[1][0])
    assert _same(runs[0][1], runs[1][1])


def test_refusals_leave_the_model_untouched(cuda):
    from photo_slam_b200 import _lib, trainer
    cam, sc = _settled("a")
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    gt, _, _, gn = _targets(H, W, cuda)
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m)
    tr.trainForOneIteration(c, gt, lambda_dn=LAMBDA_DN)
    tr.result()
    before = _state(m)
    for kw in (dict(lambda_dn=-1.0), dict(lambda_dn=math.nan), dict(lambda_dn=math.inf), dict(lambda_dn=0.05, dn_alpha_min=0.0),
               dict(lambda_dn=0.05, dn_alpha_min=1.5), dict(lambda_dn=0.05, dn_max_rel_jump=0.0), dict(lambda_dn=0.05, dn_max_rel_jump=math.inf),
               dict(lambda_dn=0.05, gt_normal=gn, lambda_normal=0.0)):
        with pytest.raises(_lib.PsbError, match="psb_trainer_step_dn"):
            tr.trainForOneIteration(c, gt, **kw)
    torch.cuda.synchronize()
    assert _same(before, _state(m))


def test_planar_scene_payoff(cuda):
    from dn_bench import planar_payoff
    res = planar_payoff(cuda, per_wall=3000, steps=300, lambda_dn=LAMBDA_DN)
    print(f"MEASURED planar payoff: {res}")
    c, d = res["colour"], res["colour+dn"]
    assert d["angle"] < GATE_ANGLE_RATIO * c["angle"], res
    assert d["psnr"] > c["psnr"] - GATE_PSNR_DROP, res
