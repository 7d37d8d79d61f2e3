"""-m gpu: depth distortion (include/psb200.h, "Depth distortion").

  1. the second depth moment M of psb_trainer_forward_moment matches tests/dist64.py on settled scenes, plain, anti-aliased and with the
     3D filter, and colour, D, A, N, radii, final T and the last blended Gaussian equal the pass without M bit for bit;
  2. backwardPixels with colour, depth, opacity and moment gradients matches autograd on the float64 restatement per raw parameter group,
     plain and anti-aliased; without dM/dz (the 2 z dL/dM of the depth sum) in the truth the position gradient misses the gate;
  3. result_dist() matches dist64 on the float64 planes of a settled scene whose walls stand at z ~ 5 (the A M - D^2 cancellation);
  4. the built-in step, alone and with depth + normal + consistency terms, equals forward_moment + psb_loss + the other terms' gradients
     + the distortion planes formed in torch float32 + backwardPixels bit for bit over 8 deterministic steps;
  5. dist == NULL is psb_trainer_step_dn bit for bit; 20 deterministic steps with the term repeat bit for bit, plain, anti-aliased and
     3D-filtered;
  6. an overflowing step is repeated with its term; the refusals, a dL/dM after a pass without the plane included, leave the model
     untouched;
  7. on the planar payoff scene the term lowers the held-out depth spread below a measured fraction of the colour-only run's, without
     growing the depth error, with PSNR within 1 dB.
"""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import torch

import contrib64
import dist64
import filter3d64 as f3d64
import photo_slam_b200.synthetic as syn
import splat64 as s64
from test_normal_gpu import _debug, _filter, _grad_of_l1, _model, _relnorm, _same, _settled, _state, _targets

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
pytestmark = pytest.mark.gpu
LAMBDA_DSSIM, LAMBDA_DEPTH, LAMBDA_NORMAL, LAMBDA_DN, LAMBDA_DIST = 0.2, 0.1, 0.05, 0.05, 1.0
ALPHA_MIN, JUMP = 0.5, 0.05
# Measured on an H100 80GB HBM3 (700 W).
GATE_MOMENT = 2e-5        # max |M - M64| / max(M64, 1): measured 3.0e-6 (scene b, plain)
GATE_GRAD = 2e-5          # rel-norm per raw parameter group: measured 1.9e-6 (xyz, scene a); 2.5e-3 (xyz, b) without dM/dz
# result_dist() against dist64 of the float64 planes, relative: measured 4.5e-5 at D / A ~ 5.05 and a median spread of 0.078 m, where
# the A M - D^2 cancellation bound eps (D / A / spread)^2 is 2.5e-4
GATE_DIST = 2e-4
# planar payoff (300 steps, 3 x 3000 Gaussians, colour only) on the held-out views: depth spread 0.117 m (colour) -> 0.059 m (colour +
# dist at lambda 1), |D / A - D_true| 0.052 -> 0.050 m, PSNR 36.01 -> 36.27 dB
GATE_SPREAD_RATIO = 0.7
GATE_PSNR_DROP = 1.0


def _planes(tr, c, dev, normal=False, depth=True):
    H, W = c["H"], c["W"]
    img, D, A, M = (torch.empty((3, H, W), device=dev), torch.empty((H, W), device=dev) if depth else None, torch.empty((H, W), device=dev),
                    torch.empty((H, W), device=dev))
    N = torch.empty((3, H, W), device=dev) if normal else None
    tr.render(c, img, out_depth=D, out_alpha=A, out_normal=N, out_depth2=M)
    return img, D, A, N, M


def _dist_planes32(D, A, M, valid, lam, gD, gA):
    """the distortion's gradient planes as the kernel forms them, in torch float32: k = lam / max(N_valid, 1) (float32), gA + k M and
    gD + (-2k) D on valid pixels, dL/dM = k A there and 0 elsewhere"""
    k = torch.tensor(lam, dtype=torch.float32, device=D.device) / torch.tensor(float(max(int(valid.sum()), 1)), dtype=torch.float32, device=D.device)
    m2k = -2.0 * k
    gA = torch.where(valid, gA + k * M, gA)
    gD = torch.where(valid, gD + m2k * D, gD)
    gM = torch.where(valid, k * A, torch.zeros_like(A))
    return gD.contiguous(), gA.contiguous(), gM.contiguous()


_F3D = {}


def _settled_f3d(name):
    """_settled(name) settled again on the splats the 3D filter widens (contrib64.settle), so that the filtered pass's decisions keep
    their margin too"""
    if name not in _F3D:
        cam, sc = _settled(name)
        sc = {k: v.copy() for k, v in sc.items()}
        packed = np.concatenate([np.asarray(cam["viewmatrix"], np.float64).reshape(-1),
                                 [cam["W"] / (2 * float(cam["tanfovx"])), cam["H"] / (2 * float(cam["tanfovy"])), cam["W"], cam["H"]]])[None]
        contrib64.settle(sc, [cam], D=1, f_of=lambda xyz: f3d64.filter3d(xyz, packed)["filter"], seed=2)
        _F3D[name] = (cam, sc)
    return _F3D[name]


@pytest.mark.parametrize("name,mode", [(n, md) for n in ("a", "b") for md in ("plain", "aa", "f3d")])
def test_moment_plane_against_truth(cuda, name, mode):
    from photo_slam_b200 import trainer
    cam, sc = _settled_f3d(name) if mode == "f3d" else _settled(name)
    c = syn.device_camera(cam, cuda)
    W, H, P = c["W"], c["H"], sc["xyz"].shape[0]
    m = _model(sc, cuda)
    if mode == "f3d":
        _filter(m, c)
    tr = trainer.GaussianTrainer(m, antialiasing=mode == "aa", filter3d=mode == "f3d")
    tr.render(c)
    outs = []
    for with_m in (False, True, "no_depth"):
        img, rad = torch.empty((3, H, W), device=cuda), torch.zeros(P, dtype=torch.int32, device=cuda)
        D, A = torch.full((H, W), -7.0, device=cuda), torch.full((H, W), -7.0, device=cuda)
        N = torch.full((3, H, W), -7.0, device=cuda)
        M = torch.full((H, W), -7.0, device=cuda) if with_m else None
        tr.render(c, img, rad, out_depth=D if with_m != "no_depth" else None, out_alpha=A, out_normal=N, out_depth2=M)
        outs.append((img, rad, D, A, N, *_debug(tr, W, H, cuda), M))
    torch.cuda.synchronize()
    for x, y in zip(outs[0][:7], outs[1][:7]):
        assert torch.equal(x, y)
    assert torch.equal(outs[1][7], outs[2][7]) and (outs[2][2] == -7.0).all()     # M without D: the same M, D not written
    M = outs[1][7]
    raw = s64.raw64(sc, cuda)
    g = contrib64.filtered(raw, m.filter3D().detach().double().cpu().numpy()) if mode == "f3d" else s64.activate(raw)
    _, M64 = dist64.render_moment(g, s64.camera64(cam, cuda), D=1, aa=mode == "aa", raw=False)
    err = float(((M.double() - M64).abs() / M64.clamp_min(1.0)).max())
    print(f"MEASURED moment plane {name} {mode}: max rel err {err:.3g}, M max {float(M64.max()):.3g}")
    assert (M64 > 1.0).any() and err < GATE_MOMENT


@pytest.mark.parametrize("name,aa", [("a", False), ("b", True)])
def test_raw_gradients_against_autograd(cuda, name, aa):
    from photo_slam_b200 import trainer
    from photo_slam_b200.parallel import GradBuffer
    cam, sc = _settled(name)
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    gen = torch.Generator().manual_seed(8)
    wc, wd, wa, wm = (torch.rand((3, H, W), generator=gen) - 0.5, 0.2 * (torch.rand((H, W), generator=gen) - 0.5),
                      torch.rand((H, W), generator=gen) - 0.5, 0.02 * (torch.rand((H, W), generator=gen) - 0.5))
    wc, wd, wa, wm = (x.to(cuda).contiguous() for x in (wc, wd, wa, wm))
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m, antialiasing=aa, deterministic=True)
    tr._apply_deterministic()
    tr.render(c)
    _planes(tr, c, cuda)
    buf = GradBuffer(m.num_points(), cuda)
    tr.backwardPixels(wc, wd, wa, grads=buf.views(), dL_ddepth2=wm)
    torch.cuda.synchronize()
    kern = [g.clone() for g in buf.views()]

    def errs_against(keep_z_grad):
        raw = {k: v.requires_grad_(True) for k, v in s64.raw64(sc, cuda).items()}
        out, M64 = dist64.render_moment(raw, s64.camera64(cam, cuda), D=1, aa=aa, keep_z_grad=keep_z_grad)
        L = (out["color"] * wc.double()).sum() + (out["depth"] * wd.double()).sum() + (out["alpha"] * wa.double()).sum() + (M64 * wm.double()).sum()
        L.backward()
        errs = {}
        for k, g in zip(s64.RAW, kern):
            ref = raw[k].grad if raw[k].grad is not None else torch.zeros_like(raw[k])
            if k == "features_rest":
                ref = ref[:, :3]
                g = g.reshape(ref.shape[0], 15, 3)[:, :3]
            errs[k] = _relnorm(g.reshape(ref.shape), ref)
        return errs

    errs = errs_against(True)
    print(f"MEASURED raw gradients {name} aa={aa}: {errs}")
    assert all(v < GATE_GRAD for v in errs.values()), errs
    errs2 = errs_against(False)
    print(f"MEASURED raw gradients without dM/dz {name} aa={aa}: {errs2}")
    assert errs2["xyz"] > 10 * GATE_GRAD


_WALLS = {}


def _walls():
    """a settled planar scene seen head-on: the back wall at z = 5 and the trainee's layers around it (synthetic.distortion_trainee)"""
    if not _WALLS:
        W, H = 64, 48
        sc, normals = syn.planar_scene(120, seed=4)
        keep = normals[:, 2] < -0.5                  # the back wall only
        sc = syn.distortion_trainee({k: v[keep] for k, v in sc.items()}, normals[keep], seed=5)
        sc["scaling"][:] = np.log(np.float32([[0.25, 0.25, 0.02]]))
        cam = syn.make_camera(W, H, 0.7 * W, 0.7 * W, *syn.random_pose(np.random.default_rng(9), max_angle=0.05, max_trans=0.1))
        s64.settle(sc, cam, D=1, aa=None, bg=(0.0, 0.0, 0.0), seed=2, dev="cuda")
        _WALLS["s"] = (cam, sc)
    return _WALLS["s"]


def test_result_dist_against_float64(cuda):
    from photo_slam_b200 import trainer
    cam, sc = _walls()
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    gt, mask, _, _ = _targets(H, W, cuda)
    out64, M64 = dist64.render_moment(s64.raw64(sc, cuda), s64.camera64(cam, cuda), D=1)
    res = []
    for msk in (None, mask):
        tr = trainer.GaussianTrainer(_model(sc, cuda), deterministic=True)
        tr.render(c)
        D, A, M = torch.empty((H, W), device=cuda), torch.empty((H, W), device=cuda), torch.empty((H, W), device=cuda)
        tr.trainForOneIteration(c, gt, msk, out_depth=D, lambda_dist=LAMBDA_DIST, out_depth2=M)
        got = tr.result_dist()[6]
        ref, nv = dist64.dist64(out64["depth"], out64["alpha"], M64, msk)
        on_planes, _ = dist64.dist64(D.double(), 1.0 - _debug(tr, W, H, cuda)[1].reshape(H, W).double(), M.double(), msk)
        res.append((got, float(ref), float(on_planes), nv))
    sel = out64["alpha"] > 0.5
    print(f"MEASURED result_dist vs float64 (kernel, float64 planes, float64 of the kernel's planes, N_valid): {res}; "
          f"median D / A {float((out64['depth'][sel] / out64['alpha'][sel]).median()):.3g}, "
          f"median spread {float(dist64.spread64(out64['depth'], out64['alpha'], M64)[sel].median()):.3g}")
    for got, ref, _, nv in res:
        assert nv > 100 and ref > 0 and abs(got - ref) <= GATE_DIST * ref, res


@pytest.mark.parametrize("others", [False, True])
def test_builtin_step_equals_the_split_path_bit_for_bit(cuda, others):
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
            img, M = torch.empty((3, H, W), device=cuda), torch.empty((H, W), device=cuda)
            kw = dict(gt_depth=gd_t, lambda_depth=LAMBDA_DEPTH, gt_normal=gn_t, lambda_normal=LAMBDA_NORMAL, lambda_dn=LAMBDA_DN,
                      dn_alpha_min=ALPHA_MIN, dn_max_rel_jump=JUMP) if others else {}
            if path == "builtin":
                tr.trainForOneIteration(c, gt, msk, out_color=img, lambda_dist=LAMBDA_DIST, out_depth2=M, **kw)
                vals.append(tr.result_dist()[6])
            else:
                img, D, A, N, M = _planes(tr, c, cuda, normal=others)
                _, _, _, g = trainer.fused_loss(img, gt, msk, LAMBDA_DSSIM)
                valid = msk[0] != 0 if msk is not None else torch.ones((H, W), dtype=torch.bool, device=cuda)
                if others:
                    vd, vn = (gd_t > 0) & valid, (gn_t != 0).any(0) & valid
                    grads = (_grad_of_l1(D, gd_t, vd, LAMBDA_DEPTH), torch.zeros_like(A), _grad_of_l1(N, gn_t, vn, LAMBDA_NORMAL))
                    _, _, grads = trainer._dn_loss(c, D, A, N, msk[0].contiguous() if msk is not None else None, LAMBDA_DN, ALPHA_MIN, JUMP,
                                                   grads=grads)
                    gD, gA, gN = grads
                else:
                    gD, gA, gN = torch.zeros_like(D), torch.zeros_like(A), None
                gD, gA, gM = _dist_planes32(D, A, M, valid, LAMBDA_DIST, gD, gA)
                vals.append(float(dist64.dist64(D, A, M, msk)[0]))
                tr.backwardPixels(g, gD, gA, dL_dnormal=gN, dL_ddepth2=gM)
                tr.result()
            imgs.append((img, M))
        torch.cuda.synchronize()
        runs.append((imgs, _state(m)))
    for (a, ma), (b, mb) in zip(runs[0][0], runs[1][0]):
        assert torch.equal(a, b) and torch.equal(ma, mb)
    assert _same(runs[0][1], runs[1][1])
    for k, s in zip(vals[:8], vals[8:]):
        assert abs(k - s) <= 1e-6 * abs(s), (k, s)
    print(f"MEASURED dist built-in vs float64 of its planes (others={others}): {list(zip(vals[:2], vals[8:10]))}")


def test_null_dist_is_the_dn_step(cuda):
    from photo_slam_b200 import _lib, trainer
    cam, sc = _settled("a")
    c = syn.device_camera(cam, cuda)
    gt, mask, gd, gn = _targets(c["H"], c["W"], cuda)
    states = []
    for fn in ("psb_trainer_step_dn", "psb_trainer_step_dist"):
        m = _model(sc, cuda)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        tr._apply_deterministic()
        tr.render(c)
        for it in range(3):
            cm, cc, cs = m._cmodel(live=m.adamLive()), trainer._ccamera(c), tr._cstep(True)
            d = trainer._Depth(gd.data_ptr(), LAMBDA_DEPTH, None)
            nrm = trainer._Normal(gn.data_ptr(), LAMBDA_NORMAL, None)
            dn = trainer._Dn(LAMBDA_DN, ALPHA_MIN, JUMP, None)
            args = (*tr._call_args(m, cm, cc, cs, gt, mask, None, None), C.byref(d), None, C.byref(nrm), C.byref(dn))
            stream = torch.cuda.current_stream().cuda_stream
            rc = tr.L.psb_trainer_step_dn(*args, stream) if fn.endswith("dn") else tr.L.psb_trainer_step_dist(*args, None, stream)
            _lib.check(rc, fn)
            m.step_ += 1
            tr.result()
        torch.cuda.synchronize()
        states.append(_state(m))
    assert _same(states[0], states[1])


@pytest.mark.parametrize("mode", ["plain", "aa", "f3d"])
def test_dist_steps_bit_identical_run_to_run(cuda, mode):
    from photo_slam_b200 import trainer
    cam, sc = _settled("b")
    c = syn.device_camera(cam, cuda)
    gt, mask, _, _ = _targets(c["H"], c["W"], cuda)
    runs = []
    for _ in range(2):
        m = _model(sc, cuda)
        if mode == "f3d":
            _filter(m, c)
        tr = trainer.GaussianTrainer(m, deterministic=True, antialiasing=mode == "aa", filter3d=mode == "f3d")
        res = []
        for it in range(20):
            tr.trainForOneIteration(c, gt, mask if it % 2 else None, lambda_dist=LAMBDA_DIST)
            res.append(tr.result_dist())
        torch.cuda.synchronize()
        runs.append((repr(res), _state(m)))
    assert runs[0][0] == runs[1][0]
    assert _same(runs[0][1], runs[1][1])


def test_overflowing_dist_step_is_repeated_with_its_term(cuda):
    """A: the first step overflows the initial binning arena and result_dist() repeats it with its term; B: a render grows the arena
    first. Same model state and dist either way."""
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
        tr.trainForOneIteration(c, gt, lambda_dist=LAMBDA_DIST)
        res = tr.result_dist()
        ov = tr._overflow_info()
        torch.cuda.synchronize()
        assert res[7] > 6 * 2_000 + 65536, "the view must overflow the initial arena"
        assert m.step_ == 1 and tr.iteration == 1 and ov[1] == 1 and res[6] > 0
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
    tr.trainForOneIteration(c, gt, lambda_dist=LAMBDA_DIST)
    tr.result()
    before = _state(m)
    for kw in (dict(lambda_dist=-1.0), dict(lambda_dist=math.nan), dict(lambda_dist=math.inf), dict(lambda_dist=LAMBDA_DIST, lambda_dn=-1.0),
               dict(lambda_dist=LAMBDA_DIST, gt_normal=gn, lambda_normal=0.0)):
        with pytest.raises(_lib.PsbError, match="psb_trainer_step_dist"):
            tr.trainForOneIteration(c, gt, **kw)
    # a dL/dM after a pass that rendered no second moment: refused by the library (the front end refuses it before the call)
    tr.render(c, out_depth=torch.empty((H, W), device=cuda))
    cm, cc, cs = m._cmodel(live=m.adamLive()), trainer._ccamera(c), tr._cstep(True)
    z3, z1 = torch.zeros((3, H, W), device=cuda), torch.zeros((H, W), device=cuda)
    px = trainer._PixelGrads(z3.data_ptr(), z1.data_ptr(), None)
    rc = tr.L.psb_trainer_backward_pixels_moment(tr.h, tr._pass, m.num_points(), 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), C.byref(px),
                                                 None, z1.data_ptr(), C.byref(cs), None, torch.cuda.current_stream().cuda_stream)
    assert rc == -1 and b"psb_trainer_backward_pixels_moment" in tr.L.psb_last_error()
    with pytest.raises(ValueError, match="dL_ddepth2"):
        tr.backwardPixels(z3, z1, dL_ddepth2=z1)
    torch.cuda.synchronize()
    assert _same(before, _state(m))


def test_planar_scene_payoff(cuda):
    from dist_bench import distortion_payoff
    res = distortion_payoff(cuda, per_wall=3000, steps=300)
    print(f"MEASURED distortion payoff: {res}")
    c, d = res["colour"], res[f"colour+dist@{LAMBDA_DIST:g}"]
    assert d["spread"] < GATE_SPREAD_RATIO * c["spread"], res
    assert d["depth_err"] <= c["depth_err"], res
    assert d["psnr"] > c["psnr"] - GATE_PSNR_DROP, res
