"""-m gpu: the whole fused training step against the float64 step of tests/step64.py, in every flag set {depth, aa, reg, f3d, normal} of
each base of gaussian_backward_kernel<MODE> (psb_train.cu), followed by frest_stream_kernel.

Instantiations and the cases that run them (flag set k: depth = bit 0, aa = bit 1, reg = bit 2, f3d = bit 3, normal = bit 4):

  MODE_ADAM_LIVE | flags(k), k = 0..31   test_live_trajectory[k]: six steps of trainForOneIteration (adam_live given)
  MODE_ADAM      | flags(k), k = 0..31   test_adam_step[k]: one psb_trainer_step_exposure / _normal with adam_live = NULL
  MODE_GRADS     | flags(k), k = 0..31   test_grads_step[k]: one backwardPixels(grads=...) fed the truth's per-pixel gradients
  MODE_PUSH      | {depth, aa}            test_dp_step[p2p-*]: one DataParallelTrainer(mode="p2p") step at world 1 for each of +-depth and
                                         +-aa (the rank pushes into its own inbox; shard_adam_small_kernel and shard_adam_frest_kernel
                                         apply Adam on the owner side, the P * 45 tail element by element)
  adam_kernel, adam_tail_kernel          test_dp_step[slabs-*]: one step of the slab pipeline at world 1 (gaussian_backward_kernel<MODE_GRADS>
                                         per slab, then psb_adam_flat per slab and tensor; P = 1537 and 1539 leave scalar tails)

Scene of case k: k even -> "terminate" (P = 1537 = 1 mod 4: pixels whose T crosses 1e-4 inside a later 128-entry batch), k odd -> "clamp"
(P = 1539 = 3 mod 4: rows whose alpha reaches the 0.99 clamp). Both hold rows behind the camera and rows outside every view. Deterministic
mode: on when k has an even number of set bits, so that each base runs both tile-backward paths.

A trajectory: three cameras in turn, a mask, a depth target with holes, a normal target with zeros, exposure rows 0 and 1 alternating, the
SH degree raised from 1 to 2 before step 3, non-zero moments on the even rows (unseen rows included) and zero moments on the odd rows,
opt.mcmc with mcmc_noise_lr = 0 for the sets with reg. Before every step the live model is settled (splat64's rule and step64's margins:
the xyz and opacity of offending rows jittered, their log-scales for the normal's axis), read into float64, stepped by the kernels and by
step64, and compared: every step starts from the kernels' own state, so errors do not compound.

Gates: measured on an H100 80GB HBM3 (700 W power limit) over all cases; the largest measured value sits in the comment beside each. The
whole file ran in 3 minutes there.
"""
import ctypes as C
import dataclasses
import math

import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn
import splat64 as s64
import step64

pytestmark = pytest.mark.gpu

W, H = 64, 48
LAMBDA_DEPTH, LAMBDA_NORMAL = 0.1, 0.05
E_ROWS = [[[1.3, 0.1, -0.08, 0.05], [0.04, 0.7, 0.09, -0.06], [-0.07, 0.05, 1.2, 0.03]],
          [[0.9, -0.05, 0.04, -0.02], [0.03, 1.1, -0.06, 0.04], [0.05, -0.04, 0.95, -0.05]]]
STEPS = 6
TINY = 1e-3               # the permitted exclusion: Adam's step of an element whose g and sqrt(v) are below TINY max|g| of its group

GATE_LOSS = 1e-5          # loss scalars, relative: measured 3.6e-6 (ssim)
GATE_STEP = 1e-5          # (|kernel - truth| - one float32 spacing) / lr, per group and for the exposure row, one step from seeded moments:
                          # measured 3.7e-6 (scaling)
GATE_STEP_TRAJ = 1e-4     # the same along a trajectory: measured 3.1e-5 (rotation). Moments made by earlier steps can be far smaller than
                          # the group's gradients, which scales the gradient's float32 error up in Adam's ratio
GATE_MOM = 4e-5           # moments, rel-norm per group: measured 7.5e-7 (xyz); the exposure row's second moment 1.4e-5
GATE_ACCUM = 1e-5         # xyz_gradient_accum: max element error / max element: measured 2.6e-6
GATE_GRAD = 1e-5          # GRADS legs: rel-norm per group: measured 1.3e-6 (xyz)
GATE_GRAD_MAX = 1e-5      # GRADS legs: max element error / max element, per group: measured 2.2e-6 (xyz)
GATE_EXCLUDED = 0.01      # excluded elements, fraction of their group


def _bits(k):
    return bin(k).count("1")


def _det(k):
    return _bits(k) % 2 == 0


# ---- scenes -------------------------------------------------------------------------------------------------------------------------
def _cams():
    f = 0.9 * W
    rot = lambda ax, a: syn.make_camera(W, H, f, f, *_pose(ax, a))
    return [syn.make_camera(W, H, f, f), rot(1, 0.03), rot(0, -0.025)]


def _pose(axis, ang):
    R = np.eye(3)
    c, s = math.cos(ang), math.sin(ang)
    i, j = [(1, 2), (0, 2), (0, 1)][axis]
    R[i, i], R[j, j], R[i, j], R[j, i] = c, c, -s, s
    return R, np.array([0.02 * axis, -0.015, 0.01])


def _random(P, cam, seed, scale_px, zr=(0.6, 8.0)):
    rng = np.random.default_rng(seed)
    fx = W / (2.0 * float(cam["tanfovx"]))
    z = zr[0] * (zr[1] / zr[0]) ** ((rng.permutation(P) + rng.uniform(0.3, 0.7, P)) / P)
    u, v = rng.uniform(-0.1 * W, 1.1 * W, P), rng.uniform(-0.1 * H, 1.1 * H, P)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return dict(xyz=f32(np.stack([(u - 0.5 * (W - 1)) / fx * z, (v - 0.5 * (H - 1)) / fx * z, z], 1)),
                features_dc=f32(((rng.uniform(0, 1, (P, 3)) - 0.5) / s64.SH_C0)[:, None]), features_rest=f32(rng.normal(0, 0.1, (P, 15, 3))),
                scaling=f32(np.log(scale_px / fx * z)[:, None] + rng.normal(0, 0.4, (P, 3))), rotation=f32(rng.normal(size=(P, 4))),
                opacity=f32(rng.normal(0.0, 1.5, (P, 1))))


def _unseen(sc, n=24):
    """the last n rows: half behind every camera, half far outside every view"""
    sc["xyz"][-n:-n // 2, 2] = -np.abs(sc["xyz"][-n:-n // 2, 2])
    sc["xyz"][-n // 2:, 0] = 4.0 * np.abs(sc["xyz"][-n // 2:, 2]) + 1.0


def _terminate():
    cam = _cams()[0]
    sc = _random(1537, cam, seed=12, scale_px=5.0)
    sc["opacity"][:] = np.abs(sc["opacity"]) + 0.5
    right = sc["xyz"][:, 0] / sc["xyz"][:, 2] > 0.6 * float(cam["tanfovx"])
    sc["xyz"][right, 2] *= -1.0
    _unseen(sc)
    return sc


def _clamp():
    cam = _cams()[0]
    sc = _random(1539, cam, seed=5, scale_px=3.0)
    rng = np.random.default_rng(5)
    fx = W / (2.0 * float(cam["tanfovx"]))
    for i in range(12):       # o = 0.9975 over a 10 px splat: alpha reaches 0.99 near its centre, with anti-aliasing too
        u, v, z = rng.integers(5, W - 5) + 0.05, rng.integers(5, H - 5) + 0.05, 0.7 + 0.01 * i
        sc["xyz"][i] = [(u - 0.5 * (W - 1)) / fx * z, (v - 0.5 * (H - 1)) / fx * z, z]
        sc["scaling"][i] = np.log(10.0 / fx * z)
        sc["rotation"][i] = [1.0, 0.0, 0.0, 0.0]
        sc["opacity"][i] = 6.0
    _unseen(sc)
    return sc


SCENES = {"terminate": _terminate, "clamp": _clamp}


def _targets(dev, seed=3):
    gen = torch.Generator().manual_seed(seed)
    gt = torch.rand((3, H, W), generator=gen)
    mask = (torch.rand((1, H, W), generator=gen) > 0.2).float().expand(3, H, W).contiguous()
    gd = 0.5 + 6 * torch.rand((H, W), generator=gen)
    gd[torch.rand((H, W), generator=gen) < 0.2] = 0.0
    n = torch.randn((3, H, W), generator=gen)
    n = n / n.norm(dim=0, keepdim=True)
    n[2] = -n[2].abs()
    n[:, torch.rand((H, W), generator=gen) < 0.2] = 0.0
    return dict(gt=gt.to(dev), mask=mask.to(dev), depth=gd.to(dev), normal=n.contiguous().to(dev))


def _targets64(t, bg):
    return dict(gt=t["gt"].double(), mask=t["mask"].double(), depth=t["depth"].double(), normal=t["normal"].double(), bg=bg,
                lambda_depth=LAMBDA_DEPTH, lambda_normal=LAMBDA_NORMAL, lambda_dssim=0.2)


BG = (0.3, 0.5, 0.7)


# ---- the model ----------------------------------------------------------------------------------------------------------------------
def _read(m, fl, exposure_id):
    """the model's state -> step64's float64 state"""
    d = lambda t: t.detach().double().clone()
    k = exposure_id
    return dict(params={g: d(t) for g, t in zip(step64.GROUPS, m.tensors())}, m={g: d(t) for g, t in zip(step64.GROUPS, m.exp_avg_)},
                v={g: d(t) for g, t in zip(step64.GROUPS, m.exp_avg_sq_)}, accum=d(m.xyz_gradient_accum_), denom=d(m.denom_),
                max_radii=d(m.max_radii2D_), step=m.step_, lr=_lrs(), D=m.active_sh_degree_,
                f=d(m.filter_3D_) if fl.f3d else None, E=d(m.exposure_[k]), E_m=d(m.exposure_exp_avg_[k]), E_v=d(m.exposure_exp_avg_sq_[k]),
                E_step=int(m.exposure_step_[k]), E_lr=float(m.exposure_lr_))


def _lrs():
    """the truth's learning rates, from the optimisation parameters themselves (spatial scale 1): f_rest at feature_lr / 20"""
    from photo_slam_b200 import trainer
    o = trainer.GaussianOptimizationParams()
    return [o.position_lr_init, o.feature_lr, o.feature_lr / 20.0, o.opacity_lr, o.scaling_lr, o.rotation_lr]


def _settle(m, st_fn, seed, tries=60, floor=s64.MIN_MARGIN):
    """jitter, in place, the xyz (~0.03 px) and opacity of every row that takes part in a decision closer than floor to its threshold
    (their log-scales for the normal's axis), until none does -> the smallest margin"""
    gen = torch.Generator(device=m.xyz_.device).manual_seed(seed)
    for _ in range(tries):
        mg = st_fn()
        axis = mg.pop("axis", None)
        bad = s64.offenders(mg, floor)
        bad_axis = axis[1][axis[0] < floor] if axis is not None else bad[:0]
        if not bad.numel() and not bad_axis.numel():
            return min(s64.min_margins(mg).values())
        if bad.numel():
            z = m.xyz_[bad].norm(dim=1, keepdim=True) + 0.1
            fx = 0.9 * W                # the cameras' focal length in pixels
            m.xyz_[bad] += 0.03 * z / fx * torch.randn((bad.numel(), 3), generator=gen, device=m.xyz_.device)
            m.opacity_[bad] += 0.02 * torch.randn((bad.numel(), 1), generator=gen, device=m.xyz_.device)
        if bad_axis.numel():
            m.scaling_[bad_axis] += 0.01 * torch.randn((bad_axis.numel(), 3), generator=gen, device=m.xyz_.device)
    raise AssertionError(f"the model did not settle: {s64.min_margins(mg)}")


def _model(sc, dev, fl, cams):
    from photo_slam_b200 import trainer
    m = trainer.GaussianModel.from_numpy({k: v.copy() for k, v in sc.items()}, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    m.setShDegree(1)
    m.ensureExposures(2)
    for k in range(2):
        m.exposure_[k] = torch.tensor(E_ROWS[k], device=dev)
    if fl.f3d:
        m.computeFilter3D([syn.device_camera(c, dev) for c in cams])
    return m


def _seed_moments(m, g64, gE):
    """moments of the size of the truth's gradient on the even rows (unseen ones included, through a floor), zero on the odd rows"""
    gen = torch.Generator(device=m.xyz_.device).manual_seed(7)
    gs, ms, vs = [g64[k] for k in step64.GROUPS], list(m.exp_avg_), list(m.exp_avg_sq_)
    if gE is not None:
        gs, ms, vs = gs + [gE], ms + [m.exposure_exp_avg_[0]], vs + [m.exposure_exp_avg_sq_[0]]
    for g, ma, va in zip(gs, ms, vs):
        rms = float(g.pow(2).mean().sqrt()) + 1e-30
        u = lambda: torch.rand(g.shape, device=g.device, generator=gen, dtype=torch.float64)
        ma.copy_((0.5 * g * (2 * u() - 1) + 0.05 * rms * (2 * u() - 1)).float())
        va.copy_((g * g * (0.5 + u()) + (0.1 * rms) ** 2).float())
        if ma.dim() > 1 and ma.shape[0] == m.num_points():
            ma[1::2] = 0.0
            va[1::2] = 0.0
    m.invalidateAdamLive()


def _trainer(m, fl, det):
    from photo_slam_b200 import trainer
    opt = trainer.GaussianOptimizationParams(mcmc=fl.reg, mcmc_noise_lr=0.0)
    return trainer.GaussianTrainer(m, opt, background=torch.tensor(BG, device=m.xyz_.device), deterministic=det, antialiasing=fl.aa,
                                   filter3d=fl.f3d)


def _relnorm(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return float((a - b).norm() / b.norm()) if b.norm() > 0 else float(a.norm())


def _maxerr(a, b):
    scale = float(b.abs().max()) if b.numel() else 0.0
    e = float((a.double() - b).abs().max()) if b.numel() else 0.0
    return e / scale if scale > 0 else e


def _step_err(p1, ref, lr, keep=None):
    p1 = p1.double()
    ulp = (torch.nextafter(p1.float(), torch.full_like(p1.float(), math.inf)).double() - p1).abs()
    e = ((p1 - ref).abs() - ulp).clamp_min(0)
    if keep is not None:
        e = e[keep]
    return float(e.max()) / lr if e.numel() else 0.0


# ---- comparison ---------------------------------------------------------------------------------------------------------------------
def _compare(m, before, r, fl, loss=None, live=False, exposure_id=0, step_gate=GATE_STEP):
    """the model after one kernel step against step64's result r (from `before`) -> errs; asserts the exact invariants"""
    nx = r["state"]
    errs, excluded = {}, {}
    if loss is not None:
        names = ["loss", "l1", "ssim"] + (["depth_l1"] if fl.depth else []) + (["normal_l1"] if fl.normal else [])
        for k, v in zip(("loss", "l1", "ssim", "depth_l1", "normal_l1"), loss):
            if k in names:
                t = r["loss"][k]
                errs[f"loss-{k}"] = abs(v - t) / abs(t)
    P = m.num_points()
    idle = torch.ones(P, dtype=torch.bool, device=m.xyz_.device)
    for i, k in enumerate(step64.GROUPS):
        p, ma, va = m.tensors()[i], m.exp_avg_[i], m.exp_avg_sq_[i]
        g = r["grads"][k]
        # Adam normalises: an element whose gradient and second moment are both below TINY max|g| of its group (a row reached for the first
        # time, or one whose only history is such gradients) steps by O(lr) at a ratio that float32 noise of the size of the group decides.
        # Those whose step misses the gate are gated on their moments only; they are counted
        gmax = float(g.abs().max())
        ill = (g.abs() < TINY * gmax) & (before["v"][k].sqrt() < TINY * gmax)
        p1 = p.detach().double()
        ulp = (torch.nextafter(p.detach(), torch.full_like(p.detach(), math.inf)).double() - p1).abs()
        miss = ((p1 - nx["params"][k]).abs() - ulp) > step_gate * before["lr"][i]
        tiny = ill & miss
        excluded[k] = int(tiny.sum())
        errs[f"step-{k}"] = _step_err(p.detach(), nx["params"][k], before["lr"][i], ~tiny)
        if errs[f"step-{k}"] > step_gate:
            e = ((p1 - nx["params"][k]).abs() * (~tiny)).reshape(-1)
            j = int(e.argmax())
            row = j // (g.numel() // P)
            f_ = lambda t: float(t.reshape(-1)[j])
            print(f"WORST {k} row={row} elem={j} kernel={f_(p.detach())} truth={f_(nx['params'][k])} before={f_(before['params'][k])} "
                  f"g={f_(g)} gmax={gmax} m0={f_(before['m'][k])} v0={f_(before['v'][k])} mk={f_(ma)} mt={f_(nx['m'][k])} "
                  f"vk={f_(va)} vt={f_(nx['v'][k])} reached={bool(r['reached'][row])} visible={bool(r['visible'][row])}")
        errs[f"mom-m-{k}"] = _relnorm(ma, nx["m"][k])
        errs[f"mom-v-{k}"] = _relnorm(va, nx["v"][k])
        assert excluded[k] <= GATE_EXCLUDED * g.numel(), (k, excluded[k], g.numel())
        idle &= (g.reshape(P, -1) == 0).all(1) & (before["m"][k].reshape(P, -1) == 0).all(1) & (before["v"][k].reshape(P, -1) == 0).all(1)
    if "E" in nx and r.get("E") is not None and exposure_id is not None:
        errs["step-exposure"] = _step_err(m.exposure_[exposure_id], nx["E"], before["E_lr"])
        errs["mom-m-exposure"] = _relnorm(m.exposure_exp_avg_[exposure_id], nx["E_m"])
        errs["mom-v-exposure"] = _relnorm(m.exposure_exp_avg_sq_[exposure_id], nx["E_v"])
    # statistics
    assert torch.equal(m.denom_.double(), nx["denom"]), "denom"
    assert torch.equal(m.max_radii2D_.double(), nx["max_radii"]), "max_radii2D"
    errs["accum"] = _maxerr(m.xyz_gradient_accum_, nx["accum"])
    # exact invariants: rows without gradient or moments keep parameters and moments; those the pass does not draw keep their statistics
    for i, k in enumerate(step64.GROUPS):
        for t, ref in ((m.tensors()[i], before["params"][k]), (m.exp_avg_[i], before["m"][k]), (m.exp_avg_sq_[i], before["v"][k])):
            assert torch.equal(t[idle].double(), ref[idle]), f"an idle row of {k} moved"
    hid = ~r["visible"]
    assert torch.equal(m.xyz_gradient_accum_[hid].double(), before["accum"][hid]) and torch.equal(m.denom_[hid].double(), before["denom"][hid])
    if live:
        nzm = torch.zeros(P, dtype=torch.bool, device=m.xyz_.device)
        for ma, va in zip(m.exp_avg_, m.exp_avg_sq_):
            nzm |= (ma.reshape(P, -1) != 0).any(1) | (va.reshape(P, -1) != 0).any(1)
        assert torch.equal(m.adam_live_.bool(), nzm), "the live byte is 'some moment of the row is non-zero'"
    return errs, excluded, int(idle.sum())


def _assert_gates(errs, step_gate=GATE_STEP):
    for k, v in errs.items():
        gate = {"loss": GATE_LOSS, "step": step_gate, "mom": GATE_MOM, "accum": GATE_ACCUM, "grad": GATE_GRAD, "gradmax": GATE_GRAD_MAX}[k.split("-")[0]]
        assert v < gate, (k, v, gate)


def _setup(k, dev):
    fl = step64.ALL_FLAGS[k]
    sc = SCENES["terminate" if k % 2 == 0 else "clamp"]()
    cams = _cams()
    tg = _targets(dev)
    tg64 = _targets64(tg, BG)
    m = _model(sc, dev, fl, cams)
    return fl, cams, tg, tg64, m


def _settled_state(m, fl, cam, tg64, seed, exposure_id=0):
    cam64 = s64.camera64(cam, m.xyz_.device)
    with torch.no_grad():
        mg = _settle(m, lambda: step64.margins(_read(m, fl, exposure_id), cam64, tg64, fl), seed)
    return _read(m, fl, exposure_id), cam64, mg


def _first_moments(m, fl, cam, tg64):
    """seed the moments from the truth's gradient of the first view"""
    st, cam64, _ = _settled_state(m, fl, cam, tg64, 0)
    g = step64.grads64(st, cam64, tg64, fl)
    _seed_moments(m, g["grads"], g["E"])


def _kernel_step(tr, m, c, tg, fl, exposure_id):
    tr.trainForOneIteration(c, tg["gt"], tg["mask"], gt_depth=tg["depth"] if fl.depth else None, lambda_depth=LAMBDA_DEPTH if fl.depth else 0.0,
                            exposure_id=exposure_id, gt_normal=tg["normal"] if fl.normal else None,
                            lambda_normal=LAMBDA_NORMAL if fl.normal else 0.0)
    out = tr.result_normal()
    torch.cuda.synchronize()
    return out[:5]


CASES = list(range(32))


@pytest.mark.parametrize("k", CASES, ids=[f"{k}-{step64.flag_name(step64.ALL_FLAGS[k])}" for k in CASES])
def test_live_trajectory(cuda, k):
    """MODE_ADAM_LIVE | flags(k): six anchored steps of trainForOneIteration against step64"""
    fl, cams, tg, tg64, m = _setup(k, cuda)
    _first_moments(m, fl, cams[0], tg64)
    tr = _trainer(m, fl, _det(k))
    worst, excl = {}, {}
    for i in range(STEPS):
        if i == 3:
            m.setShDegree(2)
        cam, e = cams[i % 3], i % 2
        st, cam64, mg = _settled_state(m, fl, cam, tg64, 100 * k + i, e)
        c = syn.device_camera(cam, cuda)
        loss = _kernel_step(tr, m, c, tg, fl, e)
        r = step64.step64(st, cam64, tg64, fl)
        errs, ex, nidle = _compare(m, st, r, fl, loss, live=True, exposure_id=e, step_gate=GATE_STEP_TRAJ)
        if i == 0:
            assert nidle > 0 and (~r["reached"]).sum() > 0
        for q, v in errs.items():
            worst[q] = max(worst.get(q, 0.0), v)
        for q, v in ex.items():
            excl[q] = excl.get(q, 0) + v
    print(f"MEASURED live {k} {step64.flag_name(fl)} det={_det(k)} margin={mg:.1e} excluded={excl} {worst}")
    _assert_gates(worst, GATE_STEP_TRAJ)


def _c_step(tr, m, c, tg, fl, exposure_id):
    """one psb_trainer_step_exposure / _normal with adam_live = NULL (MODE_ADAM)"""
    from photo_slam_b200 import _lib, trainer
    tr._hand_filter3d()
    tr._apply_deterministic()
    cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)
    d = trainer._Depth(tg["depth"].data_ptr(), LAMBDA_DEPTH, None) if fl.depth else None
    ex = trainer._Exposure(m.exposure_[exposure_id].data_ptr(), m.exposure_exp_avg_[exposure_id].data_ptr(),
                           m.exposure_exp_avg_sq_[exposure_id].data_ptr(), m.exposure_step_[exposure_id:].data_ptr(), float(m.exposure_lr_))
    args = (*tr._call_args(m, cm, cc, cs, tg["gt"], tg["mask"], None, None), C.byref(d) if d is not None else None, C.byref(ex))
    stream = torch.cuda.current_stream().cuda_stream
    if fl.normal:
        nrm = trainer._Normal(tg["normal"].data_ptr(), LAMBDA_NORMAL, None)
        _lib.check(tr.L.psb_trainer_step_normal(*args, C.byref(nrm), stream), "psb_trainer_step_normal")
    else:
        _lib.check(tr.L.psb_trainer_step_exposure(*args, stream), "psb_trainer_step_exposure")
    m.step_ += 1
    out, n = (C.c_float * 5)(), C.c_int()
    _lib.check(tr.L.psb_trainer_result_normal(tr.h, out, C.byref(n), stream), "psb_trainer_result_normal")
    torch.cuda.synchronize()
    return list(out)


@pytest.mark.parametrize("k", CASES, ids=[f"{k}-{step64.flag_name(step64.ALL_FLAGS[k])}" for k in CASES])
def test_adam_step(cuda, k):
    """MODE_ADAM | flags(k): one step through the C-ABI with adam_live = NULL (idle rows found by reading their moments)"""
    fl, cams, tg, tg64, m = _setup(k, cuda)
    _first_moments(m, fl, cams[1], tg64)
    tr = _trainer(m, fl, _det(k))
    st, cam64, mg = _settled_state(m, fl, cams[1], tg64, 7 * k)
    c = syn.device_camera(cams[1], cuda)
    tr.render(c)                     # sizes the binning arena
    loss = _c_step(tr, m, c, tg, fl, 0)
    r = step64.step64(st, cam64, tg64, fl)
    errs, ex, nidle = _compare(m, st, r, fl, loss, exposure_id=0)
    assert nidle > 0
    print(f"MEASURED adam {k} {step64.flag_name(fl)} det={_det(k)} margin={mg:.1e} excluded={ex} {errs}")
    _assert_gates(errs)


@pytest.mark.parametrize("k", CASES, ids=[f"{k}-{step64.flag_name(step64.ALL_FLAGS[k])}" for k in CASES])
def test_grads_step(cuda, k):
    """MODE_GRADS | flags(k): backwardPixels(grads=...) on the truth's per-pixel gradients -> the raw-parameter gradients (regularisers
    included) and the densification statistics"""
    fl, cams, tg, tg64, m = _setup(k, cuda)
    tr = _trainer(m, fl, _det(k))
    cam = cams[2]
    st, cam64, mg = _settled_state(m, fl, cam, tg64, 11 * k)
    r = step64.step64(st, cam64, tg64, fl)
    c = syn.device_camera(cam, cuda)
    N = torch.empty((3, H, W), device=cuda) if fl.normal else None
    tr.render(c, out_depth=torch.empty((H, W), device=cuda), out_normal=N)
    grads = [torch.zeros_like(t) for t in m.tensors()]
    px = r["pixel"]
    f32 = lambda t: t.float().contiguous()
    tr.backwardPixels(f32(px["color"]), f32(px["depth"]) if fl.depth else None, grads=grads, dL_dnormal=f32(px["normal"]) if fl.normal else None)
    tr.result()
    torch.cuda.synchronize()
    errs = {}
    n = (st["D"] + 1) ** 2 - 1
    for k_, a in zip(step64.GROUPS, grads):
        ref = r["grads"][k_]
        if k_ == "features_rest":
            assert not a[:, n:].any()
            a, ref = a[:, :n], ref[:, :n]
        errs[f"grad-{k_}"] = _relnorm(a, ref)
        errs[f"gradmax-{k_}"] = _maxerr(a, ref)
    for t, before in zip(m.tensors(), st["params"].values()):
        assert torch.equal(t.double(), before), "gradient mode leaves the parameters"
    nx = r["state"]
    assert torch.equal(m.denom_.double(), nx["denom"]) and torch.equal(m.max_radii2D_.double(), nx["max_radii"])
    errs["accum"] = _maxerr(m.xyz_gradient_accum_, nx["accum"])
    print(f"MEASURED grads {k} {step64.flag_name(fl)} det={_det(k)} margin={mg:.1e} {errs}")
    _assert_gates(errs)


def test_scenes_reach_their_edges(cuda):
    """terminate: pixels stop inside a later batch and others never stop; clamp: some blended alpha is clamped at 0.99; both: unseen rows"""
    for name in SCENES:
        fl = step64.Flags()
        m = _model(SCENES[name](), cuda, fl, _cams())
        tg64 = _targets64(_targets(cuda), BG)
        st, cam64, _ = _settled_state(m, fl, _cams()[0], tg64, 1)
        with torch.no_grad():
            out, _, _ = step64.forward(st["params"], cam64, fl, st["D"], BG)
        assert (out["radii"] == 0).sum() >= 24, name
        if name == "terminate":
            stp, nc = out["stopped"], out["n_contrib"]
            assert stp.any() and (~stp).any() and ((nc[stp] % 128 != 0) & (nc[stp] > 128)).any()
        else:
            assert out["clamped"].any()


# ---- the gates bite -----------------------------------------------------------------------------------------------------------------
PERTURB = {"eps": (dict(eps=1e-8), "step"), "no-bias-correction": (dict(bias_correction=False), "step"),
           "mean2d-pixels": (dict(mean2d_ndc=False), "accum"), "reg-all-rows": (dict(reg_reached_only=False), "step"),
           "f3d-without-c": (dict(f3d_opacity=False), "loss"), "normal-without-flip": (dict(normal_flip=False), "loss")}


@pytest.mark.parametrize("what", list(PERTURB))
def test_perturbed_truth_fails_the_gate(cuda, what):
    """one LIVE step with every flag on against a truth with one convention changed: the named gate family rejects it"""
    kw, family = PERTURB[what]
    k = 31
    fl, cams, tg, tg64, m = _setup(k, cuda)
    _first_moments(m, fl, cams[0], tg64)
    tr = _trainer(m, fl, True)
    st, cam64, _ = _settled_state(m, fl, cams[0], tg64, 5)
    loss = _kernel_step(tr, m, syn.device_camera(cams[0], cuda), tg, fl, 0)
    conv = dataclasses.replace(step64.STEP_CONV, **kw)
    r = step64.step64(st, cam64, tg64, fl, conv)
    nx = r["state"]
    if family == "accum":
        err = _maxerr(m.xyz_gradient_accum_, nx["accum"])
        gate = GATE_ACCUM
    elif family == "loss":
        err = max(abs(a - r["loss"][q]) / abs(r["loss"][q]) for a, q in zip(loss, ("loss", "l1", "ssim", "depth_l1", "normal_l1")))
        gate = GATE_LOSS
    else:
        err = max(_step_err(t.detach(), nx["params"][q], st["lr"][i]) for i, (q, t) in enumerate(zip(step64.GROUPS, m.tensors())))
        gate = GATE_STEP
    print(f"MEASURED perturbed {what}: {err:.2e} (gate {gate:.0e})")
    assert err > gate, f"{what}: the gate does not see the perturbation ({err} <= {gate})"


# ---- the data-parallel steps at world 1 ---------------------------------------------------------------------------------------------
DP_CASES = [("p2p", d, a) for d in (False, True) for a in (False, True)] + [("slabs", d, a) for d in (False, True) for a in (False, True)]


@pytest.mark.parametrize("mode,depth,aa", DP_CASES, ids=[f"{m}-{'depth' if d else 'nodepth'}-{'aa' if a else 'plain'}" for m, d, a in DP_CASES])
def test_dp_step(cuda, mode, depth, aa):
    """one DataParallelTrainer step at world 1 against step64 with {depth, aa} (the data-parallel steps take no exposure, regulariser or
    filter; their normal, consistency and distortion terms are checked in test_dp64_gpu): p2p runs gaussian_backward_kernel<MODE_PUSH |
    flags> and the owner-side Adam, the slab pipeline the per-slab gradient kernels and the flat Adam with its scalar tail"""
    from photo_slam_b200 import trainer
    fl = step64.Flags(depth=depth, aa=aa)
    k = int(depth) + 2 * int(aa)
    sc = SCENES["terminate" if mode == "p2p" else "clamp"]()
    cams = _cams()
    tg = _targets(cuda)
    tg64 = _targets64(tg, BG)
    m = _model(sc, cuda, fl, cams)
    st, cam64, _ = _settled_state(m, fl, cams[1], tg64, 31 + k)
    st["E"] = None
    g = step64.grads64(st, cam64, tg64, fl)
    _seed_moments(m, g["grads"], None)
    kw = dict(mode="p2p") if mode == "p2p" else dict(mode="nccl", pipeline=True, nslabs=3)
    tr = trainer.DataParallelTrainer(m, background=torch.tensor(BG, device=cuda), antialiasing=aa, **kw)
    assert tr.mode == kw["mode"] and (mode == "p2p" or tr.pipeline)
    c = syn.device_camera(cams[1], cuda)
    tr.render(c)                     # sizes the binning arena: an overflowing data-parallel step is dropped, not repeated
    st, cam64, mg = _settled_state(m, fl, cams[1], tg64, 41 + k)
    st["E"] = None
    tr.trainForOneIteration(c, tg["gt"], tg["mask"], gt_depth=tg["depth"] if depth else None, lambda_depth=LAMBDA_DEPTH if depth else 0.0)
    loss = tr.result_depth()[:4]
    if mode == "p2p":
        tr.sync()
    torch.cuda.synchronize()
    assert tr.dropped_views == 0 and (mode != "p2p" or tr.status() == 0)
    r = step64.step64(st, cam64, tg64, fl)
    errs, ex, nidle = _compare(m, st, r, fl, loss, exposure_id=None)
    assert nidle > 0
    if mode == "p2p":
        tr.close()
    print(f"MEASURED dp {mode} {step64.flag_name(fl)} margin={mg:.1e} excluded={ex} {errs}")
    _assert_gates(errs)
