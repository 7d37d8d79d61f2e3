"""-m gpu: the data-parallel steps with the normal, depth-normal consistency (dn) and distortion (dist) terms against the float64 step of
tests/step64.py, at world 1 on a DataParallelTrainer(geometry_terms=True):

  p2p    psb_dp_step_dist: gaussian_backward_kernel<MODE_PUSH | MODE_NORMAL [| MODE_DEPTH] [| MODE_AA]> (and MODE_PUSH | MODE_DEPTH
         [| MODE_AA] for dist alone, its dL/dz in slot 11 of the sink row) pushes each row's record into the rank's own inbox;
         shard_adam_small_kernel and shard_adam_frest_kernel apply Adam on the owner side;
  slabs  psb_trainer_backward_begin_dist -> psb_trainer_backward_slab x 3 -> psb_adam_flat per slab and tensor;
  flat   psb_trainer_backward_dist -> psb_adam_update over all P rows.

Each case is one step from a settled state (splat64's margins and step64's, the consistency term's alpha and depth-jump tests included)
with non-zero moments on the even rows, unseen rows included, checked against step64.step64 with the gates of test_step64_gpu: every
group's step and moments, the densification statistics, and the seven scalars of result_dist(). The scenes are test_step64_gpu's
"terminate" (P = 1537) and "clamp" (P = 1539) with rows inside the view moved into the partial last 128-row chunk, so that the chunk an
owner receives last, and the scalar tail of the flat Adam, hold rows the pass reaches. Deterministic mode alternates between cases.

Terms-only legs (p2p and slabs; normal alone and dist alone): the colour target is the kernel's own render and lambda_dssim = 0, so its
photometric gradient is exactly zero and the truth runs without the colour term; every row the pass reaches is reached through dL/dn or
dL/dz, the partial last chunk holds such rows, and the kernel moves exactly the rows the truth moves.

Gates: test_step64_gpu's, unchanged. Largest values measured here over all cases, on an H100 80GB HBM3 (700 W power limit); the whole
file ran in about one minute there:
  GATE_STEP 1e-5      6.5e-6 (rotation, flat, normal + depth)
  GATE_MOM 4e-5       1.3e-5 (second moments of the terms-only legs, which start from zero moments: v = (1 - beta2) g^2, and beta2 = 0.999
                      rounded to float32 makes 1 - beta2 1.3e-5 smaller than float64's 0.001); 8.8e-7 with seeded moments
  GATE_LOSS 1e-5      3.6e-6 (ssim); the terms: 2.2e-6 (dist), 1.3e-7 (dn)
  GATE_ACCUM 1e-5     4.0e-6 (p2p, normal + depth)
  GATE_GRAD 1e-5      1.6e-6 (xyz, flat gradients, every term, anti-aliased)
  GATE_GRAD_MAX 1e-5  1.9e-6 (the same)
The perturbed truths miss the step gate by five orders of magnitude (2.0: the step's sign flips).
"""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

import dn64
import photo_slam_b200.synthetic as syn
import step64
from test_step64_gpu import (BG, GATE_STEP, H, LAMBDA_DEPTH, LAMBDA_NORMAL, SCENES, W, _assert_gates, _bits, _cams, _compare, _maxerr, _model,
                             _relnorm, _seed_moments, _settled_state, _step_err, _targets, _targets64, _trainer)

pytestmark = pytest.mark.gpu

LAMBDA_DN, LAMBDA_DIST, ALPHA_MIN, JUMP = 0.05, 0.1, 0.5, 0.05
CHUNK = 128               # rows per owner chunk of the NVLink step (psb_dp_step)
NAMES = ("loss", "l1", "ssim", "depth_l1", "normal_l1", "dn", "dist")      # result_dist()'s seven scalars

PATHS = {"p2p": dict(mode="p2p"), "slabs": dict(mode="nccl", pipeline=True, nslabs=3), "flat": dict(mode="nccl", pipeline=False)}
TERMS = {"normal": step64.Flags(normal=True), "normal+depth": step64.Flags(normal=True, depth=True),
         "normal+dn": step64.Flags(normal=True, dn=True), "dist": step64.Flags(dist=True),
         "all": step64.Flags(depth=True, normal=True, dn=True, dist=True)}


def _flags(terms, aa):
    return dataclasses.replace(TERMS[terms], aa=aa)


def _scene_name(terms, aa):
    return ("terminate", "clamp")[(list(TERMS).index(terms) + int(aa)) % 2]


def _scene(name):
    """SCENES[name] with the P % 128 most opaque rows well inside the first view swapped into the partial last chunk"""
    sc = SCENES[name]()
    P = sc["xyz"].shape[0]
    k = P % CHUNK
    fx = W / (2.0 * float(_cams()[0]["tanfovx"]))
    x, y, z = sc["xyz"][:, 0], sc["xyz"][:, 1], sc["xyz"][:, 2]
    zs = np.where(z > 0, z, 1.0)
    u, v = x / zs * fx + 0.5 * (W - 1), y / zs * fx + 0.5 * (H - 1)
    inside = (z > 0.6) & (np.abs(u - 0.5 * W) < 0.3 * W) & (np.abs(v - 0.5 * H) < 0.3 * H)
    inside[P - k:] = False
    cand = np.nonzero(inside)[0]
    src = cand[np.argsort(-sc["opacity"][cand, 0], kind="stable")[:k]]
    dst = np.arange(P - k, P)
    for a in sc.values():
        a[np.concatenate([src, dst])] = a[np.concatenate([dst, src])]
    return sc


def _tg64(tg, colour=True):
    t = _targets64(tg, BG)
    t.update(lambda_dn=LAMBDA_DN, dn_alpha_min=ALPHA_MIN, dn_max_rel_jump=JUMP, lambda_dist=LAMBDA_DIST)
    if not colour:
        t.update(colour=False, mask=None, lambda_dssim=0.0)
    return t


def _kw(fl, tg):
    """trainForOneIteration's term arguments for the flags"""
    kw = {}
    if fl.depth:
        kw.update(gt_depth=tg["depth"], lambda_depth=LAMBDA_DEPTH)
    if fl.normal:
        kw.update(gt_normal=tg["normal"], lambda_normal=LAMBDA_NORMAL)
    if fl.dn:
        kw.update(lambda_dn=LAMBDA_DN, dn_alpha_min=ALPHA_MIN, dn_max_rel_jump=JUMP)
    if fl.dist:
        kw.update(lambda_dist=LAMBDA_DIST)
    return kw


def _loss_errs(res, r, fl, colour=True):
    """result_dist()'s scalars against the truth's: relative errors of the terms the step has; the others read exactly 0"""
    on = dict(loss=True, l1=colour, ssim=colour, depth_l1=fl.depth, normal_l1=fl.normal, dn=fl.dn, dist=fl.dist)
    errs = {}
    for k, v in zip(NAMES, res):
        if on[k]:
            errs[f"loss-{k}"] = abs(v - r["loss"][k]) / abs(r["loss"][k])
        elif k != "ssim":            # a colour target equal to the render: l1 reads 0, ssim about 1
            assert v == 0.0, (k, res)
    return errs


def _setup(cuda, fl, scene, seed, colour=True, seed_moments=True):
    """model of the scene, settled on the second view; moments from the truth's gradient (even rows) -> (m, tg, tg64, cam)"""
    cams = _cams()
    tg = _targets(cuda)
    tg64 = _tg64(tg, colour)
    m = _model(_scene(scene), cuda, fl, cams)
    if seed_moments:
        st, cam64, _ = _settled_state(m, fl, cams[1], tg64, seed)
        st["E"] = None
        _seed_moments(m, step64.grads64(st, cam64, tg64, fl)["grads"], None)
    return m, tg, tg64, cams[1]


def _dp_trainer(m, path, fl, det):
    from photo_slam_b200 import trainer
    tr = trainer.DataParallelTrainer(m, background=torch.tensor(BG, device=m.xyz_.device), antialiasing=fl.aa, deterministic=det,
                                     geometry_terms=True, **PATHS[path])
    assert tr.mode == PATHS[path]["mode"] and (path == "p2p" or tr.pipeline == (path == "slabs"))
    return tr


def _dp_step(cuda, path, fl, scene, det, seed, colour=True, conv=step64.STEP_CONV, truth_flags=None):
    """one DataParallelTrainer step against step64 -> (m, state before, truth, result_dist() scalars, settle margin)"""
    m, tg, tg64, cam = _setup(cuda, fl, scene, seed, colour, seed_moments=colour)
    tr = _dp_trainer(m, path, fl, det)
    c = syn.device_camera(cam, cuda)
    tr.render(c)                     # sizes the binning arena: an overflowing data-parallel step is dropped, not repeated
    st, cam64, mg = _settled_state(m, fl, cam, tg64, seed + 1)
    st["E"] = None
    if colour:
        gt, mask = tg["gt"], tg["mask"]
    else:
        tr.opt.lambda_dssim = 0.0
        gt, mask = tr.render(c).clone(), None
    tr.trainForOneIteration(c, gt, mask, **_kw(fl, tg))
    res = tr.result_dist()[:7]
    tr.sync()
    torch.cuda.synchronize()
    assert tr.dropped_views == 0 and tr.status() == 0
    if path == "p2p":
        tr.close()
    r = step64.step64(st, cam64, tg64, truth_flags or fl, conv)
    return m, st, r, res, mg


CASES = [(p, t, a) for p in PATHS for t in TERMS for a in (False, True)]


@pytest.mark.parametrize("path,terms,aa", CASES, ids=[f"{p}-{t}-{'aa' if a else 'plain'}" for p, t, a in CASES])
def test_dp_step(cuda, path, terms, aa):
    k = CASES.index((path, terms, aa))
    fl = _flags(terms, aa)
    det = _bits(k) % 2 == 0
    m, st, r, res, mg = _dp_step(cuda, path, fl, _scene_name(terms, aa), det, 1000 + 10 * k)
    errs, ex, nidle = _compare(m, st, r, fl, exposure_id=None)
    errs.update(_loss_errs(res, r, fl))
    assert nidle > 0
    print(f"MEASURED dp64 {path} {step64.flag_name(fl)} det={det} margin={mg:.1e} excluded={ex} {errs}")
    _assert_gates(errs)


@pytest.mark.parametrize("aa", [False, True], ids=["plain", "aa"])
def test_flat_gradients(cuda, aa):
    """psb_trainer_backward_dist with every term: the raw gradients against grads64 and the densification statistics"""
    from photo_slam_b200 import _lib, trainer
    from photo_slam_b200.parallel import GradBuffer
    fl = _flags("all", aa)
    m, tg, tg64, cam = _setup(cuda, fl, ("terminate", "clamp")[int(aa)], 77, seed_moments=False)
    tr = _dp_trainer(m, "flat", fl, det=aa)
    c = syn.device_camera(cam, cuda)
    tr.render(c)
    st, cam64, mg = _settled_state(m, fl, cam, tg64, 78)
    st["E"] = None
    tr._apply_deterministic()
    P = m.num_points()
    buf = GradBuffer(P, cuda)
    cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)
    d = trainer._Depth(tg["depth"].data_ptr(), LAMBDA_DEPTH, None)
    nrm = trainer._Normal(tg["normal"].data_ptr(), LAMBDA_NORMAL, None)
    dn = trainer._Dn(LAMBDA_DN, ALPHA_MIN, JUMP, None)
    ds = trainer._Dist(LAMBDA_DIST, None)
    ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in buf.segments])
    _lib.check(tr.L.psb_trainer_backward_dist(*tr._call_args(m, cm, cc, cs, tg["gt"], tg["mask"], None, None), ptrs, C.byref(d), None, None,
                                              C.byref(nrm), C.byref(dn), C.byref(ds), torch.cuda.current_stream().cuda_stream),
               "psb_trainer_backward_dist")
    res = tr.result_dist()[:7]
    torch.cuda.synchronize()
    r = step64.step64(st, cam64, tg64, fl)
    errs = _loss_errs(res, r, fl)
    n = (st["D"] + 1) ** 2 - 1
    for k_, a in zip(step64.GROUPS, buf.views()):
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
    print(f"MEASURED dp64 flat grads {step64.flag_name(fl)} margin={mg:.1e} {errs}")
    _assert_gates(errs)


ONLY = [(p, t) for p in ("p2p", "slabs") for t in ("normal", "dist")]


@pytest.mark.parametrize("path,terms", ONLY, ids=[f"{p}-{t}" for p, t in ONLY])
def test_terms_only(cuda, path, terms):
    """colour target = the render, lambda_dssim = 0, zero moments: the rows the step moves are the rows the term reaches"""
    k = ONLY.index((path, terms))
    fl = _flags(terms, False)
    m, st, r, res, mg = _dp_step(cuda, path, fl, ("terminate", "clamp")[k % 2], k % 2 == 0, 2000 + 10 * k, colour=False)
    assert res[1] == 0.0, "the colour target must equal the render"
    P = m.num_points()
    via = (r["inter"]["n"] != 0).any(1) if terms == "normal" else r["inter"]["z"] != 0
    reached = r["reached"]
    assert not r["inter"]["rgb"].any() and reached.sum() > 100
    assert torch.equal(reached & via, reached), "a row is reached other than through the term"
    assert reached[P - P % CHUNK:].any(), "the partial last chunk holds no row the term reaches"
    moved_k = torch.zeros(P, dtype=torch.bool, device=cuda)
    moved_t = torch.zeros_like(moved_k)
    for i, q in enumerate(step64.GROUPS):
        moved_k |= (m.tensors()[i].double() != st["params"][q]).reshape(P, -1).any(1)
        moved_t |= (r["state"]["params"][q] != st["params"][q]).reshape(P, -1).any(1)
    assert torch.equal(moved_t, reached)
    assert torch.equal(moved_k, moved_t), (int((moved_k & ~moved_t).sum()), int((moved_t & ~moved_k).sum()))
    errs, ex, nidle = _compare(m, st, r, fl, exposure_id=None)
    errs.update(_loss_errs(res, r, fl, colour=False))
    print(f"MEASURED dp64 terms-only {path} {terms} margin={mg:.1e} reached={int(reached.sum())} "
          f"last-chunk={int(reached[P - P % CHUNK:].sum())} excluded={ex} {errs}")
    _assert_gates(errs)


def test_scenes_reach_their_edges(cuda):
    """each scene has mask-valid pixels with and without a depth normal, rows with seeded moments that the pass does not see, and rows
    the pass reaches in the partial last chunk"""
    fl = TERMS["all"]
    for name in SCENES:
        m, tg, tg64, cam = _setup(cuda, fl, name, 5)
        st, cam64, _ = _settled_state(m, fl, cam, tg64, 6)
        r = step64.grads64(st, cam64, tg64, fl)
        out = r["out"]
        _, _, nd = dn64.dn64(out["depth"].detach(), out["alpha"].detach(), r["N"].detach(), W, H, cam64["tanfovx"], cam64["tanfovy"],
                             ALPHA_MIN, JUMP)
        inmask = tg64["mask"][0] != 0
        valid = (nd != 0).any(0) & inmask
        P = m.num_points()
        seeded = (m.exp_avg_[0] != 0).any(1)
        unseen = seeded & ~r["visible"]
        print(f"MEASURED dp64 scene {name}: dn-valid {int(valid.sum())} dn-invalid {int((inmask & ~valid).sum())} seeded-unseen "
              f"{int(unseen.sum())} reached in the last chunk {int(r['reached'][P - P % CHUNK:].sum())} of {P % CHUNK}")
        assert valid.sum() > 50 and (inmask & ~valid).sum() > 50
        assert unseen.sum() >= 10
        assert P % CHUNK and r["reached"][P - P % CHUNK:].any()


# ---- the gates bite -----------------------------------------------------------------------------------------------------------------
PERTURB = {"normal-without-flip": ("normal", dict(conv=dataclasses.replace(step64.STEP_CONV, normal_flip=False)), ["rotation"]),
           "dist-without-dz": ("dist", dict(conv=dataclasses.replace(step64.STEP_CONV, dist_dz=False)), ["xyz"]),
           "dn-dropped": ("normal+dn", dict(truth_flags=TERMS["normal"]), list(step64.GROUPS))}


@pytest.mark.parametrize("what", list(PERTURB))
def test_perturbed_truth_fails_the_gate(cuda, what):
    """one p2p step against a truth with one convention changed: the step gate of the named groups rejects it"""
    terms, kw, groups = PERTURB[what]
    m, st, r, res, _ = _dp_step(cuda, "p2p", TERMS[terms], _scene_name(terms, False), True, 3000, **kw)
    nx = r["state"]
    err = max(_step_err(t.detach(), nx["params"][q], st["lr"][i]) for i, (q, t) in enumerate(zip(step64.GROUPS, m.tensors())) if q in groups)
    print(f"MEASURED dp64 perturbed {what}: {err:.2e} (gate {GATE_STEP:.0e})")
    assert err > GATE_STEP, f"{what}: the gate does not see the perturbation ({err} <= {GATE_STEP})"


# ---- the fused step on the same terms -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("terms", list(TERMS))
def test_fused_control(cuda, terms):
    """GaussianTrainer with the same terms and gates: a data-parallel failure next to a passing fused case lies in the data-parallel path"""
    k = list(TERMS).index(terms)
    fl = _flags(terms, k % 2 == 1)
    m, tg, tg64, cam = _setup(cuda, fl, _scene_name(terms, fl.aa), 4000 + 10 * k)
    tr = _trainer(m, fl, k % 2 == 0)
    c = syn.device_camera(cam, cuda)
    tr.render(c)
    st, cam64, mg = _settled_state(m, fl, cam, tg64, 4001 + 10 * k)
    st["E"] = None
    tr.trainForOneIteration(c, tg["gt"], tg["mask"], **_kw(fl, tg))
    res = tr.result_dist()[:7]
    torch.cuda.synchronize()
    r = step64.step64(st, cam64, tg64, fl)
    errs, ex, _ = _compare(m, st, r, fl, exposure_id=None, live=True)
    errs.update(_loss_errs(res, r, fl))
    print(f"MEASURED dp64 fused {step64.flag_name(fl)} margin={mg:.1e} excluded={ex} {errs}")
    _assert_gates(errs)
