"""-m gpu: contribution scores (psb_trainer_contribution) and pruneByContribution.

  1. the score pass against the float64 restatement (tests/contrib64.py) on settled scenes over three views, plain / anti-aliased /
     3D-filtered, tight lists on: the set of rows with a score is exact, max within 1e-4, sum within 1e-4 relative plus one unit per
     blended pixel;
  2. a score pass renders what psb_trainer_render renders: colour, final T and the last splat per pixel bit for bit;
  3. determinism: two runs, a permuted view order, deterministic mode on and off, and per-view sweeps added on the host all agree bit
     for bit;
  4. a sweep whose first view overflows a fresh context's binning arena ends bit-identical to a sweep on a grown arena;
  5. the prune: rows behind every camera, outside every frustum and buried behind an opaque wall score 0 and go; no row at or above
     the threshold or younger than min_age goes; without pixels that end at the T test the scored views render bit-identical after the
     prune; training continues; a filter3d trainer needs computeFilter3D again;
  6. quality: a perturbed copy of a 20 k-row target with floaters, trained over 6 keyframes, then pruned: keyframe PSNR before and after.
"""
import math

import numpy as np
import pytest
import torch

import contrib64
import filter3d64 as f64
import splat64 as s64
import photo_slam_b200.synthetic as syn
from helpers import scene_tensors

pytestmark = pytest.mark.gpu
LRS = [0.00016, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
GATE_MAX = 1e-4            # max_weight against the float64 truth, absolute (the image tolerance of the float64 tests)
GATE_SUM_REL = 1e-4        # sum_weight: relative, plus one 2^-26 unit per blended pixel (the truncation)
# keyframe PSNR (dB) the quality run may lose through the prune, right after it and 100 steps later (DESIGN.md §5 gives the measurement)
QUALITY_MARGIN_DB = 0.05


def _views(W, H, f, n, seed, angle=0.05, trans=0.05):
    """the identity camera and n - 1 small random poses around it (numpy camera dicts)"""
    rng = np.random.default_rng(seed)
    out = [syn.make_camera(W, H, f, f)]
    for _ in range(n - 1):
        out.append(syn.make_camera(W, H, f, f, *syn.random_pose(rng, max_angle=angle, max_trans=trans)))
    return out


def _random(P, cam, seed, scale_px=2.5, logit=(0.0, 1.5), zr=(0.8, 8.0)):
    """P Gaussians in front of the identity camera, depths on a geometric ladder (no two within 1e-4 of each other)"""
    rng = np.random.default_rng(seed)
    W, H = cam["W"], cam["H"]
    fx = W / (2.0 * float(cam["tanfovx"]))
    z = zr[0] * (zr[1] / zr[0]) ** ((rng.permutation(P) + rng.uniform(0.3, 0.7, P)) / max(P, 1))
    u, v = rng.uniform(-0.1 * W, 1.1 * W, P), rng.uniform(-0.1 * H, 1.1 * H, P)
    xyz = np.stack([(u - 0.5 * (W - 1)) / fx * z, (v - 0.5 * (H - 1)) / fx * z, z], 1)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return dict(xyz=f32(xyz), features_dc=f32(((rng.uniform(0, 1, (P, 3)) - 0.5) / s64.SH_C0)[:, None]),
                features_rest=f32(rng.normal(0, 0.05, (P, 15, 3))), scaling=f32(np.log(scale_px / fx * z)[:, None] + rng.normal(0, 0.4, (P, 3))),
                rotation=f32(rng.normal(size=(P, 4))), opacity=f32(rng.normal(logit[0], logit[1], (P, 1))))


def _packed(cams):
    return np.stack([np.concatenate([np.asarray(c["viewmatrix"], np.float64).reshape(-1),
                                     [c["W"] / (2 * float(c["tanfovx"])), c["H"] / (2 * float(c["tanfovy"])), c["W"], c["H"]]]) for c in cams])


def _model(sc, dev, D=3):
    from photo_slam_b200 import trainer
    m = trainer.GaussianModel.from_numpy({k: v.copy() for k, v in sc.items()}, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    m.lr_ = list(LRS)
    m.setShDegree(D)
    return m


def _debug_state(tr, W, H, dev):
    from photo_slam_b200 import _lib
    last = torch.empty(W * H, dtype=torch.int32, device=dev)
    fT = torch.empty(W * H, dtype=torch.float32, device=dev)
    _lib.check(tr.L.psb_trainer_debug_state(tr.h, W, H, last.data_ptr(), fT.data_ptr(), None, torch.cuda.current_stream().cuda_stream),
               "psb_trainer_debug_state")
    return last, fT


def _score_pass(tr, cam, mx, sm, out):
    """one psb_trainer_contribution call into the integer arrays, the image into `out`"""
    import ctypes as C
    from photo_slam_b200 import _lib, trainer
    m = tr.model
    cm, cc = m._cmodel(False), trainer._ccamera(cam)
    _lib.check(tr.L.psb_trainer_contribution(tr.h, m.num_points(), 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), m.active_sh_degree_,
                                             mx.data_ptr(), sm.data_ptr(), out.data_ptr(), torch.cuda.current_stream().cuda_stream),
               "psb_trainer_contribution")


# ---- 1. against the restatement ----------------------------------------------------------------------------------------------------
MODES = ["plain", "aa", "filter3d"]
_SCENES = {}


def _scene(mode):
    if mode not in _SCENES:
        W, H, f = 96, 64, 80.0
        cams = _views(W, H, f, 3, seed=11)
        sc = _random(700, cams[0], seed=5)
        f_of = (lambda xyz: f64.filter3d(xyz, _packed(cams))["filter"]) if mode == "filter3d" else None
        contrib64.settle(sc, cams, D=3, aa=mode == "aa", f_of=f_of, seed=2)
        _SCENES[mode] = (sc, cams)
    return _SCENES[mode]


@pytest.mark.parametrize("mode", MODES)
def test_scores_against_the_restatement(cuda, mode):
    from photo_slam_b200 import trainer
    sc, cams = _scene(mode)
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m, background=torch.tensor([0.2, 0.3, 0.4], device=cuda), antialiasing=mode == "aa",
                                 filter3d=mode == "filter3d")
    dcams = [syn.device_camera(c, cuda) for c in cams]
    f = None
    if mode == "filter3d":
        m.computeFilter3D(dcams)
        f = m.filter_3D_.double().cpu().numpy()
    mx, sm = tr.contributionScores(dcams)
    torch.cuda.synchronize()
    ref = contrib64.scores(s64.raw64(sc, "cpu"), [s64.camera64(c, "cpu") for c in cams], D=3, aa=mode == "aa", f=f)
    kmax, ksum = mx.double().cpu(), sm.cpu()
    assert torch.equal(kmax > 0, ref["max"] > 0), "the rows with a score differ from the truth's"
    assert 0 < int((kmax > 0).sum()) < m.num_points()
    err_max = float((kmax - ref["max"]).abs().max())
    slack = (ksum - ref["sum"]).abs() - (GATE_SUM_REL * ref["sum"] + ref["pixels"].double() * trainer.CONTRIB_SUM_UNIT)
    rel_sum = float(((ksum - ref["sum"]).abs() / ref["sum"].clamp_min(1e-30))[ref["sum"] > 0].max())
    print(f"MEASURED contribution {mode}: {int((kmax > 0).sum())} of {m.num_points()} rows scored, max err {err_max:.2e}, sum rel err {rel_sum:.2e}")
    assert err_max < GATE_MAX
    assert float(slack.max()) <= 0.0


# ---- 2. the score pass renders the same ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("aa", [False, True])
def test_score_pass_renders_what_render_renders(cuda, aa):
    from photo_slam_b200 import trainer
    cam, sc, _, _, c = scene_tensors(100_000, "tum", seed=3, pose_seed=4, dev=cuda)
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m, background=torch.tensor([0.1, 0.2, 0.3], device=cuda), antialiasing=aa)
    W, H, P = c["W"], c["H"], m.num_points()
    img = tr.render(c).clone()
    last, fT = (t.clone() for t in _debug_state(tr, W, H, cuda))
    mx = torch.zeros(P, dtype=torch.int32, device=cuda)
    sm = torch.zeros(P, dtype=torch.int64, device=cuda)
    img2 = torch.empty_like(img)
    _score_pass(tr, c, mx, sm, img2)
    assert tr.result()[3] > 0
    last2, fT2 = _debug_state(tr, W, H, cuda)
    torch.cuda.synchronize()
    assert torch.equal(img, img2) and torch.equal(last, last2) and torch.equal(fT, fT2)
    # every pixel's last blended splat has a score
    shown = last[last >= 0].long().unique()
    assert (mx[shown] > 0).all() and (sm[shown] > 0).all()


# ---- 3. determinism ------------------------------------------------------------------------------------------------------------------
def test_scores_are_bit_identical_across_runs_orders_and_modes(cuda):
    from photo_slam_b200 import trainer
    cam, sc, _, _, c = scene_tensors(200_000, "tum", seed=7, pose_seed=8, dev=cuda)
    W, H = c["W"], c["H"]
    fx = W / (2 * c["tanfovx"])
    views = [syn.device_camera(v, cuda) for v in _views(W, H, fx, 5, seed=9, angle=0.1, trans=0.1)]
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m, deterministic=False)
    a = tr.contributionScores(views)
    b = tr.contributionScores(views)
    perm = tr.contributionScores([views[k] for k in (3, 0, 4, 2, 1)])
    det = trainer.GaussianTrainer(m, deterministic=True)
    d = det.contributionScores(views)
    single = [tr.contributionScores([v]) for v in views]
    torch.cuda.synchronize()
    for other in (b, perm, d):
        assert torch.equal(a[0], other[0]) and torch.equal(a[1], other[1])
    assert torch.equal(a[0], torch.stack([s[0] for s in single]).amax(0))
    units = torch.stack([(s[1] / trainer.CONTRIB_SUM_UNIT).round().long() for s in single]).sum(0)   # exact integers
    assert torch.equal((a[1] / trainer.CONTRIB_SUM_UNIT).round().long(), units)
    assert int((a[0] > 0).sum()) > 0.5 * m.num_points()


# ---- 4. overflow ---------------------------------------------------------------------------------------------------------------------
def test_overflowing_sweep_ends_as_on_a_grown_arena(cuda):
    from photo_slam_b200 import trainer
    cam, sc, _, _, c = scene_tensors(20_000, "tum", seed=5, pose_seed=6, dev=cuda, scale_px=30.0)
    W, H = c["W"], c["H"]
    views = [syn.device_camera(v, cuda) for v in _views(W, H, W / (2 * c["tanfovx"]), 3, seed=1, angle=0.1, trans=0.1)]
    m = _model(sc, cuda)
    fresh = trainer.GaussianTrainer(m)
    a = fresh.contributionScores(views)
    first, count, cur = fresh._overflow_info()
    assert count >= 1 and first == 1, "the first view did not overflow the fresh arena"
    grown = trainer.GaussianTrainer(m)
    for v in views:
        grown.render(v)                      # grows the arena (render repeats an overflowing view)
    grown_info = grown._overflow_info()[:2]
    b = grown.contributionScores(views)
    assert grown._overflow_info()[:2] == grown_info, "the sweep on the grown arena overflowed"
    torch.cuda.synchronize()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and bool((a[0] > 0).any())


# ---- 5. the prune --------------------------------------------------------------------------------------------------------------------
def _put(sc, cam, i, u, v, z, sigma_px, logit):
    fx = cam["W"] / (2.0 * float(cam["tanfovx"]))
    sc["xyz"][i] = [(u - 0.5 * (cam["W"] - 1)) / fx * z, (v - 0.5 * (cam["H"] - 1)) / fx * z, z]
    sc["scaling"][i] = np.log(sigma_px / fx * abs(z))
    sc["rotation"][i] = [1.0, 0.0, 0.0, 0.0]
    sc["opacity"][i] = logit


def _walled_scene(W=128, H=96, f=110.0):
    """an opaque wall of three layers at z ~ 1 over the whole view of every camera, 300 rows in front of it, and injected rows that no
    view shows: 40 buried behind the wall, 30 behind every camera, 30 outside every frustum. -> (scene, cams, injected rows)"""
    cams = _views(W, H, f, 3, seed=4, angle=0.02, trans=0.02)
    n_wall = 3 * (W // 8 + 5) * (H // 8 + 5)
    sc = _random(n_wall + 400, cams[0], seed=6, scale_px=2.0, zr=(0.4, 0.9))
    k = 0
    for layer in range(3):
        for gy in range(-2, H // 8 + 3):
            for gx in range(-2, W // 8 + 3):
                _put(sc, cams[0], k, 8.0 * gx + 2.0 * layer, 8.0 * gy + 2.0 * layer, 1.0 + 0.01 * layer + 1e-5 * k, 7.0, 7.0)
                k += 1
    rng = np.random.default_rng(3)
    base = n_wall + 300
    for j in range(40):            # buried: small, opaque, well behind the wall
        _put(sc, cams[0], base + j, rng.uniform(10, W - 10), rng.uniform(10, H - 10), rng.uniform(3.0, 6.0), 2.0, 4.0)
    for j in range(30):            # behind every camera
        _put(sc, cams[0], base + 40 + j, rng.uniform(0, W), rng.uniform(0, H), 2.0, 2.0, 4.0)
        sc["xyz"][base + 40 + j, 2] = -rng.uniform(1.0, 3.0)
    for j in range(30):            # far outside every frustum (to the side, in front)
        _put(sc, cams[0], base + 70 + j, 6.0 * W, rng.uniform(0, H), 2.0, 2.0, 4.0)
    return sc, cams, np.arange(base, base + 100)


def test_prune_removes_what_no_view_shows(cuda):
    from photo_slam_b200 import trainer
    sc, cams, injected = _walled_scene()
    dcams = [syn.device_camera(c, cuda) for c in cams]
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m)
    mx, sm = tr.contributionScores(dcams)
    assert (mx[injected] == 0).all() and (sm[injected] == 0).all()
    min_weight = 0.02
    P0 = m.num_points()
    ids = torch.arange(P0, device=cuda, dtype=torch.int32)
    m.features_dc_[:, 0, 0] = ids.float()         # tags the rows (colour is irrelevant to the scores' support)
    mx, _ = tr.contributionScores(dcams)
    n = tr.pruneByContribution(dcams, min_weight)
    left = m.features_dc_[:, 0, 0].round().long()
    removed = torch.ones(P0, dtype=torch.bool, device=cuda)
    removed[left] = False
    print(f"MEASURED prune: {n} of {P0} rows removed at min_weight {min_weight}")
    assert n == int(removed.sum()) == int((mx < min_weight).sum())
    assert removed[torch.from_numpy(injected).to(cuda)].all()
    assert not removed[mx >= min_weight].any()


def test_min_age_protects_fresh_rows(cuda):
    from photo_slam_b200 import trainer
    sc, cams, injected = _walled_scene()
    dcams = [syn.device_camera(c, cuda) for c in cams]
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m)
    tr.iteration = 500
    m.exist_since_iter_ = torch.zeros(m.num_points(), dtype=torch.int32, device=cuda)
    m.exist_since_iter_[injected[:50]] = 495
    n = tr.pruneByContribution(dcams, 0.02, min_age=10)
    assert m.num_points() == len(sc["xyz"]) - n
    assert int((m.exist_since_iter_ == 495).sum()) == 50      # every young row is still there


def test_pruning_unscored_rows_leaves_the_views_bit_identical(cuda):
    from photo_slam_b200 import trainer
    W, H, f = 128, 96, 110.0
    cams = _views(W, H, f, 3, seed=12)
    sc = _random(3000, cams[0], seed=8, scale_px=2.5, logit=(-2.5, 1.0))
    # rows no view blends: behind the cameras, off to the side
    sc["xyz"][:200, 2] *= -1.0
    sc["xyz"][200:400, 0] += 50.0
    ref = contrib64.scores(s64.raw64(sc, "cpu"), [s64.camera64(c, "cpu") for c in cams], D=3)
    assert not any(bool(s.any()) for s in ref["stopped"]), "the scene must have no pixel that ends at the T test"
    dcams = [syn.device_camera(c, cuda) for c in cams]
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m, background=torch.tensor([0.3, 0.2, 0.1], device=cuda))

    def views():
        out = []
        for c in dcams:
            d, a = torch.empty((H, W), device=cuda), torch.empty((H, W), device=cuda)
            out.append((tr.render(c, out_depth=d, out_alpha=a).clone(), d, a))
        return out
    before = views()
    n = tr.pruneByContribution(dcams, 1e-9)
    after = views()
    torch.cuda.synchronize()
    assert n >= 400
    for (c0, d0, a0), (c1, d1, a1) in zip(before, after):
        assert torch.equal(c0, c1) and torch.equal(d0, d1) and torch.equal(a0, a1)
    # training continues on the pruned rows
    gt = torch.rand((3, H, W), device=cuda)
    for _ in range(3):
        tr.trainForOneIteration(dcams[0], gt)
        loss = tr.result()[0]
    assert math.isfinite(loss) and m.adam_live_valid_


def test_filter3d_trainer_needs_the_filter_again(cuda):
    from photo_slam_b200 import trainer
    sc, cams, injected = _walled_scene()
    dcams = [syn.device_camera(c, cuda) for c in cams]
    m = _model(sc, cuda)
    tr = trainer.GaussianTrainer(m, filter3d=True)
    with pytest.raises(ValueError, match="computeFilter3D"):
        tr.contributionScores(dcams)
    m.computeFilter3D(dcams)
    assert tr.pruneByContribution(dcams, 0.02) > 0
    with pytest.raises(ValueError, match="computeFilter3D"):
        tr.render(dcams[0])
    m.computeFilter3D(dcams)
    tr.render(dcams[0])


# ---- 6. quality ----------------------------------------------------------------------------------------------------------------------
def test_quality_after_the_prune(cuda):
    from photo_slam_b200 import trainer
    P, W, H, fx = 20_000, 320, 240, 260.0
    cam0 = syn.make_camera(W, H, fx, fx)
    gt_scene = syn.make_scene(P, cam0, seed=31, scale_px=3.0)
    views = [syn.device_camera(v, cuda) for v in _views(W, H, fx, 6, seed=60, angle=0.06, trans=0.12)]
    gt_tr = trainer.GaussianTrainer(trainer.GaussianModel.from_numpy(gt_scene, cuda))
    gts = [gt_tr.render(c).clamp(0, 1).clone() for c in views]
    rng = np.random.default_rng(4)
    start = {k: v.copy() for k, v in gt_scene.items()}
    start["xyz"] += rng.normal(0, 0.01, start["xyz"].shape).astype(np.float32)
    start["features_dc"] += rng.normal(0, 0.5, start["features_dc"].shape).astype(np.float32)
    start["opacity"] += rng.normal(0, 0.5, start["opacity"].shape).astype(np.float32)
    # floaters: 4000 rows scattered in a box around the scene, many outside every keyframe's frustum
    fl = _random(4000, cam0, seed=9, scale_px=2.0, zr=(0.5, 12.0))
    fl["xyz"][:, :2] *= rng.uniform(0.5, 4.0, (4000, 1)).astype(np.float32)
    start = {k: np.concatenate([start[k], fl[k]]) for k in start}
    m = _model(start, cuda, D=0)
    opt = trainer.GaussianOptimizationParams()
    tr = trainer.GaussianTrainer(m, opt)

    def psnr():
        return float(np.mean([10.0 * math.log10(1.0 / ((tr.render(c) - g) ** 2).mean().item()) for c, g in zip(views, gts)]))

    def train(n):
        for it in range(n):
            k = it % len(views)
            tr.trainForOneIteration(views[k], gts[k], densify_stats=False)
            tr.result()
    train(300)
    p_before, n_before = psnr(), m.num_points()
    removed = tr.pruneByContribution(views, 0.01)
    p_after = psnr()
    train(100)
    p_later = psnr()
    print(f"MEASURED quality: {removed} of {n_before} rows removed at min_weight 0.01; keyframe PSNR {p_before:.3f} dB before, "
          f"{p_after:.3f} dB right after, {p_later:.3f} dB after 100 more steps")
    assert removed > 0
    assert p_after > p_before - QUALITY_MARGIN_DB and p_later > p_before - QUALITY_MARGIN_DB
