"""-m gpu: bounded-budget densification (3DGS-MCMC) against its float64 restatement (tests/mcmc64.py) and end to end.

  relocate / grow   with injected uniforms: picks, multiplicities, copies bit-identical to their corrected sources, corrected opacity and
                    scale to 1e-5 relative, zero moments and statistics, untouched rows bit for bit, live-byte contract; Philox draws
                    bit-identical from run to run and proportional to opacity; the rendered picture survives a relocation;
  noise             equals the restatement, skips unseen rows, is bit-identical between runs and is added once around an overflow;
  regularisers      closed form on the rows a pass updates, zero elsewhere, lambda = 0 is the plain step bit for bit, the two fused Adam
                    variants agree with depth and anti-aliasing on;
  end to end        600 steps under a cap with mcmcRefine every 100 against the same run with densifyAndPrune.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import mcmc64
import photo_slam_b200.synthetic as syn

pytestmark = pytest.mark.gpu
LRS = [0.00016, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
MIN_OP = 0.005


def _views(cuda, W, H, fx, n, seed=50):
    out = []
    for k in range(n):
        R, t = (None, None) if k == 0 else syn.random_pose(np.random.default_rng(seed + k), max_angle=0.06, max_trans=0.12)
        cam = syn.make_camera(W, H, fx, fx, R, t)
        out.append(syn.device_camera(cam, cuda))
    return out


def _state(P, seed, dev, dead_frac):
    """a model with random non-zero moments and statistics; dead rows at sigmoid(-8) = 3.4e-4, alive ones well above 0.005"""
    from photo_slam_b200 import trainer
    rng = np.random.default_rng(seed)
    sc = syn.make_scene(P, syn.make_camera(160, 120, 130.0, 130.0), seed=seed)
    sc["opacity"] = np.clip(sc["opacity"], -4.0, 6.0)                       # sigmoid(-4) = 0.018
    sc["opacity"][rng.random(P) < dead_frac] = -8.0
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    gen = torch.Generator(device=dev).manual_seed(seed)
    for t in m.exp_avg_:
        t.copy_(torch.rand(t.shape, device=dev, generator=gen) * 2 - 1)
    for t in m.exp_avg_sq_:
        t.copy_(torch.rand(t.shape, device=dev, generator=gen) + 0.1)
    m.xyz_gradient_accum_.copy_(torch.rand((P, 1), device=dev, generator=gen) + 0.1)
    m.denom_.fill_(2.0)
    m.max_radii2D_.copy_(torch.rand(P, device=dev, generator=gen) * 50 + 1)
    m.exist_since_iter_ = torch.arange(P, dtype=torch.int32, device=dev)
    m.invalidateAdamLive()
    m.adamLive()                                                            # all ones: every row has moments
    return m


def _w32(opacity_raw):
    """the weights the kernel sums: the float32 sigmoid"""
    return mcmc64.sigmoid(opacity_raw.astype(np.float32)).astype(np.float32).astype(np.float64)


def _host(m):
    n = lambda ts: [t.detach().cpu().numpy().copy() for t in ts]
    return dict(p=n(m.tensors()), m=n(m.exp_avg_), v=n(m.exp_avg_sq_), accum=m.xyz_gradient_accum_.cpu().numpy().copy(),
                denom=m.denom_.cpu().numpy().copy(), max_radii=m.max_radii2D_.cpu().numpy().copy(), exist=m.exist_since_iter_.cpu().numpy().copy())


def _safe_uniforms(weights, n, seed):
    """n uniforms none of which lands within 1e-6 * total of a cumulative boundary (there the last bit of a sigmoid may pick the neighbour)"""
    u = np.random.default_rng(seed).random(n).astype(np.float32)
    u = np.minimum(u, np.float32(0.999))
    for _ in range(20):
        _, margin = mcmc64.sample(weights, u)
        bad = margin < 1e-6
        if not bad.any():
            return u
        u[bad] = (u[bad] + np.float32(1e-3)) % np.float32(0.999)
    raise AssertionError("could not place the uniforms")


def _compare(m, before, want, picked, targets, iteration, P_old):
    """the device model against the restatement `want`; `before`: the host copy taken before the call"""
    after = _host(m)
    P = after["p"][0].shape[0]
    picked_rows = np.unique(picked)
    touched = np.zeros(P, bool)
    touched[picked_rows] = True
    touched[targets] = True
    for q in range(6):
        assert np.array_equal(after["p"][q][targets], after["p"][q][picked]), f"tensor {q}: a copy differs from its corrected source"
        for k in ("m", "v"):
            assert not after[k][q][touched].any(), f"{k}[{q}]: moments of picked / written rows must be zero"
        rest = ~touched[:P_old]
        for k in ("p", "m", "v"):
            assert np.array_equal(after[k][q][:P_old][rest], before[k][q][rest]), f"{k}[{q}]: an uninvolved row changed"
        if q not in (3, 4):
            assert np.array_equal(after["p"][q][picked_rows], before["p"][q][picked_rows])
    o_mine, o_want = mcmc64.sigmoid(after["p"][3][picked_rows, 0]), mcmc64.sigmoid(want["p"][3][picked_rows, 0])
    assert np.abs(o_mine / o_want - 1).max() < 1e-5, np.abs(o_mine / o_want - 1).max()
    s_mine, s_want = np.exp(after["p"][4][picked_rows].astype(np.float64)), np.exp(want["p"][4][picked_rows])
    assert np.abs(s_mine / s_want - 1).max() < 1e-5, np.abs(s_mine / s_want - 1).max()
    assert not after["accum"][targets].any() and not after["denom"][targets].any() and not after["max_radii"][targets].any()
    assert (after["exist"][targets] == iteration).all()
    keep = np.setdiff1d(np.arange(P_old), targets)
    for k in ("accum", "denom", "max_radii", "exist"):
        assert np.array_equal(after[k][keep], before[k][keep]), k


@pytest.mark.parametrize("P,dead_frac", [(3001, 0.2), (2049, 0.7), (50_001, 0.05)])
def test_relocate_matches_the_restatement(cuda, P, dead_frac):
    from photo_slam_b200 import _lib, trainer
    m = _state(P, 11, cuda, dead_frac)
    before = _host(m)
    o = mcmc64.sigmoid(before["p"][3][:, 0])
    n_dead = int((o <= MIN_OP).sum())
    assert (n_dead > P - n_dead) == (dead_frac > 0.5) and n_dead > 50
    u = _safe_uniforms(np.where(o > MIN_OP, _w32(before["p"][3][:, 0]), 0.0), n_dead, 5)
    want, picks, dead, _ = mcmc64.relocate(before, u, MIN_OP, iteration=42)
    n = m.relocateGaussians(MIN_OP, iteration=42, uniforms=torch.from_numpy(u))
    torch.cuda.synchronize()
    assert n == n_dead == len(dead) and m.num_points() == P
    if dead_frac > 0.5:
        assert np.bincount(picks).max() > 3, "the case must exercise multiplicities above 2"
    _compare(m, before, want, picks, dead, 42, P)
    # live bytes: cleared exactly for the rows whose moments were zeroed, and psb_adam_live_rebuild agrees
    assert m.adam_live_valid_
    live = m.adam_live_.clone()
    touched = torch.zeros(P, dtype=torch.bool, device=cuda)
    touched[torch.from_numpy(np.concatenate([picks, dead])).to(cuda)] = True
    assert torch.equal(live.bool(), ~touched)
    cm = m._cmodel()
    cm.adam_live = m.adam_live_.data_ptr()
    _lib.check(trainer._bind().psb_adam_live_rebuild(P, C.byref(cm), torch.cuda.current_stream().cuda_stream), "psb_adam_live_rebuild")
    assert torch.equal(m.adam_live_, live)
    assert int((torch.sigmoid(m.opacity_) <= MIN_OP).sum()) == 0, "no dead row is left"


def test_relocate_writes_nothing_without_dead_or_without_alive_rows(cuda):
    for dead_frac in (0.0, 1.1):
        m = _state(1500, 3, cuda, dead_frac)
        before = _host(m)
        assert m.relocateGaussians(MIN_OP, iteration=7) == 0
        after = _host(m)
        for k in ("p", "m", "v"):
            assert all(np.array_equal(a, b) for a, b in zip(after[k], before[k]))
        assert np.array_equal(after["exist"], before["exist"]) and np.array_equal(after["denom"], before["denom"])
        assert m.adam_live_.all()


@pytest.mark.parametrize("P,cap", [(3001, 10_000), (4000, 4100)])
def test_grow_matches_the_restatement_and_stops_at_the_cap(cuda, P, cap):
    m = _state(P, 13, cuda, 0.1)
    before = _host(m)
    P_new = min(cap, int(math.floor(1.05 * P)))
    o = mcmc64.sigmoid(before["p"][3][:, 0])
    u = _safe_uniforms(_w32(before["p"][3][:, 0]), P_new - P, 6)
    want, picks, _ = mcmc64.grow(before, P_new, u, MIN_OP, iteration=9)
    assert m.addNewGaussians(cap, 1.05, MIN_OP, iteration=9, uniforms=torch.from_numpy(u)) == P_new - P
    torch.cuda.synchronize()
    assert m.num_points() == P_new and m.denom_.shape == (P_new, 1) and m.exist_since_iter_.shape == (P_new,) and not m.adam_live_valid_
    _compare(m, before, want, picks, np.arange(P, P_new), 9, P)
    if P_new == cap:
        xyz = m.xyz_
        assert m.addNewGaussians(cap, 1.05, MIN_OP) == 0 and m.xyz_ is xyz, "at the cap nothing happens"


def test_philox_draw_is_repeatable_and_proportional_to_opacity(cuda):
    from photo_slam_b200 import trainer
    n_alive, n_dead = 200, 100_000

    def make():
        sc = syn.make_scene(n_alive + n_dead, syn.make_camera(160, 120, 130.0, 130.0), seed=2)
        sc["opacity"][:] = -8.0
        sc["opacity"][:n_alive, 0] = np.random.default_rng(1).uniform(-2.5, 3.0, n_alive)
        sc["xyz"][:n_alive, 0] = np.arange(n_alive)            # the copies name their source
        m = trainer.GaussianModel.from_numpy(sc, cuda)
        m.trainingSetup(trainer.GaussianOptimizationParams())
        return m
    a, b, c = make(), make(), make()
    o = torch.sigmoid(a.opacity_[:n_alive, 0]).double().cpu().numpy()
    assert a.relocateGaussians(MIN_OP, seed=7, offset=3) == n_dead and b.relocateGaussians(MIN_OP, seed=7, offset=3) == n_dead
    c.relocateGaussians(MIN_OP, seed=7, offset=4)
    assert all(torch.equal(x, y) for x, y in zip(a.tensors(), b.tensors())), "same (seed, offset): identical replicas"
    assert not torch.equal(a.xyz_, c.xyz_), "another offset: another draw"
    src = a.xyz_[n_alive:, 0].round().long().cpu().numpy()
    count = np.bincount(src, minlength=n_alive)
    assert count.sum() == n_dead and count.min() > 0
    expect = n_dead * o / o.sum()
    chi2 = float(((count - expect) ** 2 / expect).sum())
    print(f"chi-square of {n_dead} picks over {n_alive} rows: {chi2:.1f} (199 degrees of freedom)")
    assert chi2 < 290.0, chi2                                  # P(chi2_199 > 290) ~ 3e-5


def test_relocation_preserves_the_picture(cuda):
    from photo_slam_b200 import trainer
    P, W, H = 20_000, 320, 240
    view = _views(cuda, W, H, 260.0, 1)[0]
    sc = syn.make_scene(P, syn.make_camera(W, H, 260.0, 260.0), seed=8, scale_px=3.0)
    sc["opacity"] = np.clip(sc["opacity"], -3.0, 1.5)
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    tr = trainer.GaussianTrainer(m)
    img0 = tr.render(view).clone()
    assert m.relocateGaussians(MIN_OP, seed=1) == 0
    assert torch.equal(tr.render(view), img0), "nothing dead: the picture is bit-identical"
    dead = torch.from_numpy(np.random.default_rng(4).random(P) < 0.002).to(cuda)
    m.opacity_[dead] = -8.0                                  # alpha < 1/255 everywhere: these rows draw nothing
    img1 = tr.render(view).clone()
    n = m.relocateGaussians(MIN_OP, seed=1)
    img2 = tr.render(view)
    diff = (img2 - img1).abs()
    print(f"relocated {n} of {P}: max |dI| = {diff.max().item() * 255:.3f}/255, pixels changed {100 * (diff.amax(0) > 0).float().mean().item():.1f} %")
    # the correction is exact at a splat's centre only: measured 2.17/255 at the worst pixel on an H100
    assert n == int(dead.sum()) and diff.max().item() < 3.0 / 255.0
    assert (diff.amax(0) == 0).float().mean().item() > 0.2, "pixels away from the relocated splats keep their bits"


def _noise_setup(cuda, P=6000, wh=(320, 240), mcmc=True, **kw):
    from photo_slam_b200 import trainer
    view = _views(cuda, wh[0], wh[1], 260.0, 1)[0]
    sc = syn.make_scene(P, syn.make_camera(wh[0], wh[1], 260.0, 260.0), seed=5, scale_px=4.0)
    sc["opacity"][::3] = -6.0                                 # a third nearly dead: o = 0.0025, g = 0.56
    opt = trainer.GaussianOptimizationParams(mcmc=mcmc, opacity_reg=0.0, scale_reg=0.0, **kw)
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.trainingSetup(opt)
    gt = torch.from_numpy(syn.target_image(wh[1], wh[0], seed=2)).to(cuda)
    return m, trainer.GaussianTrainer(m, opt, deterministic=True), view, gt


def test_noise_matches_the_restatement_and_skips_unseen_rows(cuda):
    m, tr, view, gt = _noise_setup(cuda, mcmc=False)
    radii = torch.zeros(m.num_points(), dtype=torch.int32, device=cuda)
    tr.trainForOneIteration(view, gt, radii=radii)
    tr.result()
    torch.cuda.synchronize()
    p = [t.detach().cpu().numpy().astype(np.float64) for t in m.tensors()]
    xyz0 = m.xyz_.clone()
    seen = (radii > 0).cpu().numpy()
    assert 0.3 < seen.mean() < 0.99
    L, cm, stream = tr.L, m._cmodel(False), torch.cuda.current_stream().cuda_stream
    lr, nlr = 1.6e-4, 5e5
    for visible_only in (1, 0):
        m.xyz_.copy_(xyz0)
        assert L.psb_trainer_inject_noise(tr.h, m.num_points(), C.byref(cm), lr, nlr, 9, 4, visible_only, stream) == 0
        first = m.xyz_.clone()
        m.xyz_.copy_(xyz0)
        assert L.psb_trainer_inject_noise(tr.h, m.num_points(), C.byref(cm), lr, nlr, 9, 4, visible_only, stream) == 0
        assert torch.equal(m.xyz_, first), "bit-identical between runs"
        rows = np.nonzero(seen)[0] if visible_only else None
        want = mcmc64.noise(p[0], p[3][:, 0], p[4], p[5], lr, nlr, seed=9, step=4, rows=rows)
        mine = first.double().cpu().numpy()
        step = np.linalg.norm(want - p[0], axis=1)
        err = np.linalg.norm(mine - want, axis=1)
        # 1e-6 of the position, 1e-4 of the step: g(o) amplifies the float32 rounding of o a hundredfold
        tol = 1e-6 * np.linalg.norm(want, axis=1) + 1e-4 * step
        print(f"visible_only={visible_only}: largest step {step.max():.3e}, max error / tolerance = {(err / tol).max():.2e}")
        assert (err <= tol).all()
        assert step.max() > 1e-4, "the case must move something"
        if visible_only:
            assert torch.equal(first[torch.from_numpy(~seen).to(cuda)], xyz0[torch.from_numpy(~seen).to(cuda)])
            assert not torch.equal(first, xyz0)
    m.xyz_.copy_(xyz0)
    assert L.psb_trainer_inject_noise(tr.h, m.num_points(), C.byref(cm), lr, nlr, 9, 5, 0, stream) == 0
    assert not torch.equal(m.xyz_, first), "another step: another draw"
    assert L.psb_trainer_inject_noise(tr.h, m.num_points() - 1, C.byref(cm), lr, nlr, 9, 5, 0, stream) == -1


def test_noise_is_added_once_when_the_step_overflows_and_is_repeated(cuda):
    from helpers import scene_tensors
    from photo_slam_b200 import trainer
    P, wh = 2_000, (640, 480)
    cam, sc, act, g, c = scene_tensors(P, "tum", seed=2, pose_seed=None, dev=cuda, wh=wh, scale_px=150.0)
    sc["opacity"][::2] = -6.0
    gt = torch.rand((3, wh[1], wh[0]), device=cuda)
    opt = trainer.GaussianOptimizationParams(mcmc=True)
    models = []
    for warm in (False, True):
        m = trainer.GaussianModel.from_numpy(sc, cuda)
        m.trainingSetup(opt)
        tr = trainer.GaussianTrainer(m, opt, deterministic=True)
        if warm:                        # grows the arena before the training step
            tr.render(c)
            tr.render(c)
        tr.trainForOneIteration(c, gt)
        n = tr.result()[3]
        torch.cuda.synchronize()
        assert n > 6 * P + 65536 and m.step_ == 1
        models.append(m)
    a, b = models
    for x, y in zip(a.tensors() + a.exp_avg_, b.tensors() + b.exp_avg_):
        assert torch.equal(x, y), "the repeated step ends where the step that fitted ends: noise once"
    plain = trainer.GaussianModel.from_numpy(sc, cuda)
    plain.trainingSetup(trainer.GaussianOptimizationParams())
    tp = trainer.GaussianTrainer(plain, deterministic=True)
    tp.trainForOneIteration(c, gt)
    tp.result()
    assert not torch.equal(plain.xyz_, a.xyz_), "with mcmc the positions carry the noise"


def opt_lr(opt):
    return [opt.position_lr_init, opt.feature_lr, opt.feature_lr / 20.0, opt.opacity_lr, opt.scaling_lr, opt.rotation_lr]


def _grads(tr, m, view, dL):
    tr.render(view)
    gs = [torch.zeros_like(t) for t in m.tensors()]
    tr.backwardPixels(dL, grads=gs, densify_stats=False)
    torch.cuda.synchronize()
    return gs


def test_regularisers_add_the_closed_form_on_the_rows_the_pass_updates(cuda):
    from photo_slam_b200 import _lib
    m, tr, view, gt = _noise_setup(cuda, P=30_000, mcmc=False)
    P = m.num_points()
    dL = (torch.rand((3, view["H"], view["W"]), device=cuda, generator=torch.Generator(device=cuda).manual_seed(1)) - 0.5) / (view["H"] * view["W"])
    g0 = _grads(tr, m, view, dL)
    lam_o, lam_s = 1.0, 2.0
    _lib.check(tr.L.psb_trainer_set_regularizers(tr.h, lam_o, lam_s), "psb_trainer_set_regularizers")
    g1 = _grads(tr, m, view, dL)
    _lib.check(tr.L.psb_trainer_set_regularizers(tr.h, 0.0, 0.0), "psb_trainer_set_regularizers")
    g2 = _grads(tr, m, view, dL)
    assert all(torch.equal(a, b) for a, b in zip(g0, g2)), "lambda = 0: the plain gradients bit for bit (deterministic mode)"
    reached = torch.zeros(P, dtype=torch.bool, device=cuda)
    for g in g0:
        reached |= (g.reshape(P, -1) != 0).any(1)
    assert 0.2 < reached.float().mean().item() < 0.95
    for q in (0, 1, 2, 5):
        assert torch.equal(g0[q], g1[q]), "only opacity and scaling are regularised"
    assert torch.equal(g0[3][~reached], g1[3][~reached]) and torch.equal(g0[4][~reached], g1[4][~reached]) and not g1[3][~reached].any()
    o = torch.sigmoid(m.opacity_.double())
    s = torch.exp(m.scaling_.double())
    for mine, base, closed, lam in ((g1[3], g0[3], lam_o / P * o * (1 - o), lam_o), (g1[4], g0[4], lam_s / P * s, lam_s)):
        d = (mine.double() - base.double())[reached]
        # float32: the rounding of the sum, of the product, and of 1 - o where the opacity saturates
        tol = 2.0 ** -22 * (base.double().abs()[reached] + closed[reached]) + 1e-6 * closed[reached] + 2e-7 * lam / P
        assert ((d - closed[reached]).abs() <= tol).all(), ((d - closed[reached]).abs() / tol).max().item()


@pytest.mark.parametrize("antialiasing", [False, True])
def test_the_two_fused_adam_variants_agree_with_regularisers_depth_and_antialiasing(cuda, antialiasing):
    from photo_slam_b200 import _lib, trainer
    P, W, H = 20_000, 320, 240
    view = _views(cuda, W, H, 260.0, 1)[0]
    sc = syn.make_scene(P, syn.make_camera(W, H, 260.0, 260.0), seed=5, scale_px=4.0)
    sc["xyz"][::2, 0] += 1000.0                                # half of the rows are never reached
    gt = torch.from_numpy(syn.target_image(H, W, seed=2)).to(cuda)
    gt_depth = torch.rand((H, W), device=cuda, generator=torch.Generator(device=cuda).manual_seed(3)) * 4 + 1
    opt = trainer.GaussianOptimizationParams(mcmc=True, mcmc_noise_lr=0.0)
    out = []
    for live in (True, False):
        m = trainer.GaussianModel.from_numpy(sc, cuda)
        m.trainingSetup(opt)
        tr = trainer.GaussianTrainer(m, opt, deterministic=True, antialiasing=antialiasing)
        for k in range(8):
            if live:
                tr.trainForOneIteration(view, gt, gt_depth=gt_depth, lambda_depth=0.1)
            else:                                              # adam_live = NULL: the variant that reads the moments to find idle rows
                cm, cc, cs = m._cmodel(), trainer._ccamera(view), tr._cstep(True)
                d = trainer._Depth(gt_depth.data_ptr(), 0.1, None)
                _lib.check(tr.L.psb_trainer_step_depth(tr.h, P, 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), None, C.byref(cs),
                                                       None, None, C.byref(d), torch.cuda.current_stream().cuda_stream), "psb_trainer_step_depth")
                m.step_ += 1
            tr.result()
        torch.cuda.synchronize()
        out.append(m)
    a, b = out
    for i, (x, y) in enumerate(zip(a.tensors(), b.tensors())):     # two compilations of the same arithmetic: equal up to float contraction
        frac = ((x - y).abs() > 0.5 * opt_lr(opt)[i]).float().mean().item()
        assert frac < 2e-3, f"{trainer.GROUPS[i]}: {frac} of entries differ by more than half an Adam step"
    for x, y in zip(a.exp_avg_ + a.exp_avg_sq_, b.exp_avg_ + b.exp_avg_sq_):
        assert ((x.double() - y.double()).norm() / (y.double().norm() + 1e-30)).item() < 1e-4
    # and the regularisers were there: the same 8 steps without them end elsewhere
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    tr = trainer.GaussianTrainer(m, deterministic=True, antialiasing=antialiasing)
    for k in range(8):
        tr.trainForOneIteration(view, gt, gt_depth=gt_depth, lambda_depth=0.1)
        tr.result()
    assert not torch.equal(m.opacity_, a.opacity_) and torch.equal(m.xyz_[::2], a.xyz_[::2])


def test_capped_training_end_to_end(cuda):
    """600 steps over 6 keyframes from 20 k rows under a cap of 40 k, mcmcRefine every 100 (growth 1.2 per round, so that the cap is
    reached within the run), against the same run with densifyAndPrune every 100 until it holds as many rows."""
    from photo_slam_b200 import trainer
    P, W, H, fx, cap = 25_000, 320, 240, 260.0, 40_000
    views = _views(cuda, W, H, fx, 6)
    gt_scene = syn.make_scene(P, syn.make_camera(W, H, fx, fx), seed=21, scale_px=3.0)
    gt_tr = trainer.GaussianTrainer(trainer.GaussianModel.from_numpy(gt_scene, cuda))
    gts = [gt_tr.render(c).clamp(0, 1).clone() for c in views]
    start = syn.thinned_trainee(gt_scene)
    start["opacity"][::50] = -6.0                              # 2 % dead on arrival (o = 0.0025), as after an insertion that did not take

    def run(mcmc):
        opt = trainer.GaussianOptimizationParams(mcmc=mcmc, cap_max=cap, mcmc_grow_factor=1.2)
        m = trainer.GaussianModel.from_numpy(start, cuda)
        m.trainingSetup(opt)
        m.lr_ = list(LRS)
        tr = trainer.GaussianTrainer(m, opt)
        psnr = lambda: float(np.mean([10.0 * math.log10(1.0 / ((tr.render(c) - g) ** 2).mean().item()) for c, g in zip(views, gts)]))
        p0, log = psnr(), []
        for it in range(1, 601):
            tr.trainForOneIteration(views[it % 6], gts[it % 6])
            tr.result()
            assert m.num_points() <= cap
            if it % 100 == 0 and it <= 500:
                if mcmc:
                    dead0 = int((torch.sigmoid(m.opacity_) <= MIN_OP).sum())
                    n_rel, n_add = tr.mcmcRefine()
                    dead1 = int((torch.sigmoid(m.opacity_) <= MIN_OP).sum())
                    assert abs(n_rel - dead0) <= 2 and dead1 <= max(2, dead0 // 20), (n_rel, dead0, dead1)   # (torch's sigmoid vs the kernel's at the threshold)
                    log.append((it, dead0, dead1, n_add, m.num_points()))
                elif m.num_points() < cap:
                    grads = (m.xyz_gradient_accum_ / m.denom_).nan_to_num(0.0).squeeze()
                    tau = float(torch.quantile(grads[grads > 0], 0.8))
                    m.densifyAndPrune(tau, MIN_OP, 1.0, 20, seed=5)
                    log.append((it, m.num_points()))
        torch.cuda.synchronize()
        return p0, psnr(), m.num_points(), log
    p0, p_mcmc, n_mcmc, log_mcmc = run(True)
    _, p_base, n_base, log_base = run(False)
    print(f"PSNR start {p0:.3f} dB -> capped (mcmc) {p_mcmc:.3f} dB with {n_mcmc} rows, densifyAndPrune {p_base:.3f} dB with {n_base} rows")
    print("  mcmcRefine (iteration, dead before, dead after, added, rows):", log_mcmc)
    print("  densifyAndPrune (iteration, rows):", log_base)
    assert n_mcmc == cap, "the capped run reaches its cap and stays there"
    assert sum(d0 for _, d0, _, _, _ in log_mcmc) > 0, "the run must relocate something"
    # measured on an H100 (two runs): 17.14 dB at the start, 31.9 / 32.3 dB capped (40 000 rows), 35.5 dB with densifyAndPrune (28 500 rows). On this scene (a
    # perturbed copy of the target) every refinement disturbs rows that already fit: the bound is set from that measurement
    assert p_mcmc > p0 + 10.0 and p_mcmc > p_base - 4.5, (p0, p_mcmc, p_base)
