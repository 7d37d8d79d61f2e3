"""CPU: the session truth of tests/session64.py against itself and against independent statements: a session without surgery is chained
step64 steps, each row restatement agrees with the C oracle (oracle_c) or ref_densify where both exist, the float64 3-NN with
oracle_c.knn_mean_dist2, the learning-rate schedule with GaussianModel.exponLrFunc, and every perturbed convention changes the result."""
import dataclasses
import math

import numpy as np
import pytest
import torch

import oracle_c
import session64
import step64
from test_step64_cpu import _scene, _state, _targets


@pytest.fixture(scope="module")
def world():
    import splat64 as s64
    sc, cam = _scene()
    return sc, s64.camera64(cam, "cpu"), _targets()


def _opt(**kw):
    from photo_slam_b200 import trainer
    return trainer.GaussianOptimizationParams(**dict(dict(position_lr_init=3.2e-4, position_lr_final=3.2e-5, position_lr_max_steps=30), **kw))


def _rows(P, seed):
    """a float32-valued row state with moments and statistics (some rows never seen)"""
    rng = np.random.default_rng(seed)
    f = lambda *s: torch.from_numpy(np.float32(rng.normal(size=s))).double()
    p = [f(P, 3), f(P, 1, 3), f(P, 15, 3), f(P, 1), f(P, 3) - 3.0, f(P, 4)]
    m = [f(*t.shape) for t in p]
    v = [f(*t.shape).abs() for t in p]
    accum = torch.from_numpy(np.float32(rng.uniform(0, 0.004, (P, 1)))).double()
    denom = torch.full((P, 1), 2.0, dtype=torch.float64)
    accum[::7], denom[::7] = 0.0, 0.0
    return dict(p=p, m=m, v=v, accum=accum, denom=denom, max_radii=torch.from_numpy(np.float32(rng.uniform(0, 50, P))).double())


def test_expon_lr_closed_forms():
    """the schedule's closed forms: lr_init at 0, lr_final from max_steps on, the geometric mean half way, the delay ramp's ends"""
    i, f, n = 3.2e-4, 3.2e-5, 30
    lr = lambda step, d=0: session64.expon_lr(step, i, f, 0.01, n, d)
    assert lr(0) == pytest.approx(i, rel=1e-14) and lr(n) == pytest.approx(f, rel=1e-14) and lr(5 * n) == pytest.approx(f, rel=1e-14)
    assert lr(n / 2) == pytest.approx(math.sqrt(i * f), rel=1e-14) and lr(n / 3) == pytest.approx(i ** (2 / 3) * f ** (1 / 3), rel=1e-14)
    assert lr(-1) == 0.0 and session64.expon_lr(3, 0.0, 0.0, 0.01, n) == 0.0
    assert lr(0, 10) == pytest.approx(0.01 * i, rel=1e-14) and lr(10, 10) == pytest.approx(lr(10), rel=1e-14)
    assert lr(5, 10) == pytest.approx((0.01 + 0.99 * math.sin(math.pi / 4)) * lr(5), rel=1e-14)
    assert lr(1) < 0.95 * i, "the schedule must move measurably per step"


def test_expon_lr_is_exponlrfunc():
    from photo_slam_b200 import trainer
    for kw in (dict(), dict(position_lr_max_steps=7)):
        o = _opt(**kw)
        m = trainer.GaussianModel(device="cpu")
        m.xyz_ = torch.zeros((0, 3))
        m.features_dc_, m.features_rest_ = torch.zeros((0, 1, 3)), torch.zeros((0, 15, 3))
        m.opacity_, m.scaling_, m.rotation_ = torch.zeros((0, 1)), torch.zeros((0, 3)), torch.zeros((0, 4))
        m.trainingSetup(o)
        ses = session64.Session(o, 0)
        for step in (-1, 0, 1, 3, 7, 15, 30, 31, 100):
            assert math.isclose(ses.update_lr(step), m.updateLearningRate(step), rel_tol=1e-15, abs_tol=0.0), step


def test_session_without_surgery_is_chained_step64(world):
    sc, cam, tg = world
    fl = step64.Flags(depth=True, f3d=True)
    st = _state(sc)
    o = _opt()
    ses = session64.Session(o, 1)
    ses.set_filter(st["f"])
    ses.set_lr("opacity", 0.03)
    a = b = st
    for i in range(3):
        ses.update_lr(a["step"])
        if i == 2:
            ses.set_sh(2)
        a = ses.step(a, cam, tg, fl)["state"]
        lr = [session64.expon_lr(b["step"], o.position_lr_init, o.position_lr_final, o.position_lr_delay_mult, o.position_lr_max_steps),
              o.feature_lr, o.feature_lr / 20.0, 0.03, o.scaling_lr, o.rotation_lr]
        b = step64.step64(dict(b, lr=lr, D=2 if i == 2 else 1), cam, tg, fl)["state"]
    for k in step64.GROUPS:
        for key in ("params", "m", "v"):
            assert torch.equal(a[key][k], b[key][k]), (key, k)
    assert torch.equal(a["accum"], b["accum"]) and torch.equal(a["E"], b["E"])


def test_densify_against_the_c_oracle_and_the_parent_map():
    P, extent, tau = 600, 5.0, 0.001
    r = _rows(P, 3)
    r["p"][4][::9] = math.log(0.2)                 # large rows: split
    ns = int((((r["accum"] / r["denom"]).nan_to_num(0.0).reshape(-1) >= tau) & (torch.exp(r["p"][4]).max(1).values > 0.01 * extent)).sum())
    assert ns > 5
    z = torch.from_numpy(np.float32(np.random.default_rng(1).normal(size=(2 * ns, 3)))).double()
    want, parents, K0 = session64.densify(r, z, tau, 0.0, extent, 0, 0.01)
    host = lambda ts: [np.float32(t.numpy()) for t in ts]
    op, om, ov = oracle_c.densify_and_prune(host(r["p"]), host(r["m"]), host(r["v"]), np.float32(r["accum"].numpy()), np.float32(r["denom"].numpy()),
                                            np.float32(r["max_radii"].numpy()), tau, 0.0, extent, 0, 0.01, np.float32(z.numpy()))
    for a, c in zip(want["p"] + want["m"] + want["v"], op + om + ov):
        np.testing.assert_allclose(a.numpy(), c, rtol=1e-6, atol=1e-6)
    assert K0 == P - ns and parents.numel() == want["p"][0].shape[0] > P
    for q in (1, 2, 3, 5):                         # copies of their parent
        assert torch.equal(want["p"][q], r["p"][q][parents])
    for q in range(6):                             # survivors keep their moments, new rows start from zero
        assert torch.equal(want["m"][q][:K0], r["m"][q][parents[:K0]]) and not want["m"][q][K0:].any() and not want["v"][q][K0:].any()
    assert not want["accum"].any() and not want["denom"].any() and not want["max_radii"].any()


def test_prune_reset_and_transform_restatements():
    r = _rows(300, 4)
    mask = torch.from_numpy(np.random.default_rng(2).random(300) < 0.3)
    want = session64.prune(r, mask)
    for a, b in zip(want["p"] + want["m"] + want["v"] + [want["accum"], want["max_radii"]], r["p"] + r["m"] + r["v"] + [r["accum"], r["max_radii"]]):
        assert torch.equal(a, b[~mask])
    reset = session64.reset_opacity(r)
    np.testing.assert_allclose(reset["p"][3].numpy(), oracle_c.reset_opacity(np.float32(r["p"][3].numpy())), rtol=1e-6, atol=1e-6)
    assert not reset["m"][3].any() and torch.equal(reset["m"][0], r["m"][0])
    T = np.eye(4)
    T[:3, :3] = [[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]]
    T[:3, 3] = [1.0, 2.0, 3.0]
    t = session64.transform(r, 2.0, T)
    x = r["p"][0]
    assert torch.allclose(t["p"][0], torch.stack([-2 * x[:, 1] + 1, 2 * x[:, 0] + 2, 2 * x[:, 2] + 3], 1), rtol=0, atol=1e-12)
    assert torch.equal(t["p"][4], 2.0 * r["p"][4]) and not t["m"][0].any() and not t["v"][4].any() and torch.equal(t["m"][3], r["m"][3])


def test_knn_and_insert_against_the_c_oracle():
    rng = np.random.default_rng(5)
    pts = np.float32(rng.uniform(-1, 1, (301, 3)))
    np.testing.assert_allclose(session64.knn_mean_dist2(torch.from_numpy(pts).double()).numpy(), oracle_c.knn_mean_dist2(pts), rtol=2e-6)
    r = _rows(50, 6)
    cols = np.float32(rng.uniform(0, 1, (301, 3)))
    want = session64.insert_points(r, torch.from_numpy(pts).double(), torch.from_numpy(cols).double())
    assert want["p"][0].shape[0] == 351 and torch.equal(want["p"][0][50:], torch.from_numpy(pts).double())
    for q in range(6):
        assert torch.equal(want["p"][q][:50], r["p"][q]) and torch.equal(want["m"][q][:50], r["m"][q]) and not want["m"][q][50:].any()
    assert torch.allclose(torch.sigmoid(want["p"][3][50:]), torch.full((301, 1), 0.1, dtype=torch.float64))
    assert not want["denom"].any() and not want["p"][2][50:].any()


def test_seed_rows_are_the_plan_with_the_insert_recipe():
    import seed64
    import photo_slam_b200.synthetic as syn
    from test_seed_cpu import _planes
    A, D, G, mask = _planes()
    H, W = A.shape
    cam = syn.make_camera(W, H, 25.0, 25.0)
    img = np.random.default_rng(3).uniform(0, 1, (3, H, W))
    plan = seed64.seed(cam, A, D, G, img, mask, stride=2, max_new=17)
    r = _rows(40, 9)
    want = session64.seed_rows(r, plan)
    n = plan["n"]
    assert n == 17 and want["p"][0].shape[0] == 40 + n
    for q, key in ((0, "xyz"), (4, "scaling"), (5, "rotation")):
        assert torch.equal(want["p"][q][40:], torch.from_numpy(plan[key]).double()), key
    assert torch.equal(want["p"][1][40:, 0], torch.from_numpy(plan["features_dc"]).double())
    assert torch.equal(want["p"][3][40:, 0], torch.from_numpy(plan["opacity"]).double())
    for q in range(6):
        assert torch.equal(want["p"][q][:40], r["p"][q]) and torch.equal(want["v"][q][:40], r["v"][q]) and not want["v"][q][40:].any()
    assert not want["accum"].any() and not want["max_radii"].any()


def test_relocate_and_grow_new_rows_start_from_zero_or_inherit():
    """the wrappers' own rule on top of mcmc64: the rows they write (dead rows, grown rows) start with zero moments, or with their
    source's moments under the perturbed convention"""
    r = _rows(200, 7)
    model = dict(p=[t.numpy() for t in r["p"]], m=[t.numpy() for t in r["m"]], v=[t.numpy() for t in r["v"]], accum=r["accum"].numpy(),
                 denom=r["denom"].numpy(), max_radii=r["max_radii"].numpy(), exist=np.arange(200, dtype=np.int32))
    model["p"][3][:30] = -8.0
    u = np.float32(np.random.default_rng(8).random(200))
    inherit = dataclasses.replace(session64.SESSION_CONV, new_moments_zero=False)
    a, picks, dead = session64.relocate(model, u, 0.005, 3)
    b, picks_b, dead_b = session64.relocate(model, u, 0.005, 3, inherit)
    assert len(dead) == 30 and np.array_equal(dead, dead_b) and np.array_equal(picks, picks_b)
    for q in range(6):
        assert not a["m"][q][dead].any() and not a["v"][q][dead].any()
        assert np.array_equal(b["m"][q][dead], model["m"][q][picks]) and np.array_equal(b["v"][q][dead], model["v"][q][picks])
        assert np.array_equal(a["p"][q][dead], a["p"][q][picks]), "a relocated row is a copy of its corrected source"
    g, gp = session64.grow(model, 210, u, 0.005, 3)
    h, hp = session64.grow(model, 210, u, 0.005, 3, inherit)
    assert g["p"][0].shape[0] == 210 and np.array_equal(gp, hp)
    for q in range(6):
        assert not g["m"][q][200:].any() and np.array_equal(h["m"][q][200:], model["m"][q][gp])
        assert np.array_equal(g["p"][q][200:], g["p"][q][gp])


def test_each_perturbation_changes_the_result(world):
    sc, cam, tg = world
    fl = step64.Flags(f3d=True)
    st = _state(sc)
    o = _opt()
    base = session64.SESSION_CONV
    # new rows inherit their parent's moments
    r = _rows(300, 3)
    r["p"][4][::9] = math.log(0.2)
    ns = int((((r["accum"] / r["denom"]).nan_to_num(0.0).reshape(-1) >= 0.001) & (torch.exp(r["p"][4]).max(1).values > 0.05)).sum())
    z = torch.zeros((2 * ns, 3), dtype=torch.float64)
    a, _, K0 = session64.densify(r, z, 0.001, 0.0, 5.0, 0, 0.01)
    b, _, _ = session64.densify(r, z, 0.001, 0.0, 5.0, 0, 0.01, dataclasses.replace(base, new_moments_zero=False))
    assert not a["m"][0][K0:].any() and b["m"][0][K0:].abs().min() > 0
    # the xyz lr held at lr_init
    s1, s2 = session64.Session(o, 1), session64.Session(o, 1, dataclasses.replace(base, lr_schedule=False))
    assert s1.update_lr(8) < 0.6 * s2.update_lr(8) and s2.lr[0] == o.position_lr_init
    # the 3D filter of the pre-surgery rows stays in force
    s1, s2 = session64.Session(o, 1), session64.Session(o, 1, dataclasses.replace(base, filter_current=False))
    for s in (s1, s2):
        s.set_filter(st["f"])
        s.set_filter(2.0 * st["f"])
    assert torch.equal(s1.f, 2.0 * st["f"]) and torch.equal(s2.f, st["f"])
    l1, l2 = (s.step(st, cam, tg, fl)["loss"]["loss"] for s in (s1, s2))
    assert abs(l1 - l2) > 1e-6 * abs(l1)
    # the SH degree left at 2
    s1, s2 = session64.Session(o, 2), session64.Session(o, 2, dataclasses.replace(base, sh_raise=False))
    for s in (s1, s2):
        s.set_sh(3)
    assert (s1.D, s2.D) == (3, 2)
    l1, l2 = (s.step(st, cam, tg, step64.Flags())["loss"]["loss"] for s in (s1, s2))
    assert abs(l1 - l2) > 1e-6 * abs(l1)
