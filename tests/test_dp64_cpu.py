"""CPU: tests/step64.py's optional consistency (dn) and distortion (dist) terms, the truth the data-parallel steps with those terms are
measured against (tests/test_dp64_gpu.py): with both off the step is the one without them bit for bit; with them on its loss scalars are
dn64 and dist64 of the planes it renders, its raw-parameter gradients match central finite differences, and `margins` reports the
consistency term's alpha and depth-jump decisions where they lie."""
import dataclasses

import pytest
import torch

import dist64
import dn64
import step64
from test_step64_cpu import BG, D, H, P, W, _check_fd, _scene, _state, _targets

LAMBDA_DN, LAMBDA_DIST, ALPHA_MIN, JUMP = 0.3, 0.2, 0.5, 0.05


@pytest.fixture(scope="module")
def world():
    import splat64 as s64
    sc, cam = _scene()
    return sc, s64.camera64(cam, "cpu"), _terms(_targets())


def _terms(tg, **kw):
    return dict(tg, lambda_dn=LAMBDA_DN, dn_alpha_min=ALPHA_MIN, dn_max_rel_jump=JUMP, lambda_dist=LAMBDA_DIST, **kw)


def _same_step(a, b, skip=()):
    for k in set(a["loss"]) - set(skip):
        assert a["loss"][k] == b["loss"][k], k
    for part in ("params", "m", "v"):
        for k in step64.GROUPS:
            assert torch.equal(a["state"][part][k], b["state"][part][k]), (part, k)
    for k in ("accum", "denom", "max_radii", "E", "E_m", "E_v"):
        assert torch.equal(a["state"][k], b["state"][k]), k
    assert torch.equal(a["reached"], b["reached"])


@pytest.mark.parametrize("k", [0, 3, 17, 31])
def test_terms_off_is_the_step_without_them_bit_for_bit(world, k):
    """flags without dn and dist: the step ignores the terms' targets entirely; dL/dA and dL/dM of the render are zero"""
    sc, cam, tg = world
    fl = step64.ALL_FLAGS[k]
    plain = {q: v for q, v in tg.items() if q not in ("lambda_dn", "dn_alpha_min", "dn_max_rel_jump", "lambda_dist")}
    a = step64.step64(_state(sc), cam, plain, fl)
    b = step64.step64(_state(sc), cam, dict(tg, colour=True), fl)
    _same_step(a, b)
    assert a["loss"]["dn"] == 0.0 and a["loss"]["dist"] == 0.0
    assert not a["pixel"]["alpha"].any() and a["pixel"]["depth2"] is None and "depth2" not in a["out"]
    assert set(step64.margins(_state(sc), cam, tg, fl)) == set(step64.margins(_state(sc), cam, plain, fl))


def test_terms_at_zero_weight_leave_the_step(world):
    """dn and dist on at lambda 0: every other scalar, parameter, moment and statistic equals the step without them bit for bit"""
    sc, cam, tg = world
    base = step64.Flags(depth=True, normal=True, aa=True)
    a = step64.step64(_state(sc), cam, tg, base)
    b = step64.step64(_state(sc), cam, dict(tg, lambda_dn=0.0, lambda_dist=0.0), dataclasses.replace(base, dn=True, dist=True))
    _same_step(a, b, skip=("dn", "dist"))
    assert b["loss"]["dn"] > 0 and b["loss"]["dist"] > 0


@pytest.mark.parametrize("aa", [False, True])
def test_loss_scalars_are_dn64_and_dist64_of_the_rendered_planes(world, aa):
    sc, cam, tg = world
    st = _state(sc)
    fl = step64.Flags(depth=True, normal=True, dn=True, dist=True, aa=aa)
    r = step64.grads64(st, cam, tg, fl)
    out, N = r["out"], r["N"]
    M = out["depth2"]
    # the second moment is dist64.render_moment's (its own blend of the unfiltered splat)
    raw = {k: v.clone() for k, v in st["params"].items()}
    _, M_ref = dist64.render_moment(raw, cam, D=D, aa=aa)
    assert torch.allclose(M, M_ref, rtol=1e-13, atol=1e-15)
    dn, nv, nd = dn64.dn64(out["depth"], out["alpha"], N, W, H, cam["tanfovx"], cam["tanfovy"], ALPHA_MIN, JUMP, tg["mask"])
    dist, nvd = dist64.dist64(out["depth"], out["alpha"], M, tg["mask"])
    assert r["loss"]["dn"] == float(dn.detach()) and r["loss"]["dist"] == float(dist.detach())
    assert 0 < nv < nvd == int((tg["mask"][0] != 0).sum()), "some mask-valid pixels have a depth normal, others not"
    plain = step64.grads64(st, cam, tg, step64.Flags(depth=True, normal=True, aa=aa))["loss"]["loss"]
    assert abs(r["loss"]["loss"] - (plain + LAMBDA_DN * r["loss"]["dn"] + LAMBDA_DIST * r["loss"]["dist"])) <= 1e-14 * r["loss"]["loss"]
    # the per-pixel gradients: dist's closed form on dL/dM, and dL/dA only where a term reads A
    gA, gD, gM = dist64.grads64(out["depth"].detach(), out["alpha"].detach(), M.detach(), LAMBDA_DIST, tg["mask"])
    assert torch.allclose(r["pixel"]["depth2"], gM, rtol=1e-13, atol=0)
    assert r["pixel"]["alpha"].abs().sum() > 0


def _loss_fn(state, cam, targets, flags, conv=step64.STEP_CONV):
    def L(raw):
        out, N, _ = step64.forward(raw, cam, flags, state["D"], targets["bg"], None, conv)
        return step64.image_loss(out, N, targets, flags, state["E"], cam)[0]
    return L


TERMS = {"dn": step64.Flags(dn=True), "dist": step64.Flags(dist=True), "all": step64.Flags(depth=True, normal=True, dn=True, dist=True, aa=True)}


@pytest.mark.parametrize("name", list(TERMS))
@pytest.mark.parametrize("colour", [True, False], ids=["colour", "terms-only"])
def test_terms_against_finite_differences(world, name, colour):
    sc, cam, tg = world
    st = _state(sc)
    fl = TERMS[name]
    tg = dict(tg, colour=colour)
    mg = step64.margins(st, cam, tg, fl)
    for q in ("dn_alpha", "dn_jump", "axis", "flip"):
        if q in mg:
            assert float(mg[q][0].min()) > 1e-4, (q, float(mg[q][0].min()))
    r = step64.grads64(st, cam, tg, fl)
    assert r["reached"].any()
    if not colour:
        # no photometric term: the colour of every row is untouched, and every row the pass reaches is reached through n or z
        assert not r["grads"]["features_dc"].any() and not r["grads"]["features_rest"].any() and not r["inter"]["rgb"].any()
        via = torch.zeros(P, dtype=torch.bool)
        if "n" in r["inter"]:
            via |= (r["inter"]["n"] != 0).any(1)
        if fl.dist or fl.dn:
            via |= r["inter"]["z"] != 0
        assert torch.equal(via | r["reached"], via)
    _check_fd(_loss_fn(st, cam, tg, fl), st["params"], r["grads"], ("xyz", "opacity", "scaling", "rotation") + (("features_dc",) if colour else ()))


def test_dist_without_dz_and_dn_dropped_change_the_gradient(world):
    """the perturbed truths of the GPU suite are different truths: dist without 2 z dL/dM on dz moves dL/dxyz; dropping dn moves
    dL/drotation"""
    sc, cam, tg = world
    st = _state(sc)
    a = step64.grads64(st, cam, tg, step64.Flags(dist=True))["grads"]["xyz"]
    b = step64.grads64(st, cam, tg, step64.Flags(dist=True), step64.StepConv(dist_dz=False))["grads"]["xyz"]
    assert (a - b).norm() > 1e-3 * a.norm()
    a = step64.grads64(st, cam, tg, step64.Flags(normal=True, dn=True))["grads"]["rotation"]
    b = step64.grads64(st, cam, tg, step64.Flags(normal=True))["grads"]["rotation"]
    assert (a - b).norm() > 1e-3 * a.norm()


def test_margins_report_the_consistency_decisions(world):
    """dn_alpha and dn_jump exist with the term; moving alpha_min (max_rel_jump) onto a pixel's A (a pair's relative jump) makes that
    decision's margin zero, charged to the pixel's last blended Gaussian"""
    sc, cam, tg = world
    st = _state(sc)
    fl = step64.Flags(dn=True)
    mg = step64.margins(st, cam, tg, fl)
    assert {"dn_alpha", "dn_jump", "axis", "flip"} <= set(mg) and "normal_kink" not in mg
    for q in ("dn_alpha", "dn_jump"):
        v, ids = mg[q]
        assert v.numel() > 0 and (v >= 0).all() and ((ids >= 0) & (ids < P)).all()
    assert "dn_alpha" not in step64.margins(st, cam, tg, step64.Flags(dist=True))
    out, _, _ = step64.forward(st["params"], cam, fl, D, BG)
    A, last, Dp = out["alpha"], out["last"], out["depth"]
    y, x = H // 2, W // 2
    while A[y, x] <= 0.05:
        x += 1
    pa = step64.margins(st, cam, dict(tg, dn_alpha_min=float(A[y, x])), fl)["dn_alpha"]
    assert float(pa[0].min()) < 1e-12 and int(last[y, x]) in pa[1][pa[0] < 1e-12].tolist()
    z = dn64.normalised_depth(Dp, A, ALPHA_MIN)
    mask = tg["mask"][0] != 0
    pairs = [(yy, xx) for yy in range(1, H - 1) for xx in range(1, W - 2) if mask[yy, xx] and z[yy, xx] > 0 and z[yy, xx + 1] > 0
             and z[yy, xx + 1] != z[yy, xx]]
    yy, xx = pairs[len(pairs) // 2]
    j = float((z[yy, xx + 1] - z[yy, xx]).abs() / z[yy, xx])
    pj = step64.margins(st, cam, dict(tg, dn_max_rel_jump=j), fl)["dn_jump"]
    hit = pj[1][pj[0] < 1e-9].tolist()
    assert int(last[yy, xx]) in hit and int(last[yy, xx + 1]) in hit


# ---- dp_step64: the truth of the multi-rank step ------------------------------------------------------------------------------------
def _same_update(a, b):
    for part in ("params", "m", "v"):
        for k in step64.GROUPS:
            assert torch.equal(a[part][k], b[part][k]), (part, k)


def test_dp_step_of_one_view_is_the_step(world):
    """world 1, and world 2 with the same view on both ranks ((g + g) / 2 = g): the parameters and moments of step64, bit for bit"""
    sc, cam, tg = world
    fl = step64.Flags(normal=True, dn=True, dist=True)
    ref = step64.step64(_state(sc), cam, tg, fl)["state"]
    _same_update(step64.dp_step64(_state(sc), [(cam, tg, fl)], 1)["state"], ref)
    _same_update(step64.dp_step64(_state(sc), [(cam, tg, fl)] * 2, 2)["state"], ref)


def test_dp_step_is_the_mean_gradient_and_a_dropped_view_adds_nothing(world):
    """two views with their own targets and terms: Adam takes (g_0 + g_1) / 2; with view 1 dropped g_0 / 2, and view 1 is not evaluated;
    scale overrides 1 / world"""
    sc, cam, tg = world
    views = [(cam, tg, step64.Flags(depth=True)), (cam, _terms(_targets(seed=5)), step64.Flags(dist=True, aa=True))]
    st = _state(sc)
    g = [step64.grads64(st, *v)["grads"] for v in views]
    both = step64.dp_step64(st, views, 2)
    one = step64.dp_step64(st, [views[0], None], 2, dropped=(1,))
    unscaled = step64.dp_step64(st, views, 2, per_view=both["views"], scale=1.0)
    assert one["views"][1] is None
    for i, k in enumerate(step64.GROUPS):
        assert torch.equal(both["grads"][k], (g[0][k] + g[1][k]) * 0.5)
        assert torch.equal(one["grads"][k], g[0][k] * 0.5)
        assert torch.equal(unscaled["grads"][k], g[0][k] + g[1][k])
        p, m, v = step64.adam64(st["params"][k], both["grads"][k], st["m"][k], st["v"][k], st["lr"][i], st["step"] + 1)
        assert torch.equal(both["state"]["params"][k], p) and torch.equal(both["state"]["m"][k], m) and torch.equal(both["state"]["v"][k], v)
    assert any(not torch.equal(g[0][k], g[1][k]) for k in step64.GROUPS)


def test_stats64_is_the_step_statistics(world):
    sc, cam, tg = world
    fl = step64.Flags(depth=True)
    st = _state(sc)
    r = step64.step64(st, cam, tg, fl)
    for k, t in step64.stats64(st, r).items():
        assert torch.equal(t, r["state"][k]), k
