"""CPU: the float64 training step of tests/step64.py checked against itself and against independent statements: central finite
differences of every term it adds (the 3D filter's widening, the regularisers, the NDC mean2D of the densification statistics, the normal
term), adam64 against torch.optim.Adam, and two reductions (all flags off: splat64's loss and gradients plus torch's Adam; a zero
filter: the unfiltered step bit for bit)."""
import dataclasses

import numpy as np
import pytest
import torch

import filter3d64
import photo_slam_b200.synthetic as syn
import splat64 as s64
import step64

W, H, P, D = 24, 20, 28, 2
BG = (0.2, 0.4, 0.1)


def _scene(seed=0):
    rng = np.random.default_rng(seed)
    cam = syn.make_camera(W, H, 22.0, 22.0)
    fx = 22.0
    z = 1.0 + 3.0 * (rng.permutation(P) + rng.uniform(0.3, 0.7, P)) / P
    u, v = rng.uniform(0, W, P), rng.uniform(0, H, P)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    sc = dict(xyz=f32(np.stack([(u - 0.5 * (W - 1)) / fx * z, (v - 0.5 * (H - 1)) / fx * z, z], 1)),
              features_dc=f32(((rng.uniform(0, 1, (P, 3)) - 0.5) / s64.SH_C0)[:, None]), features_rest=f32(rng.normal(0, 0.1, (P, 15, 3))),
              scaling=f32(np.log(3.0 / fx * z)[:, None] + rng.normal(0, 0.4, (P, 3))), rotation=f32(rng.normal(size=(P, 4))),
              opacity=f32(rng.normal(0.0, 1.0, (P, 1))))
    sc["xyz"][-2:, 2] *= -1.0                      # behind the camera
    sc["xyz"][-4:-2, 0] += 3.0 * sc["xyz"][-4:-2, 2]   # outside the view
    s64.settle(sc, cam, D=D, aa=None, bg=BG, seed=seed)
    return sc, cam


def _targets(seed=1):
    gen = torch.Generator().manual_seed(seed)
    gt = torch.rand((3, H, W), generator=gen, dtype=torch.float64)
    mask = (torch.rand((1, H, W), generator=gen) > 0.2).double().expand(3, H, W).contiguous()
    depth = 1.0 + 3.0 * torch.rand((H, W), generator=gen, dtype=torch.float64)
    depth[torch.rand((H, W), generator=gen) < 0.2] = 0.0
    n = torch.randn((3, H, W), generator=gen, dtype=torch.float64)
    n = n / n.norm(dim=0, keepdim=True)
    n[2] = -n[2].abs()
    n[:, torch.rand((H, W), generator=gen) < 0.2] = 0.0
    return dict(gt=gt, mask=mask, depth=depth, normal=n, lambda_depth=0.3, lambda_normal=0.4, bg=BG, lambda_dssim=0.2)


def _state(sc, seed=2, f=None, moments=True):
    gen = torch.Generator().manual_seed(seed)
    params = {k: torch.from_numpy(sc[k]).double() for k in step64.GROUPS}
    rnd = lambda t, s: s * torch.randn(t.shape, generator=gen, dtype=torch.float64)
    m = {k: (rnd(v, 1e-3) if moments else torch.zeros_like(v)) for k, v in params.items()}
    v = {k: (rnd(x, 1e-3) ** 2 if moments else torch.zeros_like(x)) for k, x in params.items()}
    E = torch.tensor([[1.1, 0.05, -0.04, 0.02], [0.03, 0.9, 0.05, -0.03], [-0.02, 0.04, 1.05, 0.01]], dtype=torch.float64)
    return dict(params=params, m=m, v=v, accum=torch.zeros(P, 1, dtype=torch.float64), denom=torch.zeros(P, 1, dtype=torch.float64),
                max_radii=torch.zeros(P, dtype=torch.float64), step=3, lr=[1.6e-4, 2.5e-3, 1.25e-4, 0.05, 5e-3, 1e-3], D=D,
                f=f if f is not None else 0.4 * torch.exp(params["scaling"]).mean(1), E=E, E_m=rnd(E, 1e-2), E_v=rnd(E, 1e-2) ** 2, E_step=1,
                E_lr=0.01)


@pytest.fixture(scope="module")
def world():
    sc, cam = _scene()
    return sc, s64.camera64(cam, "cpu"), _targets()


def _loss_fn(state, cam, targets, flags, E=True):
    def L(raw):
        out, N, _ = step64.forward(raw, cam, flags, state["D"], targets["bg"], state["f"])
        return step64.image_loss(out, N, targets, flags, state["E"] if E else None)[0]
    return L


def _fd(L, raw, k, idx, h=1e-6):
    a = {q: t.clone() for q, t in raw.items()}
    b = {q: t.clone() for q, t in raw.items()}
    a[k].view(-1)[idx] += h
    b[k].view(-1)[idx] -= h
    return (float(L(a)) - float(L(b))) / (2 * h)


def _check_fd(L, raw, grads, groups, n=6, seed=0, tol=2e-5):
    """central differences at the n entries of largest gradient of each group against the given gradients"""
    for k in groups:
        g = grads[k].reshape(-1)
        for idx in torch.argsort(g.abs(), descending=True)[:n].tolist():
            fd = _fd(L, raw, k, idx)
            assert abs(fd - float(g[idx])) <= tol * max(abs(fd), float(g.abs().max())), (k, idx, fd, float(g[idx]))


@pytest.mark.parametrize("aa", [False, True])
def test_widening_against_finite_differences(world, aa):
    sc, cam, tg = world
    st = _state(sc)
    fl = step64.Flags(f3d=True, aa=aa)
    r = step64.grads64(st, cam, tg, fl)
    assert r["reached"].sum() > P // 2
    _check_fd(_loss_fn(st, cam, tg, fl), st["params"], r["grads"], ("scaling", "opacity", "xyz", "rotation"))
    # the chain through (s', c) is the header's closed form (filter3d64.backward)
    s = torch.exp(st["params"]["scaling"]).requires_grad_(True)
    o = torch.sigmoid(st["params"]["opacity"]).reshape(-1).requires_grad_(True)
    gen = torch.Generator().manual_seed(5)
    a, b = torch.randn(P, 3, generator=gen, dtype=torch.float64), torch.randn(P, generator=gen, dtype=torch.float64)
    sp, c = step64.widen(s, st["f"])
    ((sp * a).sum() + (o * c * b).sum()).backward()
    ds, do = filter3d64.backward(s.detach().numpy(), o.detach().numpy(), st["f"].numpy(), a.numpy(), b.numpy())
    assert np.allclose(s.grad.numpy(), ds, rtol=1e-12, atol=1e-14) and np.allclose(o.grad.numpy(), do, rtol=1e-12, atol=1e-14)
    sp_ref, c_ref = filter3d64.widen(s.detach().numpy(), st["f"].numpy())
    assert np.allclose(sp.detach().numpy(), sp_ref, rtol=1e-14) and np.allclose(c.detach().numpy(), c_ref, rtol=1e-14)


def test_regularisers_against_finite_differences(world):
    sc, cam, tg = world
    st = _state(sc)
    fl = step64.Flags(reg=True, lambda_opacity=0.7, lambda_scale=0.3)
    plain = step64.grads64(st, cam, tg, step64.Flags())
    r = step64.grads64(st, cam, tg, fl)
    rows = r["reached"]
    assert rows.any() and (~rows).any(), "some rows are not reached (outside the view or hidden)"
    dg_o = r["grads"]["opacity"] - plain["grads"]["opacity"]
    dg_s = r["grads"]["scaling"] - plain["grads"]["scaling"]
    o, s = torch.sigmoid(st["params"]["opacity"]), torch.exp(st["params"]["scaling"])
    assert torch.allclose(dg_o, torch.where(rows[:, None], 0.7 / P * o * (1 - o), torch.zeros_like(o)), rtol=1e-10, atol=1e-18)
    assert torch.allclose(dg_s, torch.where(rows[:, None], 0.3 / P * s, torch.zeros_like(s)), rtol=1e-10, atol=1e-18)
    L = lambda raw: step64.regularizer(raw, rows, fl)
    for k, g in (("opacity", dg_o), ("scaling", dg_s)):
        for idx in range(0, g.numel(), 5):
            assert abs(_fd(L, st["params"], k, idx) - float(g.reshape(-1)[idx])) < 1e-7 * float(g.abs().max())


def test_ndc_mean2d_against_finite_differences(world):
    """xyz_gradient_accum's term: dL/dmean2D in NDC units, the derivative of the loss w.r.t. a shift of each splat's NDC centre"""
    sc, cam, tg = world
    st = _state(sc)
    fl = step64.Flags(depth=True, normal=True, aa=True)
    r = step64.grads64(st, cam, tg, fl)

    def L_shift(k, idx, h):
        g = step64.splat_inputs(st["params"], fl, st["f"])
        geo = s64.geometry(g, cam, D, fl.aa)
        delta = torch.zeros(P, 2, dtype=torch.float64)
        delta.view(-1)[2 * k + idx] = h
        geo = dict(geo, means2D=geo["means2D"] + delta * torch.tensor([W / 2.0, H / 2.0], dtype=torch.float64))
        out = s64.composite(geo, W, H, tg["bg"])
        N = s64.composite(dict(geo, rgb=step64.normals(st["params"], cam)), W, H, (0.0, 0.0, 0.0))["color"]
        return float(step64.image_loss(out, N, tg, fl, st["E"])[0])

    m2 = r["mean2D"]
    big = float(m2.abs().max())
    for k in torch.argsort(m2.norm(dim=1), descending=True)[:6].tolist():
        for idx in (0, 1):
            fd = (L_shift(k, idx, 1e-7) - L_shift(k, idx, -1e-7)) / 2e-7
            assert abs(fd - float(m2[k, idx])) < 2e-5 * big, (k, idx, fd, float(m2[k, idx]))
    pix = step64.grads64(st, cam, tg, fl, step64.StepConv(mean2d_ndc=False))["mean2D"]
    assert torch.allclose(pix * torch.tensor([W / 2.0, H / 2.0], dtype=torch.float64), m2, rtol=1e-14, atol=0)


@pytest.mark.parametrize("flip", [True, False])
def test_normal_term_against_finite_differences(world, flip):
    sc, cam, tg = world
    st = _state(sc)
    fl = step64.Flags(normal=True, depth=True)
    conv = step64.StepConv(normal_flip=flip)
    r = step64.grads64(st, cam, tg, fl, conv)
    mg = step64.margins(st, cam, tg, fl, conv)
    assert min(float(mg[k][0].min()) for k in ("axis", "flip")) > 1e-4
    nl1 = r["loss"]["normal_l1"]
    assert nl1 > 0

    def L(raw):
        out, N, _ = step64.forward(raw, cam, fl, D, tg["bg"], None, conv)
        return step64.image_loss(out, N, tg, fl, st["E"])[0]
    _check_fd(L, st["params"], r["grads"], ("rotation", "opacity", "xyz", "scaling"))
    # the normals face the camera exactly when flipped
    n = step64.normals(st["params"], cam, flip)
    t = st["params"]["xyz"] @ cam["V"][:3, :3] + cam["V"][3, :3]
    if flip:
        assert ((n * t).sum(1) <= 0).all()
    else:
        assert ((n * t).sum(1) > 0).any()


def test_adam64_against_torch_adam():
    gen = torch.Generator().manual_seed(0)
    p0 = torch.randn(7, 5, generator=gen, dtype=torch.float64)
    gs = [torch.randn(7, 5, generator=gen, dtype=torch.float64) * s for s in (1.0, 0.0, 1e-3, 0.0, 0.0, 5.0)]
    gs[2][:3] = 0.0
    p = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([p], lr=0.01, betas=(0.9, 0.999), eps=1e-15, foreach=False)
    q, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
    for t, g in enumerate(gs, 1):
        p.grad = g.clone()
        opt.step()
        q, m, v = step64.adam64(q, g, m, v, 0.01, t)
        st = opt.state[p]
        assert torch.allclose(q, p.detach(), rtol=1e-14, atol=1e-16)
        assert torch.allclose(m, st["exp_avg"], rtol=1e-14, atol=0) and torch.allclose(v, st["exp_avg_sq"], rtol=1e-14, atol=0)
    # a zero gradient on zero moments is an exact no-op
    z = torch.zeros(3, dtype=torch.float64)
    x = torch.tensor([1.0, -2.0, 3.0], dtype=torch.float64)
    assert torch.equal(step64.adam64(x, z, z, z, 0.1, 1)[0], x)


def test_all_flags_off_is_splat64_and_torch_adam(world):
    sc, cam, tg = world
    st = _state(sc)
    r = step64.step64(st, cam, tg, step64.Flags())
    raw = {k: v.clone().requires_grad_(True) for k, v in st["params"].items()}
    E = st["E"].clone().requires_grad_(True)
    t = s64.render(raw, cam, BG, D=D, raw=True)
    L, l1, ss = s64.loss64(t["color"], tg["gt"], tg["mask"], 0.2, E)
    L.backward()
    assert abs(r["loss"]["loss"] - L.item()) <= 1e-15 * L.item() and r["loss"]["depth_l1"] == 0.0
    params = [raw[k] for k in step64.GROUPS] + [E]
    opt = torch.optim.Adam([dict(params=[p], lr=lr) for p, lr in zip(params, st["lr"] + [st["E_lr"]])], betas=(0.9, 0.999), eps=1e-15,
                           foreach=False)
    for i, p in enumerate(params):
        k = step64.GROUPS[i] if i < 6 else None
        opt.state[p] = dict(step=torch.tensor(float(st["step"] if k else st["E_step"])), exp_avg=(st["m"][k] if k else st["E_m"]).clone(),
                            exp_avg_sq=(st["v"][k] if k else st["E_v"]).clone())
    with torch.no_grad():
        opt.step()
    nx = r["state"]
    for i, k in enumerate(step64.GROUPS):
        assert torch.allclose(nx["params"][k], raw[k].detach(), rtol=1e-14, atol=1e-16), k
        assert torch.allclose(nx["m"][k], opt.state[raw[k]]["exp_avg"], rtol=1e-14, atol=0), k
        assert torch.allclose(nx["v"][k], opt.state[raw[k]]["exp_avg_sq"], rtol=1e-14, atol=0), k
    assert torch.allclose(nx["E"], E.detach(), rtol=1e-14, atol=1e-16) and nx["E_step"] == st["E_step"] + 1
    assert torch.allclose(nx["E_m"], opt.state[E]["exp_avg"], rtol=1e-14, atol=0)
    assert torch.allclose(nx["E_v"], opt.state[E]["exp_avg_sq"], rtol=1e-14, atol=0)
    vis = t["radii"] > 0
    assert torch.equal(nx["denom"].reshape(-1), vis.double()) and torch.equal(nx["max_radii"], t["radii"].double())


def test_zero_filter_is_the_unfiltered_step_exactly(world):
    sc, cam, tg = world
    for fl in (step64.Flags(), step64.Flags(aa=True, depth=True, normal=True, reg=True)):
        a = step64.step64(_state(sc), cam, tg, fl)
        b = step64.step64(_state(sc, f=torch.zeros(P, dtype=torch.float64)), cam, tg, dataclasses.replace(fl, f3d=True))
        assert a["loss"] == b["loss"]
        for part in ("params", "m", "v"):
            for k in step64.GROUPS:
                assert torch.equal(a["state"][part][k], b["state"][part][k]), (part, k)
        for k in ("accum", "denom", "max_radii", "E", "E_m", "E_v"):
            assert torch.equal(a["state"][k], b["state"][k]), k
        assert torch.equal(a["reached"], b["reached"])


def test_statistics_and_idle_rows(world):
    """rows the pass does not draw keep their statistics; rows without gradient or moments keep their parameters bit for bit; a row with
    moments and no gradient still moves"""
    sc, cam, tg = world
    st = _state(sc, moments=False)
    r = step64.step64(st, cam, tg, step64.Flags(depth=True))
    nx = r["state"]
    idle = ~r["reached"]
    assert idle.any()
    for k in step64.GROUPS:
        assert torch.equal(nx["params"][k][idle], st["params"][k][idle]), k
    hidden = ~r["visible"]
    assert hidden.any() and torch.equal(nx["accum"][hidden], st["accum"][hidden]) and not nx["denom"][hidden].any()
    st2 = _state(sc, moments=True)
    r2 = step64.step64(st2, cam, tg, step64.Flags(depth=True))
    assert (r2["state"]["params"]["xyz"][idle] != st2["params"]["xyz"][idle]).any(1).all()
