"""CPU: the tile-subset truth of tests/scale64.py against the dense truths it restates, without a GPU.

  * on small scenes (a posed camera, partial edge tiles, SH degree 3) the subset truth equals splat64 / step64 on the chosen tiles: colour,
    depth, A, the normal plane, the second depth moment, contributor counts, list lengths, and the gradients of weights masked to the
    kept sampled pixels; trainer parameters with anti-aliasing and the 3D filter, and the operator's activated inputs;
  * a Gaussian nudged onto each kind of threshold gets its pixels excluded (radius, rectangle edge, near plane, frustum clamp, colour clamp,
    anti-aliasing floor, alpha_min, alpha_max, T, depth tie); det and power have no such scene: with the 0.3 dilation the 2D covariance
    is positive definite in exact arithmetic, so neither decision lies near its threshold but through rounding;
  * each perturbation (a dropped contributor, two swapped contributors, truncated lists) changes the result.
"""
import dataclasses

import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn
import scale64
import splat64 as s64
import step64


def _scene(seed=0, W=72, H=40, P=700):
    rng = np.random.default_rng(seed)
    cam = syn.make_camera(W, H, 60.0, 60.0, *syn.random_pose(rng, max_angle=0.2, max_trans=0.2))
    sc = syn.make_scene(P, cam, seed=seed, scale_px=3.0, culled_frac=0.0)
    return cam, sc


def _weights(H, W, seed=0):
    gen = torch.Generator().manual_seed(seed)
    r = lambda *s: (torch.rand(s, generator=gen, dtype=torch.float64) - 0.5)
    return dict(color=r(3, H, W), depth=0.2 * r(H, W), alpha=r(H, W), normal=r(3, H, W), depth2=0.05 * r(H, W))


def _full(raw, c, bg, D, aa, f, weights, keep):
    """step64.forward's planes over the whole image and their gradient for the weights times keep"""
    fl = step64.Flags(aa=aa, f3d=f is not None, normal=True)
    out, N, _ = step64.forward(raw, c, fl, D, bg, f)
    z = out["geo"]["z"]
    M = s64.composite(dict(out["geo"], rgb=torch.stack([z * z, 0 * z, 0 * z], 1)), c["W"], c["H"], (0.0, 0.0, 0.0))["color"][0]
    planes = dict(color=out["color"], depth=out["depth"], alpha=out["alpha"], normal=N, depth2=M)
    out["geo"]["means2D"].retain_grad()
    sum((planes[k] * (w * keep)).sum() for k, w in weights.items()).backward()
    return out, planes


@pytest.mark.parametrize("aa,f3d,D", [(False, False, 3), (True, False, 1), (True, True, 3)])
def test_subset_truth_equals_full_truth(aa, f3d, D):
    cam, sc = _scene(seed=D + 2 * aa + 4 * f3d)
    c = s64.camera64(cam, "cpu")
    W, H = cam["W"], cam["H"]
    bg = (0.3, 0.5, 0.7)
    tiles = scale64.sample_tiles(W, H, 5, seed=1)
    assert any(tx == W // 16 for tx, _ in tiles) and any(ty == H // 16 for _, ty in tiles)     # the partial last column and row
    f = torch.from_numpy(np.random.default_rng(3).uniform(0.0, 0.01, sc["xyz"].shape[0])).double() if f3d else None
    raw = {k: v.requires_grad_(True) for k, v in s64.raw64(sc, "cpu").items()}
    w = _weights(H, W)
    t = scale64.tile_truth(raw, c, bg, tiles, D=D, aa=aa, f=f, planes=scale64.PLANES, weights=w)
    assert t["counts"]["excluded"] < t["counts"]["pixels"] // 4
    got = {k: v.grad.clone() for k, v in raw.items()}
    raw2 = {k: v.detach().clone().requires_grad_(True) for k, v in raw.items()}
    out, planes = _full(raw2, c, bg, D, aa, f, w, t["keep"].double())
    pix = t["pix"]
    for k in scale64.PLANES:
        ref = planes[k].detach().reshape(-1, H * W)[:, pix]
        assert torch.allclose(t[k].reshape(ref.shape), ref, rtol=1e-12, atol=1e-13), k
    assert torch.equal(t["n_contrib"], out["n_contrib"].reshape(-1)[pix]) and torch.equal(t["last"], out["last"].reshape(-1)[pix])
    gx = -(-W // 16)
    assert torch.equal(t["list_len"], out["list_len"][[ty * gx + tx for tx, ty in tiles]])
    assert torch.equal(t["radii"], out["radii"])
    for k in s64.RAW:
        assert torch.allclose(got[k], raw2[k].grad, rtol=1e-10, atol=1e-14), k
    assert torch.allclose(t["mean2D_grad"], out["geo"]["means2D"].grad, rtol=1e-10, atol=1e-14)
    # rows that are no candidate of a sampled tile get exactly zero
    other = torch.ones(sc["xyz"].shape[0], dtype=torch.bool)
    other[t["cand"]] = False
    assert other.any() and all(not got[k][other].any() for k in s64.RAW)


def test_subset_truth_equals_full_truth_operator():
    """activated inputs (raw=False): the operator's leaves, colour, depth and A"""
    cam, sc = _scene(seed=9)
    c = s64.camera64(cam, "cpu")
    W, H = cam["W"], cam["H"]
    g = {k: torch.from_numpy(np.ascontiguousarray(v)).double().requires_grad_(True) for k, v in syn.activate(sc).items()}
    tiles = scale64.sample_tiles(W, H, 4, seed=2)
    w = {k: v for k, v in _weights(H, W, 1).items() if k in ("color", "depth", "alpha")}
    t = scale64.tile_truth(g, c, (0.0, 0.0, 0.0), tiles, D=3, aa=True, raw=False, weights=w)
    got = {k: v.grad.clone() for k, v in g.items()}
    g2 = {k: v.detach().clone().requires_grad_(True) for k, v in g.items()}
    out = s64.render(g2, c, (0.0, 0.0, 0.0), D=3, aa=True)
    keep = t["keep"].double()
    sum((out[k] * (wk * keep)).sum() for k, wk in w.items()).backward()
    for k in ("color", "depth", "alpha"):
        ref = out[k].detach().reshape(-1, H * W)[:, t["pix"]]
        assert torch.allclose(t[k].reshape(ref.shape), ref, rtol=1e-12, atol=1e-13), k
    assert torch.equal(t["tiles_touched"], out["tiles_touched"])
    for k in g:
        assert torch.allclose(got[k], g2[k].grad, rtol=1e-10, atol=1e-14), k


# ---- thresholds -----------------------------------------------------------------------------------------------------------------------
def _identity_scene(P=300, seed=4):
    cam = syn.make_camera(64, 48, 50.0, 50.0)
    sc = syn.make_scene(P, cam, seed=seed, scale_px=3.0, culled_frac=0.0)
    return cam, sc


def _put(sc, cam, i, u, v, z, sigma_px, logit):
    fx = cam["W"] / (2.0 * float(cam["tanfovx"]))
    sc["xyz"][i] = [(u - 0.5 * cam["W"]) / fx * z, (v - 0.5 * cam["H"]) / fx * z, z]
    sc["scaling"][i] = np.log(sigma_px / fx * z)
    sc["rotation"][i] = [1.0, 0.0, 0.0, 0.0]
    sc["opacity"][i] = logit


def _truth(sc, cam, tiles, D=3, conv=s64.CONV, **kw):
    return scale64.tile_truth(s64.raw64(sc, "cpu"), s64.camera64(cam, "cpu"), (0.0, 0.0, 0.0), tiles, D=D, conv=conv, **kw)


def _pixels_of(t, i, W):
    """the sampled pixels at which Gaussian i reaches the alpha test (its truth alpha >= 1/255)"""
    g = t["geo"]
    px, py = (t["pix"] % W).double(), (t["pix"] // W).double()
    dx, dy = g["means2D"][i, 0] - px, g["means2D"][i, 1] - py
    cn = g["conic"][i]
    a = g["o"][i] * torch.exp(-0.5 * (cn[0] * dx * dx + cn[2] * dy * dy) - cn[1] * dx * dy)
    return a >= 1.0 / 255.0


def test_gaussian_on_radius_threshold_excludes_its_pixels():
    cam, sc = _identity_scene()
    _put(sc, cam, 0, 24.3, 20.6, 2.0, 2.0, 1.0)
    c = s64.camera64(cam, "cpu")
    lo, hi = np.log(1.5), np.log(2.5)
    base = sc["scaling"][0].copy()
    target = None
    for _ in range(80):       # bisect an isotropic scale onto r3 = an integer from above
        mid = 0.5 * (lo + hi)
        sc["scaling"][0] = base + np.float32(mid - np.log(2.0))
        r3 = float(s64.geometry(s64.activate(s64.raw64(sc, "cpu")), c, 3)["r3"][0])
        target = target or np.ceil(r3)
        lo, hi = (mid, hi) if r3 < target else (lo, mid)
    sc["scaling"][0] = base + np.float32(hi - np.log(2.0))
    tiles = [(tx, ty) for ty in range(3) for tx in range(4)]
    t = _truth(sc, cam, tiles)
    assert t["offender"][0] and t["counts"]["gauss"]["radius"] >= 1
    # a radius step moves the rectangle's edges lying within 1/16 tile of an integer: the tile row or column there is ambiguous
    g = t["geo"]
    e = g["edges"][0]
    near = ((e - torch.round(e)).abs() < 1.0 / 16 + 1e-6).nonzero().reshape(-1).tolist()
    assert near and t["list_ambiguous"].any()
    line = int(torch.round(e[near[0]])) - 1
    amb_tiles = [i for i, (tx, ty) in enumerate(tiles) if (tx if near[0] % 2 == 0 else ty) == line]
    assert all(bool(t["list_ambiguous"][i]) for i in amb_tiles if 0 <= line)
    on = _pixels_of(t, 0, cam["W"]) & torch.isin(t["tile"], torch.tensor(amb_tiles, dtype=torch.long))
    assert t["excluded"][on].all()


def test_gaussian_on_colour_clamp_and_near_plane_excludes_its_pixels():
    cam, sc = _identity_scene()
    _put(sc, cam, 0, 20.0, 20.0, 1.5, 2.5, 1.0)
    sc["features_dc"][0, 0, 1] = np.float32(-0.5 / s64.SH_C0)        # green before the clamp ~ 0
    _put(sc, cam, 1, 40.0, 25.0, 0.2 + 5e-6, 2.5, 1.0)                # on the near plane, in front of it
    t = _truth(sc, cam, [(1, 1), (2, 1)], D=0)
    assert t["counts"]["gauss"]["colour"] >= 1 and t["counts"]["gauss"]["near"] >= 1
    for i in (0, 1):
        on = _pixels_of(t, i, cam["W"])
        assert on.any() and t["excluded"][on].all(), i
    sc["xyz"][1, 2] = np.float32(0.2 - 5e-6)                             # behind it: refused
    with pytest.raises(ValueError, match="near plane"):
        _truth(sc, cam, [(1, 1), (2, 1)], D=0)


def test_rectangle_edge_on_an_integer_makes_its_tile_column_ambiguous():
    """a splat whose left rectangle edge (x - radius) / 16 lands on 2: tile column 1 may or may not list it"""
    cam, sc = _identity_scene()
    _put(sc, cam, 0, 40.0, 24.0, 2.0, 2.0, 2.0)
    c = s64.camera64(cam, "cpu")
    fx = cam["W"] / (2.0 * float(cam["tanfovx"]))
    for _ in range(3):        # move the mean onto 32 + radius
        g = s64.geometry(s64.activate(s64.raw64(sc, "cpu")), c, 3)
        du = 32.0 + float(g["radius"][0]) - float(g["means2D"][0, 0])
        sc["xyz"][0, 0] += np.float32(du / fx * 2.0)
    tiles = [(tx, ty) for ty in range(3) for tx in range(4)]
    t = _truth(sc, cam, tiles)
    assert t["offender"][0] and t["counts"]["gauss"]["rect"] >= 1
    r = t["geo"]["rect"][0]
    col1 = [i for i, (tx, ty) in enumerate(tiles) if tx == 1 and int(r[1]) - 1 <= ty <= int(r[3])]
    assert col1 and all(bool(t["list_ambiguous"][i]) for i in col1)
    on = _pixels_of(t, 0, cam["W"]) & torch.isin(t["tile"], torch.tensor(col1))
    assert t["excluded"][on].all()


def test_frustum_clamp_alpha_clamp_and_aa_floor_exclude_their_pixels():
    cam, sc = _identity_scene()
    c = s64.camera64(cam, "cpu")
    tan = float(cam["tanfovx"])
    # a wide splat whose mean sits on the 1.3 tan(fovx) clamp, reaching into the image
    _put(sc, cam, 0, 30.0, 24.0, 2.0, 30.0, 2.0)
    sc["xyz"][0, 0] = np.float32(1.3 * tan * 2.0)
    t = _truth(sc, cam, [(tx, ty) for ty in range(3) for tx in range(4)])
    assert t["counts"]["gauss"]["frustum"] >= 1 and t["offender"][0]
    on = _pixels_of(t, 0, cam["W"])
    assert on.any() and t["excluded"][on].all()
    # alpha reaching 0.99 exactly: opacity logit(0.99), its mean on a pixel centre
    cam, sc = _identity_scene()
    _put(sc, cam, 1, 20.0, 20.0, 1.0, 2.0, float(np.log(0.99 / 0.01)))
    g = s64.geometry(s64.activate(s64.raw64(sc, "cpu")), c, 3)
    u, v = (int(round(float(x))) for x in g["means2D"][1])
    sc["xyz"][1, :2] += ((np.array([u, v]) - g["means2D"][1].numpy()) / (cam["W"] / (2.0 * tan))).astype(np.float32)
    t = _truth(sc, cam, [(u // 16, v // 16)])
    assert t["counts"]["alpha_max"] >= 1 and t["excluded"][t["pix"] == v * cam["W"] + u].all()
    # the anti-aliasing floor: a tiny splat whose det0 / det1 sits on 2.5e-5, opaque enough to pass the alpha test at its centre pixel
    cam, sc = _identity_scene()
    _put(sc, cam, 0, 20.0, 20.0, 2.0, 0.04, 6.0)
    g = s64.geometry(s64.activate(s64.raw64(sc, "cpu")), c, 3)
    sc["xyz"][0, :2] += ((np.round(g["means2D"][0].numpy()) - g["means2D"][0].numpy()) / (cam["W"] / (2.0 * tan)) * 2.0).astype(np.float32)
    lo, hi = np.log(0.01), np.log(0.1)
    base = sc["scaling"][0].copy()
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        sc["scaling"][0] = base + np.float32(mid - np.log(0.04))
        ratio = float(s64.geometry(s64.activate(s64.raw64(sc, "cpu")), c, 3, aa=True)["ratio"][0])
        lo, hi = (mid, hi) if ratio < s64.MIN_RATIO else (lo, mid)
    t = _truth(sc, cam, [(1, 1)], aa=True)
    assert t["counts"]["gauss"]["aa"] >= 1 and t["offender"][0]
    on = _pixels_of(t, 0, cam["W"])
    assert on.any() and t["excluded"][on].all()


def test_pair_decisions_on_their_thresholds_exclude_the_pixel():
    cam, sc = _identity_scene()
    tiles = [(1, 1)]
    t0 = _truth(sc, cam, tiles)
    assert not t0["excluded"].all()
    # alpha_min: the threshold moved onto the alpha of one pair of one pixel
    g, k = t0["geo"], int((~t0["excluded"] & (t0["n_contrib"] > 0)).nonzero()[0])
    i, p = int(t0["last"][k]), int(t0["pix"][k])
    dx, dy = g["means2D"][i, 0] - p % cam["W"], g["means2D"][i, 1] - p // cam["W"]
    cn = g["conic"][i]
    a = float(g["o"][i] * torch.exp(-0.5 * (cn[0] * dx * dx + cn[2] * dy * dy) - cn[1] * dx * dy))
    t = _truth(sc, cam, tiles, conv=dataclasses.replace(s64.CONV, alpha_min=a))
    assert t["excluded"][k] and t["counts"]["alpha_min"] >= 1
    # T: the termination threshold moved onto the final T of a pixel whose list the T test does not end
    k2 = int(((~t0["stopped"]) & (t0["alpha"] > 0.5) & ~t0["excluded"]).nonzero()[0])
    t = _truth(sc, cam, tiles, conv=dataclasses.replace(s64.CONV, t_min=float(1.0 - t0["alpha"][k2])))
    assert t["excluded"][k2] and t["counts"]["T"] >= 1
    # depth tie: a second splat at the same depth as the last contributor of pixel k, over it
    j = int((torch.arange(sc["xyz"].shape[0]) != i).nonzero()[-1])
    _put(sc, cam, j, float(g["means2D"][i, 0]) + 0.5, float(g["means2D"][i, 1]), float(sc["xyz"][i, 2]), 3.0, 2.0)
    sc["xyz"][j, 2] = sc["xyz"][i, 2]
    t = _truth(sc, cam, tiles)
    assert t["counts"]["depth_tie"] >= 1 and t["excluded"][k]


def test_t_margin_grows_with_the_blended_factors(monkeypatch):
    """the T rule's second arm, T_ULPS 2^-24 sum 1 / (1 - alpha) over the blended factors, excludes pixels whose margin clears
    MIN_MARGIN: the longer the blend, the wider the excluded band"""
    cam, sc = _identity_scene(P=1200, seed=6)
    sc["opacity"][:] = np.abs(sc["opacity"]) + 1.0
    t0 = _truth(sc, cam, [(1, 1), (2, 1)])
    assert t0["stopped"].any()
    monkeypatch.setattr(scale64, "T_ULPS", 1e4)
    t1 = _truth(sc, cam, [(1, 1), (2, 1)])
    assert t1["counts"]["T"] > t0["counts"]["T"] and (t1["excluded"] | ~t0["excluded"]).all()


# ---- perturbations --------------------------------------------------------------------------------------------------------------------
def test_each_perturbation_changes_the_result():
    cam, sc = _identity_scene(P=1500, seed=8)
    tiles = [(1, 1), (2, 1)]
    t0 = _truth(sc, cam, tiles)
    k = int((t0["n_contrib"] > 2).nonzero()[0])
    gid = int(t0["last"][k])
    td = _truth(sc, cam, tiles, perturb=dict(drop=(int(t0["tile"][k]), gid)))
    assert not torch.equal(td["color"], t0["color"]) and not torch.equal(td["last"], t0["last"])
    # swap: the last contributor of pixel k and the contributor of pixel k before it
    g = t0["geo"]
    ti = int(t0["tile"][k])
    tx, ty = tiles[ti]
    r = g["rect"]
    lst = (g["alive"] & (r[:, 0] <= tx) & (tx < r[:, 2]) & (r[:, 1] <= ty) & (ty < r[:, 3])).nonzero().reshape(-1)
    lst = lst[torch.argsort(g["zd"][lst], stable=True)]
    at = int((lst == gid).nonzero())
    before = [int(j) for j in lst[:at] if _pixels_of(t0, int(j), cam["W"])[k]]
    ts = _truth(sc, cam, tiles, perturb=dict(swap=(ti, gid, before[-1])))
    assert not torch.equal(ts["color"], t0["color"])
    n = int(t0["list_len"].max())
    tt = _truth(sc, cam, tiles, perturb=dict(truncate=n // 2))
    assert not torch.equal(tt["color"], t0["color"])
