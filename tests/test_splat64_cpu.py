"""CPU: the float64 truth of tests/splat64.py pinned on its own, without a GPU.

  * gradcheck of colour, depth and A with respect to the trainer's raw parameters, on a dozen Gaussians away from every threshold:
    SH degrees 0-3, anti-aliasing on and off, and the exposure affine of the loss;
  * against oracle_c (the float32 C port that test_oracle_golden.py pins to the reference's kernels) on oracle cases a and b: radii,
    tile-list lengths and per-pixel contributor counts equal, image and gradients within float32 rounding;
  * the loss truth against oracle_c.loss at odd sizes;
  * margins() reports a decision that sits on its threshold.
"""
import dataclasses

import numpy as np
import pytest
import torch

import oracle_c
import photo_slam_b200.synthetic as syn
import splat64 as s64
from helpers import ORACLE_CASES

RAW = s64.RAW


def _small_scene(seed, n=12, W=40, H=24):
    rng = np.random.default_rng(seed)
    cam = syn.make_camera(W, H, 30.0, 30.0, *syn.random_pose(rng, max_angle=0.2, max_trans=0.2))
    sc = syn.make_scene(n, cam, seed=seed, scale_px=3.0, culled_frac=0.0)
    sc["opacity"] = np.clip(sc["opacity"], -3.0, 2.0)      # o <= 0.88: the 0.99 clamp (straight through) never acts
    sc["features_rest"] *= 4.0                            # higher-order SH terms of a size that moves the colour
    return cam, sc


@pytest.mark.parametrize("D,aa", [(0, False), (1, True), (2, False), (3, True)])
def test_gradcheck_colour_depth_alpha(D, aa):
    cam, sc = _small_scene(D)
    mm = s64.settle(sc, cam, D=D, aa=aa, bg=(0.2, 0.4, 0.6), seed=D, floor=1e-3)
    assert mm["alpha_max"] > 1e-3 and mm["frustum"] > 1e-3
    c = s64.camera64(cam, "cpu")
    raw = s64.raw64(sc, "cpu")
    assert (s64.render(raw, c, (0.2, 0.4, 0.6), D=D, aa=aa, raw=True)["n_contrib"] > 0).any()

    def f(*leaves):
        o = s64.render(dict(zip(RAW, leaves)), c, (0.2, 0.4, 0.6), D=D, aa=aa, raw=True)
        return o["color"], o["depth"], o["alpha"]
    leaves = tuple(raw[k].clone().requires_grad_(True) for k in RAW)
    assert torch.autograd.gradcheck(f, leaves, eps=1e-7, atol=1e-6, rtol=1e-5, fast_mode=True)


def test_gradcheck_loss_with_exposure_and_mask():
    gen = torch.Generator().manual_seed(0)
    I = torch.rand((3, 13, 17), generator=gen, dtype=torch.float64, requires_grad=True)
    G = torch.rand((3, 13, 17), generator=gen, dtype=torch.float64)
    mask = (torch.rand((1, 13, 17), generator=gen, dtype=torch.float64) > 0.3).double().expand(3, 13, 17)
    E = torch.tensor([[1.4, 0.1, -0.2, 0.1], [0.05, 0.6, 0.1, -0.1], [-0.1, 0.2, 1.3, 0.05]], dtype=torch.float64, requires_grad=True)
    assert torch.autograd.gradcheck(lambda i, e: s64.loss64(i, G, mask, 0.2, e)[0], (I, E), eps=1e-7, atol=1e-7, rtol=1e-5)


def _oracle_case(case):
    k = ORACLE_CASES[case]
    W, H = k["wh"]
    _, _, fx, fy = syn.CAMERAS["tum"]
    cam = syn.make_camera(W, H, fx * W / 640, fy * H / 480, *syn.random_pose(np.random.default_rng(k["pose_seed"])))
    sc = syn.make_scene(k["P"], cam, seed=k["seed"], scale_px=k["scale_px"])
    s64.settle(sc, cam, D=k["D"], bg=k["bg"], seed=1)
    return k, cam, sc


@pytest.mark.parametrize("case", ["a", "b"])
def test_truth_matches_the_oracle(case):
    k, cam, sc = _oracle_case(case)
    W, H = k["wh"]
    act = syn.activate(sc)
    o = oracle_c.forward(cam, act, D=k["D"], bg=k["bg"])
    g = {n: torch.tensor(v, dtype=torch.float64, requires_grad=True) for n, v in act.items()}
    tr = s64.render(g, s64.camera64(cam, "cpu"), k["bg"], D=k["D"])
    assert torch.equal(tr["radii"], torch.from_numpy(o["radii"]).long())
    assert torch.equal(tr["tiles_touched"], torch.from_numpy(o["tiles_touched"].astype(np.int64)))
    ranges = o["ranges"].astype(np.int64)
    assert torch.equal(tr["list_len"], torch.from_numpy(ranges[:, 1] - ranges[:, 0]))
    assert torch.equal(tr["n_contrib"].reshape(-1), torch.from_numpy(o["n_contrib"].astype(np.int64)))
    assert (tr["n_contrib"] > 0).float().mean() > 0.5
    # float32 rounding of a forward over lists of ~100 entries: measured max 9.1e-7 (a) / 5.7e-7 (b)
    assert np.abs(tr["color"].detach().numpy() - o["out_color"]).max() < 4e-6
    assert np.abs(1.0 - tr["alpha"].detach().numpy().reshape(-1) - o["final_T"]).max() < 4e-7
    dpix = np.random.default_rng(0).uniform(-1, 1, (3, H, W)).astype(np.float32)
    b = oracle_c.backward(cam, act, o, dpix, D=k["D"])
    (tr["color"] * torch.from_numpy(dpix).double()).sum().backward()
    # rel-norm of float32 against float64 gradients: measured <= 1.7e-6 on every group
    for name, key in (("means3D", "dL_dmean3D"), ("shs", "dL_dsh"), ("opacities", "dL_dopacity"), ("scales", "dL_dscale"),
                      ("rotations", "dL_drot")):
        a, r = torch.from_numpy(b[key]).double().reshape(-1), g[name].grad.reshape(-1)
        assert ((a - r).norm() / r.norm()).item() < 1e-5, name


@pytest.mark.parametrize("H,W", [(1, 1), (5, 7), (11, 11), (17, 33), (241, 17)])
def test_loss_truth_matches_the_oracle(H, W):
    rng = np.random.default_rng(H * 100 + W)
    img, gt = rng.uniform(0, 1, (3, H, W)).astype(np.float32), rng.uniform(0, 1, (3, H, W)).astype(np.float32)
    gt[:, :, : W // 3] = img[:, :, : W // 3]     # ties: sign(0) = 0
    val, l1, ss, grad = oracle_c.loss(img, gt, 0.2)
    I = torch.from_numpy(img).double().requires_grad_(True)
    L, l1t, sst = s64.loss64(I, torch.from_numpy(gt).double(), lam=0.2)
    L.backward()
    assert abs(L.item() - val) < 1e-6 and abs(l1t.item() - l1) < 1e-6 and abs(sst.item() - ss) < 1e-6
    assert np.abs(I.grad.numpy() - grad).max() <= 1e-6 * np.abs(I.grad.numpy()).max() + 1e-10


def test_margins_flag_a_decision_on_its_threshold():
    cam, sc = _small_scene(5)
    s64.settle(sc, cam, D=1, seed=5)
    c = s64.camera64(cam, "cpu")
    raw = s64.raw64(sc, "cpu")
    tr = s64.render(raw, c, (0, 0, 0), D=1, raw=True)
    # move Gaussian i's termination threshold onto one of its T tests: the margin of T must see it
    mg = s64.margins(raw, c, D=1, raw=True)
    v, ids = mg["T"]
    j = int(torch.argmin(v))
    moved = [s64.margins(raw, c, D=1, raw=True, conv=dataclasses.replace(s64.CONV, t_min=s64.CONV.t_min * (1.0 + sgn * float(v[j]))))
             for sgn in (1, -1)]
    mg2 = min(moved, key=lambda m: s64.min_margins(m)["T"])
    assert s64.min_margins(mg2)["T"] < 1e-8 and int(ids[j]) in s64.offenders(mg2).tolist()
    assert tr["n_contrib"].any()
