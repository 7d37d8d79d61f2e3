"""-m gpu: the kernels against the float64 truth of tests/splat64.py, on a catalogue of scenes each built to reach one edge of the tile
kernels, with every decision of every scene at least splat64.MIN_MARGIN (relative) from its threshold.

  * operator forward (RasterizeGaussiansCUDA and RasterizeGaussiansDepthCUDA, plain and anti-aliased): colour, depth, radii,
    tiles_touched, tile-list lengths and per-pixel contributor counts; operator backward (atomic, deterministic, anti-aliased) against
    float64 autograd on the activated leaves, with random weights on colour and depth, dL_dmeans2D (the densification signal, in NDC
    units) included; at scale_modifier = 0.6 the forward and the backward, whose dL_dscales is the gradient with respect to 0.6 s;
  * trainer render (colour, depth, A, radii, last contributor and final T of psb_trainer_debug_state) and backwardPixels against
    float64 autograd on the raw parameters, default and deterministic modes, anti-aliasing on and off;
  * the built-in loss: psb_trainer_backward, _depth and _exposure in gradient mode (loss scalars, raw-parameter gradients, the 12
    exposure sums), default and deterministic; one psb_trainer_step_exposure against the float64 gradients and a float64 Adam step;
  * psb_loss (fused_loss) against the float64 loss and its gradient at odd sizes, with masks and ties;
  * each gate family fails against a deliberately perturbed truth.

There is no scene for a splat whose dilated conic is not positive definite (`power > 0` inside the kernels' reach test). In exact
arithmetic the dilated 2D covariance is always positive definite: det = det0 + 0.3 (a0 + c0) + 0.09 > 0 for a covariance with det0 >= 0.
Such a splat exists only through float32 rounding, so its decision lies within rounding of its threshold and breaks the margin rule
every scene here keeps. The `power` decision is still checked on every pair through margins()["power"].

Gates: measured on an H100 SXM (80 GB, 700 W) over the whole catalogue; the largest measured error sits in the comment beside each.
Gradient groups are gated twice: rel-norm, and the largest element error relative to the largest element of the group.
"""
import dataclasses
import math

import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn
import splat64 as s64

pytestmark = pytest.mark.gpu

BG = {"black": (0.0, 0.0, 0.0), "colour": (0.3, 0.5, 0.7)}
# forward: max |kernel - truth| over the image (depth relative to the largest depth)
GATE_COLOR = 1e-5         # measured 3.4e-6 (rect-33)
GATE_DEPTH = 1e-5         # measured 3.4e-6 (rect-32)
GATE_ALPHA = 1.5e-5       # measured 4.4e-6 (rect-33, trainer)
# gradients: rel-norm per parameter group, operator (activated leaves) and trainer (raw parameters), every mode
GATE_GRAD = 2e-5          # measured 5.5e-6 (trainer xyz, odd-P-1); operator 4.5e-6 (scales, rect-33); built-in loss 1.3e-6; Adam moments 4.6e-7
GATE_GRAD_MAX = 3e-5      # max |kernel - truth| / max |truth| per group: measured 8.3e-6 (operator, rect-33); trainer 4.9e-6; built-in 2.1e-6
GATE_STEP = 5e-6          # one Adam step: max |kernel - truth| / lr beyond one float32 spacing of the parameter: measured 1.3e-6
GATE_LOSS = 8e-5          # loss scalars, relative: measured 2.5e-5 (psb_loss at 480x640, a float32 mean of 0.9M terms); built-in 3.3e-6
GATE_LOSS_GRAD = 3e-6     # dL/dimage, max abs relative to its largest entry: measured 7.5e-7


# ---- scenes -------------------------------------------------------------------------------------------------------------------------
def _cam(W, H, f=None):
    f = f if f is not None else 0.9 * max(W, H)
    return syn.make_camera(W, H, f, f)


def _put(sc, cam, i, u, v, z, sigma_px, logit, rgb=None, aniso=(1.0, 1.0, 1.0)):
    """Gaussian i at pixel (u, v), view depth z (identity pose), isotropic size sigma_px pixels"""
    fx = cam["W"] / (2.0 * float(cam["tanfovx"]))
    sc["xyz"][i] = [(u - 0.5 * (cam["W"] - 1)) / fx * z, (v - 0.5 * (cam["H"] - 1)) / fx * z, z]
    sc["scaling"][i] = np.log(sigma_px / fx * abs(z) * np.asarray(aniso))
    sc["rotation"][i] = [1.0, 0.0, 0.0, 0.0]
    sc["opacity"][i] = logit
    if rgb is not None:
        sc["features_dc"][i, 0] = (np.asarray(rgb) - 0.5) / s64.SH_C0
        sc["features_rest"][i] = 0.0


def _random(P, cam, seed, scale_px=2.5, rest=0.05, zr=(0.6, 8.0)):
    """P Gaussians in front of the camera, depths on a geometric ladder (no two within 1e-4 of each other)"""
    rng = np.random.default_rng(seed)
    W, H = cam["W"], cam["H"]
    fx = W / (2.0 * float(cam["tanfovx"]))
    z = zr[0] * (zr[1] / zr[0]) ** ((rng.permutation(P) + rng.uniform(0.3, 0.7, P)) / max(P, 1))
    u, v = rng.uniform(-0.1 * W, 1.1 * W, P), rng.uniform(-0.1 * H, 1.1 * H, P)
    xyz = np.stack([(u - 0.5 * (W - 1)) / fx * z, (v - 0.5 * (H - 1)) / fx * z, z], 1)
    f32 = lambda a: np.ascontiguousarray(a, dtype=np.float32)
    return dict(xyz=f32(xyz), features_dc=f32(((rng.uniform(0, 1, (P, 3)) - 0.5) / s64.SH_C0)[:, None]),
                features_rest=f32(rng.normal(0, rest, (P, 15, 3))), scaling=f32(np.log(scale_px / fx * z)[:, None] + rng.normal(0, 0.4, (P, 3))),
                rotation=f32(rng.normal(size=(P, 4))), opacity=f32(rng.normal(0.0, 1.5, (P, 1))))


def _stack(n):
    """n small splats stacked in front of the centre of tile (1, 1) of a 48x48 image: one tile list of exactly n entries"""
    cam = _cam(48, 48)
    sc = _random(n + 40, cam, seed=n)
    rng = np.random.default_rng(n + 1)
    for i in range(n):
        _put(sc, cam, i, 23.5 + rng.uniform(-2.5, 2.5), 23.5 + rng.uniform(-2.5, 2.5), 1.0 + 2.0 * i / n + 1e-3 * rng.uniform(), 1.2,
             rng.uniform(-3.5, -1.5))
    # the other 40 stay away from tile (1, 1)'s rectangle: small and in the outer ring of tiles
    for i in range(n, n + 40):
        k = i - n
        _put(sc, cam, i, [3.0, 44.0][k % 2] + rng.uniform(-2, 2), 3.0 + (k // 2) * 2.1, 2.0 + 0.05 * k, 1.0, rng.uniform(-2, 2))
    return dict(cam=cam, sc=sc, D=1, edge=("list", (1, 1), n))


def _rect(area):
    """one splat whose tile rectangle holds exactly `area` tiles (8 x 4 for 32, 11 x 3 for 33) over a few small ones"""
    W, H = 256, (64 if area == 32 else 48)
    cam = _cam(W, H, f=200.0)
    sc = _random(150, cam, seed=area, scale_px=1.5)
    for sig in np.linspace(8.0, 60.0, 400):
        _put(sc, cam, 0, 130.3, H / 2 + 0.3, 3.01, sig, 2.0)
        g = s64.geometry(s64.activate(s64.raw64(sc, "cpu")), s64.camera64(cam, "cpu"), D=0)
        if int(g["tiles_touched"][0]) == area:
            break
    return dict(cam=cam, sc=sc, D=0, edge=("area", 0, area))


def _dense(seed=3, W=64, H=48, P=900, D=3, rest=0.05, scale_px=3.0):
    cam = _cam(W, H)
    return dict(cam=cam, sc=_random(P, cam, seed, scale_px=scale_px, rest=rest), D=D, edge=None)


def _alpha_clamp():
    s = _dense(seed=5, P=300)
    rng = np.random.default_rng(5)
    for i in range(12):
        # o = 0.9975 on a whole pixel: alpha = o G reaches 0.99 near the centre, with anti-aliasing too (h > 0.997 at 10 px)
        _put(s["sc"], s["cam"], i, rng.integers(5, 59) + 0.05, rng.integers(5, 43) + 0.05, 0.7 + 0.01 * i, 10.0, 6.0)
    s.update(edge=("alpha_max",))
    return s


def _colour_clamp(D):
    s = _dense(seed=10 + D, P=400, D=D, rest=0.6)
    s["sc"]["features_dc"][:] *= 0.3
    s["edge"] = ("colour",)
    return s


def _frustum():
    s = _dense(seed=7, P=300)
    W, H = 64, 48
    for i, (u, v) in enumerate([(-0.35 * W, 20), (1.35 * W, 30), (30, -0.4 * H), (20, 1.4 * H)]):
        _put(s["sc"], s["cam"], i, u, v, 0.9 + 0.05 * i, 22.0, 1.0, aniso=(1.0, 0.6, 0.8))
    s.update(edge=("frustum", range(4)))
    return s


def _near():
    s = _dense(seed=8, P=300)
    cam = s["cam"]
    for i, z in enumerate([0.2002, 0.2004, 0.2006, -0.5, 0.1999, 0.0, -3.0]):
        _put(s["sc"], cam, i, 10 + 7 * i, 12 + 3 * i, z if z != 0 else 1e-3, 1.0, 1.0)
        if z <= 0:
            s["sc"]["xyz"][i, 2] = z
    s.update(edge=("near", range(3), range(3, 7)))
    return s


def _huge():
    s = _dense(seed=9, P=1000, scale_px=1.5)
    _put(s["sc"], s["cam"], 0, 31.0, 23.0, 5.5, 60.0, 0.0)
    s.update(edge=("area", 0, 12))
    return s


def _terminate():
    s = _dense(seed=12, P=2000, scale_px=5.0)
    sc = s["sc"]
    sc["opacity"][:] = np.abs(sc["opacity"]) + 0.5
    # the right fifth of the view sees only the tails of the others: pixels there never reach T < 1e-4 (the moved ones are culled)
    right = sc["xyz"][:, 0] / sc["xyz"][:, 2] > 0.6 * float(s["cam"]["tanfovx"])
    sc["xyz"][right, 2] *= -1.0
    s["edge"] = ("terminate",)
    return s


def _small(W, H):
    cam = _cam(W, H, f=max(W, H, 8) * 0.9)
    return dict(cam=cam, sc=_random(200, cam, seed=W * 7 + H, scale_px=2.0), D=2, edge=None)


def _odd(P):
    cam = _cam(64, 48)
    sc = _random(P, cam, seed=P, scale_px=3.0 if P < 1000 else 1.2)
    return dict(cam=cam, sc=sc, D=3, edge=None)


SCENES = {**{f"list-{n}": (lambda n=n: _stack(n)) for n in (127, 128, 129, 256, 257)},
          "rect-32": lambda: _rect(32), "rect-33": lambda: _rect(33),
          "terminate-mid-batch": _terminate, "alpha-clamp": _alpha_clamp,
          **{f"colour-clamp-sh{d}": (lambda d=d: _colour_clamp(d)) for d in (1, 2, 3)},
          "frustum-clamp": _frustum, "near-plane-behind": _near, "huge": _huge,
          **{f"small-{w}x{h}": (lambda w=w, h=h: _small(w, h)) for w, h in ((1, 1), (1, 37), (15, 9), (16, 16), (17, 33), (250, 15))},
          **{f"sh-degree-{d}": (lambda d=d: dict(_dense(seed=20), D=d)) for d in (0, 1, 2, 3)},
          **{f"odd-P-{p}": (lambda p=p: _odd(p)) for p in (1, 127, 129, 4097)}}
_CACHE = {}


def _scene(name):
    if name not in _CACHE:
        s = SCENES[name]()
        s["margins"] = s64.settle(s["sc"], s["cam"], D=s["D"], aa=None, bg=(0.3, 0.5, 0.7), seed=1, dev="cuda")
        _CACHE[name] = s
    return _CACHE[name]


def _bg(name):
    return BG["black" if sum(map(ord, name)) % 2 else "colour"]


def _weights(H, W, dev, seed=0):
    gen = torch.Generator().manual_seed(seed)
    return ((torch.rand((3, H, W), generator=gen) - 0.5).to(dev), (0.2 * (torch.rand((H, W), generator=gen) - 0.5)).to(dev),
            (torch.rand((H, W), generator=gen) - 0.5).to(dev))


def _relnorm(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    if b.norm() == 0:
        return float(a.norm())
    return float((a - b).norm() / b.norm())


def _maxerr(a, b, scale=1.0):
    """max |a - b| / scale; an all-zero reference (scale 0) wants an all-zero a"""
    if not a.numel():
        return 0.0
    e = float((a.double() - b.double()).abs().max())
    return e / scale if scale > 0 else e


# ---- the operator -------------------------------------------------------------------------------------------------------------------
def _op_inputs(sc, dev):
    import photo_slam_b200.synthetic as syn
    act = syn.activate(sc)
    return {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in act.items()}


def _op_forward(g, c, bg, D, aa, mod=1.0):
    from photo_slam_b200 import rasterizer
    return rasterizer.RasterizeGaussiansDepthCUDA(bg, g["means3D"], None, g["opacities"], g["scales"], g["rotations"], mod, None, c["viewmatrix"],
                                                  c["projmatrix"], c["tanfovx"], c["tanfovy"], c["H"], c["W"], g["shs"], D, c["campos"], False,
                                                  antialiasing=aa)


def _export(P, R, W, H, geom, binning, img):
    from photo_slam_b200 import _lib
    dev = geom.device
    tt = torch.zeros(P, dtype=torch.int32, device=dev)
    ranges = torch.zeros((-(-W // 16)) * (-(-H // 16)), 2, dtype=torch.int32, device=dev)
    nc = torch.zeros(W * H, dtype=torch.int32, device=dev)
    _lib.check(_lib.lib().psb_debug_export(P, R, W, H, geom.data_ptr(), binning.data_ptr() if R else None, img.data_ptr(), None, None, None, None,
                                           None, tt.data_ptr(), None, None, ranges.data_ptr(), nc.data_ptr(), None, None), "psb_debug_export")
    torch.cuda.synchronize()
    return tt.long(), (ranges[:, 1] - ranges[:, 0]).long(), nc.long().reshape(H, W)


def _truth_op(g, cam, bg, D, aa, conv=s64.CONV, mod=1.0):
    """float64 leaves and the truth's render of them; the NDC mean2D is kept for its gradient (dL_dmeans2D)"""
    leaves = {k: v.double().clone().requires_grad_(True) for k, v in g.items()}
    tr = s64.render(leaves, s64.camera64(cam, g["means3D"].device), bg, D=D, aa=aa, scale_modifier=mod, conv=conv)
    tr["geo"]["means2D"].retain_grad()
    return leaves, tr


def _ndc_mean2d_grad(tr, W, H):
    """dL/dmean2D of the truth in the operator's NDC units: dL/dpixel * (W/2, H/2)"""
    return tr["geo"]["means2D"].grad * torch.tensor([0.5 * W, 0.5 * H], dtype=torch.float64, device=tr["geo"]["means2D"].device)


def _check_edge(s, name, tt, list_len, nc, radii, truth):
    """the scene reaches the edge it was built for (kernel side)"""
    e = s["edge"]
    W = s["cam"]["W"]
    if e is None:
        return
    if e[0] == "list":
        gx = -(-W // 16)
        assert int(list_len[e[1][1] * gx + e[1][0]]) == e[2], name
    elif e[0] == "area":
        assert int(tt[e[1]]) == e[2], name
    elif e[0] == "alpha_max":
        assert truth["clamped"].any(), "alpha reaches the 0.99 clamp on some pixels"
    elif e[0] == "colour":
        assert (truth["geo"]["rgb_pre"][truth["geo"]["alive"]] < 0).any(), name
    elif e[0] == "frustum":
        rx, ry = truth["geo"]["ratios"]
        lim = (s64.FRUSTUM * float(s["cam"]["tanfovx"]), s64.FRUSTUM * float(s["cam"]["tanfovy"]))
        idx = list(e[1])
        out = (rx[idx].abs() > lim[0]) | (ry[idx].abs() > lim[1])
        assert out.all() and (radii[idx] > 0).all(), "clamped means whose splats still touch the image"
    elif e[0] == "near":
        assert (radii[list(e[1])] > 0).all() and (radii[list(e[2])] == 0).all()
    elif e[0] == "terminate":
        # pixels whose T crosses 1e-4 inside a 128-entry batch of the second or a later batch, and pixels that never stop
        st = truth["stopped"]
        assert st.any() and (~st).any() and ((nc[st] % 128 != 0) & (nc[st] > 128)).any(), name


OP_CASES = [(n, aa) for n in SCENES for aa in (False, True)]


@pytest.mark.parametrize("name,aa", OP_CASES, ids=[f"{n}-{'aa' if a else 'plain'}" for n, a in OP_CASES])
def test_operator_against_truth(cuda, name, aa):
    s = _scene(name)
    cam, D, bg = s["cam"], s["D"], _bg(name)
    c, g = syn.device_camera(cam, cuda), _op_inputs(s["sc"], cuda)
    bgt = torch.tensor(bg, device=cuda)
    P, W, H = g["means3D"].shape[0], cam["W"], cam["H"]
    R, color, depth, radii, geom, binning, img = _op_forward(g, c, bgt, D, aa)
    tt, list_len, nc = _export(P, R, W, H, geom, binning, img)
    leaves, tr = _truth_op(g, cam, bg, D, aa)
    _check_edge(s, name, tt, list_len, nc, radii, tr)
    assert torch.equal(radii.long(), tr["radii"]) and torch.equal(tt, tr["tiles_touched"])
    assert torch.equal(list_len, tr["list_len"]) and torch.equal(nc, tr["n_contrib"])
    zmax = max(float(tr["depth"].detach().abs().max()), 1e-30)
    errs = dict(color=_maxerr(color, tr["color"].detach()), depth=_maxerr(depth, tr["depth"].detach(), zmax))
    # the colour-only entry RasterizeGaussiansCUDA
    from photo_slam_b200 import rasterizer
    R2, color2, radii2, _, _, _ = rasterizer.RasterizeGaussiansCUDA(bgt, g["means3D"], None, g["opacities"], g["scales"], g["rotations"], 1.0, None,
                                                                    c["viewmatrix"], c["projmatrix"], c["tanfovx"], c["tanfovy"], H, W, g["shs"], D,
                                                                    c["campos"], False, antialiasing=aa)
    assert R2 == R and torch.equal(radii2.long(), tr["radii"])
    errs["color_plain_entry"] = _maxerr(color2, tr["color"].detach())
    wc, wd, _ = _weights(H, W, cuda)
    ((tr["color"] * wc.double()).sum() + (tr["depth"] * wd.double()).sum()).backward()
    for det in (False, True):
        out = rasterizer.RasterizeGaussiansBackwardDepthCUDA(bgt, g["means3D"], radii, None, g["scales"], g["rotations"], 1.0, None, c["viewmatrix"],
                                                             c["projmatrix"], c["tanfovx"], c["tanfovy"], wc, wd, g["shs"], D, c["campos"], geom, R,
                                                             binning, img, deterministic=det, antialiasing=aa)
        d_m2, _, d_op, d_m3, _, d_sh, d_sc, d_rot = out
        m2 = _ndc_mean2d_grad(tr, W, H)
        for k, a, ref in (("means3D", d_m3, leaves["means3D"].grad), ("shs", d_sh, leaves["shs"].grad), ("opacities", d_op, leaves["opacities"].grad),
                          ("scales", d_sc, leaves["scales"].grad), ("rotations", d_rot, leaves["rotations"].grad), ("means2D", d_m2[:, :2], m2)):
            errs[f"grad-{k}-{'det' if det else 'atomic'}"] = _relnorm(a, ref)
            errs[f"gradmax-{k}-{'det' if det else 'atomic'}"] = _maxerr(a, ref, float(ref.abs().max()))
    torch.cuda.synchronize()
    print(f"MEASURED operator {name} aa={aa} margins={min(s['margins'].values()):.2e} {errs}")
    assert errs["color"] < GATE_COLOR and errs["color_plain_entry"] < GATE_COLOR and errs["depth"] < GATE_DEPTH, errs
    _assert_grad_gates(errs)


MOD = 0.6
MOD_CASES = [(n, aa) for n in ("odd-P-129", "alpha-clamp", "terminate-mid-batch", "frustum-clamp") for aa in (False, True)]


def _op_mod_pass(cuda, name, aa):
    """forward and backward of the operator at scale_modifier = MOD, and the truth's render at MOD with its autograd"""
    from photo_slam_b200 import rasterizer
    s = _scene(name)
    cam, D, bg = s["cam"], s["D"], _bg(name)
    c, g = syn.device_camera(cam, cuda), _op_inputs(s["sc"], cuda)
    bgt = torch.tensor(bg, device=cuda)
    R, color, depth, radii, geom, binning, img = _op_forward(g, c, bgt, D, aa, mod=MOD)
    leaves, tr = _truth_op(g, cam, bg, D, aa, mod=MOD)
    wc, wd, _ = _weights(cam["H"], cam["W"], cuda)
    ((tr["color"] * wc.double()).sum() + (tr["depth"] * wd.double()).sum()).backward()
    out = rasterizer.RasterizeGaussiansBackwardDepthCUDA(bgt, g["means3D"], radii, None, g["scales"], g["rotations"], MOD, None, c["viewmatrix"],
                                                         c["projmatrix"], c["tanfovx"], c["tanfovy"], wc, wd, g["shs"], D, c["campos"], geom, R,
                                                         binning, img, antialiasing=aa)
    torch.cuda.synchronize()
    return s, (color, depth, radii), out, leaves, tr


@pytest.mark.parametrize("name,aa", MOD_CASES, ids=[f"{n}-{'aa' if a else 'plain'}" for n, a in MOD_CASES])
def test_operator_scale_modifier_against_truth(cuda, name, aa):
    """scale_modifier = 0.6: the forward draws the splats at 0.6 s; the backward's dL_dscales is the gradient with respect to the modified
    scale 0.6 s (the reference's convention, RasterizeGaussiansBackwardCUDA), i.e. the truth's dL/ds / 0.6"""
    s, (color, depth, radii), out, leaves, tr = _op_mod_pass(cuda, name, aa)
    W, H = s["cam"]["W"], s["cam"]["H"]
    assert torch.equal(radii.long(), tr["radii"])
    zmax = max(float(tr["depth"].detach().abs().max()), 1e-30)
    errs = dict(color=_maxerr(color, tr["color"].detach()), depth=_maxerr(depth, tr["depth"].detach(), zmax))
    d_m2, _, d_op, d_m3, _, d_sh, d_sc, d_rot = out
    for k, a, ref in (("means3D", d_m3, leaves["means3D"].grad), ("shs", d_sh, leaves["shs"].grad), ("opacities", d_op, leaves["opacities"].grad),
                      ("scales", d_sc, leaves["scales"].grad / MOD), ("rotations", d_rot, leaves["rotations"].grad),
                      ("means2D", d_m2[:, :2], _ndc_mean2d_grad(tr, W, H))):
        errs[f"grad-{k}"] = _relnorm(a, ref)
        errs[f"gradmax-{k}"] = _maxerr(a, ref, float(ref.abs().max()))
    print(f"MEASURED operator scale_modifier {name} aa={aa} {errs}")
    assert errs["color"] < GATE_COLOR and errs["depth"] < GATE_DEPTH, errs
    _assert_grad_gates(errs)


# ---- the trainer --------------------------------------------------------------------------------------------------------------------
def _model(sc, dev, D):
    from photo_slam_b200 import trainer
    m = trainer.GaussianModel.from_numpy({k: v.copy() for k, v in sc.items()}, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    m.setShDegree(D)
    return m


def _debug_state(tr, W, H, dev):
    """psb_trainer_debug_state: per pixel the Gaussian index of the last blended splat (-1 = none) and the final transmittance"""
    import ctypes as C
    from photo_slam_b200 import _lib
    last = torch.empty(W * H, dtype=torch.int32, device=dev)
    fT = torch.empty(W * H, dtype=torch.float32, device=dev)
    _lib.check(tr.L.psb_trainer_debug_state(tr.h, W, H, last.data_ptr(), fT.data_ptr(), None, torch.cuda.current_stream().cuda_stream),
               "psb_trainer_debug_state")
    return last.long().reshape(H, W), fT.reshape(H, W)


def _raw_grad_errs(errs, grads, raw, D, prefix="grad"):
    """rel-norm and max-element errors of the six raw-parameter gradient groups against the truth's autograd"""
    for k, a in zip(s64.RAW, grads):
        ref = raw[k].grad
        if k == "features_rest":       # rows of the degrees above the active one get no gradient
            n = (D + 1) ** 2 - 1
            assert not a[:, n:].any()
            a, ref = a[:, :n], ref[:, :n]
        if ref.numel() and ref.abs().max() > 0:
            errs[f"{prefix}-{k}"] = _relnorm(a, ref)
            errs[f"{prefix}max-{k}"] = _maxerr(a, ref, float(ref.abs().max()))
    return errs


def _assert_grad_gates(errs):
    for k, v in errs.items():
        if k.startswith("grad-"):
            assert v < GATE_GRAD, (k, v)
        if k.startswith("gradmax-"):
            assert v < GATE_GRAD_MAX, (k, v)


TR_CASES = [(n, aa, det) for n in SCENES for aa in (False, True) for det in (False, True)]


def _trainer_pass(s, name, cuda, aa, det, conv=s64.CONV):
    """render + backwardPixels(random wc, wd, wa) on the trainer, and the same on the truth -> (kernel outputs, truth, raw leaves)"""
    from photo_slam_b200 import trainer
    cam, D, bg = s["cam"], s["D"], _bg(name)
    c = syn.device_camera(cam, cuda)
    W, H = cam["W"], cam["H"]
    m = _model(s["sc"], cuda, D)
    P = m.num_points()
    tr = trainer.GaussianTrainer(m, background=torch.tensor(bg, device=cuda), deterministic=det, antialiasing=aa)
    img, rad = torch.empty((3, H, W), device=cuda), torch.zeros(P, dtype=torch.int32, device=cuda)
    dep, A = torch.empty((H, W), device=cuda), torch.empty((H, W), device=cuda)
    tr.render(c, img, rad, out_depth=dep, out_alpha=A)
    last, fT = _debug_state(tr, W, H, cuda)
    wc, wd, wa = _weights(H, W, cuda, seed=1)
    grads = [torch.zeros_like(t) for t in m.tensors()]
    tr.backwardPixels(wc, wd, wa, grads=grads)
    tr.result()
    torch.cuda.synchronize()
    raw = {k: v.requires_grad_(True) for k, v in s64.raw64(s["sc"], cuda).items()}
    t = s64.render(raw, s64.camera64(cam, cuda), bg, D=D, aa=aa, raw=True, conv=conv)
    ((t["color"] * wc.double()).sum() + (t["depth"] * wd.double()).sum() + (t["alpha"] * wa.double()).sum()).backward()
    return dict(img=img, rad=rad, dep=dep, A=A, last=last, fT=fT, grads=grads), t, raw


@pytest.mark.parametrize("name,aa,det", TR_CASES, ids=[f"{n}-{'aa' if a else 'plain'}-{'det' if d else 'default'}" for n, a, d in TR_CASES])
def test_trainer_against_truth(cuda, name, aa, det):
    """The trainer blends tight tile lists (only the tiles a splat can reach, for rectangles of at most TIGHT_MAX_AREA tiles), so its
    list lengths differ from the rectangle lists of the truth. That it walks the scene's edge the same way is asserted through
    psb_trainer_debug_state: the last blended Gaussian of every pixel is the truth's and the final T agrees."""
    s = _scene(name)
    k, t, raw = _trainer_pass(s, name, cuda, aa, det)
    assert torch.equal(k["rad"].long(), t["radii"])
    assert torch.equal(k["last"], t["last"]), "the last blended Gaussian of a pixel differs from the truth's"
    if s["edge"] is not None and s["edge"][0] == "terminate":
        assert t["stopped"].any() and (~t["stopped"]).any()
    zmax = max(float(t["depth"].detach().abs().max()), 1e-30)
    errs = dict(color=_maxerr(k["img"], t["color"].detach()), depth=_maxerr(k["dep"], t["depth"].detach(), zmax),
                alpha=_maxerr(k["A"], t["alpha"].detach()), final_T=_maxerr(k["fT"], 1.0 - t["alpha"].detach()))
    _raw_grad_errs(errs, k["grads"], raw, s["D"])
    print(f"MEASURED trainer {name} aa={aa} det={det} {errs}")
    assert errs["color"] < GATE_COLOR and errs["depth"] < GATE_DEPTH and errs["alpha"] < GATE_ALPHA and errs["final_T"] < GATE_ALPHA, errs
    _assert_grad_gates(errs)


# ---- the built-in loss --------------------------------------------------------------------------------------------------------------
E_TEST = [[1.3, 0.1, -0.08, 0.05], [0.04, 0.7, 0.09, -0.06], [-0.07, 0.05, 1.2, 0.03]]    # far from the identity row
LAMBDA_DEPTH = 0.1


def _targets(H, W, dev, seed=3):
    gen = torch.Generator().manual_seed(seed)
    gt = torch.rand((3, H, W), generator=gen).to(dev)
    mask = (torch.rand((1, H, W), generator=gen) > 0.2).float().expand(3, H, W).contiguous().to(dev)
    gd = (0.5 + 6 * torch.rand((H, W), generator=gen)).to(dev)
    gd[(torch.rand((H, W), generator=gen) < 0.2).to(dev)] = 0.0
    return gt, mask, gd


def _truth_loss(s, name, cuda, aa, entry, gt, mask, gd, conv=s64.CONV):
    """float64 loss of the truth's render and its gradients on the raw parameters (and on E with the exposure entry)"""
    raw = {k: v.requires_grad_(True) for k, v in s64.raw64(s["sc"], cuda).items()}
    t = s64.render(raw, s64.camera64(s["cam"], cuda), _bg(name), D=s["D"], aa=aa, raw=True)
    E = torch.tensor(E_TEST, dtype=torch.float64, device=cuda, requires_grad=True) if entry == "exposure" else None
    L, l1, ss = s64.loss64(t["color"], gt.double(), mask.double(), 0.2, E, conv)
    dl1 = s64.depth_l1_64(t["depth"], gd.double(), mask.double()) if entry != "plain" else torch.zeros((), dtype=torch.float64, device=cuda)
    total = L + LAMBDA_DEPTH * dl1
    total.backward()
    return dict(loss=total.item(), l1=l1.item(), ssim=ss.item(), depth_l1=dl1.item(), raw=raw, E=E)


BUILTIN = [("plain", False, False), ("plain", True, True), ("depth", False, True), ("depth", True, False), ("exposure", False, False),
           ("exposure", True, True)]
BUILTIN_CASES = [(n, e, d, a) for n in ("terminate-mid-batch", "alpha-clamp", "colour-clamp-sh2", "small-17x33") for e, d, a in BUILTIN]


def _builtin_backward(s, name, cuda, entry, det, aa, gt, mask, gd):
    """psb_trainer_backward / _depth / _exposure (gradient mode) -> (raw-parameter gradients, dL/dE or None, result_depth())"""
    import ctypes as C
    from photo_slam_b200 import _lib, trainer
    from photo_slam_b200.parallel import GradBuffer
    m = _model(s["sc"], cuda, s["D"])
    tr = trainer.GaussianTrainer(m, background=torch.tensor(_bg(name), device=cuda), deterministic=det, antialiasing=aa)
    tr._apply_deterministic()
    c = syn.device_camera(s["cam"], cuda)       # held until the call has run: _ccamera keeps only its device pointers
    tr.render(c)
    buf = GradBuffer(m.num_points(), cuda)
    cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)
    ptrs = (C.c_void_p * 6)(*[x.data_ptr() for x in buf.segments])
    args = (tr.h, m.num_points(), 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), mask.data_ptr(), C.byref(cs), None, None, ptrs)
    stream = torch.cuda.current_stream().cuda_stream
    egrad = None
    if entry == "plain":
        _lib.check(tr.L.psb_trainer_backward(*args, stream), "psb_trainer_backward")
    elif entry == "depth":
        d = trainer._Depth(gd.data_ptr(), LAMBDA_DEPTH, None)
        _lib.check(tr.L.psb_trainer_backward_depth(*args, C.byref(d), stream), "psb_trainer_backward_depth")
    else:
        d = trainer._Depth(gd.data_ptr(), LAMBDA_DEPTH, None)
        E = torch.tensor(E_TEST, device=cuda)
        ex = trainer._Exposure(E.data_ptr(), None, None, None, 0.01)
        egrad = torch.full((3, 4), float("nan"), device=cuda)
        _lib.check(tr.L.psb_trainer_backward_exposure(*args, C.byref(d), C.byref(ex), egrad.data_ptr(), stream), "psb_trainer_backward_exposure")
    res = tr.result_depth()
    torch.cuda.synchronize()
    return buf.views(), egrad, res


@pytest.mark.parametrize("name,entry,det,aa", BUILTIN_CASES, ids=[f"{n}-{e}-{'det' if d else 'default'}-{'aa' if a else 'plain'}" for n, e, d, a in BUILTIN_CASES])
def test_builtin_loss_gradients_against_truth(cuda, name, entry, det, aa):
    """psb_trainer_backward (plain), _depth (+ 0.1 depth L1) and _exposure (+ the depth term, loss through a far-from-identity E):
    the loss scalars, the raw-parameter gradients and the 12 exposure sums dL/dE, against float64 autograd of the truth"""
    s = _scene(name)
    H, W = s["cam"]["H"], s["cam"]["W"]
    gt, mask, gd = _targets(H, W, cuda)
    grads, egrad, (loss, l1, ssim, dl1, _) = _builtin_backward(s, name, cuda, entry, det, aa, gt, mask, gd)
    t = _truth_loss(s, name, cuda, aa, entry, gt, mask, gd)
    errs = dict(loss=abs(loss - t["loss"]) / t["loss"], l1=abs(l1 - t["l1"]) / t["l1"], ssim=abs(ssim - t["ssim"]) / abs(t["ssim"]))
    if entry != "plain":
        errs["depth_l1"] = abs(dl1 - t["depth_l1"]) / t["depth_l1"]
    _raw_grad_errs(errs, grads, t["raw"], s["D"])
    if egrad is not None:
        errs["grad-E"] = _relnorm(egrad, t["E"].grad)
        errs["gradmax-E"] = _maxerr(egrad, t["E"].grad, float(t["E"].grad.abs().max()))
    print(f"MEASURED builtin {name} {entry} det={det} aa={aa} {errs}")
    for k in ("loss", "l1", "ssim", "depth_l1"):
        assert errs.get(k, 0.0) < GATE_LOSS, errs
    _assert_grad_gates(errs)


def _adam64(p, g, m, v, lr, t, b1=0.9, b2=0.999, eps=1e-15):
    m1 = b1 * m + (1 - b1) * g
    v1 = b2 * v + (1 - b2) * g * g
    return p - lr / (1 - b1 ** t) * m1 / (v1.sqrt() / math.sqrt(1 - b2 ** t) + eps), m1, v1


def _step_err(p1, ref, lr):
    """max over elements of (|kernel - truth| - one float32 spacing of the result) / lr: the update gated relative to lr, less the
    rounding of storing the parameter itself"""
    p1, ref = p1.double(), ref
    ulp = (torch.nextafter(p1.float(), torch.full_like(p1.float(), math.inf)).double() - p1).abs()
    return float(((p1 - ref).abs() - ulp).clamp_min(0).max()) / lr


@pytest.mark.parametrize("name,det", [(n, d) for n in ("terminate-mid-batch", "colour-clamp-sh2") for d in (False, True)],
                         ids=[f"{n}-{'det' if d else 'default'}" for n in ("terminate-mid-batch", "colour-clamp-sh2") for d in (False, True)])
def test_builtin_step_against_float64_adam(cuda, name, det):
    """one psb_trainer_step_exposure (mask, depth target, exposure row 0 = E_TEST) on non-zero Adam moments: every parameter, both
    moments and the exposure row against the float64 gradients of the truth followed by a float64 Adam step"""
    from photo_slam_b200 import trainer
    s = _scene(name)
    cam, D = s["cam"], s["D"]
    H, W = cam["H"], cam["W"]
    gt, mask, gd = _targets(H, W, cuda)
    t = _truth_loss(s, name, cuda, False, "exposure", gt, mask, gd)
    m = _model(s["sc"], cuda, D)
    m.ensureExposures(1)
    m.exposure_[0] = torch.tensor(E_TEST, device=cuda)
    gen = torch.Generator(device=cuda).manual_seed(7)
    refs = [t["raw"][k].grad for k in s64.RAW] + [t["E"].grad]
    params = m.tensors() + [m.exposure_[0]]
    moms = list(zip(m.exp_avg_ + [m.exposure_exp_avg_[0]], m.exp_avg_sq_ + [m.exposure_exp_avg_sq_[0]]))
    for g, (ma, va) in zip(refs, moms):     # moments of the size of the gradient, so that every update is well conditioned
        rms = float(g.pow(2).mean().sqrt()) + 1e-30
        ma.copy_((0.5 * g * (2 * torch.rand(g.shape, device=cuda, generator=gen, dtype=torch.float64) - 1)).float())
        va.copy_((g * g * (0.5 + torch.rand(g.shape, device=cuda, generator=gen, dtype=torch.float64)) + (0.1 * rms) ** 2).float())
        live = (g != 0)
        ma.mul_(live.float())
        va.mul_(live.float())
    m.exposure_step_[0] = 2
    m.invalidateAdamLive()
    p0 = [p.detach().double().clone() for p in params]
    mv0 = [(a.double().clone(), b.double().clone()) for a, b in moms]
    tr = trainer.GaussianTrainer(m, background=torch.tensor(_bg(name), device=cuda), deterministic=det)
    c = syn.device_camera(cam, cuda)
    tr.render(c)
    tr.trainForOneIteration(c, gt, mask, gt_depth=gd, lambda_depth=LAMBDA_DEPTH, exposure_id=0)
    loss = tr.result_depth()[0]
    torch.cuda.synchronize()
    lrs = list(m.lr_) + [m.exposure_lr_]
    steps = [1] * 6 + [3]
    errs = dict(loss=abs(loss - t["loss"]) / t["loss"])
    for k, p, g, (m0, v0), (ma, va), p_0, lr, st in zip(s64.RAW + ("exposure",), params, refs, mv0, moms, p0, lrs, steps):
        p1, m1, v1 = _adam64(p_0, g, m0, v0, lr, st)
        errs[f"step-{k}"] = _step_err(p.detach(), p1, lr)
        errs[f"grad-m-{k}"] = _relnorm(ma, m1)
        errs[f"grad-v-{k}"] = _relnorm(va, v1)
    print(f"MEASURED step {name} det={det} {errs}")
    assert errs["loss"] < GATE_LOSS, errs
    for k, v in errs.items():
        if k.startswith("step-"):
            assert v < GATE_STEP, (k, v)
        if k.startswith("grad-"):
            assert v < GATE_GRAD, (k, v)


# ---- the loss -----------------------------------------------------------------------------------------------------------------------
LOSS_CASES = [((1, 1), "none"), ((1, 37), "none"), ((5, 7), "mask"), ((10, 10), "none"), ((11, 11), "mask"), ((16, 16), "ties"),
              ((17, 33), "mask"), ((241, 17), "ties"), ((480, 640), "mask"), ((17, 33), "zero-mask"), ((480, 640), "none")]


@pytest.mark.parametrize("hw,kind", LOSS_CASES, ids=[f"{h}x{w}-{k}" for (h, w), k in LOSS_CASES])
def test_fused_loss_against_truth(cuda, hw, kind):
    from photo_slam_b200 import trainer
    H, W = hw
    gen = torch.Generator().manual_seed(H * 1000 + W)
    img, gt = torch.rand((3, H, W), generator=gen).to(cuda), torch.rand((3, H, W), generator=gen).to(cuda)
    mask = None
    if kind in ("mask", "zero-mask"):
        mask = (torch.rand((1, H, W), generator=gen) > 0.3).float().expand(3, H, W).contiguous().to(cuda)
        if kind == "zero-mask":
            mask.zero_()
    if kind == "ties":
        gt[:, : H // 2] = img[:, : H // 2]
    loss, l1, ssim, grad = trainer.fused_loss(img, gt, mask, 0.2)
    torch.cuda.synchronize()
    I = img.double().requires_grad_(True)
    L, l1t, sst = s64.loss64(I, gt.double(), mask.double() if mask is not None else None, 0.2)
    L.backward()
    err = max(abs(loss - L.item()) / L.item(), abs(l1 - l1t.item()) / max(l1t.item(), 1e-30), abs(ssim - sst.item()) / abs(sst.item()))
    gerr = _maxerr(grad, I.grad, max(float(I.grad.abs().max()), 1e-30))
    print(f"MEASURED loss {H}x{W} {kind} scalars={err:.2e} grad={gerr:.2e}")
    assert err < GATE_LOSS and gerr < GATE_LOSS_GRAD, (err, gerr)
    if kind == "zero-mask":
        assert not grad.any()


# ---- the gates bite -----------------------------------------------------------------------------------------------------------------
PERTURB = {"dilation": (dict(dilation=0.29), "odd-P-4097", "color"), "alpha_min": (dict(alpha_min=1.0 / 256.0), "terminate-mid-batch", "color"),
           "termination": (dict(t_min=2e-4), "terminate-mid-batch", "color"),
           "clamp-autograd": (dict(straight_through=False), "alpha-clamp", "grad-opacities"),
           "depth-unweighted": (dict(depth_weighted=False), "odd-P-129", "depth")}


@pytest.mark.parametrize("what", list(PERTURB))
def test_perturbed_truth_fails_the_gate(cuda, what):
    """the kernel output against a truth with one convention changed: the gate of that output must reject it"""
    kw, name, out = PERTURB[what]
    s = _scene(name)
    cam, D, bg = s["cam"], s["D"], _bg(name)
    c, g = syn.device_camera(cam, cuda), _op_inputs(s["sc"], cuda)
    bgt = torch.tensor(bg, device=cuda)
    R, color, depth, radii, geom, binning, img = _op_forward(g, c, bgt, D, False)
    leaves, tr = _truth_op(g, cam, bg, D, False, conv=dataclasses.replace(s64.CONV, **kw))
    if out == "color":
        err, gate = _maxerr(color, tr["color"].detach()), GATE_COLOR
    elif out == "depth":
        err, gate = _maxerr(depth, tr["depth"].detach(), float(tr["depth"].detach().abs().max())), GATE_DEPTH
    else:
        from photo_slam_b200 import rasterizer
        wc = _weights(cam["H"], cam["W"], cuda)[0]
        (tr["color"] * wc.double()).sum().backward()
        d_op = rasterizer.RasterizeGaussiansBackwardCUDA(bgt, g["means3D"], radii, None, g["scales"], g["rotations"], 1.0, None, c["viewmatrix"],
                                                         c["projmatrix"], c["tanfovx"], c["tanfovy"], wc, g["shs"], D, c["campos"], geom, R, binning,
                                                         img)[2]
        err, gate = _relnorm(d_op, leaves["opacities"].grad), GATE_GRAD
        errmax = _maxerr(d_op, leaves["opacities"].grad, float(leaves["opacities"].grad.abs().max()))
        assert errmax > GATE_GRAD_MAX, errmax
    print(f"MEASURED perturbed {what}: {err:.2e} (gate {gate:.0e})")
    assert err > gate, f"{what}: the gate does not see the perturbation ({err} <= {gate})"


def test_perturbed_scale_modifier_convention_fails_the_gate(cuda):
    """dL_dscales at scale_modifier = 0.6 against the true dL/ds (the factor applied): the scales gates reject it"""
    _, _, out, leaves, _ = _op_mod_pass(cuda, "odd-P-129", False)
    d_sc, ref = out[6], leaves["scales"].grad
    err, errmax = _relnorm(d_sc, ref), _maxerr(d_sc, ref, float(ref.abs().max()))
    print(f"MEASURED perturbed scale_modifier convention: {err:.2e} (gate {GATE_GRAD:.0e}), max {errmax:.2e} (gate {GATE_GRAD_MAX:.0e})")
    assert err > GATE_GRAD and errmax > GATE_GRAD_MAX


def test_perturbed_ndc_mean2d_fails_the_gate(cuda):
    """dL_dmeans2D against the truth's gradient in pixels instead of NDC: the means2D gate rejects it"""
    name = "odd-P-129"
    s = _scene(name)
    cam, D, bg = s["cam"], s["D"], _bg(name)
    c, g = syn.device_camera(cam, cuda), _op_inputs(s["sc"], cuda)
    bgt = torch.tensor(bg, device=cuda)
    R, color, depth, radii, geom, binning, img = _op_forward(g, c, bgt, D, False)
    leaves, tr = _truth_op(g, cam, bg, D, False)
    wc, wd, _ = _weights(cam["H"], cam["W"], cuda)
    ((tr["color"] * wc.double()).sum() + (tr["depth"] * wd.double()).sum()).backward()
    from photo_slam_b200 import rasterizer
    d_m2 = rasterizer.RasterizeGaussiansBackwardDepthCUDA(bgt, g["means3D"], radii, None, g["scales"], g["rotations"], 1.0, None, c["viewmatrix"],
                                                          c["projmatrix"], c["tanfovx"], c["tanfovy"], wc, wd, g["shs"], D, c["campos"], geom, R,
                                                          binning, img)[0]
    err = _relnorm(d_m2[:, :2], tr["geo"]["means2D"].grad)
    print(f"MEASURED perturbed mean2D in pixels: {err:.2e} (gate {GATE_GRAD:.0e})")
    assert err > GATE_GRAD


@pytest.mark.parametrize("what", ["termination", "clamp-autograd"])
def test_perturbed_truth_fails_the_trainer_gates(cuda, what):
    """termination 2e-4: A and final T; the clamp differentiated by autograd: the raw opacity gradient (rel-norm and max element)"""
    name = "terminate-mid-batch" if what == "termination" else "alpha-clamp"
    conv = dataclasses.replace(s64.CONV, **(dict(t_min=2e-4) if what == "termination" else dict(straight_through=False)))
    k, t, raw = _trainer_pass(_scene(name), name, cuda, False, True, conv=conv)
    if what == "termination":
        errs = dict(alpha=_maxerr(k["A"], t["alpha"].detach()), final_T=_maxerr(k["fT"], 1.0 - t["alpha"].detach()))
        print(f"MEASURED perturbed trainer {what}: {errs}")
        assert errs["alpha"] > GATE_ALPHA and errs["final_T"] > GATE_ALPHA, errs
    else:
        errs = _raw_grad_errs({}, k["grads"], raw, _scene(name)["D"])
        print(f"MEASURED perturbed trainer {what}: {errs}")
        assert errs["grad-opacity"] > GATE_GRAD and errs["gradmax-opacity"] > GATE_GRAD_MAX, errs


def test_perturbed_ssim_window_fails_the_builtin_gradient_and_step_gates(cuda):
    """the SSIM window at sigma 1.4: the built-in loss gradients; a float64 Adam with beta2 = 0.99: the step gate"""
    name = "terminate-mid-batch"
    s = _scene(name)
    gt, mask, gd = _targets(s["cam"]["H"], s["cam"]["W"], cuda)
    grads, egrad, _ = _builtin_backward(s, name, cuda, "exposure", True, False, gt, mask, gd)
    t = _truth_loss(s, name, cuda, False, "exposure", gt, mask, gd, conv=dataclasses.replace(s64.CONV, ssim_sigma=1.4))
    errs = _raw_grad_errs({}, grads, t["raw"], s["D"])
    errs["grad-E"] = _relnorm(egrad, t["E"].grad)
    print(f"MEASURED perturbed builtin ssim_sigma: {errs}")
    assert min(v for k, v in errs.items() if k.startswith("grad-")) > GATE_GRAD, errs
    assert min(v for k, v in errs.items() if k.startswith("gradmax-")) > GATE_GRAD_MAX, errs
    # Adam: the same moments and gradient, beta2 = 0.999 against 0.99
    g = t["raw"]["opacity"].grad
    m0, v0 = 0.5 * g, g * g + 1e-12
    p, lr = torch.zeros_like(g), 0.05
    a = _adam64(p, g, m0, v0, lr, 1)[0]
    b = _adam64(p, g, m0, v0, lr, 1, b2=0.99)[0]
    err = _step_err(b.float(), a, lr)
    print(f"MEASURED perturbed adam beta2: {err:.2e} (gate {GATE_STEP:.0e})")
    assert err > GATE_STEP


def test_perturbed_ssim_window_fails_the_loss_gate(cuda):
    from photo_slam_b200 import trainer
    gen = torch.Generator().manual_seed(0)
    img, gt = torch.rand((3, 41, 37), generator=gen).to(cuda), torch.rand((3, 41, 37), generator=gen).to(cuda)
    loss, _, _, _ = trainer.fused_loss(img, gt, None, 0.2, want_grad=False)
    L, _, _ = s64.loss64(img.double(), gt.double(), None, 0.2, conv=dataclasses.replace(s64.CONV, ssim_sigma=1.4))
    err = abs(loss - L.item()) / L.item()
    _, _, _, grad = trainer.fused_loss(img, gt, None, 0.2)
    I = img.double().requires_grad_(True)
    s64.loss64(I, gt.double(), None, 0.2, conv=dataclasses.replace(s64.CONV, ssim_sigma=1.4))[0].backward()
    gerr = _maxerr(grad, I.grad, float(I.grad.abs().max()))
    print(f"MEASURED perturbed ssim_sigma: {err:.2e} (gate {GATE_LOSS:.0e}), grad {gerr:.2e} (gate {GATE_LOSS_GRAD:.0e})")
    assert err > GATE_LOSS and gerr > GATE_LOSS_GRAD
