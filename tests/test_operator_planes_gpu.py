"""-m gpu: the accumulated opacity A, the normal plane N and the second depth moment M on the rasterizer operator path
(psb_rasterize_forward_planes / psb_rasterize_backward_planes, the B1 glue, GaussianRasterizer(..., return_alpha / return_normal /
return_depth2), renderer.render and the LibTorch drop-in).

A, N and M blend exactly like a colour whose per-Gaussian value is (1, 1, 1), n_i or (z^2, 0, 0) with a black background. Their
reference chain is therefore the reference's own rasterizer called once for the colour and once per plane with those colours, n_i
formed in torch from the scales, rotations and view matrix, and autograd through torch (test_depth_operator_gpu.py's method). Its
outputs are stored in tests/golden/test_operator_planes_gpu.npz, written on an H100 by
`python tests/golden/make_ref_golden.py test_operator_planes_gpu` (reference_cases() below). The reference has no anti-aliasing, so the
anti-aliased cases are checked against the same chain on this project's plain operator. Beyond that: the planes and gradients against
the float64 restatement (normal64, dist64, splat64) on settled scenes, the operator's raw-parameter gradients against the fused
backward, and renderer.render in every branch against the fused render."""
import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn
import dist64
import normal64
import splat64 as s64
from helpers import Gold, rel_close
from test_depth_operator_gpu import CASES, _RefRasterize, _export, _few, _inputs, _rn

MODULE = "test_operator_planes_gpu"

pytestmark = pytest.mark.gpu

LEAVES = ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")


def _settings(c, bg, D, aa):
    from photo_slam_b200 import rasterizer
    return rasterizer.GaussianRasterizationSettings(c["H"], c["W"], c["tanfovx"], c["tanfovy"], bg, 1.0, c["viewmatrix"], c["projmatrix"], D,
                                                    c["campos"], False, aa)


def _leaves(x):
    out = {k: v.clone().requires_grad_(True) for k, v in x.items()}
    out["means2D"] = torch.zeros_like(x["means3D"], requires_grad=True)
    return out


def _grads(lv):
    d = {k: v.grad for k, v in lv.items() if k != "means2D"}
    d["means2D"] = lv["means2D"].grad[:, :2]
    return d


def torch_normals(means3D, scales, rotations, viewmatrix):
    """n_i of include/psb200.h in torch: column k = argmin(scales) of R(q) for q as given, turned by V and signed towards the camera; the
    arg-min and the sign are constants of the graph, so the gradient reaches the rotations only."""
    V = viewmatrix.reshape(4, 4)        # column-major storage: V[c, r] is row r, column c of the view matrix
    Rv = V[:3, :3].t()
    w, x, y, z = rotations.unbind(1)
    cols = torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + w * z), 2 * (x * z - w * y)], 1),
        torch.stack([2 * (x * y - w * z), 1 - 2 * (x * x + z * z), 2 * (y * z + w * x)], 1),
        torch.stack([2 * (x * z + w * y), 2 * (y * z - w * x), 1 - 2 * (x * x + y * y)], 1)], 1)   # [P, k, 3]
    k = torch.argmin(scales.detach(), dim=1)
    r = cols[torch.arange(len(k), device=k.device), k]
    m = r @ Rv.t()
    t = means3D.detach() @ Rv.t() + V[3, :3]
    sign = torch.where((m.detach() * t).sum(1) <= 0, 1.0, -1.0)
    return m * sign[:, None]


def _weights(H, W, dev, seed=31):
    g = torch.Generator().manual_seed(seed)
    f = lambda *s: (torch.rand(s, generator=g) - 0.5).to(dev)
    return dict(color=f(3, H, W), depth=f(H, W), alpha=f(H, W), normal=f(3, H, W), depth2=f(H, W) * 0.1)


def _mine(c, x, bg, aa, wts, planes, deterministic=False):
    from photo_slam_b200 import rasterizer
    lv = _leaves(x)
    r = rasterizer.GaussianRasterizer(_settings(c, bg, 3 if "shs" in x else 0, aa))
    kw = {k: lv[k] for k in LEAVES if k in lv and k not in ("means3D", "opacities")}
    flags = dict(return_depth="depth" in planes, return_alpha="alpha" in planes, return_normal="normal" in planes,
                 return_depth2="depth2" in planes)
    out = r(lv["means3D"], lv["means2D"], lv["opacities"], deterministic=deterministic, **kw, **flags)
    got = dict(color=out[0], **dict(zip([p for p in ("depth", "alpha", "normal", "depth2") if p in planes], out[2:])))
    sum((wts[k] * v).sum() for k, v in got.items()).backward()
    torch.cuda.synchronize()
    return {k: v.detach() for k, v in got.items()}, out[1], _grads(lv)


def _plane_colours(lv, c, planes):
    """the per-Gaussian colour each plane blends: (z, 0, 0), (1, 1, 1), n_i, (z^2, 0, 0)"""
    V = c["viewmatrix"].reshape(-1)
    z = lv["means3D"] @ V[[2, 6, 10]] + V[14]
    zero = torch.zeros_like(z)
    cols = dict(depth=torch.stack([z, zero, zero], 1), alpha=torch.ones_like(lv["means3D"]), depth2=torch.stack([z * z, zero, zero], 1))
    if "normal" in planes:
        cols["normal"] = torch_normals(lv["means3D"], lv["scales"], lv["rotations"], c["viewmatrix"])
    return cols


def _chain(c, x, bg, aa, wts, planes):
    """each plane as a colour of the plain operator with a black background, n_i / z from torch, autograd through all of them"""
    from photo_slam_b200 import rasterizer
    lv = _leaves(x)
    D = 3 if "shs" in x else 0
    geo = {k: lv[k] for k in ("scales", "rotations", "cov3D_precomp") if k in lv}
    img, radii = rasterizer.GaussianRasterizer(_settings(c, bg, D, aa))(
        lv["means3D"], lv["means2D"], lv["opacities"], shs=lv.get("shs"), colors_precomp=lv.get("colors_precomp"), **geo)
    got = dict(color=img)
    black = rasterizer.GaussianRasterizer(_settings(c, torch.zeros(3, device=bg.device), 0, aa))
    cols = _plane_colours(lv, c, planes)
    for p in planes:
        o, _ = black(lv["means3D"], lv["means2D"], lv["opacities"], colors_precomp=cols[p].contiguous(), **geo)
        got[p] = o if p == "normal" else o[0]
    sum((wts[k] * v).sum() for k, v in got.items()).backward()
    torch.cuda.synchronize()
    return {k: v.detach() for k, v in got.items()}, radii, _grads(lv)


def _planes_of(case):
    return ("depth", "alpha", "depth2") if case == "cov3d" else ("depth", "alpha", "normal", "depth2")


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("case", CASES)
def test_planes_and_gradients_match_the_colour_chain(cuda, case, aa):
    _, c, x, bg, _, _ = _inputs(cuda, case)
    planes = _planes_of(case)
    wts = _weights(c["H"], c["W"], cuda)
    mine, radii, gm = _mine(c, x, bg, aa, wts, planes)
    ref, radii_ref, gr = _chain(c, x, bg, aa, wts, planes)
    _, _, gr2 = _chain(c, x, bg, aa, wts, planes)      # the chain's own run-to-run spread (float atomics) is the floor
    assert torch.equal(radii, radii_ref)
    assert torch.equal(mine["color"], ref["color"])
    for p in planes:
        assert rel_close(mine[p], ref[p], rtol=1e-4, atol=1e-6) <= 5e-4, p
    vis = radii > 0
    for k in gr:
        a, b, b2 = gm[k][vis].reshape(-1), gr[k][vis].reshape(-1), gr2[k][vis].reshape(-1)
        scale = b.abs().max().item() + 1e-30
        self_frac = rel_close(b2, b, rtol=1e-4, atol=1e-6 * scale)
        frac = rel_close(a, b, rtol=1e-4, atol=1e-6 * scale)
        print(f"{case} aa={aa}: grad {k}: frac>1e-4 {frac:.2e} (chain vs itself {self_frac:.2e}), rel-norm {_rn(a, b):.2e}")
        assert _rn(a, b) <= 1e-4, (k, _rn(a, b))
        assert frac <= max(1e-3, 3 * self_frac), (k, frac, self_frac)
        assert not gm[k][~vis].any(), k


def _b1_fwd(c, x, bg, aa, **planes):
    from photo_slam_b200 import rasterizer
    e = torch.empty(0, device=bg.device)
    get = lambda k: x.get(k, e)
    return rasterizer.RasterizeGaussiansPlanesCUDA(bg, x["means3D"], get("colors_precomp"), x["opacities"], get("scales"), get("rotations"), 1.0,
                                                   get("cov3D_precomp"), c["viewmatrix"], c["projmatrix"], c["tanfovx"], c["tanfovy"], c["H"],
                                                   c["W"], get("shs"), 3 if "shs" in x else 0, c["campos"], False, antialiasing=aa, **planes)


def _b1_bwd(c, x, bg, aa, fwd, dpix, grads, deterministic):
    from photo_slam_b200 import rasterizer
    e = torch.empty(0, device=bg.device)
    get = lambda k: x.get(k, e)
    R, radii, gb, bb, ib = fwd[0], fwd[6], fwd[7], fwd[8], fwd[9]
    return rasterizer.RasterizeGaussiansBackwardPlanesCUDA(
        bg, x["means3D"], radii, get("colors_precomp"), get("scales"), get("rotations"), 1.0, get("cov3D_precomp"), c["viewmatrix"],
        c["projmatrix"], c["tanfovx"], c["tanfovy"], dpix, grads.get("depth"), grads.get("alpha"), grads.get("normal"), grads.get("depth2"),
        get("shs"), 3 if "shs" in x else 0, c["campos"], gb, R, bb, ib, deterministic=deterministic, antialiasing=aa)


@pytest.mark.parametrize("aa", [False, True])
@pytest.mark.parametrize("case", CASES)
def test_unchanged_when_unused_and_bit_identical_beside_the_planes(cuda, case, aa):
    from photo_slam_b200 import rasterizer
    _, c, x, bg, _, _ = _inputs(cuda, case)
    W, H, P = c["W"], c["H"], x["means3D"].shape[0]
    plain = _b1_fwd(c, x, bg, aa, depth=True)
    none = _c_planes_forward(c, x, bg, aa)               # psb_rasterize_forward_planes with every field of the record NULL
    kw = {p: True for p in _planes_of(case)}
    full = _b1_fwd(c, x, bg, aa, **kw)
    e0 = _export(P, plain[0], W, H, plain[7], plain[8], plain[9])
    for other, depth_too in ((none, False), (full, True)):
        assert other[0] == plain[0] and torch.equal(other[1], plain[1]) and torch.equal(other[6], plain[6])
        if depth_too:
            assert torch.equal(other[2], plain[2])
        e1 = _export(P, other[0], W, H, other[7], other[8], other[9])
        for k in e0:
            assert torch.equal(e0[k], e1[k]), k
    assert torch.equal(full[3], 1.0 - e0["final_T"].reshape(H, W))    # A = 1 - T_final, bit for bit
    # no gradient: the deterministic planes backward is psb_rasterize_backward_aa's, bit for bit
    g = torch.Generator().manual_seed(41)
    dpix = torch.rand((3, H, W), generator=g).to(cuda)
    ddep = torch.rand((H, W), generator=g).to(cuda)
    b = rasterizer.RasterizeGaussiansBackwardDepthCUDA(*_plain_bwd_args(c, x, bg, full, dpix, ddep), deterministic=True, antialiasing=aa)
    b0 = rasterizer.RasterizeGaussiansBackwardDepthCUDA(*_plain_bwd_args(c, x, bg, full, dpix, None), deterministic=True, antialiasing=aa)
    for a, ref in ((_c_planes_backward(c, x, bg, aa, full, dpix, ddep), b),          # the depth gradient alone in the record
                   (_c_planes_backward(c, x, bg, aa, full, dpix, None), b0),         # every field NULL
                   (_c_planes_backward(c, x, bg, aa, full, dpix, None, record=False), b0)):   # a NULL record
        for u, v in zip(a, ref):
            assert torch.equal(u, v)
    # the atomic mode with a NULL record is psb_rasterize_backward_aa's atomic backward (equal up to the order of float atomics)
    a = _c_planes_backward(c, x, bg, aa, full, dpix, None, record=False, det=False)
    ref = rasterizer.RasterizeGaussiansBackwardDepthCUDA(*_plain_bwd_args(c, x, bg, full, dpix, None), antialiasing=aa)
    for u, v in zip(a, ref):
        if v.numel():
            assert _rn(u, v) <= 1e-5


def _c_planes_forward(c, x, bg, aa):
    from photo_slam_b200 import _lib, rasterizer
    L = _lib.lib()
    e = torch.empty(0, device=bg.device)
    get = lambda k: x.get(k, e)
    P, H, W = x["means3D"].shape[0], c["H"], c["W"]
    out = torch.zeros((3, H, W), device=bg.device)
    radii = torch.zeros((P,), dtype=torch.int32, device=bg.device)
    geom, binning, img = (rasterizer._Scratch(bg.device) for _ in range(3))
    p = rasterizer._ptr
    rec = _lib.RasterPlanes(None, None, None, None)
    R = _lib.check(L.psb_rasterize_forward_planes(
        geom.cb, None, binning.cb, None, img.cb, None, P, 3 if "shs" in x else 0, 16 if "shs" in x else 0, p(bg), W, H, p(x["means3D"]),
        p(get("shs")), p(get("colors_precomp")), p(x["opacities"]), p(get("scales")), 1.0, p(get("rotations")), p(get("cov3D_precomp")),
        p(c["viewmatrix"]), p(c["projmatrix"]), p(c["campos"]), c["tanfovx"], c["tanfovy"], 0, out.data_ptr(), radii.data_ptr(),
        rasterizer.C.byref(rec), None, 0, int(aa), rasterizer._stream()), "psb_rasterize_forward_planes")
    return (R, out, None, None, None, None, radii, geom.tensor, binning.tensor, img.tensor)


def _c_planes_backward(c, x, bg, aa, fwd, dpix, ddep, record=True, det=True):
    """psb_rasterize_backward_planes with the depth gradient (or None) alone in the record; record=False: a NULL record; det: the
    deterministic mode over psb_rasterize_backward_det_bytes(P, R), else the atomic one without det_scratch"""
    from photo_slam_b200 import _lib, rasterizer
    L = _lib.lib()
    e = torch.empty(0, device=bg.device)
    get = lambda k: x.get(k, e)
    P, H, W, R = x["means3D"].shape[0], c["H"], c["W"], fwd[0]
    M = 16 if "shs" in x else 0
    z = lambda *s: torch.zeros(s, device=bg.device)
    outs = [z(P, 3), z(P, 2, 2), z(P, 1), z(P, 3), z(P, 3), z(P, 6), z(P, M, 3), z(P, 3), z(P, 4)]
    dz = z(P) if ddep is not None else None
    nbytes = L.psb_rasterize_backward_det_bytes(P, R) if det else 0
    scratch = torch.empty((nbytes,), dtype=torch.uint8, device=bg.device) if det else None
    p = rasterizer._ptr
    rec = _lib.RasterPlaneGrads(p(ddep), None, None, None)
    _lib.check(L.psb_rasterize_backward_planes(
        P, 3 if "shs" in x else 0, M, R, p(bg), W, H, p(x["means3D"]), p(get("shs")), p(get("colors_precomp")), p(get("scales")), 1.0,
        p(get("rotations")), p(get("cov3D_precomp")), p(c["viewmatrix"]), p(c["projmatrix"]), p(c["campos"]), c["tanfovx"], c["tanfovy"],
        fwd[6].data_ptr(), fwd[7].data_ptr(), p(fwd[8]), fwd[9].data_ptr(), dpix.data_ptr(), *[p(t) for t in outs],
        rasterizer.C.byref(rec) if record else None, p(dz), p(scratch), nbytes, None, 0, int(aa), int(det), rasterizer._stream()),
        "psb_rasterize_backward_planes")
    dm2, dconic, dop, dcol, dm3, dcov, dsh, dsc, drot = outs
    return dm2, dcol, dop, dm3, dcov, dsh, dsc, drot


def _plain_bwd_args(c, x, bg, fwd, dpix, ddep):
    e = torch.empty(0, device=bg.device)
    get = lambda k: x.get(k, e)
    return (bg, x["means3D"], fwd[6], get("colors_precomp"), get("scales"), get("rotations"), 1.0, get("cov3D_precomp"), c["viewmatrix"],
            c["projmatrix"], c["tanfovx"], c["tanfovy"], dpix, ddep, get("shs"), 3 if "shs" in x else 0, c["campos"], fwd[7], fwd[0], fwd[8],
            fwd[9])


@pytest.mark.parametrize("aa", [False, True])
def test_deterministic_backward_with_every_plane_is_bit_identical(cuda, aa):
    _, c, x, bg, _, _ = _inputs(cuda, "sh3")
    wts = _weights(c["H"], c["W"], cuda)
    planes = _planes_of("sh3")
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        runs = [_mine(c, x, bg, aa, wts, planes, deterministic=True)[2] for _ in range(3)]
    finally:
        torch.use_deterministic_algorithms(prev)
    for r in runs[1:]:
        for k in r:
            assert torch.equal(r[k], runs[0][k]), k
    # and the deterministic sums are the atomic ones up to summation order
    atomic = _mine(c, x, bg, aa, wts, planes)[2]
    for k in atomic:
        assert _rn(atomic[k], runs[0][k]) <= 1e-5, k


def test_a_loss_that_ignores_the_planes_runs_the_plain_backward(cuda):
    _, c, x, bg, _, _ = _inputs(cuda, "sh3")
    wts = _weights(c["H"], c["W"], cuda)
    a = _mine(c, x, bg, False, {"color": wts["color"]}, (), deterministic=True)[2]
    from photo_slam_b200 import rasterizer
    lv = _leaves(x)
    r = rasterizer.GaussianRasterizer(_settings(c, bg, 3, False))
    kw = {k: lv[k] for k in LEAVES if k in lv and k not in ("means3D", "opacities")}
    out = r(lv["means3D"], lv["means2D"], lv["opacities"], deterministic=True, return_alpha=True, return_normal=True, return_depth2=True, **kw)
    (wts["color"] * out[0]).sum().backward()     # the planes get no gradient: they arrive as None
    b = _grads(lv)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_libtorch_planes_ops_equal_the_ctypes_path(cuda):
    import os
    from photo_slam_b200 import _lib
    lib = os.path.join(os.path.dirname(_lib.LIB_PATH), "libcuda_rasterizer.so")
    torch.ops.load_library(lib)
    for case in ("sh3", "cov3d"):
        _, c, x, bg, _, _ = _inputs(cuda, case)
        kw = {p: True for p in _planes_of(case)}
        for aa in (False, True):
            py = _b1_fwd(c, x, bg, aa, **kw)
            e = torch.empty(0, device=cuda)
            get = lambda k: x.get(k, e)
            cc = torch.ops.psb200.rasterize_gaussians_planes(
                bg, x["means3D"], get("colors_precomp"), x["opacities"], get("scales"), get("rotations"), 1.0, get("cov3D_precomp"),
                c["viewmatrix"], c["projmatrix"], c["tanfovx"], c["tanfovy"], c["H"], c["W"], get("shs"), 3 if "shs" in x else 0, c["campos"],
                False, kw.get("depth", False), kw.get("alpha", False), kw.get("normal", False), kw.get("depth2", False), aa)
            assert cc[0] == py[0]
            for i in (1, 2, 3, 4, 5, 6):
                assert (py[i] is None and (cc[i] is None or cc[i].numel() == 0)) or torch.equal(cc[i], py[i]), (case, aa, i)
            g = torch.Generator().manual_seed(43)
            H, W = c["H"], c["W"]
            dpix = torch.rand((3, H, W), generator=g).to(cuda)
            grads = {p: torch.rand((3, H, W) if p == "normal" else (H, W), generator=g).to(cuda) for p in kw}
            a = _b1_bwd(c, x, bg, aa, py, dpix, grads, True)
            b = torch.ops.psb200.rasterize_gaussians_backward_planes(
                bg, x["means3D"], py[6], get("colors_precomp"), get("scales"), get("rotations"), 1.0, get("cov3D_precomp"), c["viewmatrix"],
                c["projmatrix"], c["tanfovx"], c["tanfovy"], dpix, grads.get("depth"), grads.get("alpha"), grads.get("normal"),
                grads.get("depth2"), get("shs"), 3 if "shs" in x else 0, c["campos"], py[7], py[0], py[8], py[9], aa, True)
            for u, v in zip(a, b):
                assert torch.equal(u, v), (case, aa)


def test_empty_and_fully_culled_scenes(cuda):
    _, c, x, bg, _, _ = _inputs(cuda, "sh3")
    H, W = c["H"], c["W"]
    wts = _weights(H, W, cuda)
    planes = _planes_of("sh3")
    empty = {k: v[:0].contiguous() for k, v in x.items()}
    out = _b1_fwd(c, empty, bg, False, depth=True, alpha=True, normal=True, depth2=True)
    assert out[0] == 0 and all(out[i].abs().max().item() == 0.0 for i in (2, 3, 4, 5))
    behind = dict(x)
    V = c["viewmatrix"].reshape(4, 4)
    # every mean behind the camera: view z = -1 for all of them
    Rv, tv = V[:3, :3].t(), V[3, :3]
    behind["means3D"] = ((torch.tensor([0.0, 0.0, -1.0], device=cuda) - tv) @ Rv).expand_as(x["means3D"]).contiguous()
    for det in (False, True):
        got, radii, g = _mine(c, behind, bg, False, wts, planes, deterministic=det)
        assert int((radii > 0).sum()) == 0
        for p in planes:
            assert got[p].abs().max().item() == 0.0
        for k, v in g.items():
            assert v.abs().max().item() == 0.0, k
    assert np.isfinite(got["color"].cpu().numpy()).all()


def _ref_chain_once(c, x, bg, wts, planes):
    """the reference's rasterizer: once for the colour, once per plane with its colours on a black background; autograd through all"""
    lv = _leaves(x)
    e = torch.empty(0, device=bg.device)
    get = lambda k: lv.get(k, e)
    rs = dict(bg=bg, viewmatrix=c["viewmatrix"], projmatrix=c["projmatrix"], campos=c["campos"], tanfovx=c["tanfovx"], tanfovy=c["tanfovy"],
              H=c["H"], W=c["W"], D=3 if "shs" in x else 0)
    geo = (get("scales"), get("rotations"), get("cov3D_precomp"))
    img, radii = _RefRasterize.apply(lv["means3D"], lv["means2D"], get("shs"), get("colors_precomp"), lv["opacities"], *geo, rs)
    got = dict(color=img)
    rs_black = dict(rs, bg=torch.zeros(3, device=bg.device), D=0)
    cols = _plane_colours(lv, c, planes)
    for p in planes:
        o, _ = _RefRasterize.apply(lv["means3D"], lv["means2D"], e, cols[p].contiguous(), lv["opacities"], *geo, rs_black)
        got[p] = o if p == "normal" else o[0]
    sum((wts[k] * v).sum() for k, v in got.items()).backward()
    torch.cuda.synchronize()
    return {k: v.detach() for k, v in got.items()}, radii, _grads(lv)


def _reference(cuda, case):
    _, c, x, bg, _, _ = _inputs(cuda, case)
    planes = _planes_of(case)
    wts = _weights(c["H"], c["W"], cuda)
    got, radii, grads = _ref_chain_once(c, x, bg, wts, planes)
    _, _, grads2 = _ref_chain_once(c, x, bg, wts, planes)     # the reference's own run-to-run spread (float atomics) is the floor
    d = dict(radii=radii, **got)
    vis = radii > 0
    for k, b in grads.items():
        b, b2 = b.reshape(b.shape[0], -1), grads2[k].reshape(b.shape[0], -1)
        scale = b.abs().max().item()
        d["grad_" + k], d["grad_" + k + "#max"] = b, scale
        d["grad_" + k + "#self"] = rel_close(b2[vis], b[vis], rtol=1e-4, atol=1e-6 * (scale + 1e-30))
    return d


@pytest.mark.parametrize("case", CASES)
def test_planes_and_gradients_match_the_reference_chain(cuda, case):
    """GaussianRasterizer with every plane of the case under a random linear loss on colour, D, A, N and M vs autograd of the reference
    chain (stored): each plane per element at 1e-4, and the gradients of every input the case has plus means2D.grad[:, :2] per element
    at 1e-4 against the reference-vs-itself floor, with the bounds of test_depth_operator_gpu.py."""
    r = Gold(MODULE, case)
    _, c, x, bg, _, _ = _inputs(cuda, case)
    planes = _planes_of(case)
    P = x["means3D"].size(0)
    mine, radii, grads = _mine(c, x, bg, False, _weights(c["H"], c["W"], cuda), planes)
    a, b = r.pair("radii", radii)
    assert (a != b).double().mean().item() <= _few(1 / 5000)
    assert r.frac("color", mine["color"], atol=1e-6) <= _few(5e-4)
    for p in planes:
        frac = r.frac(p, mine[p], rtol=1e-4, atol=1e-6)
        print(f"{case}: {p}: {frac:.2e} of the sampled pixels outside 1e-4")
        assert frac <= _few(5e-4), p
    vis = radii > 0
    for k, g in grads.items():
        g = g.reshape(P, -1)
        key = "grad_" + k
        scale, self_frac = r[key + "#max"] + 1e-30, r[key + "#self"]
        xm, ym = r.pair(key, g)
        live = (xm != 0) | (ym != 0)
        frac = rel_close(xm[live], ym[live], rtol=1e-4, atol=1e-6 * scale)
        nrm = ((xm - ym).norm() / (ym.norm() + 1e-30)).item()
        print(f"{case}: grad {k}: frac>1e-4 {frac:.2e} (reference vs itself {self_frac:.2e}), rel-norm {nrm:.2e}")
        assert nrm < 2e-4, f"{k}: relative norm error {nrm}"
        assert frac <= _few(max(1e-3, 3 * self_frac)), f"{k}: {frac} of the sampled entries outside 1e-4 (reference vs itself: {self_frac})"
        assert not g[~vis].any(), f"{k}: rows of invisible Gaussians must be zero"


def _fused_planes(m, c, aa):
    """the fused render's colour, D, A, N, M of model m (psb_trainer_forward_moment with the normal plane) and its trainer"""
    from photo_slam_b200 import trainer
    H, W = c["H"], c["W"]
    tr = trainer.GaussianTrainer(m, antialiasing=aa, deterministic=True)
    tr._apply_deterministic()
    out = dict(color=torch.empty((3, H, W), device=m.device), depth=torch.empty((H, W), device=m.device),
               alpha=torch.empty((H, W), device=m.device), normal=torch.empty((3, H, W), device=m.device),
               depth2=torch.empty((H, W), device=m.device))
    tr.render(c, out["color"], out_depth=out["depth"], out_alpha=out["alpha"], out_normal=out["normal"], out_depth2=out["depth2"])
    torch.cuda.synchronize()
    return tr, out


def _render_planes(m, c, pipe, **kw):
    from photo_slam_b200 import renderer
    flags = dict(return_depth=True, return_alpha=True, return_normal=not pipe.compute_cov3D, return_depth2=True)
    out = renderer.render(c, c["H"], c["W"], m, pipe, **flags, **kw)
    names = ["depth", "alpha"] + (["normal"] if flags["return_normal"] else []) + ["depth2"]
    return dict(color=out[0], **dict(zip(names, out[4:])))


@pytest.mark.parametrize("aa", [False, True])
def test_operator_plane_gradients_match_the_fused_backward(cuda, aa):
    """Default branch: autograd's raw-parameter gradients of a random linear loss on colour, D, A, N and M through renderer.render (the
    operator, chained through torch's sigmoid, exp and normalize) equal psb_trainer_backward_pixels_moment's (gradient mode, with the
    normal gradient) for the same per-pixel gradients. The two share no kernel of the plane backward, and the operator forms n_i from
    activated scales and the rotation as given, the fused step from log-scales and the normalised rotation."""
    from photo_slam_b200 import renderer, trainer
    from photo_slam_b200.parallel import GradBuffer
    sc, c, _, _, _, _ = _inputs(cuda, "sh3")
    wts = _weights(c["H"], c["W"], cuda)
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    for t in m.tensors():
        t.requires_grad_(True)
    got = _render_planes(m, c, renderer.GaussianPipelineParams(antialiasing=aa))
    sum((wts[k] * v).sum() for k, v in got.items()).backward()
    torch.cuda.synchronize()
    fm = trainer.GaussianModel.from_numpy(sc, cuda)
    fm.trainingSetup(trainer.GaussianOptimizationParams())
    tr, fused = _fused_planes(fm, c, aa)
    for k in got:
        print(f"aa={aa}: {k}: rel-norm vs fused render {_rn(got[k], fused[k]):.2e}")
        assert _rn(got[k], fused[k]) < 1e-5, k
    buf = GradBuffer(fm.num_points(), cuda)
    tr.backwardPixels(wts["color"], wts["depth"], wts["alpha"], grads=buf.views(), dL_dnormal=wts["normal"], dL_ddepth2=wts["depth2"])
    torch.cuda.synchronize()
    for name, t, g in zip(trainer.GROUPS, m.tensors(), buf.views()):
        rn = _rn(t.grad.reshape(-1), g.reshape(-1))
        print(f"aa={aa}: grad {name}: operator path vs fused backward, rel-norm {rn:.2e}")
        assert rn <= 1e-4, (name, rn)


def test_renderer_planes_in_every_branch_match_the_fused_render(cuda):
    """renderer.render's A, N and M in every pipeline branch equal the fused render's (psb_trainer_forward_moment with the normal plane);
    N with compute_cov3D is refused, and gradients reach the model from every plane in every branch."""
    from photo_slam_b200 import renderer, trainer
    sc, c, _, _, _, _ = _inputs(cuda, "sh3")
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    _, fused = _fused_planes(trainer.GaussianModel.from_numpy(sc, cuda), c, False)
    col = torch.rand((m.num_points(), 3), device=cuda, generator=torch.Generator(device=cuda).manual_seed(3))
    branches = (("default", renderer.GaussianPipelineParams(), {}, 1e-5), ("convert_SHs", renderer.GaussianPipelineParams(convert_SHs=True), {}, 1e-5),
                ("override_color", renderer.GaussianPipelineParams(), dict(override_color=col, use_override_color=True), 1e-5),
                ("compute_cov3D", renderer.GaussianPipelineParams(compute_cov3D=True), {}, 1e-4))
    with torch.no_grad():
        plain = renderer.render(c, c["H"], c["W"], m)
        for name, pipe, kw, tol in branches:
            got = _render_planes(m, c, pipe, **kw)
            if name == "default":
                assert torch.equal(got["color"], plain[0])
            for k in ("depth", "alpha", "normal", "depth2"):
                if k in got:
                    print(f"renderer {name}: {k}: rel-norm vs fused render {_rn(got[k], fused[k]):.2e}")
                    assert _rn(got[k], fused[k]) < tol, (name, k, _rn(got[k], fused[k]))
    with pytest.raises(RuntimeError, match="return_normal needs scales and rotations"):
        renderer.render(c, c["H"], c["W"], m, renderer.GaussianPipelineParams(compute_cov3D=True), return_normal=True)
    wts = _weights(c["H"], c["W"], cuda)
    for name, pipe, kw, _ in branches:
        for t in m.tensors():
            t.requires_grad_(True)
            t.grad = None
        got = _render_planes(m, c, pipe, **kw)
        sum((wts[k] * v).sum() for k, v in got.items() if k != "color").backward()
        assert m.xyz_.grad.abs().sum().item() > 0 and m.opacity_.grad.abs().sum().item() > 0, name
        if name != "compute_cov3D":
            assert m.rotation_.grad.abs().sum().item() > 0, name
        for t in m.tensors():
            t.requires_grad_(False)


_SETTLED = {}


def _settled(name):
    """small dense scenes (splat64.settle: every decision at least 1e-4 from its threshold), as tests/test_normal_gpu.py builds them"""
    if name not in _SETTLED:
        seed, P, W, H = {"a": (5, 700, 64, 48), "b": (6, 1500, 80, 56)}[name]
        cam = syn.make_camera(W, H, 0.9 * W, 0.9 * W, *syn.random_pose(np.random.default_rng(seed)))
        sc = syn.make_scene(P, cam, seed=seed, scale_px=3.0)
        s64.settle(sc, cam, D=1, aa=None, bg=(0.0, 0.0, 0.0), seed=1, dev="cuda")
        _SETTLED[name] = (cam, sc)
    return _SETTLED[name]


@pytest.mark.parametrize("name,aa", [("a", False), ("b", False), ("a", True), ("b", True)])
def test_planes_and_gradients_against_float64(cuda, name, aa):
    """renderer.render's D, A, N, M on settled scenes against the float64 restatement (splat64, normal64, dist64), and the raw-parameter
    gradients of a random linear loss on colour and every plane against autograd on it."""
    from photo_slam_b200 import renderer, trainer
    cam, sc = _settled(name)
    c = syn.device_camera(cam, cuda)
    W, H = c["W"], c["H"]
    wts = _weights(H, W, cuda, seed=7)
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.setShDegree(1)
    for t in m.tensors():
        t.requires_grad_(True)
    got = _render_planes(m, c, renderer.GaussianPipelineParams(antialiasing=aa))
    sum((wts[k] * v).sum() for k, v in got.items()).backward()
    torch.cuda.synchronize()
    raw = {k: v.requires_grad_(True) for k, v in s64.raw64(sc, cuda).items()}
    cam64 = s64.camera64(cam, cuda)
    out, N64 = normal64.render_normal(raw, cam64, D=1, aa=aa)
    _, M64 = dist64.render_moment(raw, cam64, D=1, aa=aa)
    truth = dict(color=out["color"], depth=out["depth"], alpha=out["alpha"], normal=N64, depth2=M64)
    for k, v in truth.items():
        err = float(((got[k].double() - v).abs() / v.abs().clamp_min(1.0)).max())
        print(f"MEASURED {name} aa={aa}: {k}: max rel err vs float64 {err:.2e}")
        assert err < 2e-5, (k, err)
    sum((wts[k].double() * v).sum() for k, v in truth.items()).backward()
    for k, t in zip(s64.RAW, m.tensors()):
        ref = raw[k].grad
        g = t.grad.reshape(ref.shape)
        if k == "features_rest":
            ref, g = ref[:, :3], g[:, :3]
        rn = _rn(g, ref)
        print(f"MEASURED {name} aa={aa}: grad {k}: rel-norm vs float64 {rn:.2e}")
        assert rn < 1e-4, (k, rn)


def reference_cases(cuda):
    """(case, {name: array | scalar}) of the reference chain for test_planes_and_gradients_match_the_reference_chain
    (python tests/golden/make_ref_golden.py test_operator_planes_gpu)."""
    for case in CASES:
        yield case, _reference(cuda, case)
