"""-m gpu: the deterministic backward of the rasterizer operator (psb_rasterize_backward_deterministic through the B1 glue,
GaussianRasterizer(..., deterministic=True), renderer.render(..., deterministic=True) and the LibTorch drop-in).

Its gradients must be bit-identical from call to call, and otherwise be the operator's: the same per-element gates against the reference's
stored outputs as the atomic backward (tests/golden/test_parity_ref_gpu.npz, tests/golden/test_depth_operator_gpu.npz), and a difference
from the atomic backward no larger than a change of summation order."""
import contextlib
import functools
import os
import warnings

import pytest
import torch

import test_depth_operator_gpu as dop
import test_parity_ref_gpu as par
from helpers import Gold, rel_close

pytestmark = pytest.mark.gpu

CASES = dop.CASES
TEETH = 0.9   # share of the visible Gaussians that must have >= 2 instances (tiles): their gradients are sums of several flushes


def _rn(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


@contextlib.contextmanager
def _torch_deterministic():
    """torch.use_deterministic_algorithms(True) with every warning an error; the previous setting is restored."""
    before, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        with warnings.catch_warnings():
            warnings.simplefilter("error")
            yield
    finally:
        torch.use_deterministic_algorithms(before, warn_only=warn)


def _b1_fwd(c, x, bg, depth):
    from photo_slam_b200 import rasterizer
    fwd = (rasterizer.RasterizeGaussiansDepthCUDA if depth else rasterizer.RasterizeGaussiansCUDA)(*dop._b1_args(c, x, bg))
    if not depth:   # the depth forward's 7-tuple layout, without the depth image
        fwd = (fwd[0], fwd[1], None, fwd[2], fwd[3], fwd[4], fwd[5])
    return fwd


def _b1_bwd(c, x, bg, fwd, dpix, ddep, deterministic):
    from photo_slam_b200 import rasterizer
    args = dop._b1_bwd_args(c, x, bg, fwd[3], fwd, dpix, ddep)
    if ddep is None:
        args = args[:13] + args[14:]
        return rasterizer.RasterizeGaussiansBackwardCUDA(*args, deterministic=deterministic)
    return rasterizer.RasterizeGaussiansBackwardDepthCUDA(*args, deterministic=deterministic)


def _pixel_grads(c, cuda):
    gen = torch.Generator().manual_seed(31)
    dpix = (torch.randn((3, c["H"], c["W"]), generator=gen) / (3 * c["H"] * c["W"])).to(cuda)
    ddep = (torch.randn((c["H"], c["W"]), generator=gen) / (c["H"] * c["W"])).to(cuda)
    return dpix, ddep


def _instances(P, fwd, W, H):
    from photo_slam_b200 import _lib
    tt = torch.zeros(P, dtype=torch.int32, device=fwd[4].device)
    _lib.check(_lib.lib().psb_debug_export(P, fwd[0], W, H, fwd[4].data_ptr(), None, None, None, None, None, None, None, tt.data_ptr(), None,
                                           None, None, None, None, None), "psb_debug_export")
    torch.cuda.synchronize()
    return tt


@pytest.mark.parametrize("depth", [False, True], ids=["colour", "depth"])
@pytest.mark.parametrize("case", CASES)
def test_repeated_calls_and_runs_are_bit_identical(cuda, case, depth):
    sc, c, x, bg, gt, gd = dop._inputs(cuda, case)
    P = x["means3D"].size(0)
    dpix, ddep = _pixel_grads(c, cuda)
    ddep = ddep if depth else None
    fwd = _b1_fwd(c, x, bg, depth)
    tt = _instances(P, fwd, c["W"], c["H"])
    vis = tt > 0
    share = (tt[vis] >= 2).double().mean().item()
    print(f"{case}: {int(vis.sum())} visible Gaussians, {share:.3f} of them with >= 2 instances, {fwd[0]} instances")
    assert share >= TEETH, share
    first = _b1_bwd(c, x, bg, fwd, dpix, ddep, True)
    torch.cuda.synchronize()
    assert first[0].abs().sum().item() > 0 and first[3].abs().sum().item() > 0
    for _ in range(4):      # five calls on the same forward buffers
        again = _b1_bwd(c, x, bg, fwd, dpix, ddep, True)
        for i, (a, b) in enumerate(zip(first, again)):
            assert torch.equal(a, b), (case, i)
    for _ in range(2):      # two independent forward + backward runs
        fwd2 = _b1_fwd(c, x, bg, depth)
        assert fwd2[0] == fwd[0]
        again = _b1_bwd(c, x, bg, fwd2, dpix, ddep, True)
        for i, (a, b) in enumerate(zip(first, again)):
            assert torch.equal(a, b), (case, i)
    # against the atomic backward: the same sums in another order
    atomic = _b1_bwd(c, x, bg, fwd, dpix, ddep, False)
    for name, a, b in zip(par.NAMES, first, atomic):
        if b.numel():
            assert _rn(a, b) <= 2e-5, (case, name, _rn(a, b))
            assert not a[~vis].any(), (case, name)


@pytest.mark.parametrize("P,camname,wh,pose_seed,D,bg,scale_px", par.CONFIGS)
def test_deterministic_backward_matches_reference(cuda, P, camname, wh, pose_seed, D, bg, scale_px):
    """test_parity_ref_gpu.py::test_backward_matches_reference's gates on the deterministic backward, and its distance from the atomic
    backward."""
    from photo_slam_b200 import rasterizer
    gold = Gold(par.MODULE, "bwd-" + par._cid(P, camname, wh, pose_seed, D, bg, scale_px))
    cam, sc, act, g, c = par._scene(cuda, P, camname, wh, pose_seed, scale_px)
    bgt = torch.tensor(bg, dtype=torch.float32, device=cuda)
    mine, extra = par._run_mine(g, c, D, bgt)
    assert gold.exact("radii", mine[2])
    dL = par._loss_grad(mine[1], par._rand((3, c["H"], c["W"]), 1, cuda))
    det = functools.partial(rasterizer.RasterizeGaussiansBackwardCUDA, deterministic=True)
    gm = par._backward(det, mine, g, c, D, bgt, extra, dL)
    atomic = par._backward_mine(mine, g, c, D, bgt, extra, dL)
    vis = mine[2] > 0
    for name, a, b in zip(par.NAMES, gm, atomic):
        scale, self_frac = gold[name + "#max"] + 1e-30, gold[name + "#self"]
        frac = gold.frac(name, a[vis], rtol=1e-4, atol=1e-6 * scale)
        nrm = gold.relnorm(name, a[vis])
        d = _rn(a, b)
        print(f"{name}: frac>1e-4 vs ref {frac:.2e} (ref-vs-ref {self_frac:.2e}), rel-norm vs ref {nrm:.2e}, vs atomic {d:.2e}")
        assert nrm < 2e-5, f"{name}: relative norm error {nrm}"
        assert frac <= max(5e-4, 3 * self_frac), f"{name}: {frac} of visible entries outside 1e-4 (reference vs itself: {self_frac})"
        assert torch.equal(a[~vis], torch.zeros_like(a[~vis])), f"{name}: rows of invisible Gaussians must stay zero"
        assert d <= 2e-5, f"{name}: {d} from the atomic backward"


def _mine_det(c, x, bg, gt, gd, return_depth=True):
    """test_depth_operator_gpu._mine through GaussianRasterizer(..., deterministic=True), under torch's deterministic flag."""
    from photo_slam_b200 import rasterizer
    lv = dop._leaves(x)
    r = rasterizer.GaussianRasterizer(dop._settings(c, bg, 3 if "shs" in x else 0))
    kw = {k: lv[k] for k in dop.LEAVES if k in lv and k not in ("means3D", "opacities")}
    with _torch_deterministic():
        out = r(lv["means3D"], lv["means2D"], lv["opacities"], return_depth=return_depth, deterministic=True, **kw)
        loss = dop._loss(out[0], out[2], gt, gd) if return_depth else (out[0] - gt).abs().mean()
        loss.backward()
    torch.cuda.synchronize()
    return out[0].detach(), (out[2].detach() if return_depth else None), out[1], dop._grads(lv)


@pytest.mark.parametrize("case", CASES)
def test_deterministic_depth_gradients_match_reference_chain(cuda, case):
    """test_depth_operator_gpu.py::test_depth_and_gradients_match_reference_chain's gates through the deterministic autograd path."""
    r = Gold(dop.MODULE, case)
    sc, c, x, bg, gt, gd = dop._inputs(cuda, case)
    P = x["means3D"].size(0)
    img, depth, radii, grads = _mine_det(c, x, bg, gt, gd)
    a, b = r.pair("radii", radii)
    assert (a != b).double().mean().item() <= dop._few(1 / 5000)
    assert r.frac("image", img, atol=1e-6) <= dop._few(5e-4)
    assert r.frac("depth", depth, rtol=1e-4, atol=1e-6) <= dop._few(5e-4)
    vis = radii > 0
    _, _, _, atomic = dop._mine(c, x, bg, gt, gd)
    for k, g in grads.items():
        g = g.reshape(P, -1)
        key = "grad_" + k
        scale, self_frac = r[key + "#max"] + 1e-30, r[key + "#self"]
        xm, ym = r.pair(key, g)
        live = (xm != 0) | (ym != 0)
        frac = rel_close(xm[live], ym[live], rtol=1e-4, atol=1e-6 * scale)
        nrm = ((xm - ym).norm() / (ym.norm() + 1e-30)).item()
        d = _rn(g, atomic[k].reshape(P, -1))
        print(f"{case}: grad {k}: frac>1e-4 {frac:.2e} (reference vs itself {self_frac:.2e}), rel-norm {nrm:.2e}, vs atomic {d:.2e}")
        assert nrm < 2e-4, f"{k}: relative norm error {nrm}"
        assert frac <= dop._few(max(1e-3, 3 * self_frac)), f"{k}: {frac} of the sampled entries outside 1e-4 (reference vs itself: {self_frac})"
        assert not g[~vis].any(), f"{k}: rows of invisible Gaussians must be zero"
        assert d <= 2e-5, f"{k}: {d} from the atomic backward"


@pytest.mark.parametrize("return_depth", [False, True], ids=["colour", "depth"])
def test_autograd_is_silent_under_torch_deterministic_algorithms_and_repeats(cuda, return_depth):
    """GaussianRasterizer(rs)(..., deterministic=True) neither raises nor warns under torch.use_deterministic_algorithms(True), and its
    leaf gradients are bit-identical to a second run's."""
    sc, c, x, bg, gt, gd = dop._inputs(cuda, "sh3")
    first = _mine_det(c, x, bg, gt, gd, return_depth)
    second = _mine_det(c, x, bg, gt, gd, return_depth)
    assert torch.equal(first[0], second[0]) and torch.equal(first[2], second[2])
    for k, g in first[3].items():
        assert g.abs().sum().item() > 0, k
        assert torch.equal(g, second[3][k]), k


def _train(c, H, W, sc, gt, gd, cuda, pipe, override):
    """10 Adam steps of L1 + 0.1 depth L1 through renderer.render(..., deterministic=True): final parameters and the accumulated
    screen-space gradient."""
    from photo_slam_b200 import renderer, trainer
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    params = m.tensors()
    kw = {}
    if override:
        col = torch.rand((m.num_points(), 3), generator=torch.Generator().manual_seed(41)).to(cuda)
        params = params + [col]
        kw = dict(override_color=col, use_override_color=True)
    for t in params:
        t.requires_grad_(True)
    opt = torch.optim.Adam(params, lr=1e-3)
    acc = torch.zeros_like(m.xyz_)
    for _ in range(10):
        opt.zero_grad()
        img, viewspace, vis, radii, D = renderer.render(c, H, W, m, pipe, return_depth=True, deterministic=True, **kw)
        dop._loss(img, D, gt, gd).backward()
        acc += viewspace.grad
        opt.step()
    torch.cuda.synchronize()
    return [t.detach().clone() for t in params], acc


@pytest.mark.parametrize("branch", ["default", "convert_SHs", "compute_cov3D", "override_color"])
def test_renderer_training_is_bit_identical(cuda, branch):
    """renderer.render(..., deterministic=True) under torch.optim.Adam, twice from the same start, in every pipeline branch. torch's global
    deterministic flag is on for the default branch only: the compute_cov3D branch's batched matmul would need CUBLAS_WORKSPACE_CONFIG set
    before CUDA started."""
    from photo_slam_b200 import renderer
    sc, c, x, bg, gt, gd = dop._inputs(cuda, "sh3")
    pipe = renderer.GaussianPipelineParams(convert_SHs=branch == "convert_SHs", compute_cov3D=branch == "compute_cov3D")
    ctx = _torch_deterministic if branch == "default" else contextlib.nullcontext
    runs = []
    for _ in range(2):
        with ctx():
            runs.append(_train(c, c["H"], c["W"], sc, gt, gd, cuda, pipe, branch == "override_color"))
    (p0, a0), (p1, a1) = runs
    assert a0.abs().sum().item() > 0
    assert torch.equal(a0, a1), branch
    for i, (u, v) in enumerate(zip(p0, p1)):
        assert torch.equal(u, v), (branch, i)


def test_libtorch_op_equals_the_ctypes_path(cuda):
    from photo_slam_b200 import _lib
    torch.ops.load_library(os.path.join(os.path.dirname(_lib.LIB_PATH), "libcuda_rasterizer.so"))
    for case in ("sh3", "colors", "cov3d"):
        sc, c, x, bg, gt, gd = dop._inputs(cuda, case)
        dpix, ddep = _pixel_grads(c, cuda)
        fwd = _b1_fwd(c, x, bg, True)
        for dd in (ddep, None):
            a = _b1_bwd(c, x, bg, fwd, dpix, dd, True)
            b = torch.ops.psb200.rasterize_gaussians_backward_deterministic(*dop._b1_bwd_args(c, x, bg, fwd[3], fwd, dpix, dd))
            torch.cuda.synchronize()
            assert len(a) == len(b) == 8
            for i, (u, v) in enumerate(zip(a, b)):
                assert u.shape == v.shape and torch.equal(u, v), (case, dd is None, i)
        # an empty depth gradient is colour only
        e = torch.ops.psb200.rasterize_gaussians_backward_deterministic(*dop._b1_bwd_args(c, x, bg, fwd[3], fwd, dpix,
                                                                                          torch.empty(0, device=cuda)))
        for u, v in zip(a, e):
            assert torch.equal(u, v), case


def test_empty_and_fully_culled_scenes(cuda):
    from photo_slam_b200 import _lib
    torch.ops.load_library(os.path.join(os.path.dirname(_lib.LIB_PATH), "libcuda_rasterizer.so"))
    sc, c, x, bg, gt, gd = dop._inputs(cuda, "sh3")
    H, W = c["H"], c["W"]
    V = c["viewmatrix"].reshape(-1)
    zrow = V[[2, 6, 10]]
    z = x["means3D"] @ zrow + V[14]
    behind = dict(x, means3D=(x["means3D"] - (z + 1.0).unsqueeze(1) * zrow / zrow.dot(zrow)).contiguous())  # view z = -1: all culled
    empty = {k: v[:0].contiguous() for k, v in x.items()}
    ones, ones_d = torch.ones((3, H, W), device=cuda), torch.ones((H, W), device=cuda)
    for name, xs in (("empty", empty), ("culled", behind)):
        P = xs["means3D"].size(0)
        fwd = _b1_fwd(c, xs, bg, True)
        assert fwd[0] == 0, name
        for dd in (ones_d, None):
            g = _b1_bwd(c, xs, bg, fwd, ones, dd, True)
            torch.cuda.synchronize()
            assert all(not t.any() for t in g), name
            g = torch.ops.psb200.rasterize_gaussians_backward_deterministic(*dop._b1_bwd_args(c, xs, bg, fwd[3], fwd, ones, dd))
            torch.cuda.synchronize()
            assert all(not t.any() for t in g), name
        if P == 0:
            continue      # (the front-end, like the reference's, cannot tell empty SHs from absent ones)
        lv = dop._leaves(xs)
        r = dop._settings(c, bg, 3)
        from photo_slam_b200 import rasterizer
        with _torch_deterministic():
            img, radii, D = rasterizer.GaussianRasterizer(r)(lv["means3D"], lv["means2D"], lv["opacities"], shs=lv["shs"], scales=lv["scales"],
                                                             rotations=lv["rotations"], return_depth=True, deterministic=True)
            (img.sum() + D.sum()).backward()
        torch.cuda.synchronize()
        assert not D.any() and (radii == 0).all()
        assert all(not t.grad.any() for t in lv.values()), name
