"""-m gpu: rendered depth on the rasterizer operator path (psb_rasterize_forward_depth / psb_rasterize_backward_depth, the B1 glue,
GaussianRasterizer(..., return_depth=True), renderer.render(..., return_depth=True) and the LibTorch drop-in).

The reference renders no depth, but depth blends exactly like a colour channel whose per-Gaussian value is the view-space depth z. Its
chain is therefore test_depth_gpu.py's: the reference's own rasterizer called once for the colour and once with colors_precomp =
(z, 0, 0) and a black background, z computed in torch from means3D and the view matrix, and autograd through both. The reference
outputs are stored in tests/golden/test_depth_operator_gpu.npz, written on an H100 by
`python tests/golden/make_ref_golden.py test_depth_operator_gpu` (which runs reference_cases() below)."""
import os

import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn
from helpers import SAMPLE, Gold, rel_close

pytestmark = pytest.mark.gpu

MODULE = "test_depth_operator_gpu"
LAMBDA_DEPTH = 0.1
CASES = ("sh3", "colors", "cov3d", "background", "culled")
LEAVES = ("means3D", "shs", "colors_precomp", "opacities", "scales", "rotations", "cov3D_precomp")


def _rn(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def _few(bound):
    """a bound on a fraction of elements, applied to the stored sample"""
    return max(bound, 2 / SAMPLE)


def _cov3d(scales, rotations):
    from photo_slam_b200 import renderer
    Lm = renderer.build_rotation(rotations) * scales.unsqueeze(1)
    cov = Lm @ Lm.transpose(1, 2)
    return torch.stack((cov[:, 0, 0], cov[:, 0, 1], cov[:, 0, 2], cov[:, 1, 1], cov[:, 1, 2], cov[:, 2, 2]), dim=1).contiguous()


def _inputs(cuda, case):
    """30 k Gaussians at 320x240 (a general pose), the operator inputs of `case`, a colour target and a depth target with ~10 % holes
    and some negative (invalid) values."""
    P, W, H = 30_000, 320, 240
    W0, H0, fx, fy = syn.CAMERAS["tum"]
    cam = syn.make_camera(W, H, fx * W / W0, fy * H / H0, *syn.random_pose(np.random.default_rng(22)))
    sc = syn.make_scene(P, cam, seed=21, scale_px=5.0, culled_frac=0.4 if case == "culled" else 0.05)
    act = syn.activate(sc)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    c = syn.device_camera(cam, cuda)
    x = dict(means3D=T(act["means3D"]), opacities=T(act["opacities"]), shs=T(act["shs"]), scales=T(act["scales"]),
             rotations=T(act["rotations"]))
    if case == "colors":
        x["colors_precomp"] = torch.rand((P, 3), generator=torch.Generator().manual_seed(23)).to(cuda)
        del x["shs"]
    if case == "cov3d":
        x["cov3D_precomp"] = _cov3d(x.pop("scales"), x.pop("rotations"))
    bg = torch.tensor([0.3, 0.5, 0.7] if case == "background" else [0.0, 0.0, 0.0], device=cuda)
    gen = torch.Generator().manual_seed(24)
    gt = torch.rand((3, H, W), generator=gen).to(cuda)
    V = c["viewmatrix"].reshape(-1)
    z = x["means3D"] @ V[[2, 6, 10]] + V[14]
    zs = torch.quantile(z[z > 0.2], torch.tensor([0.1, 0.9], device=cuda)).cpu()
    depth = zs[0] + (zs[1] - zs[0]) * torch.rand((H, W), generator=gen)
    r = torch.rand((H, W), generator=gen)
    depth[r < 0.1] = 0.0
    depth[(r >= 0.1) & (r < 0.12)] = -1.0
    return sc, c, x, bg, gt, depth.float().contiguous().to(cuda)


def _settings(c, bg, D):
    from photo_slam_b200 import rasterizer
    return rasterizer.GaussianRasterizationSettings(c["H"], c["W"], c["tanfovx"], c["tanfovy"], bg, 1.0, c["viewmatrix"], c["projmatrix"], D,
                                                    c["campos"], False)


def _loss(img, D, gt, gd):
    """colour L1 plus LAMBDA_DEPTH x depth L1 over the valid target pixels (target > 0)"""
    valid = gd > 0
    return (img - gt).abs().mean() + LAMBDA_DEPTH * ((D - gd).abs() * valid).sum() / max(int(valid.sum().item()), 1)


def _leaves(x):
    out = {k: v.clone().requires_grad_(True) for k, v in x.items()}
    out["means2D"] = torch.zeros_like(x["means3D"], requires_grad=True)
    return out


def _grads(lv):
    d = {k: v.grad for k, v in lv.items() if k != "means2D"}
    d["means2D"] = lv["means2D"].grad[:, :2]
    return d


class _RefRasterize(torch.autograd.Function):
    """The reference's rasterizer with every input differentiable (sh, colors_precomp, scales, rotations, cov3D_precomp: empty = absent)."""

    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors, opacities, scales, rotations, cov3D, rs):
        import ref_gpu
        R, img, radii, gb, bb, ib = ref_gpu.rasterize_forward(rs["bg"], means3D, colors, opacities, scales, rotations, 1.0, cov3D, rs["viewmatrix"],
                                                              rs["projmatrix"], rs["tanfovx"], rs["tanfovy"], rs["H"], rs["W"], sh, rs["D"],
                                                              rs["campos"])
        ctx.rs, ctx.R = rs, R
        ctx.save_for_backward(means3D, sh, colors, scales, rotations, cov3D, radii, gb, bb, ib)
        ctx.mark_non_differentiable(radii)
        return img, radii

    @staticmethod
    def backward(ctx, grad_out, _):
        import ref_gpu
        rs = ctx.rs
        means3D, sh, colors, scales, rotations, cov3D, radii, gb, bb, ib = ctx.saved_tensors
        dm2, dcol, dop, dm3, dcov, dsh, dsc, drot, _ = ref_gpu.rasterize_backward(
            rs["bg"], means3D, radii, colors, scales, rotations, 1.0, cov3D, rs["viewmatrix"], rs["projmatrix"], rs["tanfovx"], rs["tanfovy"],
            grad_out.contiguous(), sh, rs["D"], rs["campos"], gb, ctx.R, bb, ib)
        g = lambda t, ref: t if ref.numel() else None
        return dm3, dm2, g(dsh, sh), g(dcol, colors), dop, g(dsc, scales), g(drot, rotations), g(dcov, cov3D), None


def _reference_once(c, x, bg, gt, gd):
    lv = _leaves(x)
    e = torch.empty(0, device=gt.device)
    get = lambda k: lv.get(k, e)
    rs = dict(bg=bg, viewmatrix=c["viewmatrix"], projmatrix=c["projmatrix"], campos=c["campos"], tanfovx=c["tanfovx"], tanfovy=c["tanfovy"],
              H=c["H"], W=c["W"], D=3 if "shs" in x else 0)
    img, radii = _RefRasterize.apply(lv["means3D"], lv["means2D"], get("shs"), get("colors_precomp"), lv["opacities"], get("scales"),
                                     get("rotations"), get("cov3D_precomp"), rs)
    V = c["viewmatrix"].reshape(-1)   # column-major: the view-space z row is V[2], V[6], V[10], V[14]
    z = lv["means3D"] @ V[[2, 6, 10]] + V[14]
    cols = torch.stack([z, torch.zeros_like(z), torch.zeros_like(z)], dim=1).contiguous()
    rs_d = dict(rs, bg=torch.zeros(3, device=gt.device), D=0)
    dimg, _ = _RefRasterize.apply(lv["means3D"], lv["means2D"], e, cols, lv["opacities"], get("scales"), get("rotations"), get("cov3D_precomp"),
                                  rs_d)
    _loss(img, dimg[0], gt, gd).backward()
    torch.cuda.synchronize()
    return img.detach(), dimg[0].detach(), radii, _grads(lv)


def _reference(cuda, case):
    sc, c, x, bg, gt, gd = _inputs(cuda, case)
    image, depth, radii, grads = _reference_once(c, x, bg, gt, gd)
    _, _, _, grads2 = _reference_once(c, x, bg, gt, gd)      # the reference's own run-to-run spread (float atomics) is the floor
    d = dict(image=image, depth=depth, radii=radii)
    vis = radii > 0
    for k, b in grads.items():
        b, b2 = b.reshape(b.shape[0], -1), grads2[k].reshape(b.shape[0], -1)
        scale = b.abs().max().item()
        d["grad_" + k], d["grad_" + k + "#max"] = b, scale
        d["grad_" + k + "#self"] = rel_close(b2[vis], b[vis], rtol=1e-4, atol=1e-6 * (scale + 1e-30))
    return d


def _mine(c, x, bg, gt, gd, return_depth=True, depth_loss=True):
    from photo_slam_b200 import rasterizer
    lv = _leaves(x)
    r = rasterizer.GaussianRasterizer(_settings(c, bg, 3 if "shs" in x else 0))
    kw = {k: lv[k] for k in LEAVES if k in lv and k not in ("means3D", "opacities")}
    out = r(lv["means3D"], lv["means2D"], lv["opacities"], return_depth=return_depth, **kw)
    img, radii = out[0], out[1]
    if depth_loss:
        _loss(img, out[2], gt, gd).backward()
    else:
        (img - gt).abs().mean().backward()
    torch.cuda.synchronize()
    return img.detach(), (out[2].detach() if return_depth else None), radii, _grads(lv)


def _b1_args(c, x, bg):
    e = torch.empty(0, device=bg.device)
    get = lambda k: x.get(k, e)
    return (bg, x["means3D"], get("colors_precomp"), x["opacities"], get("scales"), get("rotations"), 1.0, get("cov3D_precomp"), c["viewmatrix"],
            c["projmatrix"], c["tanfovx"], c["tanfovy"], c["H"], c["W"], get("shs"), 3 if "shs" in x else 0, c["campos"], False)


def _b1_bwd_args(c, x, bg, radii, fwd, dpix, ddep):
    """arguments of RasterizeGaussiansBackwardDepthCUDA (fwd = the 7-tuple of the depth forward)"""
    e = torch.empty(0, device=bg.device)
    get = lambda k: x.get(k, e)
    R, gb, bb, ib = fwd[0], fwd[4], fwd[5], fwd[6]
    return (bg, x["means3D"], radii, get("colors_precomp"), get("scales"), get("rotations"), 1.0, get("cov3D_precomp"), c["viewmatrix"],
            c["projmatrix"], c["tanfovx"], c["tanfovy"], dpix, ddep, get("shs"), 3 if "shs" in x else 0, c["campos"], gb, R, bb, ib)


def _export(P, R, W, H, geom, binning, img):
    from photo_slam_b200 import _lib
    L = _lib.lib()
    dev = geom.device
    o = dict(keys_sorted=torch.zeros(max(R, 1), dtype=torch.int64, device=dev), values_sorted=torch.zeros(max(R, 1), dtype=torch.int32, device=dev),
             n_contrib=torch.zeros(W * H, dtype=torch.int32, device=dev), final_T=torch.zeros(W * H, device=dev))
    _lib.check(L.psb_debug_export(P, R, W, H, geom.data_ptr(), binning.data_ptr() if R else None, img.data_ptr(), None, None, None, None, None,
                                  None, o["keys_sorted"].data_ptr(), o["values_sorted"].data_ptr(), None, o["n_contrib"].data_ptr(),
                                  o["final_T"].data_ptr(), None), "psb_debug_export")
    torch.cuda.synchronize()
    return o


@pytest.mark.parametrize("case", CASES)
def test_depth_forward_leaves_the_plain_forward_bit_identical(cuda, case):
    from photo_slam_b200 import rasterizer
    sc, c, x, bg, gt, gd = _inputs(cuda, case)
    P, W, H = x["means3D"].size(0), c["W"], c["H"]
    a = rasterizer.RasterizeGaussiansCUDA(*_b1_args(c, x, bg))
    b = rasterizer.RasterizeGaussiansDepthCUDA(*_b1_args(c, x, bg))
    torch.cuda.synchronize()
    assert a[0] == b[0] and a[0] > 0
    assert torch.equal(a[1], b[1]) and torch.equal(a[2], b[3])
    ea, eb = _export(P, a[0], W, H, *a[3:]), _export(P, b[0], W, H, *b[4:])
    for k in ea:
        assert torch.equal(ea[k], eb[k]), k
    assert b[2].shape == (H, W) and (b[2] >= 0).all()
    if case == "culled":
        assert (a[2] == 0).sum().item() > P // 4


@pytest.mark.parametrize("case", CASES)
def test_depth_and_gradients_match_reference_chain(cuda, case):
    """GaussianRasterizer(..., return_depth=True) under a colour L1 + LAMBDA_DEPTH x depth L1 loss vs autograd of the reference chain: the
    depth plane per element at 1e-4, and the gradients of every input the case has (which together cover all eight operator gradients)
    and means2D.grad[:, :2] per element at 1e-4 against the reference-vs-itself floor."""
    r = Gold(MODULE, case)
    sc, c, x, bg, gt, gd = _inputs(cuda, case)
    P = x["means3D"].size(0)
    img, depth, radii, grads = _mine(c, x, bg, gt, gd)
    a, b = r.pair("radii", radii)
    assert (a != b).double().mean().item() <= _few(1 / 5000)
    assert r.frac("image", img, atol=1e-6) <= _few(5e-4)
    frac_d = r.frac("depth", depth, rtol=1e-4, atol=1e-6)
    print(f"{case}: depth: {frac_d:.2e} of the sampled pixels outside 1e-4")
    assert frac_d <= _few(5e-4)
    if case == "background":   # no background term: pixels that show only the background have depth 0
        uncovered = (img == bg.view(3, 1, 1)).all(dim=0)
        assert not depth[uncovered].any()
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


@pytest.mark.parametrize("case", ("sh3", "cov3d"))
def test_colour_only_loss_with_depth_output_equals_plain_operator(cuda, case):
    """return_depth=True with a loss on the colour only: the depth output gets no gradient, backward is the plain one."""
    sc, c, x, bg, gt, gd = _inputs(cuda, case)
    img0, _, radii0, g0 = _mine(c, x, bg, gt, gd, return_depth=False, depth_loss=False)
    img1, _, radii1, g1 = _mine(c, x, bg, gt, gd, return_depth=True, depth_loss=False)
    assert torch.equal(img0, img1) and torch.equal(radii0, radii1)
    for k in g0:
        assert _rn(g1[k], g0[k]) < 1e-5, (k, _rn(g1[k], g0[k]))
        assert rel_close(g1[k], g0[k], rtol=1e-4, atol=1e-6 * (g0[k].abs().max().item() + 1e-30)) < 1e-3, k


def _fused_depth(model, c):
    from photo_slam_b200 import trainer
    dep = torch.empty((c["H"], c["W"]), device=model.device)
    trainer.GaussianTrainer(model).render(c, out_depth=dep)
    torch.cuda.synchronize()
    return dep


def test_renderer_depth_in_every_branch_matches_the_fused_render(cuda):
    from photo_slam_b200 import renderer, trainer
    sc, c, x, bg, gt, gd = _inputs(cuda, "sh3")
    H, W = c["H"], c["W"]
    model = trainer.GaussianModel.from_numpy(sc, cuda)
    fused = _fused_depth(model, c)
    P = model.num_points()
    col = torch.rand((P, 3), device=cuda, generator=torch.Generator(device=cuda).manual_seed(3))
    with torch.no_grad():
        plain = renderer.render(c, H, W, model)
        d0 = renderer.render(c, H, W, model, return_depth=True)
        d_sh = renderer.render(c, H, W, model, renderer.GaussianPipelineParams(convert_SHs=True), return_depth=True)[4]
        d_cov = renderer.render(c, H, W, model, renderer.GaussianPipelineParams(compute_cov3D=True), return_depth=True)[4]
        d_over = renderer.render(c, H, W, model, override_color=col, use_override_color=True, return_depth=True)[4]
    assert len(plain) == 4 and len(d0) == 5
    assert torch.equal(plain[0], d0[0]) and torch.equal(plain[3], d0[3])
    for name, d, tol in (("default", d0[4], 1e-5), ("convert_SHs", d_sh, 1e-5), ("override_color", d_over, 1e-5), ("compute_cov3D", d_cov, 1e-4)):
        print(f"renderer depth, {name}: rel-norm vs fused render {_rn(d, fused):.2e}")
        assert _rn(d, fused) < tol, (name, _rn(d, fused))
    # gradients flow from the depth image into the model tensors in every branch
    for pipe, kw in ((renderer.GaussianPipelineParams(), {}), (renderer.GaussianPipelineParams(convert_SHs=True), {}),
                     (renderer.GaussianPipelineParams(compute_cov3D=True), {}), (renderer.GaussianPipelineParams(), dict(override_color=col,
                                                                                                                        use_override_color=True))):
        for t in model.tensors():
            t.requires_grad_(True)
            t.grad = None
        img, viewspace, vis, radii, D = renderer.render(c, H, W, model, pipe, return_depth=True, **kw)
        (D - gd).abs().mean().backward()
        assert model.xyz_.grad.abs().sum().item() > 0 and model.opacity_.grad.abs().sum().item() > 0
        assert viewspace.grad[:, :2].abs().sum().item() > 0
        for t in model.tensors():
            t.requires_grad_(False)


def test_operator_depth_gradients_match_the_fused_depth_backward(cuda):
    """Default branch: autograd's raw-parameter gradients of (0.8 L1 + 0.2 (1 - SSIM) + LAMBDA_DEPTH depth_l1) through renderer.render equal
    psb_trainer_backward_depth's on the same model and target. The two implementations share no kernel of the depth backward."""
    import ref_trainer
    from photo_slam_b200 import renderer, trainer
    sc, c, x, bg, gt, gd = _inputs(cuda, "sh3")
    H, W = c["H"], c["W"]
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    for t in m.tensors():
        t.requires_grad_(True)
    img, viewspace, vis, radii, D = renderer.render(c, H, W, m, return_depth=True)
    valid = gd > 0
    dl1 = ((D - gd).abs() * valid).sum() / max(int(valid.sum().item()), 1)
    (0.8 * (img - gt).abs().mean() + 0.2 * (1 - ref_trainer.ssim(img, gt)) + LAMBDA_DEPTH * dl1).backward()
    torch.cuda.synchronize()
    fm = trainer.GaussianModel.from_numpy(sc, cuda)
    fm.trainingSetup(trainer.GaussianOptimizationParams())
    dp = trainer.DataParallelTrainer(fm)      # world == 1: backward -> (no all-reduce) -> Adam; dp.segs keeps the raw gradients
    dp.trainForOneIteration(c, gt, gt_depth=gd, lambda_depth=LAMBDA_DEPTH)
    l, l1, ss, fdl1, n = dp.result_depth()
    torch.cuda.synchronize()
    assert abs(fdl1 - dl1.item()) < 1e-5 * max(1.0, dl1.item())
    for name, t, seg in zip(trainer.GROUPS, m.tensors(), dp.segs):
        rn = _rn(seg.reshape(-1), t.grad.reshape(-1))
        print(f"grad {name}: operator path vs fused depth backward, rel-norm {rn:.2e}")
        assert rn < 1e-4, (name, rn)


def test_libtorch_depth_ops_equal_the_ctypes_path(cuda):
    from photo_slam_b200 import _lib, rasterizer
    shim = os.path.join(os.path.dirname(_lib.LIB_PATH), "libcuda_rasterizer.so")
    torch.ops.load_library(shim)
    for case in ("sh3", "colors", "cov3d"):
        sc, c, x, bg, gt, gd = _inputs(cuda, case)
        a = rasterizer.RasterizeGaussiansDepthCUDA(*_b1_args(c, x, bg))
        b = torch.ops.psb200.rasterize_gaussians_depth(*_b1_args(c, x, bg))
        torch.cuda.synchronize()
        assert a[0] == b[0] and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]) and torch.equal(a[3], b[3]), case
        dpix = torch.randn((3, c["H"], c["W"]), device=cuda, generator=torch.Generator(device=cuda).manual_seed(5)) / 1e4
        ddep = torch.randn((c["H"], c["W"]), device=cuda, generator=torch.Generator(device=cuda).manual_seed(6)) / 1e4
        ga = rasterizer.RasterizeGaussiansBackwardDepthCUDA(*_b1_bwd_args(c, x, bg, a[3], a, dpix, ddep))
        gb = torch.ops.psb200.rasterize_gaussians_backward_depth(*_b1_bwd_args(c, x, bg, b[3], b, dpix, ddep))
        plain = rasterizer.RasterizeGaussiansBackwardDepthCUDA(*_b1_bwd_args(c, x, bg, a[3], a, dpix, None))
        torch.cuda.synchronize()
        assert len(ga) == len(gb) == 8
        for i, (u, v) in enumerate(zip(ga, gb)):
            assert u.shape == v.shape
            if v.numel():
                assert _rn(u, v) < 1e-5, (case, i, _rn(u, v))
        # the depth gradient reaches dL/dmean3D and dL/dmean2D, and only through depth
        assert _rn(ga[3], plain[3]) > 1e-3 and _rn(ga[0], plain[0]) > 1e-3


def test_empty_and_fully_culled_scenes(cuda):
    from photo_slam_b200 import rasterizer
    sc, c, x, bg, gt, gd = _inputs(cuda, "sh3")
    H, W = c["H"], c["W"]
    V = c["viewmatrix"].reshape(-1)
    zrow = V[[2, 6, 10]]
    z = x["means3D"] @ zrow + V[14]
    behind = dict(x, means3D=(x["means3D"] - (z + 1.0).unsqueeze(1) * zrow / zrow.dot(zrow)).contiguous())  # view z = -1: all culled
    empty = {k: v[:0].contiguous() for k, v in x.items()}
    for name, xs in (("empty", empty), ("culled", behind)):
        P = xs["means3D"].size(0)
        fwd = rasterizer.RasterizeGaussiansDepthCUDA(*_b1_args(c, xs, bg))
        assert fwd[0] == 0 and fwd[2].shape == (H, W) and not fwd[2].any(), name
        g = rasterizer.RasterizeGaussiansBackwardDepthCUDA(*_b1_bwd_args(c, xs, bg, fwd[3], fwd, torch.ones((3, H, W), device=cuda),
                                                                          torch.ones((H, W), device=cuda)))
        assert all(not t.any() for t in g), name
        if P == 0:
            continue      # (the front-end, like the reference's, cannot tell empty SHs from absent ones)
        lv = _leaves(xs)
        r = rasterizer.GaussianRasterizer(_settings(c, bg, 3))
        img, radii, D = r(lv["means3D"], lv["means2D"], lv["opacities"], shs=lv["shs"], scales=lv["scales"], rotations=lv["rotations"],
                          return_depth=True)
        (img.sum() + D.sum()).backward()      # expanded, zero-stride output gradients
        torch.cuda.synchronize()
        assert not D.any() and (radii == 0).all() and P == radii.numel()
        assert all(not t.grad.any() for t in lv.values()), name


def reference_cases(cuda):
    """(case, {name: array | scalar}) of the reference chain for the comparisons above (python tests/golden/make_ref_golden.py
    test_depth_operator_gpu)."""
    for case in CASES:
        yield case, _reference(cuda, case)
