"""CPU: anti-aliasing (the 2D Mip filter, o' = o h with h = sqrt(max(det0 / det1, 2.5e-5))).

  * a float64 spec of h and of dh/d(a0, b, c0), the formulas the kernels implement, against central finite differences, including
    near-degenerate covariances and the clamped region (gradient 0);
  * the torch restatement of projection -> cov2D -> h that the GPU tests use as their oracle passes gradcheck in float64, with the
    1.3 tanfov clamp of the mean and its gradient quirk (SURVEY.md Appendix A);
  * psb_rasterize_forward_aa / psb_rasterize_backward_aa / psb_trainer_set_antialiasing reject bad arguments before any CUDA call;
  * the LibTorch drop-in exports the new symbols; the settings field defaults to False and the B1 positional lists are unchanged.
"""
import os
import subprocess

import numpy as np
import pytest
import torch

from photo_slam_b200 import _lib
from splat64 import h_torch, quat_cov as _quat_cov

DILATION = 0.3
MIN_RATIO = 2.5e-5
ONE = 4096  # fake non-null pointer; never dereferenced because validation fails first


# ---- the spec ----------------------------------------------------------------------------------------------------------------------
def aa_h(a0, b, c0):
    det0 = a0 * c0 - b * b
    det1 = (a0 + DILATION) * (c0 + DILATION) - b * b
    return np.sqrt(np.maximum(det0 / det1, MIN_RATIO))


def aa_dh(a0, b, c0):
    """(dh/da0, dh/db, dh/dc0) as the kernels compute them: 0 where the clamp is active"""
    a1, c1 = a0 + DILATION, c0 + DILATION
    det0, det1 = a0 * c0 - b * b, a1 * c1 - b * b
    h = aa_h(a0, b, c0)
    live = det0 / det1 > MIN_RATIO
    da = np.where(live, 0.5 * h * (c0 / det0 - c1 / det1), 0.0)
    dc = np.where(live, 0.5 * h * (a0 / det0 - a1 / det1), 0.0)
    db = np.where(live, h * b * (1.0 / det1 - 1.0 / det0), 0.0)
    return da, db, dc


def _covs(rng, n, cond):
    """n random SPD 2x2 covariances (a0, b, c0) with eigenvalue ratio up to `cond`"""
    lam1 = np.exp(rng.uniform(np.log(0.01), np.log(400.0), n))
    lam2 = lam1 / np.exp(rng.uniform(0.0, np.log(cond), n))
    th = rng.uniform(0, np.pi, n)
    c, s = np.cos(th), np.sin(th)
    return lam1 * c * c + lam2 * s * s, (lam1 - lam2) * c * s, lam1 * s * s + lam2 * c * c


@pytest.mark.parametrize("cond", [1.0 + 1e-9, 10.0, 1e3, 1e5], ids=["round", "moderate", "thin", "near-degenerate"])
def test_h_and_its_derivatives_against_finite_differences(cond):
    rng = np.random.default_rng(int(cond) % 1000)
    a0, b, c0 = _covs(rng, 4000, cond)
    h = aa_h(a0, b, c0)
    assert (h >= np.sqrt(MIN_RATIO) - 1e-15).all() and (h <= 1.0).all()
    da, db, dc = aa_dh(a0, b, c0)
    ratio = (a0 * c0 - b * b) / ((a0 + DILATION) * (c0 + DILATION) - b * b)
    # away from the kink of the clamp, where a central difference is well defined
    ok = np.abs(ratio / MIN_RATIO - 1.0) > 1e-3
    for k, d in enumerate((da, db, dc)):
        x = [a0.copy(), b.copy(), c0.copy()]
        det0 = a0 * c0 - b * b
        eps = 1e-5 * det0 / (np.abs(a0) + np.abs(b) + np.abs(c0))    # moves det0 by ~1e-5 of itself, however thin the splat
        xp = [v.copy() for v in x]
        xm = [v.copy() for v in x]
        xp[k] += eps
        xm[k] -= eps
        fd = (aa_h(*xp) - aa_h(*xm)) / (2 * eps)
        err = np.abs(fd - d)[ok]
        scale = (np.abs(d) + np.abs(fd) + h * (np.abs(a0) + np.abs(b) + np.abs(c0)) / det0 * 1e-3)[ok]
        assert (err <= 1e-5 * scale).all(), (cond, k, float((err / scale).max()))
    clamped = ratio < MIN_RATIO
    if cond >= 1e5:
        assert clamped.any() and (~clamped).any(), "want both sides of the clamp"
    for d in (da, db, dc):
        assert (d[clamped] == 0).all()


def test_h_is_one_minus_dilation_effect_for_large_splats_and_the_clamp_for_thin_ones():
    # a round splat of variance v: h = v / (v + 0.3)
    v = np.array([0.01, 0.3, 10.0, 1e4])
    assert np.allclose(aa_h(v, 0 * v, v), v / (v + DILATION), rtol=1e-14)
    # a degenerate line: det0 = 0 -> the clamp
    assert np.allclose(aa_h(np.array([4.0]), np.array([2.0]), np.array([1.0])), np.sqrt(MIN_RATIO))


# ---- the torch restatement (splat64.h_torch, the GPU tests' oracle) --------------------------------------------------------------------------------
def _gradcheck_inputs(n=12, seed=0):
    import photo_slam_b200.synthetic as syn
    rng = np.random.default_rng(seed)
    cam = syn.make_camera(64, 48, 50.0, 50.0, *syn.random_pose(rng))
    sc = syn.make_scene(n, cam, seed=seed, scale_px=3.0, culled_frac=0.2)
    act = syn.activate(sc)
    m = torch.tensor(act["means3D"], dtype=torch.float64)
    # push two Gaussians far outside the frustum: the clamp of the mean is active for them
    V = torch.tensor(cam["viewmatrix"], dtype=torch.float64).reshape(4, 4)
    t = m @ V[:3, :3] + V[3, :3]
    t[0, 0] = 3.0 * float(cam["tanfovx"]) * abs(float(t[0, 2])) + 0.5
    t[1, 1] = -3.0 * float(cam["tanfovy"]) * abs(float(t[1, 2])) - 0.5
    t[0, 2], t[1, 2] = 2.0, 3.0
    m = (t - V[3, :3]) @ torch.linalg.inv(V[:3, :3])
    s = torch.tensor(act["scales"], dtype=torch.float64)
    q = torch.tensor(act["rotations"], dtype=torch.float64)
    return cam, m, s, q


def test_torch_oracle_passes_gradcheck():
    cam, m, s, q = _gradcheck_inputs()
    vm = torch.tensor(cam["viewmatrix"], dtype=torch.float64)
    args = (64, 48, float(cam["tanfovx"]), float(cam["tanfovy"]))
    h = h_torch(m, _quat_cov(s, q), vm, *args)
    assert (h < 1).any() and (h == 1).any(), "want visible and culled Gaussians"
    # Gaussians 0 and 1 have a clamped mean, whose gradient follows the kernels, not the exact derivative: the full chain is checked
    # on the others, the covariance path (exact either way) on all of them
    m2, s2, q2 = (x[2:].clone().requires_grad_(True) for x in (m, s, q))
    assert torch.autograd.gradcheck(lambda m_, s_, q_: h_torch(m_, _quat_cov(s_, q_), vm, *args), (m2, s2, q2), eps=1e-7, atol=1e-6, rtol=1e-5)
    cov = _quat_cov(s, q).detach().clone().requires_grad_(True)
    assert torch.autograd.gradcheck(lambda c_: h_torch(m, c_, vm, *args), (cov,), eps=1e-7, atol=1e-6, rtol=1e-5)
    # the clamped coordinates pass no gradient to the mean along x (Gaussian 0) / y (Gaussian 1) in view space
    mm = m.detach().clone().requires_grad_(True)
    h_torch(mm, cov.detach(), vm, *args)[:2].sum().backward()
    V = vm.reshape(4, 4)
    g_view = mm.grad[:2] @ V[:3, :3]     # dL/dt = R dL/dm for t = m V[:3,:3] + ...  (R orthonormal)
    assert abs(float(g_view[0, 0])) < 1e-6 * float(g_view[0].norm()) and abs(float(g_view[1, 1])) < 1e-6 * float(g_view[1].norm())


def test_torch_oracle_matches_the_spec_on_the_2d_covariance():
    cam, m, s, q = _gradcheck_inputs(n=200, seed=4)
    vm = torch.tensor(cam["viewmatrix"], dtype=torch.float64)
    h = h_torch(m, _quat_cov(s, q), vm, 64, 48, float(cam["tanfovx"]), float(cam["tanfovy"]))
    assert ((h >= np.sqrt(MIN_RATIO) - 1e-12) & (h <= 1)).all()
    assert (h < 1).sum() > 100


# ---- host-side validation -----------------------------------------------------------------------------------------------------------
def _fwd(L, P=10, antialiasing=1, geom=True, shs=ONE, colors=None, depth=ONE):
    cb = _lib.ALLOC_FN(lambda n, u: 0)
    return L.psb_rasterize_forward_aa(cb if geom else _lib.ALLOC_FN(), None, cb, None, cb, None, P, 3, 16, ONE, 64, 64, ONE, shs, colors, ONE, ONE, 1.0, ONE,
                                      None, ONE, ONE, ONE, 1.0, 1.0, 0, ONE, ONE, depth, antialiasing, None)


def _bwd(L, P=10, R=100, dL_dpix=ONE, dL_ddepth=None, dL_dz=None, scratch=None, nbytes=0, antialiasing=1):
    return L.psb_rasterize_backward_aa(P, 3, 16, R, ONE, 64, 64, ONE, ONE, None, ONE, 1.0, ONE, None, ONE, ONE, ONE, 1.0, 1.0,
                                       None, ONE, ONE, ONE, dL_dpix, ONE, ONE, ONE, ONE, ONE, ONE, ONE, ONE, ONE, dL_ddepth, dL_dz,
                                       scratch, nbytes, antialiasing, None)


def test_forward_aa_validates_before_any_cuda_call():
    L = _lib.lib()
    name = b"psb_rasterize_forward_aa: "
    for bad in (2, -1, 7):
        assert _fwd(L, antialiasing=bad) == -1 and L.psb_last_error() == name + b"antialiasing must be 0 or 1"
    for aa in (0, 1):
        assert _fwd(L, antialiasing=aa, geom=False) == -1 and L.psb_last_error() == name + b"bad argument"
        assert _fwd(L, antialiasing=aa, P=-1) == -1 and L.psb_last_error() == name + b"bad argument"
        assert _fwd(L, antialiasing=aa, colors=ONE) == -1 and L.psb_last_error() == name + b"provide exactly one of shs / colors_precomp"
        assert _fwd(L, antialiasing=aa, shs=None) == -1 and L.psb_last_error() == name + b"provide exactly one of shs / colors_precomp"


def test_backward_aa_validates_before_any_cuda_call():
    L = _lib.lib()
    name = b"psb_rasterize_backward_aa: "
    for bad in (2, -1):
        assert _bwd(L, antialiasing=bad) == -1 and L.psb_last_error() == name + b"antialiasing must be 0 or 1"
    need = L.psb_rasterize_backward_det_bytes(10, 100)
    for aa in (0, 1):
        for P in (10, 0):
            assert _bwd(L, P=P, dL_ddepth=ONE, antialiasing=aa) == -1 and L.psb_last_error() == name + b"dL_ddepth needs a dL_dz array"
        assert _bwd(L, dL_dpix=None, antialiasing=aa) == -1 and L.psb_last_error() == name + b"bad argument"
        assert _bwd(L, P=-3, antialiasing=aa) == -1 and L.psb_last_error() == name + b"bad argument"
        assert _bwd(L, R=-1, antialiasing=aa) == -1 and L.psb_last_error() == name + b"bad argument"
        # the deterministic backward's scratch check
        assert _bwd(L, scratch=ONE, nbytes=need - 1, antialiasing=aa) == -1 and L.psb_last_error().startswith(name + b"det_scratch holds")
        assert _bwd(L, P=0, antialiasing=aa) == 0
    # the existing entry points' messages are unchanged
    assert L.psb_rasterize_backward(10, 3, 16, 100, ONE, 64, 64, ONE, ONE, None, ONE, 1.0, ONE, None, ONE, ONE, ONE, 1.0, 1.0, None, ONE, ONE,
                                    ONE, None, ONE, ONE, ONE, ONE, ONE, ONE, ONE, ONE, ONE, None) == -1
    assert L.psb_last_error() == b"psb_rasterize_backward: bad argument"


def test_trainer_set_antialiasing_rejects_a_null_context():
    from photo_slam_b200 import trainer
    L = trainer._bind()
    assert L.psb_trainer_set_antialiasing(None, 1) == -1
    assert L.psb_last_error() == b"psb_trainer_set_antialiasing: null context"


def test_header_declares_and_library_exports_the_new_calls():
    names = _lib.exported_symbols()
    for n in ("psb_rasterize_forward_aa", "psb_rasterize_backward_aa", "psb_trainer_set_antialiasing"):
        assert n in names and hasattr(_lib.lib(), n), n


def test_libtorch_shim_exports_the_antialiased_symbols():
    lib = os.path.join(os.path.dirname(_lib.LIB_PATH), "libcuda_rasterizer.so")
    assert os.path.exists(lib), "build it with `python photo-slam_b200/build.py --torch`"
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    for sym in (# the signature and 7-tuple of RasterizeGaussiansDepthCUDA
                "_Z33RasterizeGaussiansAntialiasedCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffiiS2_iS2_b",
                # RasterizeGaussiansBackwardDeterministicCUDA's signature plus a trailing bool
                "_Z41RasterizeGaussiansBackwardAntialiasedCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffS2_S2_S2_iS2_S2_iS2_S2_b",
                "_Z27RasterizeGaussiansDepthCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffiiS2_iS2_b",
                "_Z43RasterizeGaussiansBackwardDeterministicCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffS2_S2_S2_iS2_S2_iS2_S2_",
                # the reference's own symbols stay
                "_Z22RasterizeGaussiansCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffiiS2_iS2_b",
                "_Z30RasterizeGaussiansBackwardCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffS2_S2_iS2_S2_iS2_S2_"):
        assert sym in out, sym


def test_python_front_end_defaults_and_positional_lists():
    import dataclasses
    import inspect
    from photo_slam_b200 import rasterizer, renderer, trainer
    z = torch.zeros
    rs = rasterizer.GaussianRasterizationSettings(32, 32, 1.0, 1.0, z(3), 1.0, torch.eye(4).flatten(), torch.eye(4).flatten(), 3, z(3))
    assert rs.antialiasing is False
    names = [f.name for f in dataclasses.fields(rasterizer.GaussianRasterizationSettings)]
    assert names[-2:] == ["prefiltered", "antialiasing"]
    assert renderer.GaussianPipelineParams().antialiasing is False
    for fn, npos in ((rasterizer.RasterizeGaussiansCUDA, 18), (rasterizer.RasterizeGaussiansDepthCUDA, 18),
                     (rasterizer.RasterizeGaussiansBackwardCUDA, 20), (rasterizer.RasterizeGaussiansBackwardDepthCUDA, 21)):
        ps = inspect.signature(fn).parameters
        pos = [p for p in ps.values() if p.kind == p.POSITIONAL_OR_KEYWORD]
        assert len(pos) == npos, fn.__name__
        assert ps["antialiasing"].kind == ps["antialiasing"].KEYWORD_ONLY and ps["antialiasing"].default is False, fn.__name__
    with pytest.raises(TypeError):
        rasterizer.RasterizeGaussiansCUDA(*([None] * 18), True)
    for cls in (trainer.GaussianTrainer, trainer.DataParallelTrainer):
        assert inspect.signature(cls.__init__).parameters["antialiasing"].default is False
    assert isinstance(trainer.GaussianTrainer.antialiasing, property)
