"""CPU: the opacity / normal / second-moment entry points of the rasterizer operator (psb_rasterize_forward_planes /
psb_rasterize_backward_planes, the B1 glue, the autograd front end, the renderer and the LibTorch drop-in) reject bad arguments on the
host, before any CUDA call."""
import ctypes as C
import os
import subprocess

import pytest

from photo_slam_b200 import _lib

ONE = 4096  # fake non-null pointer; never dereferenced because validation fails first


def _fwd(L, P=10, shs=ONE, colors=None, scales=ONE, rotations=ONE, cov=None, planes=None, scratch=None, nbytes=0, aa=0):
    cb = _lib.ALLOC_FN(lambda n, u: 0)
    rec = C.byref(planes) if planes is not None else None
    return L.psb_rasterize_forward_planes(cb, None, cb, None, cb, None, P, 3, 16, ONE, 64, 64, ONE, shs, colors, ONE, scales, 1.0, rotations, cov,
                                          ONE, ONE, ONE, 1.0, 1.0, 0, ONE, None, rec, scratch, nbytes, aa, None)


def _bwd(L, P=10, R=100, grads=None, dL_dz=ONE, det_scratch=None, det_bytes=0, scratch=None, nbytes=0, aa=0, det=0, scales=ONE,
         rotations=ONE, cov=None, dL_dpix=ONE, dL_drot=ONE):
    rec = C.byref(grads) if grads is not None else None
    return L.psb_rasterize_backward_planes(P, 3, 16, R, ONE, 64, 64, ONE, ONE, None, scales, 1.0, rotations, cov, ONE, ONE, ONE, 1.0, 1.0, None,
                                           ONE, ONE, ONE, dL_dpix, ONE, ONE, ONE, ONE, ONE, ONE, ONE, ONE, dL_drot, rec, dL_dz, det_scratch,
                                           det_bytes, scratch, nbytes, aa, det, None)


def _err(L):
    return L.psb_last_error()


def test_planes_forward_validates_before_any_cuda_call():
    L = _lib.lib()
    P = _lib.RasterPlanes
    # everything the plain forward rejects, under this entry point's name
    assert _fwd(L, colors=ONE) == -1 and b"psb_rasterize_forward_planes: provide exactly one of shs" in _err(L)
    assert _fwd(L, P=-1, planes=P(ONE, ONE, None, ONE)) == -1 and b"bad argument" in _err(L)
    assert _fwd(L, aa=2) == -1 and b"antialiasing must be 0 or 1" in _err(L)
    # the normal plane needs scales and rotations, and its scratch
    assert _fwd(L, scales=None, rotations=None, cov=ONE, planes=P(None, None, ONE, None), scratch=ONE, nbytes=1 << 30) == -1
    assert b"the normal plane needs scales and rotations, not cov3D_precomp" in _err(L)
    need = L.psb_rasterize_planes_bytes(10, 0)
    assert _fwd(L, planes=P(None, None, ONE, None)) == -1 and b"plane_scratch" in _err(L)
    assert _fwd(L, planes=P(None, None, ONE, None), scratch=ONE, nbytes=need - 1) == -1 and str(need).encode() in _err(L)
    # opacity and the second moment work with cov3D_precomp; the allocator (which returns NULL here) is the first thing that fails
    assert _fwd(L, scales=None, rotations=None, cov=ONE, planes=P(None, ONE, None, ONE)) == -1 and b"allocator returned null" in _err(L)


def test_planes_backward_validates_before_any_cuda_call():
    L = _lib.lib()
    G = _lib.RasterPlaneGrads
    assert _bwd(L, aa=3) == -1 and b"antialiasing must be 0 or 1" in _err(L)
    assert _bwd(L, det=2) == -1 and b"deterministic must be 0 or 1" in _err(L)
    # a gradient with nowhere to go, whatever P is
    for P in (10, 0):
        assert _bwd(L, P=P, grads=G(ONE, None, None, None), dL_dz=None) == -1 and b"dL_ddepth needs a dL_dz array" in _err(L)
        assert _bwd(L, P=P, grads=G(None, None, None, ONE), dL_dz=None) == -1 and b"dL_ddepth2 needs a dL_dz array" in _err(L)
        assert _bwd(L, P=P, grads=G(None, None, ONE, None), scales=None, rotations=None, cov=ONE, scratch=ONE, nbytes=1 << 30) == -1
        assert b"dL_dnormal needs scales and rotations, not cov3D_precomp" in _err(L)
        assert _bwd(L, P=P, grads=G(None, None, ONE, None), dL_drot=None, scratch=ONE, nbytes=1 << 30) == -1
        assert b"dL_dnormal needs a dL_drot array" in _err(L)
    # the normal gradient's scratch: psb_rasterize_planes_bytes(P, 0), or (P, R) in deterministic mode
    assert _bwd(L, grads=G(None, None, ONE, None)) == -1 and b"plane_scratch" in _err(L)
    need0, needR = L.psb_rasterize_planes_bytes(10, 0), L.psb_rasterize_planes_bytes(10, 100)
    assert needR >= need0 + 64 * 100
    assert _bwd(L, grads=G(None, None, ONE, None), scratch=ONE, nbytes=need0 - 1) == -1 and str(need0).encode() in _err(L)
    det_need = L.psb_rasterize_backward_det_bytes(10, 100)
    assert _bwd(L, grads=G(None, None, ONE, None), det=1, det_scratch=ONE, det_bytes=det_need, scratch=ONE, nbytes=need0) == -1
    assert str(needR).encode() in _err(L)
    # deterministic mode needs its own scratch, as psb_rasterize_backward_deterministic
    assert _bwd(L, grads=G(None, ONE, None, None), det=1) == -1 and b"det_scratch is NULL" in _err(L)
    assert _bwd(L, grads=G(None, ONE, None, None), det=1, det_scratch=ONE, det_bytes=det_need - 1) == -1 and b"det_scratch holds" in _err(L)
    # everything the plain backward rejects
    assert _bwd(L, dL_dpix=None) == -1 and b"psb_rasterize_backward_planes: bad argument" in _err(L)
    assert _bwd(L, P=0) == 0 and _bwd(L, P=0, grads=G(ONE, ONE, ONE, ONE), scratch=ONE, nbytes=0) == 0   # nothing to do


def test_planes_bytes_is_a_pure_function_of_P_and_R():
    L = _lib.lib()
    assert L.psb_rasterize_planes_bytes(-1, 0) == 0 and L.psb_rasterize_planes_bytes(1, -1) == 0
    assert L.psb_rasterize_planes_bytes(1000, 0) >= 1000 * 28
    assert L.psb_rasterize_planes_bytes(1000, 5000) - L.psb_rasterize_planes_bytes(1000, 0) >= 5000 * 64
    # the existing scratch sizes are untouched by the planes
    assert L.psb_rasterize_backward_det_bytes(1000, 5000) < L.psb_rasterize_planes_bytes(1000, 5000)


def test_python_front_ends_refuse_normals_with_a_covariance_before_any_c_call():
    import torch
    from photo_slam_b200 import rasterizer, renderer, trainer
    P = 4
    z = torch.zeros
    rs = rasterizer.GaussianRasterizationSettings(32, 32, 1.0, 1.0, z(3), 1.0, torch.eye(4).flatten(), torch.eye(4).flatten(), 3, z(3))
    r = rasterizer.GaussianRasterizer(rs)
    with pytest.raises(RuntimeError, match="normal plane needs scales and rotations"):
        r(z(P, 3), z(P, 3), z(P, 1), colors_precomp=z(P, 3), cov3D_precomp=z(P, 6), return_normal=True)
    with pytest.raises(RuntimeError, match="normal plane needs scales and rotations"):
        rasterizer.RasterizeGaussiansPlanesCUDA(z(3), z(P, 3), z(P, 3), z(P, 1), None, None, 1.0, z(P, 6), None, None, 1.0, 1.0, 8, 8, None, 0,
                                                None, False, normal=True)
    with pytest.raises(RuntimeError, match="normal plane needs scales and rotations"):
        rasterizer.RasterizeGaussiansBackwardPlanesCUDA(z(3), z(P, 3), None, z(P, 3), None, None, 1.0, z(P, 6), None, None, 1.0, 1.0, z(3, 8, 8),
                                                        None, None, z(3, 8, 8), None, None, 0, None, None, 0, None, None)
    with pytest.raises(RuntimeError, match="num_points, 3"):
        rasterizer.RasterizeGaussiansPlanesCUDA(z(3), z(P, 2), None, None, None, None, 1.0, None, None, None, 1.0, 1.0, 8, 8, None, 0, None,
                                                False, alpha=True)
    model = trainer.GaussianModel.__new__(trainer.GaussianModel)
    model.xyz_ = z(P, 3)
    cam = dict(viewmatrix=torch.eye(4).flatten(), projmatrix=torch.eye(4).flatten(), campos=z(3), tanfovx=1.0, tanfovy=1.0)
    with pytest.raises(RuntimeError, match="return_normal needs scales and rotations"):
        renderer.render(cam, 8, 8, model, renderer.GaussianPipelineParams(compute_cov3D=True), return_normal=True)


def test_libtorch_shim_exports_the_planes_symbols():
    lib = os.path.join(os.path.dirname(_lib.LIB_PATH), "libcuda_rasterizer.so")
    assert os.path.exists(lib), "build it with `python photo-slam_b200/build.py --torch`"
    out = subprocess.run(["nm", "-D", "--defined-only", "-C", lib], capture_output=True, text=True, check=True).stdout
    for sym in ("RasterizeGaussiansPlanesCUDA(", "RasterizeGaussiansBackwardPlanesCUDA(",
                "RasterizeGaussiansCUDA(", "RasterizeGaussiansBackwardCUDA(", "markVisible(", "CudaRasterizer::Rasterizer::forward(",
                "CudaRasterizer::Rasterizer::backward("):
        assert sym in out, sym
