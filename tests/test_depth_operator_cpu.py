"""CPU: the depth entry points of the rasterizer operator (psb_rasterize_forward_depth / psb_rasterize_backward_depth, the B1 glue, the
autograd front-end and the LibTorch drop-in) reject bad arguments on the host, before any CUDA call."""
import os
import subprocess

import pytest

from photo_slam_b200 import _lib

ONE = 4096  # fake non-null pointer; never dereferenced because validation fails first


def _fwd(L, P=10, D=3, M=16, shs=ONE, colors=None, out_depth=ONE):
    cb = _lib.ALLOC_FN(lambda n, u: 0)
    return L.psb_rasterize_forward_depth(cb, None, cb, None, cb, None, P, D, M, ONE, 64, 64, ONE, shs, colors, ONE, ONE, 1.0, ONE, None,
                                         ONE, ONE, ONE, 1.0, 1.0, 0, ONE, None, out_depth, None)


def _bwd(L, P=10, dL_dpix=ONE, dL_ddepth=ONE, dL_dz=ONE):
    return L.psb_rasterize_backward_depth(P, 3, 16, 100, ONE, 64, 64, ONE, ONE, None, ONE, 1.0, ONE, None, ONE, ONE, ONE, 1.0, 1.0, None,
                                          ONE, ONE, ONE, dL_dpix, ONE, ONE, ONE, ONE, ONE, ONE, ONE, ONE, ONE, dL_ddepth, dL_dz, None)


def test_depth_entry_points_validate_before_any_cuda_call():
    L = _lib.lib()
    # everything the plain forward rejects, reported under the depth entry point's name
    assert _fwd(L, colors=ONE) == -1 and b"psb_rasterize_forward_depth: provide exactly one of shs" in L.psb_last_error()
    assert _fwd(L, M=4) == -1 and b"SH degree" in L.psb_last_error()
    assert _fwd(L, P=-1) == -1 and b"bad argument" in L.psb_last_error()
    assert _fwd(L, colors=ONE, out_depth=None) == -1          # NULL out_depth: the plain forward, with its own checks
    # the plain forward's messages are unchanged
    cb = _lib.ALLOC_FN(lambda n, u: 0)
    assert L.psb_rasterize_forward(cb, None, cb, None, cb, None, 10, 3, 16, ONE, 64, 64, ONE, ONE, ONE, ONE, ONE, 1.0, ONE, None, ONE, ONE,
                                   ONE, 1.0, 1.0, 0, ONE, None, None) == -1
    assert L.psb_last_error().startswith(b"psb_rasterize_forward: provide exactly one of shs")
    # a depth gradient needs somewhere to put dL/dz, whatever P is
    for P in (10, 0):
        assert _bwd(L, P=P, dL_dz=None) == -1 and b"psb_rasterize_backward_depth: dL_ddepth needs a dL_dz array" in L.psb_last_error()
    # everything the plain backward rejects
    assert _bwd(L, dL_dpix=None) == -1 and b"psb_rasterize_backward_depth: bad argument" in L.psb_last_error()
    assert _bwd(L, P=-3) == -1
    assert _bwd(L, P=0) == 0                                  # nothing to do, as psb_rasterize_backward


def test_depth_rasterizer_frontend_validation_is_host_side():
    import torch
    from photo_slam_b200 import rasterizer
    P = 4
    z = torch.zeros
    rs = rasterizer.GaussianRasterizationSettings(32, 32, 1.0, 1.0, z(3), 1.0, torch.eye(4).flatten(), torch.eye(4).flatten(), 3, z(3))
    r = rasterizer.GaussianRasterizer(rs)
    with pytest.raises(RuntimeError, match="SHs or precomputed colors"):
        r(z(P, 3), z(P, 3), z(P, 1), shs=z(P, 16, 3), colors_precomp=z(P, 3), scales=z(P, 3), rotations=z(P, 4), return_depth=True)
    with pytest.raises(RuntimeError, match="scale/rotation pair or precomputed 3D covariance"):
        r(z(P, 3), z(P, 3), z(P, 1), shs=z(P, 16, 3), scales=z(P, 3), return_depth=True)
    with pytest.raises(RuntimeError, match="num_points, 3"):
        rasterizer.RasterizeGaussiansDepthCUDA(z(3), z(P, 2), None, None, None, None, 1.0, None, None, None, 1.0, 1.0, 8, 8, None, 0, None,
                                               False)


def test_libtorch_shim_exports_the_depth_symbols():
    """The two C++ depth functions of the LibTorch drop-in are exported next to the reference's symbols (signatures: the reference's
    RasterizeGaussiansCUDA / RasterizeGaussiansBackwardCUDA, the latter with dL_dout_depth after dL_dout_color)."""
    lib = os.path.join(os.path.dirname(_lib.LIB_PATH), "libcuda_rasterizer.so")
    assert os.path.exists(lib), "build it with `python photo-slam_b200/build.py --torch`"
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    for sym in ("_Z27RasterizeGaussiansDepthCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffiiS2_iS2_b",
                "_Z35RasterizeGaussiansBackwardDepthCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffS2_S2_S2_iS2_S2_iS2_S2_",
                # the reference's own symbols stay
                "_Z22RasterizeGaussiansCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffiiS2_iS2_b",
                "_Z30RasterizeGaussiansBackwardCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffS2_S2_iS2_S2_iS2_S2_"):
        assert sym in out, sym
