"""CPU: the deterministic backward of the rasterizer operator (psb_rasterize_backward_deterministic, its scratch size, the LibTorch
drop-in's RasterizeGaussiansBackwardDeterministicCUDA and GaussianRasterizer(..., deterministic=True)) rejects bad arguments on the
host, before any CUDA call."""
import os
import subprocess

import pytest

from photo_slam_b200 import _lib

ONE = 4096  # fake non-null pointer; never dereferenced because validation fails first
P0, R0 = 10, 100


def _bwd(L, P=P0, R=R0, dL_dpix=ONE, dL_ddepth=None, dL_dz=None, scratch=ONE, nbytes=None):
    if nbytes is None:
        nbytes = L.psb_rasterize_backward_det_bytes(P, R)
    return L.psb_rasterize_backward_deterministic(P, 3, 16, R, ONE, 64, 64, ONE, ONE, None, ONE, 1.0, ONE, None, ONE, ONE, ONE, 1.0, 1.0,
                                                  None, ONE, ONE, ONE, dL_dpix, ONE, ONE, ONE, ONE, ONE, ONE, ONE, ONE, ONE, dL_ddepth, dL_dz,
                                                  scratch, nbytes, None)


def test_deterministic_backward_validates_before_any_cuda_call():
    L = _lib.lib()
    name = b"psb_rasterize_backward_deterministic: "
    assert _bwd(L, scratch=None) == -1 and L.psb_last_error() == name + b"det_scratch is NULL"
    need = L.psb_rasterize_backward_det_bytes(P0, R0)
    assert _bwd(L, nbytes=need - 1) == -1 and L.psb_last_error().startswith(name + b"det_scratch holds")
    assert str(need).encode() in L.psb_last_error()
    assert _bwd(L, dL_ddepth=ONE, dL_dz=ONE, nbytes=need - 1) == -1          # with a depth gradient too
    # a depth gradient needs somewhere to put dL/dz, whatever P is
    for P in (P0, 0):
        assert _bwd(L, P=P, dL_ddepth=ONE) == -1 and L.psb_last_error() == name + b"dL_ddepth needs a dL_dz array"
    # everything the plain backward rejects, under the new name
    assert _bwd(L, dL_dpix=None) == -1 and L.psb_last_error() == name + b"bad argument"
    assert _bwd(L, P=-3) == -1 and L.psb_last_error() == name + b"bad argument"
    assert _bwd(L, R=-1, nbytes=0) == -1 and L.psb_last_error() == name + b"bad argument"
    # nothing to do, as psb_rasterize_backward: no scratch is needed either
    assert _bwd(L, P=0) == 0
    assert _bwd(L, P=0, scratch=None, nbytes=0) == 0
    # the plain entry points' messages are unchanged
    assert L.psb_rasterize_backward(P0, 3, 16, R0, ONE, 64, 64, ONE, ONE, None, ONE, 1.0, ONE, None, ONE, ONE, ONE, 1.0, 1.0, None, ONE, ONE,
                                    ONE, None, ONE, ONE, ONE, ONE, ONE, ONE, ONE, ONE, ONE, None) == -1
    assert L.psb_last_error() == b"psb_rasterize_backward: bad argument"


def test_det_scratch_bytes_cover_slots_and_bases_and_grow_with_both_sizes():
    L = _lib.lib()
    f = L.psb_rasterize_backward_det_bytes
    sizes = (0, 1, 7, 100, 4097, 1_000_003, 13_000_000)
    for P in sizes:
        for R in sizes:
            assert f(P, R) >= 48 * R + 4 * P, (P, R)
    for a, b in zip(sizes, sizes[1:]):
        for n in sizes:
            assert f(b, n) >= f(a, n) and f(n, b) >= f(n, a), (a, b, n)
    assert f(10, 1_000_100) > f(10, 1_000_000) and f(1_000_100, 10) > f(1_000_000, 10)
    assert f(-1, 5) == 0 and f(5, -1) == 0


def test_libtorch_shim_exports_the_deterministic_symbol():
    """RasterizeGaussiansBackwardDeterministicCUDA (the signature of RasterizeGaussiansBackwardDepthCUDA) is exported next to the
    reference's symbols."""
    lib = os.path.join(os.path.dirname(_lib.LIB_PATH), "libcuda_rasterizer.so")
    assert os.path.exists(lib), "build it with `python photo-slam_b200/build.py --torch`"
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True).stdout
    for sym in ("_Z43RasterizeGaussiansBackwardDeterministicCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffS2_S2_S2_iS2_S2_iS2_S2_",
                "_Z35RasterizeGaussiansBackwardDepthCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffS2_S2_S2_iS2_S2_iS2_S2_",
                # the reference's own symbols stay
                "_Z22RasterizeGaussiansCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffiiS2_iS2_b",
                "_Z30RasterizeGaussiansBackwardCUDARKN2at6TensorES2_S2_S2_S2_S2_fS2_S2_S2_ffS2_S2_iS2_S2_iS2_S2_"):
        assert sym in out, sym


def test_deterministic_rasterizer_frontend_validation_is_host_side():
    import torch
    from photo_slam_b200 import rasterizer
    P = 4
    z = torch.zeros
    rs = rasterizer.GaussianRasterizationSettings(32, 32, 1.0, 1.0, z(3), 1.0, torch.eye(4).flatten(), torch.eye(4).flatten(), 3, z(3))
    r = rasterizer.GaussianRasterizer(rs)
    for depth in (False, True):
        with pytest.raises(RuntimeError, match="SHs or precomputed colors"):
            r(z(P, 3), z(P, 3), z(P, 1), shs=z(P, 16, 3), colors_precomp=z(P, 3), scales=z(P, 3), rotations=z(P, 4), return_depth=depth,
              deterministic=True)
        with pytest.raises(RuntimeError, match="scale/rotation pair or precomputed 3D covariance"):
            r(z(P, 3), z(P, 3), z(P, 1), shs=z(P, 16, 3), scales=z(P, 3), return_depth=depth, deterministic=True)
    with pytest.raises(RuntimeError, match="num_points, 3"):
        rasterizer.RasterizeGaussiansCUDA(z(3), z(P, 2), None, None, None, None, 1.0, None, None, None, 1.0, 1.0, 8, 8, None, 0, None, False)
    # the flag is keyword-only on the B1 functions: their positional argument lists stay the reference's
    with pytest.raises(TypeError):
        rasterizer.RasterizeGaussiansBackwardCUDA(*([None] * 20), True)
