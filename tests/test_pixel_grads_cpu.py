"""CPU: the caller's-loss entry points (psb_trainer_forward, psb_trainer_backward_pixels) are declared, exported and validate their
arguments before any CUDA call; the Python front end checks its inputs on the host, and DataParallelTrainer refuses trainWithLoss."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from photo_slam_b200 import _lib, trainer

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "psb200.h")


def test_declared_and_exported():
    hdr = open(HEADER).read()
    for name in ("psb_trainer_forward", "psb_trainer_backward_pixels"):
        assert name in _lib.exported_symbols()
        assert hasattr(_lib.lib(), name)
    assert "typedef struct psb_pixel_grads" in hdr
    assert [f for f, _ in trainer._PixelGrads._fields_] == ["dL_dcolor", "dL_ddepth", "dL_dalpha"]


def test_c_argument_checks_need_no_device():
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        assert L.psb_trainer_forward(h, 10, 16, None, None, None, 0, None, None, None, None, None, None) == -1
        assert b"psb_trainer_forward: null argument" in L.psb_last_error()
        step = trainer._Step()
        px = trainer._PixelGrads(4096, None, None)
        cam, model = trainer._Camera(), trainer._Model()
        bwd = lambda pass_no, pg: L.psb_trainer_backward_pixels(h, pass_no, 10, 16, C.byref(model), C.byref(cam), 4096, pg, C.byref(step), None, None)
        assert bwd(1, None) == -1 and b"null argument" in L.psb_last_error()
        assert bwd(1, C.byref(trainer._PixelGrads(None, None, None))) == -1 and b"dL_dcolor is required" in L.psb_last_error()
        # a fresh context has run no forward pass
        for p in (0, 1):
            assert bwd(p, C.byref(px)) == -1 and b"latest forward pass" in L.psb_last_error()
    finally:
        L.psb_trainer_destroy(h)


def _cpu_trainer(P=40, W=32, H=24):
    import photo_slam_b200.synthetic as syn
    cam = syn.make_camera(W, H, 30.0, 30.0, *syn.random_pose(np.random.default_rng(0)))
    sc = syn.make_scene(P, cam, seed=1, scale_px=2.0)
    m = trainer.GaussianModel.from_numpy(sc, "cpu")
    m.trainingSetup(trainer.GaussianOptimizationParams())
    tr = trainer.GaussianTrainer(m, background=torch.zeros(3))
    c = dict(viewmatrix=torch.zeros(16), projmatrix=torch.zeros(16), campos=torch.zeros(3), tanfovx=1.0, tanfovy=1.0, W=W, H=H)
    return tr, m, c


def test_backward_pixels_checks_its_inputs_on_the_host():
    tr, m, c = _cpu_trainer()
    H, W = c["H"], c["W"]
    with pytest.raises(_lib.PsbError, match="call render"):
        tr.backwardPixels(torch.zeros((3, H, W)))
    tr._last_render, tr._pass = (c, None, None, None, None), 1     # as after a render of this view
    bad = [dict(dL_dcolor=None), dict(dL_dcolor=torch.zeros((3, W, H))), dict(dL_dcolor=torch.zeros((3, H, W), dtype=torch.float64)),
           dict(dL_dcolor=torch.zeros((3, H, W)), dL_ddepth=torch.zeros((1, H, W))),
           dict(dL_dcolor=torch.zeros((3, H, W)), dL_dalpha=torch.zeros((W, H)).t()),
           dict(dL_dcolor=torch.zeros((3, H, W)), grads=[torch.zeros_like(t) for t in m.tensors()][:5]),
           dict(dL_dcolor=torch.zeros((3, H, W)), grads=[torch.zeros_like(t) for t in m.tensors()][::-1])]
    for kw in bad:
        with pytest.raises(ValueError):
            tr.backwardPixels(**kw)
    assert m.step_ == 0 and tr.iteration == 0


def test_train_with_loss_needs_a_callable():
    tr, m, c = _cpu_trainer()
    with pytest.raises(TypeError, match="callable"):
        tr.trainWithLoss(c, None)


def test_data_parallel_trainer_refuses_a_callers_loss():
    dp = trainer.DataParallelTrainer.__new__(trainer.DataParallelTrainer)   # (the refusal needs no context)
    with pytest.raises(NotImplementedError, match="trainWithLoss"):
        dp.trainWithLoss({}, lambda image: image.sum())
    with pytest.raises(NotImplementedError, match="grads="):
        dp.backwardPixels(torch.zeros((3, 4, 4)))
