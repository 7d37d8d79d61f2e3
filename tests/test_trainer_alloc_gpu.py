"""-m gpu: a trainer context survives an allocation that fails.

A forward pass over more rows than the card can hold returns PSB_ERR_CUDA before any launch. The context must stay usable. The pass's
scratch must not be back-propagated. The next render of the small model must give the same image bit for bit, and a training step must
still work. The failing request is larger than the card's memory, so it fails at once and reserves nothing.
"""
import ctypes as C

import pytest
import torch

from helpers import scene_tensors

pytestmark = pytest.mark.gpu
PSB_ERR_CUDA = -2


def _huge_P(L, total):
    for p in (1 << 28, 1 << 29, 1 << 30, (1 << 31) - 1):
        if L.psb_geometry_bytes(p) > total:
            return p
    return None


def test_failed_allocation_leaves_the_context_usable(cuda):
    from photo_slam_b200 import trainer
    cam, sc, act, g, c = scene_tensors(20_000, "replica", seed=5, pose_seed=6, dev=cuda, wh=(320, 240), scale_px=6.0)
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    m.setShDegree(1)
    P, H, W = m.num_points(), c["H"], c["W"]
    tr = trainer.GaussianTrainer(m)
    huge = _huge_P(tr.L, torch.cuda.get_device_properties(0).total_memory)
    if huge is None:
        pytest.skip("no int row count whose geometry scratch exceeds this card's memory")

    img0, rad0 = torch.empty((3, H, W), device=cuda), torch.zeros(P, dtype=torch.int32, device=cuda)
    tr.render(c, img0, rad0)
    torch.cuda.synchronize()
    pass0 = tr._pass

    # the same small tensors, declared as `huge` rows: the geometry chunk cannot be allocated, and nothing is launched
    cm, cc = m._cmodel(False), trainer._ccamera(c)
    out = torch.empty((3, H, W), device=cuda)
    pass_no = C.c_uint()
    stream = torch.cuda.current_stream().cuda_stream
    rc = tr.L.psb_trainer_forward(tr.h, huge, 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), m.active_sh_degree_, out.data_ptr(), None,
                                  None, None, C.byref(pass_no), stream)
    assert rc == PSB_ERR_CUDA and b"out of memory" in tr.L.psb_last_error()

    # the failed pass has no scratch to back-propagate through
    gc = torch.full((3, H, W), 1e-3, device=cuda)
    cm, cs = m._cmodel(live=m.adamLive()), tr._cstep(True)
    px = trainer._PixelGrads(gc.data_ptr(), None, None)
    rc = tr.L.psb_trainer_backward_pixels(tr.h, pass0, P, 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), C.byref(px), C.byref(cs),
                                          None, stream)
    assert rc == -1 and b"latest forward pass" in tr.L.psb_last_error()

    img1, rad1 = torch.empty((3, H, W), device=cuda), torch.zeros(P, dtype=torch.int32, device=cuda)
    tr.render(c, img1, rad1)
    torch.cuda.synchronize()
    assert torch.equal(img0, img1) and torch.equal(rad0, rad1)

    before = m.xyz_.clone()
    gen = torch.Generator().manual_seed(7)
    gt = torch.rand((3, H, W), generator=gen).to(cuda)
    tr.trainForOneIteration(c, gt)
    loss = tr.result()
    torch.cuda.synchronize()
    assert m.step_ == 1 and loss[0] > 0 and not torch.equal(before, m.xyz_)
