"""-m gpu: the per-row live byte of the fused step (psb_model.adam_live).

Contract: a row whose byte is 0 has all 118 moments exactly zero. The fused step skips such rows unless a gradient
reaches them, so (a) the contract must survive every entry point that touches the model, (b) rows no gradient has
reached stay untouched, and (c) a step with the byte computes what the step without it (moments read to find idle
rows) computes."""
import ctypes as C

import numpy as np
import pytest
import torch

import photo_slam_b200.synthetic as syn

pytestmark = pytest.mark.gpu

LRS = [0.00032, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]


def _setup(cuda, P=40_000, W=320, H=240, seed=5):
    from photo_slam_b200 import trainer
    cam0 = syn.make_camera(W, H, 260.0, 260.0)
    sc = syn.make_scene(P, cam0, seed=seed)
    sc["xyz"][::2, 0] += 1000.0          # half of the rows far outside the view: never reached
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    c = syn.device_camera(cam0, cuda)
    gt = torch.from_numpy(syn.target_image(H, W, seed=2)).to(cuda)
    return m, trainer.GaussianTrainer(m), c, gt


def _moment_rows(m):
    """bool [P]: any of the row's 118 moments is non-zero"""
    nz = torch.zeros(m.num_points(), dtype=torch.bool, device=m.device)
    for t in m.exp_avg_ + m.exp_avg_sq_:
        nz |= (t.reshape(t.size(0), -1) != 0).any(dim=1)
    return nz


def _assert_contract(m, what):
    assert m.adam_live_valid_, what
    live = m.adam_live_.bool()
    nz = _moment_rows(m)
    assert not (nz & ~live).any(), f"{what}: {(nz & ~live).sum().item()} rows with non-zero moments have adam_live == 0"


def _step(tr, c, gt, n=1):
    for _ in range(n):
        tr.trainForOneIteration(c, gt)
        tr.result()
    torch.cuda.synchronize()


def test_contract_holds_after_every_entry_point(cuda):
    from photo_slam_b200 import trainer
    m, tr, c, gt = _setup(cuda)
    _step(tr, c, gt, 6)
    _assert_contract(m, "fused steps")
    live = m.adam_live_.bool()
    assert 0 < live.sum().item() < m.num_points() // 2, "the scene must leave most rows without a gradient"
    snap = m.snapshot()

    m.resetOpacity()                      # zeroes moments: the bytes stay conservative
    _assert_contract(m, "resetOpacity")
    _step(tr, c, gt, 2)
    _assert_contract(m, "step after resetOpacity")

    m.restore(snap)
    _assert_contract(m, "restore")
    assert torch.equal(m.adam_live_, snap["live"])
    _step(tr, c, gt, 2)
    _assert_contract(m, "step after restore")

    m.densifyAndPrune(1e-6, 0.005, 2.0, 0, seed=1)
    assert not m.adam_live_valid_
    _step(tr, c, gt, 2)
    _assert_contract(m, "densifyAndPrune + step")

    g = torch.Generator(device=cuda).manual_seed(3)
    m.prunePoints(torch.rand(m.num_points(), device=cuda, generator=g) < 0.1)
    _step(tr, c, gt, 2)
    _assert_contract(m, "prunePoints + step")

    pts = m.xyz_[:500].detach().clone() + 0.01
    m.increasePcd(pts, torch.rand(500, 3, device=cuda, generator=g), iteration=10)
    _step(tr, c, gt, 2)
    _assert_contract(m, "increasePcd + step")

    dp = trainer.DataParallelTrainer(m)   # world 1: backward -> Adam split path, moments written without the bytes
    dp.trainForOneIteration(c, gt)
    dp.result()
    assert not m.adam_live_valid_
    _step(tr, c, gt, 2)
    _assert_contract(m, "DataParallelTrainer step + fused step")


def test_rows_never_reached_are_untouched(cuda):
    m, tr, c, gt = _setup(cuda)
    p0 = [t.clone() for t in m.tensors()]
    _step(tr, c, gt, 6)
    idle = ~m.adam_live_.bool()
    assert idle.sum().item() >= m.num_points() // 2
    for a, b in zip(m.tensors(), p0):
        assert torch.equal(a[idle], b[idle])
    for t in m.exp_avg_ + m.exp_avg_sq_:
        assert not t[idle].any()


def test_step_with_live_bytes_matches_step_without(cuda):
    from photo_slam_b200 import _lib, trainer
    m, tr, c, gt = _setup(cuda)
    _step(tr, c, gt, 5)
    snap = m.snapshot()
    _step(tr, c, gt, 1)                   # with the live bytes
    with_live = [t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_]
    m.restore(snap)
    cm, cc, cs = m._cmodel(), trainer._ccamera(c), tr._cstep(True)   # adam_live = NULL
    _lib.check(tr.L.psb_trainer_step(tr.h, m.num_points(), 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), gt.data_ptr(), None, C.byref(cs),
                                     None, None, torch.cuda.current_stream().cuda_stream), "psb_trainer_step")
    torch.cuda.synchronize()
    without = m.tensors() + m.exp_avg_ + m.exp_avg_sq_
    for i, (a, b) in enumerate(zip(with_live[:6], without[:6])):
        frac = ((a - b).abs() > 0.5 * LRS[i]).float().mean().item()
        assert frac < 2e-3, f"{trainer.GROUPS[i]}: {frac} of entries differ by more than half an Adam step"
    for a, b in zip(with_live[6:], without[6:]):
        assert ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item() < 1e-4
        assert torch.equal(a == 0, b == 0) or ((a == 0) != (b == 0)).float().mean().item() < 1e-3
