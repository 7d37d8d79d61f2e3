"""-m gpu: the NVLink data-parallel step (psb_dp_step) — single-GPU equivalence with the fused step, and K ranks over real peer memory
(one per GPU when the box has >= 2, three processes sharing the GPU otherwise): replicas bit-identical and equal to the 1-rank step on
the summed gradients."""
import os
import subprocess
import sys

import pytest
import torch

import photo_slam_b200.synthetic as syn
import shared_device
from helpers import scene_tensors

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LRS = [0.00032, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]


@pytest.mark.parametrize("P", [20_000, 12_345])
def test_p2p_step_world1_equals_fused_step(cuda, P):
    """world == 1: push into the own inbox -> owner-side Adam must reproduce psb_trainer_step (same arithmetic, other kernels)."""
    from photo_slam_b200 import trainer
    wh = (320, 240)
    cam, sc, act, g, c = scene_tensors(P, "tum", seed=5, pose_seed=6, dev=cuda, wh=wh, scale_px=4.0)
    gt = torch.rand((3, wh[1], wh[0]), device=cuda)
    a = trainer.GaussianModel.from_numpy(sc, cuda)
    b = trainer.GaussianModel.from_numpy(sc, cuda)
    for m in (a, b):
        m.trainingSetup(trainer.GaussianOptimizationParams())
    ta = trainer.GaussianTrainer(a)
    tb = trainer.DataParallelTrainer(b, mode="p2p")
    assert tb.mode == "p2p"
    for it in range(4):
        ta.trainForOneIteration(c, gt)
        la = ta.result()[0]
        tb.trainForOneIteration(c, gt)
        lb = tb.result()[0]
        assert abs(la - lb) <= 2e-5 * max(1.0, abs(la)), (it, la, lb)
    tb.sync()
    torch.cuda.synchronize()
    assert tb.status() == 0
    for x, y, lr, name in zip(a.tensors(), b.tensors(), LRS, trainer.GROUPS):
        frac = ((x - y).abs() > 0.5 * lr).float().mean().item()
        assert frac < 2e-3, (name, frac)
    for x, y in zip(a.exp_avg_ + a.exp_avg_sq_, b.exp_avg_ + b.exp_avg_sq_):
        rn = ((x.double() - y.double()).norm() / (x.double().norm() + 1e-30)).item()
        assert rn < 1e-4, rn
    for x, y in zip((a.max_radii2D_, a.denom_), (b.max_radii2D_, b.denom_)):
        assert torch.equal(x, y)
    tb.close()


def _launch(world, mode, P, steps=3, timeout=420):
    port = 29500 + (os.getpid() % 400)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(ROOT, "tests", "dp_worker.py"), mode, str(P), str(steps)]
    env = dict(os.environ, PSB_DP_TIMEOUT_MS="15000")
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=env)
    return r


@pytest.mark.parametrize("mode", ["p2p", "nccl"])
def test_multi_rank_replicas_identical_and_equal_summed_gradient_step(cuda, mode):
    """One rank per GPU; on a single GPU, p2p runs three ranks sharing it (tests/shared_device.py)"""
    n = torch.cuda.device_count()
    if n < 2:
        if mode != "p2p":
            pytest.skip("NCCL needs one GPU per rank: >= 2 GPUs")
        why = shared_device.unavailable()
        if why:
            pytest.skip(why)
        codes, out, tails = shared_device.launch(os.path.join(ROOT, "tests", "dp_worker.py"), [mode, 30_001, 3], 3, timeout=600)
        assert codes == [0, 0, 0] and "DP_WORKER_OK" in out, tails
        print(out.strip().splitlines()[-1])
        return
    world = 2 if n < 4 else (4 if n < 8 else 8)
    r = _launch(world, mode, 30_001)
    assert r.returncode == 0 and "DP_WORKER_OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])
    print(r.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("kw", [dict(mode="nccl", pipeline=False), dict(mode="nccl", pipeline=True, nslabs=3), dict(mode="p2p")],
                         ids=["nccl-flat", "nccl-slabs", "p2p"])
def test_split_paths_with_P_not_multiple_of_4(cuda, kw):
    """Gradient segments / slab blocks are padded to 16-byte boundaries: P = 12 345 (odd) must not fault and must match the fused step."""
    from photo_slam_b200 import trainer
    P, wh = 12_345, (320, 240)
    cam, sc, act, g, c = scene_tensors(P, "tum", seed=8, pose_seed=9, dev=cuda, wh=wh, scale_px=4.0)
    gt = torch.rand((3, wh[1], wh[0]), device=cuda)
    a = trainer.GaussianModel.from_numpy(sc, cuda)
    b = trainer.GaussianModel.from_numpy(sc, cuda)
    for m in (a, b):
        m.trainingSetup(trainer.GaussianOptimizationParams())
    ta, tb = trainer.GaussianTrainer(a), trainer.DataParallelTrainer(b, **kw)
    for it in range(3):
        ta.trainForOneIteration(c, gt)
        ta.result()
        tb.trainForOneIteration(c, gt)
        tb.result()
    tb.sync()
    torch.cuda.synchronize()
    for x, y, lr, name in zip(a.tensors(), b.tensors(), LRS, trainer.GROUPS):
        frac = ((x - y).abs() > 0.5 * lr).float().mean().item()
        assert frac < 2e-3, (name, frac)
    tb.close()


@pytest.mark.parametrize("mode", ["nccl", "p2p"])
def test_overflowing_view_is_dropped_not_retried_on_the_data_parallel_path(cuda, mode):
    """A view that overflows the binning arena contributes a ZERO gradient (no stale gradients, no one-rank retry that would
    desynchronise the group); the arena grows and the next step of the same view trains normally."""
    from photo_slam_b200 import trainer
    P, wh = 2_000, (640, 480)
    cam, sc, act, g, c = scene_tensors(P, "tum", seed=2, pose_seed=None, dev=cuda, wh=wh, scale_px=150.0)
    gt = torch.rand((3, wh[1], wh[0]), device=cuda)
    m = trainer.GaussianModel.from_numpy(sc, cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    tr = trainer.DataParallelTrainer(m, mode=mode, pipeline=False) if mode == "nccl" else trainer.DataParallelTrainer(m, mode=mode)
    before = [t.clone() for t in m.tensors()]
    tr.trainForOneIteration(c, gt)
    loss, _, _, n = tr.result()
    tr.sync()
    torch.cuda.synchronize()
    assert n > 6 * P + 65536 and tr.dropped_views == 1 and loss != loss
    for x, y in zip(before, m.tensors()):
        assert torch.equal(x, y), "a dropped view must not move the parameters (zero gradient, zero moments)"
    assert not any(t.any() for t in m.exp_avg_ + m.exp_avg_sq_)
    tr.trainForOneIteration(c, gt)
    loss2 = tr.result()[0]
    tr.sync()
    torch.cuda.synchronize()
    assert loss2 == loss2 and tr.dropped_views == 1
    assert not torch.equal(before[0], m.xyz_)
    tr.close()


def test_queued_overflow_is_reported(cuda):
    """psb_trainer_result reports an overflow of ANY step queued since the last collection (sticky device-side record)."""
    from photo_slam_b200 import _lib, trainer
    P, wh = 2_000, (640, 480)
    cam, big, act, g, c = scene_tensors(P, "tum", seed=2, pose_seed=None, dev=cuda, wh=wh, scale_px=150.0)
    cam2, small, _, _, c2 = scene_tensors(P, "tum", seed=2, pose_seed=None, dev=cuda, wh=wh, scale_px=2.0)
    gt = torch.rand((3, wh[1], wh[0]), device=cuda)
    m = trainer.GaussianModel.from_numpy(small, cuda)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    tr = trainer.GaussianTrainer(m)
    tr.trainForOneIteration(c2, gt)
    tr.result()                                     # fits
    m.scaling_.copy_(torch.from_numpy(big["scaling"]).to(cuda))   # splats now cover hundreds of tiles: the next step overflows
    tr.trainForOneIteration(c2, gt)                 # overflows (queued, not collected)
    m.scaling_.copy_(torch.from_numpy(small["scaling"]).to(cuda))
    tr.trainForOneIteration(c2, gt)                 # fits again
    step_before = m.step_
    with pytest.raises(_lib.PsbError, match="overflowed the binning arena"):
        tr.result()
    assert m.step_ == step_before - 1
    tr.trainForOneIteration(c2, gt)
    assert tr.result()[0] == tr.result()[0]
