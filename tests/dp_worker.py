"""Worker of tests/test_dp_gpu.py (one process per GPU, launched with torch.distributed.run; or K processes on one GPU, launched by
tests/shared_device.py, p2p only): K data-parallel steps through
DataParallelTrainer(mode=...) on world ranks, then
  (1) every rank's parameter replica must be BIT-identical,
  (2) they must equal the 1-rank step on the summed gradients of the same K views (SURVEY §8e): rank 0 recomputes every view's
      dense gradient with psb_trainer_backward, sums them and applies psb_adam_update(grad_scale = 1/world),
  (3) the Adam moments gathered from their owners must equal that reference's.
Prints one line `DP_WORKER_OK ...` from rank 0 on success; any assertion fails the launch."""
import ctypes as C
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import photo_slam_b200.synthetic as syn  # noqa: E402
import shared_device  # noqa: E402
from photo_slam_b200 import _lib, trainer  # noqa: E402

LRS = [0.00032, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]


def view(rank, W, H, fx, fy, dev):
    R, t = syn.random_pose(np.random.default_rng(100 + rank), max_angle=0.08, max_trans=0.15)
    cam = syn.make_camera(W, H, fx, fy, R, t)
    c = syn.device_camera(cam, dev)
    gt = torch.from_numpy(syn.target_image(H, W, seed=7 + rank)).to(dev)
    return c, gt


def main():
    mode = sys.argv[1] if len(sys.argv) > 1 else "p2p"
    P = int(sys.argv[2]) if len(sys.argv) > 2 else 30_001
    steps = int(sys.argv[3]) if len(sys.argv) > 3 else 3
    shared = shared_device.init_rank()
    if shared:      # every rank on device 0 (tests/shared_device.py): gloo, and the NVLink step only
        assert mode == "p2p", "ranks sharing one device run the p2p step only: NCCL refuses two ranks on one device"
        rank, world, dev = shared
    else:
        rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
        torch.cuda.set_device(local)
        dev = torch.device("cuda", local)
        dist.init_process_group("nccl", device_id=dev)
    W, H, fx, fy = 320, 240, 260.0, 260.0
    sc = syn.make_scene(P, syn.make_camera(W, H, fx, fy), seed=11, scale_px=4.0)
    model = trainer.GaussianModel.from_numpy(sc, dev)
    model.trainingSetup(trainer.GaussianOptimizationParams())
    tr = trainer.DataParallelTrainer(model, mode=mode)
    assert tr.mode == mode, f"requested {mode}, running {tr.mode}: {getattr(tr, '_p2p_error', '')}"
    c, gt = view(rank, W, H, fx, fy, dev)
    losses = []
    for _ in range(steps):
        tr.trainForOneIteration(c, gt)
        losses.append(tr.result()[0])
    tr.sync()
    torch.cuda.synchronize()
    dist.barrier()
    assert tr.status() == 0, "a cross-rank wait timed out"
    tr.gather_moments()
    torch.cuda.synchronize()
    # (1) bit-identical replicas
    for name, t in zip(trainer.GROUPS, model.tensors()):
        ref0 = t.clone()
        dist.broadcast(ref0, src=0)
        assert torch.equal(ref0, t), f"rank {rank}: replica of {name} differs from rank 0"
    for t in model.exp_avg_ + model.exp_avg_sq_:
        ref0 = t.clone()
        dist.broadcast(ref0, src=0)
        assert torch.equal(ref0, t), f"rank {rank}: gathered moments differ from rank 0"
    # (2)+(3) vs the 1-rank step on the summed gradients
    if rank == 0:
        ref = trainer.GaussianModel.from_numpy(sc, dev)
        ref.trainingSetup(trainer.GaussianOptimizationParams())
        rt = trainer.DataParallelTrainer(ref, mode="nccl", pipeline=False)   # world-agnostic use of backward / adam_update below
        from photo_slam_b200.parallel import GradBuffer
        views = [view(r, W, H, fx, fy, dev) for r in range(world)]
        total = GradBuffer(P, dev)
        for _ in range(steps):
            total.flat.zero_()
            cm, cs = ref._cmodel(), rt._cstep(True)
            for (cc_, gt_) in views:
                ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in rt.segs])
                cc = trainer._ccamera(cc_)
                _lib.check(rt.L.psb_trainer_backward(rt.h, P, 16, C.byref(cm), C.byref(cc), rt.background.data_ptr(), gt_.data_ptr(), None, C.byref(cs),
                                                     None, None, ptrs, torch.cuda.current_stream().cuda_stream), "psb_trainer_backward")
                total.flat += rt.flat
            ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in total.segments])
            _lib.check(rt.L.psb_adam_update(P, 16, C.byref(cm), ptrs, C.byref(cs), 1.0 / world, torch.cuda.current_stream().cuda_stream), "psb_adam_update")
            ref.step_ += 1
        torch.cuda.synchronize()
        worst = 0.0
        for name, a, b, lr in zip(trainer.GROUPS, model.tensors(), ref.tensors(), LRS):
            frac = ((a - b).abs() > 0.5 * lr).float().mean().item()
            worst = max(worst, frac)
            assert frac < 2e-3, f"{name}: {frac} of the entries differ from the summed-gradient step by more than half an Adam step"
        for name, a, b in zip(trainer.GROUPS, model.exp_avg_, ref.exp_avg_):
            rn = ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()
            assert rn < 1e-4, f"exp_avg {name}: rel-norm {rn}"
        for name, a, b in zip(trainer.GROUPS, model.exp_avg_sq_, ref.exp_avg_sq_):
            rn = ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()
            assert rn < 1e-4, f"exp_avg_sq {name}: rel-norm {rn}"
        print(f"DP_WORKER_OK mode={mode} world={world} P={P} steps={steps} losses={losses} worst_frac={worst:.2e}", flush=True)
    dist.barrier()
    tr.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
