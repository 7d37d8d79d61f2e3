"""Worker of tests/test_deterministic_gpu.py (one process per GPU, launched with torch.distributed.run): K NVLink data-parallel
steps (DataParallelTrainer(mode="p2p", deterministic=True); even ranks with a depth target, odd ranks without), then every rank's
parameter replica must be BIT-identical to rank 0's. Rank 0 prints `DP_DET_WORKER_OK ... digest=<sha1>` of the replica and the
step losses, which the test compares across two launches."""
import hashlib
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import photo_slam_b200.synthetic as syn  # noqa: E402
from photo_slam_b200 import trainer  # noqa: E402


def main():
    P = int(sys.argv[1]) if len(sys.argv) > 1 else 30_001
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 4
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    W, H, fx, fy = 320, 240, 260.0, 260.0
    sc = syn.make_scene(P, syn.make_camera(W, H, fx, fy), seed=11, scale_px=6.0)
    model = trainer.GaussianModel.from_numpy(sc, dev)
    model.trainingSetup(trainer.GaussianOptimizationParams())
    tr = trainer.DataParallelTrainer(model, mode="p2p", deterministic=True)
    assert tr.mode == "p2p", getattr(tr, "_p2p_error", "")
    R, t = syn.random_pose(np.random.default_rng(100 + rank), max_angle=0.08, max_trans=0.15)
    cam = syn.make_camera(W, H, fx, fy, R, t)
    c = syn.device_camera(cam, dev)
    gt = torch.from_numpy(syn.target_image(H, W, seed=7 + rank)).to(dev)
    gd = (1.0 + 6.0 * torch.rand((H, W), generator=torch.Generator().manual_seed(rank))).to(dev)
    tr.render(c)        # grows the binning arena: no step is a dropped view
    losses = []
    for _ in range(steps):
        kw = dict(gt_depth=gd, lambda_depth=0.1) if rank % 2 == 0 else {}
        tr.trainForOneIteration(c, gt, **kw)
        losses.append(tr.result()[0])
    tr.sync()
    torch.cuda.synchronize()
    dist.barrier()
    assert tr.status() == 0, "a cross-rank wait timed out"
    h = hashlib.sha1()
    for name, p in zip(trainer.GROUPS, model.tensors()):
        ref0 = p.clone()
        dist.broadcast(ref0, src=0)
        assert torch.equal(ref0, p), f"rank {rank}: replica of {name} differs from rank 0"
        h.update(p.cpu().numpy().tobytes())
    all_losses = [None] * world
    dist.all_gather_object(all_losses, losses)
    h.update(repr(all_losses).encode())
    if rank == 0:
        print(f"DP_DET_WORKER_OK world={world} P={P} steps={steps} digest={h.hexdigest()} losses={all_losses}", flush=True)
    dist.barrier()
    tr.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
