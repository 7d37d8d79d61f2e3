"""Worker of tests/test_dp_terms_gpu.py (one process per GPU, launched with torch.distributed.run; or K processes on one GPU, launched
by tests/shared_device.py, p2p only): K data-parallel steps through
DataParallelTrainer(mode=..., geometry_terms=True) on world ranks, rank r training with the terms TERMS[r % 4] (normal + consistency,
distortion, none, all of depth, normal, consistency and distortion), then
  (1) every rank's parameter replica, and the Adam moments gathered from their owners, must be BIT-identical,
  (2) they must equal the 1-rank step on the summed gradients of the same K views: rank 0 recomputes every view's dense gradient with
      psb_trainer_backward_dist and that view's terms, sums them and applies psb_adam_update(grad_scale = 1/world).
Prints one line `DP_TERMS_WORKER_OK ...` from rank 0 on success; any assertion fails the launch."""
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
LAMBDA_DEPTH, LAMBDA_NORMAL, LAMBDA_DN, LAMBDA_DIST = 0.1, 0.05, 0.05, 0.1
ALPHA_MIN, JUMP = 0.5, 0.05
TERMS = ("normal_dn", "dist", "plain", "all")


def view(rank, sc, W, H, fx, fy, dev):
    """dp_depth_worker.py's view of this rank with a depth target for every rank, a normal target (the sensor normals of that depth
    without its holes) and the name of this rank's terms"""
    R, t = syn.random_pose(np.random.default_rng(100 + rank), max_angle=0.08, max_trans=0.15)
    cam = syn.make_camera(W, H, fx, fy, R, t)
    c = syn.device_camera(cam, dev)
    gt = torch.from_numpy(syn.target_image(H, W, seed=7 + rank)).to(dev)
    V = cam["viewmatrix"].reshape(-1)
    z = sc["xyz"] @ V[[2, 6, 10]] + V[14]
    zs = np.quantile(z[z > 0.2], [0.1, 0.9])
    gen = torch.Generator().manual_seed(300 + rank)
    smooth = torch.linspace(float(zs[0]), float(zs[1]), W)[None, :].expand(H, W).contiguous().to(dev)
    gn = trainer.normals_from_depth(c, smooth, JUMP)
    depth = (zs[0] + (zs[1] - zs[0]) * torch.rand((H, W), generator=gen)).float()
    depth[torch.rand((H, W), generator=gen) < 0.1] = 0.0
    return c, gt, depth.contiguous().to(dev), gn.contiguous(), TERMS[rank % len(TERMS)]


def kwargs(name, gd, gn):
    n = dict(gt_normal=gn, lambda_normal=LAMBDA_NORMAL)
    dn = dict(lambda_dn=LAMBDA_DN, dn_alpha_min=ALPHA_MIN, dn_max_rel_jump=JUMP)
    return {"plain": {}, "normal_dn": dict(n, **dn), "dist": dict(lambda_dist=LAMBDA_DIST),
            "all": dict(n, **dn, gt_depth=gd, lambda_depth=LAMBDA_DEPTH, lambda_dist=LAMBDA_DIST)}[name]


def records(name, gd, gn):
    """the C records of kwargs(name): (depth, normal, dn, dist), None for a term the view does not have"""
    kw = kwargs(name, gd, gn)
    depth = trainer._Depth(gd.data_ptr(), LAMBDA_DEPTH, None) if "gt_depth" in kw else None
    normal = trainer._Normal(gn.data_ptr(), LAMBDA_NORMAL, None) if "gt_normal" in kw else None
    dn = trainer._Dn(LAMBDA_DN, ALPHA_MIN, JUMP, None) if "lambda_dn" in kw else None
    ds = trainer._Dist(LAMBDA_DIST, None) if "lambda_dist" in kw else None
    return depth, normal, dn, ds


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
    tr = trainer.DataParallelTrainer(model, mode=mode, geometry_terms=True)
    assert tr.mode == mode, f"requested {mode}, running {tr.mode}: {getattr(tr, '_p2p_error', '')}"
    assert mode == "p2p" or tr.pipeline, "the nccl mode must run the slab pipeline at world > 1"
    c, gt, gd, gn, name = view(rank, sc, W, H, fx, fy, dev)
    losses = []
    for _ in range(steps):
        tr.trainForOneIteration(c, gt, **kwargs(name, gd, gn))
        r = tr.result_dist()
        assert (r[4] > 0.0) == (name in ("normal_dn", "all")) and (r[6] > 0.0) == (name in ("dist", "all")), (name, r)
        losses.append(r[0])
    tr.sync()
    torch.cuda.synchronize()
    dist.barrier()
    assert tr.status() == 0, "a cross-rank wait timed out"
    tr.gather_moments()
    torch.cuda.synchronize()
    # (1) bit-identical replicas and moments
    for gname, t in zip(trainer.GROUPS, model.tensors()):
        ref0 = t.clone()
        dist.broadcast(ref0, src=0)
        assert torch.equal(ref0, t), f"rank {rank}: replica of {gname} differs from rank 0"
    for t in model.exp_avg_ + model.exp_avg_sq_:
        ref0 = t.clone()
        dist.broadcast(ref0, src=0)
        assert torch.equal(ref0, t), f"rank {rank}: gathered moments differ from rank 0"
    # (2) vs the 1-rank step on the summed gradients
    if rank == 0:
        ref = trainer.GaussianModel.from_numpy(sc, dev)
        ref.trainingSetup(trainer.GaussianOptimizationParams())
        rt = trainer.DataParallelTrainer(ref, mode="nccl", pipeline=False)   # world-agnostic use of backward / adam_update below
        from photo_slam_b200.parallel import GradBuffer
        views = [view(r, sc, W, H, fx, fy, dev) for r in range(world)]
        total = GradBuffer(P, dev)
        stream = torch.cuda.current_stream().cuda_stream
        byref = lambda x: C.byref(x) if x is not None else None
        for _ in range(steps):
            total.flat.zero_()
            cm, cs = ref._cmodel(), rt._cstep(True)
            for (cc_, gt_, gd_, gn_, name_) in views:
                ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in rt.segs])
                cc = trainer._ccamera(cc_)
                depth, normal, dn, ds = records(name_, gd_, gn_)
                _lib.check(rt.L.psb_trainer_backward_dist(rt.h, P, 16, C.byref(cm), C.byref(cc), rt.background.data_ptr(), gt_.data_ptr(), None,
                                                          C.byref(cs), None, None, ptrs, byref(depth), None, None, byref(normal), byref(dn),
                                                          byref(ds), stream), "psb_trainer_backward_dist")
                total.flat += rt.flat
            ptrs = (C.c_void_p * 6)(*[s.data_ptr() for s in total.segments])
            _lib.check(rt.L.psb_adam_update(P, 16, C.byref(cm), ptrs, C.byref(cs), 1.0 / world, stream), "psb_adam_update")
            ref.step_ += 1
        torch.cuda.synchronize()
        worst = 0.0
        for gname, a, b, lr in zip(trainer.GROUPS, model.tensors(), ref.tensors(), LRS):
            frac = ((a - b).abs() > 0.5 * lr).float().mean().item()
            worst = max(worst, frac)
            assert frac < 2e-3, f"{gname}: {frac} of the entries differ from the summed-gradient step by more than half an Adam step"
        for gname, a, b in zip(trainer.GROUPS, model.exp_avg_, ref.exp_avg_):
            rn = ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()
            assert rn < 1e-4, f"exp_avg {gname}: rel-norm {rn}"
        for gname, a, b in zip(trainer.GROUPS, model.exp_avg_sq_, ref.exp_avg_sq_):
            rn = ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()
            assert rn < 1e-4, f"exp_avg_sq {gname}: rel-norm {rn}"
        print(f"DP_TERMS_WORKER_OK mode={mode} world={world} P={P} steps={steps} terms={[TERMS[r % len(TERMS)] for r in range(world)]} "
              f"losses={losses} worst_frac={worst:.2e}", flush=True)
    dist.barrier()
    tr.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
