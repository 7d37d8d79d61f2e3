"""Cost and payoff of depth-guided seeding: python tools/seed_bench.py [--reps 20] [--steps 300]

Cost: psb_seed_plan + psb_seed_apply (CUDA events around both, the plan's host read-back included; median over --reps after a warm-up) at
1200x680 with stride 1, 2 and 4, on a 500 k-row model whose rendered planes and a synthetic sensor depth select every grid pixel (the
most rows one call can add), next to one fused step (trainForOneIteration) on the same model. Payoff: the experiment of
tests/test_seed_gpu.py (payoff() below): the scene of tests/test_quality_gpu.py (200 k rows, 6 keyframes at 640x480), a trainee that
lacks every row in a box the keyframes see, seeded once per keyframe or not, then 300 fused steps each; mean keyframe PSNR of both runs.
Prints one JSON object with the card's name and power limit. Writes nothing."""
import argparse
import ctypes as C
import json
import math

import numpy as np
import torch

import harness
import photo_slam_b200.synthetic as syn
from photo_slam_b200 import trainer

LRS = [0.00016, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
BOX = ((-0.6, 0.6), (-0.45, 0.45), (1.0, 4.0))   # world box (the scene lies in front of the identity view) the trainee lacks


def sensor_depth(tr, cam):
    """What an RGB-D sensor would see of tr's map from cam: the normalised depth D / A where A >= 0.5, else no measurement (0)."""
    H, W = cam["H"], cam["W"]
    A = torch.empty((H, W), device=tr.model.device)
    D = torch.empty((H, W), device=tr.model.device)
    img = tr.render(cam, out_depth=D, out_alpha=A).clamp(0, 1).clone()
    return img, torch.where(A >= 0.5, D / A.clamp_min(1e-12), torch.zeros_like(D)).contiguous(), A


def payoff(dev, seeded, steps=300, stride=2):
    """The scene of tests/test_quality_gpu.py, a trainee without the rows in BOX, optionally seeded once per keyframe, `steps` fused steps.
    -> dict(psnr_start, psnr (mean over the 6 keyframes after the steps), rows_removed, seeded (rows added), points)."""
    gt_scene, cams = syn.quality_scene()
    views = [syn.device_camera(cam, dev) for cam in cams]
    gt_tr = trainer.GaussianTrainer(trainer.GaussianModel.from_numpy(gt_scene, dev))
    frames = [sensor_depth(gt_tr, c)[:2] for c in views]
    x = gt_scene["xyz"]
    inside = np.ones(len(x), dtype=bool)
    for a, (lo, hi) in enumerate(BOX):
        inside &= (x[:, a] > lo) & (x[:, a] < hi)
    start = {k: v[~inside].copy() for k, v in gt_scene.items()}
    start["features_rest"] *= 0
    opt = trainer.GaussianOptimizationParams()
    model = trainer.GaussianModel.from_numpy(start, dev)
    model.trainingSetup(opt)
    model.lr_ = list(LRS)
    model.setShDegree(0)
    tr = trainer.GaussianTrainer(model, opt)

    def psnr():
        return float(np.mean([10.0 * math.log10(1.0 / ((tr.render(c) - g) ** 2).mean().item()) for c, (g, _) in zip(views, frames)]))

    p_start = psnr()
    added = 0
    if seeded:
        for c, (g, d) in zip(views, frames):
            added += tr.seedFromDepth(c, g, d, stride=stride)[0]
    for it in range(1, steps + 1):
        c, (g, _) = views[it % 6], frames[it % 6]
        tr.trainForOneIteration(c, g)
        tr.result()
    torch.cuda.synchronize()
    return dict(psnr_start=p_start, psnr=psnr(), rows_removed=int(inside.sum()), seeded=int(added), points=model.num_points())


def cost(dev, reps):
    sc, _, _, c, _ = harness.workload("B", dev)
    P, W, H = len(sc["xyz"]), c["W"], c["H"]
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    tr = trainer.GaussianTrainer(m)
    A = torch.empty((H, W), device=dev)
    D = torch.empty((H, W), device=dev)
    img = tr.render(c, out_depth=D, out_alpha=A).clamp(0, 1).clone()
    # nearer than the map where it is opaque (in front), some depth elsewhere (hole): every grid pixel is selected
    G = torch.where(A >= 0.5, 0.85 * D / A.clamp_min(1e-12), torch.full_like(D, 3.0)).contiguous()
    L = trainer._bind()
    stream = torch.cuda.current_stream().cuda_stream
    cc = trainer._ccamera(c)
    src = trainer._cmodel_of(**m._rows())
    out = {}
    for stride in (1, 2, 4):
        cfg = trainer._SeedCfg(0.5, 0.1, 0.2, 40.0, stride, 2 ** 31 - 1)
        ws = torch.empty(L.psb_seed_workspace_bytes(W, H, stride), dtype=torch.uint8, device=dev)
        counts = (C.c_int * 3)()
        trainer._lib.check(L.psb_seed_plan(C.byref(cc), A.data_ptr(), D.data_ptr(), G.data_ptr(), None, C.byref(cfg), ws.data_ptr(), counts, stream),
                           "psb_seed_plan")
        n = counts[0]
        d = m._blank(P + n)
        dst = trainer._cmodel_of(**d)

        def call():
            trainer._lib.check(L.psb_seed_plan(C.byref(cc), A.data_ptr(), D.data_ptr(), G.data_ptr(), None, C.byref(cfg), ws.data_ptr(), counts,
                                               stream), "psb_seed_plan")
            trainer._lib.check(L.psb_seed_apply(P, C.byref(src), C.byref(dst), n, C.byref(cc), img.data_ptr(), G.data_ptr(), C.byref(cfg),
                                                ws.data_ptr(), 0, stream), "psb_seed_apply")
        out[f"stride{stride}"] = dict(ms=harness.cuda_ms(call, reps, warmup=3), rows_added=n, holes=counts[1], in_front=counts[2])
        del d
    step = lambda: tr.trainForOneIteration(c, img)
    out["fused_step_ms"] = harness.cuda_ms(step, reps, warmup=5)
    out["P"] = P
    out["size"] = [W, H]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--steps", type=int, default=300)
    a = ap.parse_args()
    dev = harness.device()
    res = dict(card=harness.card(), cost=cost(dev, a.reps))
    base, seeded = payoff(dev, False, a.steps), payoff(dev, True, a.steps)
    res["payoff"] = dict(steps=a.steps, unseeded=base, seeded=seeded, gain_db=seeded["psnr"] - base["psnr"])
    print(json.dumps(res))


if __name__ == "__main__":
    main()
