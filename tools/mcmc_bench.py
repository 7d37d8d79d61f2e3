"""Cost of bounded-budget densification (3DGS-MCMC): python tools/mcmc_bench.py [--configs B D] [--steps 30] [--quality-steps 600]

Step: at each config the fused step runs with opt.mcmc off and on (regularisers in the per-Gaussian stage + the position-noise kernel behind
the step), legs alternating in one process and each starting from the same model snapshot; it reports it/s, the per-stage times
(psb_trainer_stage_times) and the noise kernel's time (CUDA events around 20 launches) with the bytes it moves (56 B per visible row).
Refinement: relocateGaussians and addNewGaussians on the largest config with 5 % dead rows, and densifyAndPrune on the same model for scale
(CUDA events, the host round trip of each included).
Quality (--quality-steps > 0): the scene of tests/test_quality_gpu.py (200 k rows, 640x480, 6 keyframes) trained with the default
densification and under a cap of 400 k with mcmcRefine every 100 steps: PSNR and row count every 100 steps.
Prints one JSON object. Writes nothing."""
import argparse
import json
import math

import numpy as np
import torch

import harness
import photo_slam_b200.synthetic as syn
from photo_slam_b200 import trainer


def step_cost(dev, config, steps, warmup, rounds):
    sc, _, _, c, gt = harness.workload(config, dev)
    P = len(sc["xyz"])
    m = trainer.GaussianModel.from_numpy(sc, dev)
    opts = {"off": trainer.GaussianOptimizationParams(), "on": trainer.GaussianOptimizationParams(mcmc=True, cap_max=P)}
    m.trainingSetup(opts["off"])
    trs = {k: trainer.GaussianTrainer(m, o) for k, o in opts.items()}
    rewind = harness.rewinder(m, *trs.values())   # every leg starts from the untrained model: the warm-up grows the arenas
    for _ in range(warmup):
        for tr in trs.values():
            tr.trainForOneIteration(c, gt)
            tr.result()
    res = harness.alternate({k: (lambda tr=tr: harness.step_leg(tr, c, gt, steps, rewind)) for k, tr in trs.items()}, rounds, rewind)
    rewind()
    out = {k: {"it_s": [round(x[0], 1) for x in legs], "stage_ms": {s: round(v, 4) for s, v in harness.mean_stages([x[1] for x in legs]).items()}}
           for k, legs in res.items()}
    # the noise kernel alone, behind a pass of the mcmc trainer, on the model as one "on" leg leaves it (its warm-up, timed and 5
    # profiled steps); refine_cost then works on that model
    tr = trs["on"]
    for _ in range(warmup + steps + 5):
        tr.trainForOneIteration(c, gt)
    tr.result()
    radii = torch.zeros(P, dtype=torch.int32, device=dev)
    tr.trainForOneIteration(c, gt, radii=radii)
    tr.result()
    ms = harness.window_ms(tr._inject_noise, 20)     # back to back: one launch is shorter than its host side
    visible = int((radii > 0).sum())
    out["noise_kernel"] = {"ms": round(ms, 4), "rows": P, "visible_rows": visible, "bytes": 16 * P + 56 * visible,
                           "GB_s": round((16 * P + 56 * visible) / ms / 1e6, 1)}
    return out, m


def refine_cost(dev, m, rounds=3):
    P = m.num_points()
    dead = torch.rand(P, device=dev, generator=torch.Generator(device=dev).manual_seed(1)) < 0.05
    m.opacity_[dead] = -8.0
    m.xyz_gradient_accum_.copy_(torch.rand((P, 1), device=dev) * 0.004)
    m.denom_.fill_(2.0)
    snap = m.snapshot()
    out = {"rows": P, "dead_rows": int(dead.sum()), "relocate_ms": [], "grow_ms": [], "densify_and_prune_ms": []}
    for _ in range(rounds):
        m.restore(snap)
        out["relocate_ms"].append(round(harness.window_ms(lambda: m.relocateGaussians(0.005, seed=1), 1), 3))
    keep = {k: [t.clone() for t in snap[k]] for k in ("p", "stats")}
    for fn, key in ((lambda mm: mm.addNewGaussians(2 * P, 1.05, seed=1), "grow_ms"),
                    (lambda mm: mm.densifyAndPrune(0.0019, 0.005, 5.0, 0, seed=1), "densify_and_prune_ms")):
        for _ in range(rounds):
            mm = trainer.GaussianModel(device=dev)
            mm._set([t.clone() for t in keep["p"]])
            mm.trainingSetup(trainer.GaussianOptimizationParams())
            mm.xyz_gradient_accum_, mm.denom_ = keep["stats"][0].clone(), keep["stats"][1].clone()
            out[key].append(round(harness.window_ms(lambda: fn(mm), 1), 3))
            out[key + "_rows_after"] = mm.num_points()
            del mm
    return out


def quality(dev, steps, cap=400_000):
    gt_scene, cams = syn.quality_scene()
    views = [syn.device_camera(cam, dev) for cam in cams]
    gt_tr = trainer.GaussianTrainer(trainer.GaussianModel.from_numpy(gt_scene, dev))
    gts = [gt_tr.render(c).clamp(0, 1).clone() for c in views]
    start = syn.thinned_trainee(gt_scene)
    out = {}
    for mcmc in (False, True):
        opt = trainer.GaussianOptimizationParams(mcmc=mcmc, cap_max=cap, mcmc_grow_factor=1.2)
        m = trainer.GaussianModel.from_numpy(start, dev)
        m.trainingSetup(opt)
        m.lr_ = [0.00016, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]
        tr = trainer.GaussianTrainer(m, opt)
        psnr = lambda: float(np.mean([10.0 * math.log10(1.0 / ((tr.render(c) - g) ** 2).mean().item()) for c, g in zip(views, gts)]))
        log = [(0, round(psnr(), 3), m.num_points())]
        for it in range(1, steps + 1):
            tr.trainForOneIteration(views[it % 6], gts[it % 6])
            tr.result()
            if it % 100 == 0:
                if it < steps:
                    if mcmc:
                        tr.mcmcRefine()
                    else:
                        grads = (m.xyz_gradient_accum_ / m.denom_).nan_to_num(0.0).squeeze()
                        m.densifyAndPrune(float(torch.quantile(grads[grads > 0][:1_000_000], 0.95)), 0.005, 1.0, 20, seed=5)
                log.append((it, round(psnr(), 3), m.num_points()))
        out["capped" if mcmc else "default"] = log
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="*", default=["B", "D"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--quality-steps", type=int, default=600)
    a = ap.parse_args()
    dev = harness.device()
    res = {"card": harness.card(), "step": {}}
    m = None
    for cfg in a.configs:
        res["step"][cfg], m = step_cost(dev, cfg, a.steps, a.warmup, a.rounds)
    if m is not None:
        res["refine"] = refine_cost(dev, m)
        del m
    if a.quality_steps > 0:
        res["quality"] = quality(dev, a.quality_steps)
    print(json.dumps(res))
