"""Cost and evidence of the 3D smoothing filter (Mip-Splatting): python tools/filter3d_bench.py [--configs B D] [--steps 30]

Cost: psb_filter3d at P = 500 k / 3 M rows and K = 100 / 300 / 1000 cameras (CUDA events, median of 5 after a warm-up); at each config the
fused step with the filter off and on, legs alternating in one process and each starting from the same model snapshot: it/s, the per-stage
times (psb_trainer_stage_times) and the instance count. Evidence (the zoom-in case the filter is for): a seeded synthetic target scene is
rendered at 1200x680 from 8 poses; models are trained with anti-aliasing on the 2x2 area-averaged 600x340 views, without and with the
filter (recomputed from the 8 full-resolution cameras every 100 steps and after each densification), and rendered at 600x340 and at 1200x680
against the targets (PSNR). Prints one JSON object with the card's name and power limit. Writes nothing."""
import argparse
import json

import numpy as np
import torch

import harness
import photo_slam_b200.synthetic as syn
from photo_slam_b200 import _lib, trainer


def _views(dev, K, W, H, f, seed=0):
    rng = np.random.default_rng(seed)
    return [syn.device_camera(syn.make_camera(W, H, f, f, *syn.random_pose(rng, max_angle=0.3, max_trans=0.5)), dev) for _ in range(K)]


def filter_cost(dev):
    out = {}
    L = trainer._bind()
    for config in ("B", "D"):
        sc, _, _, c, _ = harness.workload(config, dev)
        P, (W, H, fx, _) = len(sc["xyz"]), syn.CAMERAS[harness.CONFIGS[config][1]]
        m = trainer.GaussianModel.from_numpy(sc, dev)
        f = torch.empty(P, device=dev)
        for K in (100, 300, 1000):
            views = _views(dev, K, W, H, fx)
            m.computeFilter3D(views)   # (packs the cameras; the timed calls below reuse the packed array)
            packed = torch.tensor(np.stack([np.concatenate([v["viewmatrix"].cpu().numpy().reshape(-1), [W / (2 * v["tanfovx"]), H / (2 * v["tanfovy"]), W, H]])
                                            for v in views]), dtype=torch.float32, device=dev)
            s = torch.cuda.current_stream()
            call = lambda: _lib.check(L.psb_filter3d(P, m.xyz_.data_ptr(), K, packed.data_ptr(), f.data_ptr(), None, s.cuda_stream), "psb_filter3d")
            times = [harness.window_ms(call, 1) for _ in range(7)][2:]      # each call from an idle device, after 2 warm-up calls
            out[f"P={P},K={K}"] = {"ms": round(float(np.median(times)), 3), "rows_seen": m.computeFilter3D(views)}
    return out


def step_cost(dev, config, steps, warmup, rounds):
    sc, _, _, c, gt = harness.workload(config, dev)
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    W, H, fx, _ = syn.CAMERAS[harness.CONFIGS[config][1]]
    m.computeFilter3D([c] + _views(dev, 31, W, H, fx))
    trs = {"off": trainer.GaussianTrainer(m, filter3d=False), "on": trainer.GaussianTrainer(m, filter3d=True)}
    rewind = harness.rewinder(m, *trs.values())   # every leg starts from the untrained model: the warm-up grows the arenas
    for _ in range(warmup):
        for tr in trs.values():
            tr.trainForOneIteration(c, gt)
            tr.result()
    res = harness.alternate({k: (lambda tr=tr: harness.step_leg(tr, c, gt, steps, rewind)) for k, tr in trs.items()}, rounds, rewind)
    instances = {}
    for k, tr in trs.items():      # read after as many steps as a leg used to take: its warm-up, timed and 5 profiled steps
        rewind()
        for _ in range(warmup + steps + 5):
            tr.trainForOneIteration(c, gt)
        instances[k] = int(tr.result()[3])
    rewind()
    return {k: {"it_s": [round(x[0], 1) for x in legs], "stage_ms": {s: round(v, 3) for s, v in harness.mean_stages([x[1] for x in legs]).items()},
                "instances": instances[k]} for k, legs in res.items()}


def _psnr(a, b):
    return 10 * np.log10(1.0 / max(((a - b) ** 2).mean().item(), 1e-12))


def evidence(dev, steps=600):
    Wf, Hf, ff = 1200, 680, 600.0
    rng = np.random.default_rng(1)
    poses = [syn.random_pose(rng, max_angle=0.1, max_trans=0.1) for _ in range(8)]
    full = [(cam, syn.device_camera(cam, dev)) for cam in (syn.make_camera(Wf, Hf, ff, ff, *p) for p in poses)]
    half = [syn.device_camera(syn.make_camera(Wf // 2, Hf // 2, ff / 2, ff / 2, *p), dev) for p in poses]
    target = trainer.GaussianModel.from_numpy(syn.make_scene(100_000, full[0][0], seed=11, scale_px=1.5), dev)
    gts_full = [trainer.GaussianTrainer(target, antialiasing=True).render(c) for _, c in full]
    gts_half = [torch.nn.functional.avg_pool2d(g[None], 2)[0].contiguous() for g in gts_full]
    out = {}
    for on in (False, True):
        m = trainer.GaussianModel.from_numpy(syn.make_scene(100_000, full[0][0], seed=12, scale_px=1.5), dev)
        opt = trainer.GaussianOptimizationParams()
        m.trainingSetup(opt)
        tr = trainer.GaussianTrainer(m, opt, antialiasing=True, filter3d=on)
        refresh = lambda: m.computeFilter3D([c for _, c in full])
        if on:
            refresh()
        for it in range(1, steps + 1):
            k = it % len(poses)
            tr.trainForOneIteration(half[k], gts_half[k])
            tr.result()
            densify = it % 200 == 0 and it < steps
            if densify:
                m.densifyAndPrune(opt.densify_grad_threshold, 0.005, 2.0, 0)
            if on and (densify or it % 100 == 0):
                refresh()
        out["filter" if on else "plain"] = {
            "rows": m.num_points(),
            "psnr_600x340": round(float(np.mean([_psnr(tr.render(c), g) for c, g in zip(half, gts_half)])), 3),
            "psnr_1200x680": round(float(np.mean([_psnr(tr.render(c), g) for (_, c), g in zip(full, gts_full)])), 3)}
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="*", default=["B", "D"])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--evidence-steps", type=int, default=600)
    a = ap.parse_args()
    dev = harness.device()
    res = {"card": harness.card(), "filter3d": filter_cost(dev), "step": {cfg: step_cost(dev, cfg, a.steps, a.warmup, a.rounds) for cfg in a.configs}}
    if a.evidence_steps > 0:
        res["evidence"] = evidence(dev, a.evidence_steps)
    print(json.dumps(res))
