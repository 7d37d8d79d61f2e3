"""Cost and evidence of the 3D smoothing filter (Mip-Splatting): python tools/filter3d_bench.py [--configs B D] [--steps 30]

Cost: psb_filter3d at P = 500 k / 3 M rows and K = 100 / 300 / 1000 cameras (CUDA events, median of 5 after a warm-up); at each config the
fused step with the filter off and on, legs alternating in one process and each starting from the same model snapshot: it/s, the per-stage
times (psb_trainer_stage_times) and the instance count. Evidence (the zoom-in case the filter is for): a seeded synthetic target scene is
rendered at 1200x680 from 8 poses; models are trained with anti-aliasing on the 2x2 area-averaged 600x340 views, without and with the
filter (recomputed from the 8 full-resolution cameras every 100 steps and after each densification), and rendered at 600x340 and at 1200x680
against the targets (PSNR). Prints one JSON object with the card's name and power limit. Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import photo_slam_b200.synthetic as syn  # noqa: E402
from photo_slam_b200 import _lib, trainer  # noqa: E402

CONFIGS = {"B": (500_000, "replica"), "D": (3_000_000, "replica")}


def _cam(dev, W, H, fx, fy, pose=None):
    cam = syn.make_camera(W, H, fx, fy, *(pose or (None, None)))
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return cam, dict(viewmatrix=T(cam["viewmatrix"]), projmatrix=T(cam["projmatrix"]), campos=T(cam["campos"]), tanfovx=float(cam["tanfovx"]),
                     tanfovy=float(cam["tanfovy"]), W=W, H=H)


def _views(dev, K, W, H, f, seed=0):
    rng = np.random.default_rng(seed)
    return [_cam(dev, W, H, f, f, syn.random_pose(rng, max_angle=0.3, max_trans=0.5))[1] for _ in range(K)]


def filter_cost(dev):
    out = {}
    L = trainer._bind()
    for P, camname in ((500_000, "replica"), (3_000_000, "replica")):
        W, H, fx, fy = syn.CAMERAS[camname]
        cam, c = _cam(dev, W, H, fx, fy)
        m = trainer.GaussianModel.from_numpy(syn.make_scene(P, cam, seed=0), dev)
        f = torch.empty(P, device=dev)
        for K in (100, 300, 1000):
            views = _views(dev, K, W, H, fx)
            m.computeFilter3D(views)   # (packs the cameras; the timed calls below reuse the packed array)
            packed = torch.tensor(np.stack([np.concatenate([v["viewmatrix"].cpu().numpy().reshape(-1), [W / (2 * v["tanfovx"]), H / (2 * v["tanfovy"]), W, H]])
                                            for v in views]), dtype=torch.float32, device=dev)
            s = torch.cuda.current_stream()
            times = []
            for i in range(7):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(s)
                _lib.check(L.psb_filter3d(P, m.xyz_.data_ptr(), K, packed.data_ptr(), f.data_ptr(), None, s.cuda_stream), "psb_filter3d")
                e1.record(s)
                e1.synchronize()
                if i >= 2:
                    times.append(e0.elapsed_time(e1))
            out[f"P={P},K={K}"] = {"ms": round(float(np.median(times)), 3), "rows_seen": m.computeFilter3D(views)}
    return out


def _leg(sc, c, gt, dev, views, on, steps, warmup):
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    if on:
        m.computeFilter3D(views)
    tr = trainer.GaussianTrainer(m, filter3d=on)
    tr.render(c)
    for _ in range(warmup):
        tr.trainForOneIteration(c, gt)
        tr.result()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        tr.trainForOneIteration(c, gt)
    tr.result()
    torch.cuda.synchronize()
    its = steps / (time.perf_counter() - t0)
    tr.set_profiling(True)
    st = {}
    for _ in range(5):
        tr.trainForOneIteration(c, gt)
        tr.result()
        for k, v in tr.stage_times().items():
            st[k] = st.get(k, 0.0) + v / 5
    return its, st, int(tr.result()[3])


def step_cost(dev, config, steps, warmup, rounds):
    P, camname = CONFIGS[config]
    W, H, fx, fy = syn.CAMERAS[camname]
    cam, c = _cam(dev, W, H, fx, fy)
    sc = syn.make_scene(P, cam, seed=0)
    gt = torch.from_numpy(syn.target_image(H, W)).to(dev)
    views = [c] + _views(dev, 31, W, H, fx)
    res = {"off": [], "on": []}
    for _ in range(rounds):
        for on in (False, True):
            res["on" if on else "off"].append(_leg(sc, c, gt, dev, views, on, steps, warmup))
    out = {}
    for k, legs in res.items():
        out[k] = {"it_s": [round(x[0], 1) for x in legs], "stage_ms": {s: round(float(np.mean([x[1][s] for x in legs])), 3) for s in legs[0][1]},
                  "instances": legs[-1][2]}
    return out


def _psnr(a, b):
    return 10 * np.log10(1.0 / max(((a - b) ** 2).mean().item(), 1e-12))


def evidence(dev, steps=600):
    Wf, Hf, ff = 1200, 680, 600.0
    rng = np.random.default_rng(1)
    poses = [syn.random_pose(rng, max_angle=0.1, max_trans=0.1) for _ in range(8)]
    full = [_cam(dev, Wf, Hf, ff, ff, p) for p in poses]
    half = [_cam(dev, Wf // 2, Hf // 2, ff / 2, ff / 2, p)[1] for p in poses]
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
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    res = {"gpu": torch.cuda.get_device_name(dev), "nvidia_smi": q.stdout.strip(), "filter3d": filter_cost(dev),
           "step": {cfg: step_cost(dev, cfg, a.steps, a.warmup, a.rounds) for cfg in a.configs}}
    if a.evidence_steps > 0:
        res["evidence"] = evidence(dev, a.evidence_steps)
    print(json.dumps(res))
