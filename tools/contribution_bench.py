"""Cost and payoff of contribution pruning: python tools/contribution_bench.py [--configs B D] [--reps 20]

Cost: one score pass (psb_trainer_contribution) against one render (psb_trainer_render) of the same view at each config, legs alternating
in one process on the same model (CUDA events, median over --reps after a warm-up), with the instance count; a sweep over K = 32 and 128
keyframes at the last config (contributionScores: one host round trip). Payoff: the scene of tests/test_quality_gpu.py (200 k rows, 6
keyframes at 640x480), trained for 600 fused steps, then pruned at several thresholds from the same snapshot: rows removed, mean keyframe
PSNR right after the prune and after 100 more steps, and the fused step's it/s before and after. Prints one JSON object with the card's name
and power limit. Writes nothing."""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import photo_slam_b200.synthetic as syn  # noqa: E402
from photo_slam_b200 import trainer  # noqa: E402

CONFIGS = {"B": (500_000, "replica"), "D": (3_000_000, "replica")}
LRS = [0.00016, 0.0025, 0.0025 / 20, 0.05, 0.005, 0.001]


def _dev_cam(cam, dev):
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return dict(viewmatrix=T(cam["viewmatrix"]), projmatrix=T(cam["projmatrix"]), campos=T(cam["campos"]), tanfovx=float(cam["tanfovx"]),
                tanfovy=float(cam["tanfovy"]), W=int(cam["W"]), H=int(cam["H"]))


def _views(dev, K, W, H, fx, fy, seed, angle=0.3, trans=0.5):
    rng = np.random.default_rng(seed)
    return [_dev_cam(syn.make_camera(W, H, fx, fy, *syn.random_pose(rng, max_angle=angle, max_trans=trans)), dev) for _ in range(K)]


def _time(fn, reps):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def pass_cost(dev, configs, reps):
    out = {}
    for name in configs:
        P, camname = CONFIGS[name]
        W, H, fx, fy = syn.CAMERAS[camname]
        cam = syn.make_camera(W, H, fx, fy)
        m = trainer.GaussianModel.from_numpy(syn.make_scene(P, cam, seed=0), dev)
        tr = trainer.GaussianTrainer(m)
        c = _dev_cam(cam, dev)
        img = torch.empty((3, H, W), device=dev)
        mx = torch.zeros(m.num_points(), dtype=torch.int32, device=dev)
        sm = torch.zeros(m.num_points(), dtype=torch.int64, device=dev)
        import ctypes as C
        cm, cc = m._cmodel(False), trainer._ccamera(c)
        stream = torch.cuda.current_stream().cuda_stream

        def render():
            tr.L.psb_trainer_render(tr.h, m.num_points(), 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), m.active_sh_degree_,
                                    img.data_ptr(), None, stream)

        def score():
            tr.L.psb_trainer_contribution(tr.h, m.num_points(), 16, C.byref(cm), C.byref(cc), tr.background.data_ptr(), m.active_sh_degree_,
                                          mx.data_ptr(), sm.data_ptr(), img.data_ptr(), stream)
        tr.render(c)
        n = tr.result()[3]
        for f in (render, score):
            _time(f, 3)
        legs = {"render": [], "score": []}
        for _ in range(4):                       # alternate the legs
            legs["render"].append(_time(render, reps))
            legs["score"].append(_time(score, reps))
        assert tr.result()[3] == n
        r, s = float(np.median(legs["render"])), float(np.median(legs["score"]))
        out[name] = dict(P=P, W=W, H=H, instances=n, render_ms=round(r, 4), score_ms=round(s, 4), overhead=round(s / r - 1.0, 4))
    return out


def sweep_cost(dev, name, Ks):
    P, camname = CONFIGS[name]
    W, H, fx, fy = syn.CAMERAS[camname]
    cam = syn.make_camera(W, H, fx, fy)
    m = trainer.GaussianModel.from_numpy(syn.make_scene(P, cam, seed=0), dev)
    tr = trainer.GaussianTrainer(m)
    out = {}
    for K in Ks:
        views = _views(dev, K, W, H, fx, fy, seed=K, angle=0.05, trans=0.05)
        tr.contributionScores(views)           # warm-up, grows the arena
        times = []
        for _ in range(3):
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            mx, _ = tr.contributionScores(views)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        out[f"K{K}"] = dict(config=name, ms=round(float(np.median(times)), 3), per_view_ms=round(float(np.median(times)) / K, 4),
                            rows_scored=int((mx > 0).sum()), P=P)
    return out


def payoff(dev, thresholds, steps=600, more=100):
    """the scene and trainee of tests/test_quality_gpu.py, trained without densification (the SH degree rises every 200 steps)"""
    P, W, H, fx = 200_000, 640, 480, 520.9
    cam0 = syn.make_camera(W, H, fx, fx)
    gt_scene = syn.make_scene(P, cam0, seed=21, scale_px=3.0)
    views = []
    for k in range(6):
        R, t = syn.random_pose(np.random.default_rng(50 + k), max_angle=0.06, max_trans=0.12)
        views.append(_dev_cam(syn.make_camera(W, H, fx, fx, R, t), dev))
    gt_tr = trainer.GaussianTrainer(trainer.GaussianModel.from_numpy(gt_scene, dev))
    gts = [gt_tr.render(c).clamp(0, 1).clone() for c in views]
    rng = np.random.default_rng(3)
    keep = rng.random(P) < 0.8
    start = {k: v[keep].copy() for k, v in gt_scene.items()}
    start["xyz"] += rng.normal(0, 0.01, start["xyz"].shape).astype(np.float32)
    start["features_dc"] += rng.normal(0, 0.6, start["features_dc"].shape).astype(np.float32)
    start["features_rest"] *= 0
    start["opacity"] += rng.normal(0, 0.7, start["opacity"].shape).astype(np.float32)
    start["scaling"] += np.float32(0.15)
    opt = trainer.GaussianOptimizationParams()
    m = trainer.GaussianModel.from_numpy(start, dev)
    m.trainingSetup(opt)
    m.lr_ = list(LRS)
    m.setShDegree(0)
    tr = trainer.GaussianTrainer(m, opt)

    def train(n, it0=0):
        for it in range(n):
            if (it0 + it) % 200 == 0 and it0 + it > 0:
                m.oneUpShDegree()
            k = (it0 + it) % len(views)
            tr.trainForOneIteration(views[k], gts[k], densify_stats=False)
            tr.result()

    def psnr():
        return float(np.mean([10.0 * math.log10(1.0 / ((tr.render(c) - g) ** 2).mean().item()) for c, g in zip(views, gts)]))

    def its(n=60):
        train(5, steps)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for it in range(n):
            k = it % len(views)
            tr.trainForOneIteration(views[k], gts[k], densify_stats=False)
        b.record()
        torch.cuda.synchronize()
        tr.result()
        return n * 1000.0 / a.elapsed_time(b)

    train(steps)
    copy = lambda d: {k: [t.clone() for t in v] if isinstance(v, list) else v.clone() for k, v in d.items()}
    saved, step, sh = copy(m._rows()), m.step_, m.active_sh_degree_
    out = dict(rows=m.num_points(), psnr_trained=round(psnr(), 3), rows_unseen=None, legs=[])
    mx, _ = tr.contributionScores(views)
    out["rows_unseen"] = int((mx == 0).sum())
    base = None
    for th in [None] + list(thresholds):
        m._adopt(copy(saved))             # every leg starts from the same trained rows
        m.step_, m.active_sh_degree_, tr.iteration = step, sh, steps
        removed = tr.pruneByContribution(views, th) if th is not None else 0
        after = psnr()
        train(more, steps)
        later = psnr()
        rate = its()
        leg = dict(min_weight=th, removed=removed, rows=m.num_points(), psnr_after=round(after, 3),
                   psnr_after_100=round(later, 3), it_s=round(rate, 1))
        if th is None:
            base = leg
        out["legs"].append(leg)
    for leg in out["legs"]:
        leg["it_s_vs_unpruned"] = round(leg["it_s"] / base["it_s"], 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["B", "D"], choices=list(CONFIGS))
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--thresholds", nargs="+", type=float, default=[0.001, 0.01, 0.05])
    a = ap.parse_args()
    assert torch.cuda.is_available(), "contribution_bench needs a CUDA device"
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = dict(gpu=smi.splitlines()[0] if smi else torch.cuda.get_device_name(0))
    res["pass"] = pass_cost(dev, a.configs, a.reps)
    res["sweep"] = sweep_cost(dev, a.configs[-1], [32, 128])
    res["payoff"] = payoff(dev, a.thresholds)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
