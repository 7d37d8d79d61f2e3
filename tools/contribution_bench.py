"""Cost and payoff of contribution pruning: python tools/contribution_bench.py [--configs B D] [--reps 20]

Cost: one score pass (psb_trainer_contribution) against one render (psb_trainer_render) of the same view at each config, legs alternating
in one process on the same model (CUDA events, median over --reps after a warm-up), with the instance count; a sweep over K = 32 and 128
keyframes at the last config (contributionScores: one host round trip). Payoff: the scene of tests/test_quality_gpu.py (200 k rows, 6
keyframes at 640x480), trained for 600 fused steps, then pruned at several thresholds from the same snapshot: rows removed, mean keyframe
PSNR right after the prune and after 100 more steps, and the fused step's it/s before and after. Prints one JSON object with the card's name
and power limit. Writes nothing."""
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


def _views(dev, K, W, H, fx, fy, seed, angle=0.3, trans=0.5):
    rng = np.random.default_rng(seed)
    return [syn.device_camera(syn.make_camera(W, H, fx, fy, *syn.random_pose(rng, max_angle=angle, max_trans=trans)), dev) for _ in range(K)]


def pass_cost(dev, configs, reps):
    out = {}
    for name in configs:
        sc, _, _, c, _ = harness.workload(name, dev)
        W, H = c["W"], c["H"]
        m = trainer.GaussianModel.from_numpy(sc, dev)
        tr = trainer.GaussianTrainer(m)
        img = torch.empty((3, H, W), device=dev)
        mx = torch.zeros(m.num_points(), dtype=torch.int32, device=dev)
        sm = torch.zeros(m.num_points(), dtype=torch.int64, device=dev)
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
        legs = harness.alternate({"render": lambda: harness.cuda_ms(render, reps), "score": lambda: harness.cuda_ms(score, reps)}, 4)
        assert tr.result()[3] == n
        r, s = float(np.median(legs["render"])), float(np.median(legs["score"]))
        out[name] = dict(P=m.num_points(), W=W, H=H, instances=n, render_ms=round(r, 4), score_ms=round(s, 4), overhead=round(s / r - 1.0, 4))
    return out


def sweep_cost(dev, name, Ks):
    sc, _, _, c, _ = harness.workload(name, dev)
    W, H, fx, fy = syn.CAMERAS[harness.CONFIGS[name][1]]
    m = trainer.GaussianModel.from_numpy(sc, dev)
    tr = trainer.GaussianTrainer(m)
    out = {}
    for K in Ks:
        views = _views(dev, K, W, H, fx, fy, seed=K, angle=0.05, trans=0.05)
        ms = harness.cuda_ms(lambda: tr.contributionScores(views), 3)      # the warm-up call grows the arena
        mx, _ = tr.contributionScores(views)
        out[f"K{K}"] = dict(config=name, ms=round(ms, 3), per_view_ms=round(ms / K, 4), rows_scored=int((mx > 0).sum()), P=m.num_points())
    return out


def payoff(dev, thresholds, steps=600, more=100):
    """the scene and trainee of tests/test_quality_gpu.py, trained without densification (the SH degree rises every 200 steps)"""
    gt_scene, cams = syn.quality_scene()
    views = [syn.device_camera(cam, dev) for cam in cams]
    gt_tr = trainer.GaussianTrainer(trainer.GaussianModel.from_numpy(gt_scene, dev))
    gts = [gt_tr.render(c).clamp(0, 1).clone() for c in views]
    start = syn.thinned_trainee(gt_scene)
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

        def window():
            for it in range(n):
                k = it % len(views)
                tr.trainForOneIteration(views[k], gts[k], densify_stats=False)
        rate = n * 1000.0 / harness.window_ms(window, 1)
        tr.result()
        return rate

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
    ap.add_argument("--configs", nargs="+", default=["B", "D"], choices=["B", "D"])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--thresholds", nargs="+", type=float, default=[0.001, 0.01, 0.05])
    a = ap.parse_args()
    dev = harness.device()
    res = dict(card=harness.card())
    res["pass"] = pass_cost(dev, a.configs, a.reps)
    res["sweep"] = sweep_cost(dev, a.configs[-1], [32, 128])
    res["payoff"] = payoff(dev, a.thresholds)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
