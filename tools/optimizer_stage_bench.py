"""Optimizer stage of the fused step: python tools/optimizer_stage_bench.py [--configs B D] [--steps 30] [--warmup 10] [--rounds 2]

At each config two legs alternate from the same model snapshot: "one view" (bench.py's camera every step) and "two views" (that camera
and a second one, turned by 0.25 rad and shifted, on alternate steps: the SLAM-like case, where many live rows have no staged f_rest row
in a given step). Per leg it reports it/s, the two stage times of the optimizer stage (gaussian_backward: the per-Gaussian backward with
the Adam of the staged SH rows; frest_adam: frest_momentum_kernel) and, from one extra step, the rows of that step:
  live       rows whose live byte is set after the step;
  staged     live rows whose f_rest moments moved by more than the momentum decay (a non-zero f_rest gradient: their row was staged);
  momentum   the other live rows (g = 0: momentum-only).
Bytes of the f_rest Adam under the fused accounting: staged rows 900 B (m, v read; p, m, v written; p comes from the staged copy the
backward reads anyway), momentum rows 1084 B (p, m, v read and written, one list entry). GB/s = those bytes over the stage that moves
them is given for frest_adam (momentum rows only) and for the whole stage (bench.py's gaussian_backward bytes + both f_rest terms).
Prints one JSON object. Writes nothing."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import harness  # noqa: E402
import bench  # noqa: E402
import photo_slam_b200.synthetic as syn  # noqa: E402
from photo_slam_b200 import trainer  # noqa: E402


def second_camera(host, dev):
    R, _ = syn.random_pose(np.random.default_rng(11), max_angle=0.25, max_trans=0.0)
    c = syn.make_camera(host["W"], host["H"], host["W"] / (2 * float(host["tanfovx"])), host["H"] / (2 * float(host["tanfovy"])), R,
                        np.array([0.15, -0.1, 0.0]))
    return syn.device_camera(c, dev)


def row_counts(m, tr, cam, gt):
    """One step on `cam`: -> (live, staged, momentum-only) rows of it."""
    m0 = m.exp_avg_[2].clone()
    tr.trainForOneIteration(cam, gt)
    tr.result()
    torch.cuda.synchronize()
    live = m.adam_live_.bool()
    decayed = (m.exp_avg_[2] == m0 * 0.9).reshape(m.num_points(), -1).all(dim=1)
    staged = live & ~decayed
    return int(live.sum()), int(staged.sum()), int((live & decayed).sum())


def config_run(dev, config, steps, warmup, rounds):
    sc, host, _, cam, gt = harness.workload(config, dev)   # host: the make_camera dict
    cam2 = second_camera(host, dev)
    P = len(sc["xyz"])
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    tr = trainer.GaussianTrainer(m)
    for i in range(warmup):
        tr.trainForOneIteration(cam2 if i % 2 else cam, gt)
        tr.result()
    rewind = harness.rewinder(m, tr)
    cams = {"one view": [cam], "two views": [cam, cam2]}

    def leg(cs):
        def run():
            its_e0, its_e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            its_e0.record()
            for i in range(steps):
                tr.trainForOneIteration(cs[i % len(cs)], gt)
            its_e1.record()
            tr.result()
            torch.cuda.synchronize()
            its = 1000.0 * steps / its_e0.elapsed_time(its_e1)
            rewind()
            k = [0]

            def step():
                tr.trainForOneIteration(cs[k[0] % len(cs)], gt)
                k[0] += 1
            st = harness.stage_ms(tr, step, steps)
            rewind()
            for i in range(steps):     # the rows of the step after `steps` steps of this leg
                tr.trainForOneIteration(cs[i % len(cs)], gt)
            tr.result()
            return its, st, row_counts(m, tr, cs[steps % len(cs)], gt)
        return run

    res = harness.alternate({k: leg(cs) for k, cs in cams.items()}, rounds, rewind)
    rewind()
    out = {}
    for k, legs in res.items():
        st = harness.mean_stages([x[1] for x in legs])
        live, staged, mom = legs[-1][2]
        gb, fa = st["gaussian_backward"], st["frest_adam"]
        bytes_stage = bench.algorithmic_bytes(P, live, 0, 1, 1, 0, P_touched=live)["gaussian_backward"] + 900 * staged + 1084 * mom
        out[k] = {"it_s": [round(x[0], 1) for x in legs], "gaussian_backward_ms": round(gb, 4), "frest_adam_ms": round(fa, 4),
                  "rows": {"P": P, "live": live, "staged": staged, "momentum_only": mom},
                  "frest_adam_GBps": round(1084 * mom / 1e6 / fa, 1) if fa > 0 else None,
                  "optimizer_stage_GBps": round(bytes_stage / 1e6 / (gb + fa), 1)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["B", "D"])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    dev = harness.device()
    out = {"card": harness.card()}
    for cfg in a.configs:
        out[cfg] = config_run(dev, cfg, a.steps, a.warmup, a.rounds)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
