"""Cost of the deterministic mode of the fused step (GaussianTrainer(deterministic=True)) on bench.py's workloads.

    python tools/deterministic_bench.py [--configs B,D] [--steps K] [--warmup W] [--rounds R]

Per config, one model and two trainers on it — the default mode and the deterministic mode, each with its own context and arena.
The two legs alternate R times in one process (the order alternates from round to round), every leg restarting from the same
training state, so both time the same K iterations. Per leg: value = K device-input steps / their CUDA-event time (iters/s), and
the mean per-stage times of K profiled steps (the ordered gather is inside "render_bwd"). The card's name and power limit are read
in the same run. Prints one JSON line; writes nothing.

A lower bound from bytes, for comparison: the slots cost 48 B written + 48 B read per instance, plus 48 B per visible Gaussian for
the sink row the gather writes (and 16 + 4 B of tile_info / base it reads); divided by 3.35 TB/s (H100 SXM data sheet)."""
import argparse
import json

import numpy as np
import torch

import harness


def run_config(cfg, a, dev):
    from photo_slam_b200 import trainer as T
    scene, cam, host, devcam, gt_dev = harness.workload(cfg, dev)
    model = T.GaussianModel.from_numpy(scene, dev)
    model.trainingSetup(T.GaussianOptimizationParams())
    legs = {"default": T.GaussianTrainer(model, deterministic=False), "deterministic": T.GaussianTrainer(model, deterministic=True)}
    for _ in range(max(a.warmup, 3)):           # also grows both binning arenas (and the slot buffer)
        for tr in legs.values():
            tr.trainForOneIteration(devcam, gt_dev)
            tr.result()
    rewind = harness.rewinder(model, *legs.values())
    n_inst = legs["default"].result()[3]
    radii = torch.empty(model.num_points(), dtype=torch.int32, device=dev)
    legs["default"].render(devcam, radii=radii)
    visible = int((radii > 0).sum())
    res = harness.alternate({k: (lambda tr=tr: harness.step_leg(tr, devcam, gt_dev, a.steps, rewind)) for k, tr in legs.items()}, a.rounds, rewind)
    rewind()
    out = {"gaussians": model.num_points(), "width": devcam["W"], "height": devcam["H"], "instances": n_inst, "visible": visible}
    for name, r in res.items():
        value, stages = [x[0] for x in r], [x[1] for x in r]
        out[name] = {"value": value, "value_median": float(np.median(value)), "stages_per_round": stages, "stages": harness.mean_stages(stages)}
    out["stage_cost_ms"] = {k: out["deterministic"]["stages"][k] - out["default"]["stages"][k] for k in out["default"]["stages"]}
    out["value_ratio"] = out["deterministic"]["value_median"] / out["default"]["value_median"]
    slot_bytes = 96 * n_inst + 68 * visible
    out["byte_lower_bound_ms"] = {"bytes": slot_bytes, "ms_at_3.35TBps": slot_bytes / 3.35e12 * 1e3,
                                  "note": "data-sheet bandwidth, a bound from bytes; not a measurement"}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="B,D")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=4)
    a = ap.parse_args()
    dev = harness.device()
    out = {"card": harness.card(), "steps": a.steps, "rounds": a.rounds, "unit": "iters/s (value), ms (stages)"}
    for cfg in a.configs.split(","):
        out[cfg] = run_config(cfg, a, dev)
        torch.cuda.empty_cache()
    out["card_after"] = harness.card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
