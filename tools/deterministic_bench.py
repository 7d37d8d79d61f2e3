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
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import bench  # noqa: E402  (its workload: make_inputs)

CONFIGS = {"B": (500_000, "replica"), "C": (1_000_000, "tum"), "D": (3_000_000, "replica")}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"not read: {e}"
    return {"device": torch.cuda.get_device_name(0), "nvidia_smi": q}


def run_config(cfg, a, dev):
    from photo_slam_b200 import trainer as T
    a.points, a.camera = CONFIGS[cfg]
    scene, cam, host, devcam, gt_dev = bench.make_inputs(a, 0, dev)
    model = T.GaussianModel.from_numpy(scene, dev)
    model.trainingSetup(T.GaussianOptimizationParams())
    legs = {"default": T.GaussianTrainer(model, deterministic=False), "deterministic": T.GaussianTrainer(model, deterministic=True)}
    for _ in range(max(a.warmup, 3)):           # also grows both binning arenas (and the slot buffer)
        for tr in legs.values():
            tr.trainForOneIteration(devcam, gt_dev)
            tr.result()
    snap = model.snapshot()
    n_inst = legs["default"].result()[3]
    radii = torch.empty(model.num_points(), dtype=torch.int32, device=dev)
    legs["default"].render(devcam, radii=radii)
    visible = int((radii > 0).sum())

    def rewind():
        torch.cuda.synchronize()
        model.restore(snap)

    res = {k: dict(value=[], stages=[]) for k in legs}
    for rnd in range(a.rounds):
        for name in (("default", "deterministic") if rnd % 2 == 0 else ("deterministic", "default")):
            tr = legs[name]
            rewind()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                tr.trainForOneIteration(devcam, gt_dev)
            e1.record()
            tr.result()
            torch.cuda.synchronize()
            res[name]["value"].append(1000.0 * a.steps / e0.elapsed_time(e1))
            rewind()
            tr.set_profiling(True)
            acc = {}
            for _ in range(a.steps):
                tr.trainForOneIteration(devcam, gt_dev)
                tr.result()
                for k, v in tr.stage_times().items():
                    acc.setdefault(k, []).append(v)
            tr.set_profiling(False)
            res[name]["stages"].append({k: float(np.mean(v)) for k, v in acc.items()})
    rewind()
    out = {"gaussians": a.points, "width": devcam["W"], "height": devcam["H"], "instances": n_inst, "visible": visible}
    for name, r in res.items():
        out[name] = {"value": r["value"], "value_median": float(np.median(r["value"])), "stages_per_round": r["stages"],
                     "stages": {k: float(np.mean([s[k] for s in r["stages"]])) for k in r["stages"][0]}}
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
    assert torch.cuda.is_available(), "deterministic_bench needs a CUDA device"
    dev = torch.device("cuda", 0)
    out = {"card": card(), "steps": a.steps, "rounds": a.rounds, "unit": "iters/s (value), ms (stages)"}
    for cfg in a.configs.split(","):
        out[cfg] = run_config(cfg, a, dev)
        torch.cuda.empty_cache()
    out["card_after"] = card()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
