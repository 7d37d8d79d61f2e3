"""Cost of exposure compensation on the NVLink data-parallel step at world 1, on bench.py's workloads (default: configs B and D).

    python tools/dp_exposure_bench.py [--configs B,D] [--steps K] [--warmup W] [--rounds R]

For each config two legs alternate R times in one process, each restarting from the same training state: "off"
(DataParallelTrainer(mode="p2p"), psb_dp_step_depth without exposure) and "exposure" (DataParallelTrainer(mode="p2p", exposure=True),
psb_dp_step_table through row 0 of a one-row table: the exposure mix and update kernels, the exposure record in the meta row and
exposure_apply_kernel). Each leg has its own model and trainer, built from the same scene. The order of the legs flips from round to
round. Per leg: value (K device-input steps, CUDA events) and the per-stage times of K profiled steps. World 1 times the kernels of the
step, not the exchange between ranks. Prints one JSON line per config, with the card's name and power limit; writes nothing."""
import argparse
import json

import torch

import harness

LEGS = ("off", "exposure")


def run_config(config, a, dev):
    from photo_slam_b200 import trainer as T
    scene, cam, host, devcam, gt_dev = harness.workload(config, dev)
    out = {"config": config, "gaussians": int(scene["xyz"].shape[0]), "width": devcam["W"], "height": devcam["H"], "steps": a.steps,
           "rounds": a.rounds, "card": harness.card(), "world": 1, "multi_gpu": "not measured: world 1 only",
           "unit": "iters/s (value), ms (stages)"}
    legs, kws = {}, {"off": {}, "exposure": {"exposure_id": 0}}
    for name in LEGS:
        model = T.GaussianModel.from_numpy(scene, dev)
        model.trainingSetup(T.GaussianOptimizationParams())
        model.ensureExposures(1)
        tr = T.DataParallelTrainer(model, mode="p2p", exposure=(name == "exposure"))
        assert tr.mode == "p2p", getattr(tr, "_p2p_error", "")
        for _ in range(max(a.warmup, 3)):          # also grows the binning arena
            tr.trainForOneIteration(devcam, gt_dev, **kws[name])
            tr.result()
        legs[name] = (model, tr, harness.rewinder(model, tr))

    def leg(name):
        model, tr, rewind = legs[name]
        rewind()
        value, _ = harness.step_leg(tr, devcam, gt_dev, a.steps, profile=False, **kws[name])
        rewind()
        stages = harness.stage_ms(tr, lambda: tr.trainForOneIteration(devcam, gt_dev, **kws[name]), a.steps)
        return value, stages

    res = harness.alternate({k: (lambda k=k: leg(k)) for k in LEGS}, a.rounds)
    for name, r in res.items():
        out[name] = {"value": [x[0] for x in r], "stages": harness.mean_stages([x[1] for x in r])}
    mean = lambda v: sum(v) / len(v)
    out["exposure"]["step_cost_ms"] = 1000.0 / mean(out["exposure"]["value"]) - 1000.0 / mean(out["off"]["value"])
    out["exposure"]["stage_cost_ms"] = {k: out["exposure"]["stages"][k] - out["off"]["stages"][k] for k in out["off"]["stages"]}
    print(json.dumps(out), flush=True)
    for model, tr, _ in legs.values():
        tr.close()
    del legs
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="B,D")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=4)
    a = ap.parse_args()
    configs = [c.strip() for c in a.configs.split(",") if c.strip()]
    for c in configs:
        if c not in harness.CONFIGS:
            ap.error(f"unknown config {c}: choose from {sorted(harness.CONFIGS)}")
    dev = harness.device()
    for c in configs:
        run_config(c, a, dev)


if __name__ == "__main__":
    main()
