"""Cost of the RGB-D depth term of the fused step, or of a data-parallel step at world 1, on bench.py's workload (default: config D).

    python tools/depth_bench.py [--config B|C|D] [--steps K] [--warmup W] [--rounds R] [--lambda-depth L] [--dp p2p|slabs]

The target depth is the model's own rendered depth at the start x 1.02 with ~10 % of the pixels zeroed (no measurement). The
plain step and the depth step alternate R times in one process, every leg restarting from the same training state, so both time
the same K iterations; the order of the two legs alternates from round to round. Per leg: value (K device-input steps, CUDA events), e2e (GaussianTrainer.trainHost: pinned host inputs,
the loss read back every step) and the per-stage times of K profiled steps. Prints one JSON line; writes nothing.

--dp p2p times DataParallelTrainer(mode="p2p") (psb_dp_step / psb_dp_step_depth; stages: DataParallelTrainer.DP_STAGES), --dp slabs
the slab pipeline (mode="nccl", pipeline=True; psb_trainer_backward_begin / _begin_depth -> _slab; it reports no stage times).
Both run at world 1 on one GPU: they time the kernels of the data-parallel step, not the exchange between ranks."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import bench  # noqa: E402  (its workload: make_inputs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="D", choices=["B", "C", "D"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--lambda-depth", type=float, default=0.1)
    ap.add_argument("--dp", choices=["p2p", "slabs"], default=None, help="time a data-parallel step at world 1 instead of the fused step")
    a = ap.parse_args()
    a.points, a.camera = {"B": (500_000, "replica"), "C": (1_000_000, "tum"), "D": (3_000_000, "replica")}[a.config]
    from photo_slam_b200 import trainer as T
    dev = torch.device("cuda", 0)
    scene, cam, host, devcam, gt_dev = bench.make_inputs(a, 0, dev)
    model = T.GaussianModel.from_numpy(scene, dev)
    model.trainingSetup(T.GaussianOptimizationParams())
    if a.dp is None:
        tr = T.GaussianTrainer(model)
    else:
        tr = T.DataParallelTrainer(model, mode="p2p") if a.dp == "p2p" else T.DataParallelTrainer(model, mode="nccl", pipeline=True)
        assert tr.mode == ("p2p" if a.dp == "p2p" else "nccl"), getattr(tr, "_p2p_error", "")
    sync = getattr(tr, "sync", lambda: None)   # p2p at world 1 with one group: everything is on the caller's stream already
    W, H = devcam["W"], devcam["H"]
    d0 = torch.empty((H, W), device=dev)
    tr.render(devcam, torch.empty((3, H, W), device=dev), out_depth=d0)
    keep = torch.rand((H, W), generator=torch.Generator().manual_seed(1)) >= 0.1
    gt_depth = (d0 * 1.02 * keep.to(dev)).contiguous()
    host_depth = gt_depth.cpu().pin_memory()
    legs = {"plain": (dict(), dict()),
            "depth": (dict(gt_depth=gt_depth, lambda_depth=a.lambda_depth), dict(host_depth=host_depth, lambda_depth=a.lambda_depth))}
    for _ in range(max(a.warmup, 3)):          # also grows the binning arena
        for dkw, _h in legs.values():
            tr.trainForOneIteration(devcam, gt_dev, **dkw)
            tr.result()
    snap, it0 = model.snapshot(), tr.iteration

    def rewind():
        sync()
        torch.cuda.synchronize()
        model.restore(snap)
        tr.iteration = it0

    hostcam = dict(devcam, viewmatrix=host["viewmatrix"], projmatrix=host["projmatrix"], campos=host["campos"])
    res = {k: dict(value=[], e2e=[], stages=[]) for k in legs}
    for rnd in range(a.rounds):
        for name in (("plain", "depth") if rnd % 2 == 0 else ("depth", "plain")):   # alternate the order: no drift bias
            dkw, hkw = legs[name]
            rewind()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.steps):
                tr.trainForOneIteration(devcam, gt_dev, **dkw)
            sync()
            e1.record()
            tr.result()
            torch.cuda.synchronize()
            res[name]["value"].append(1000.0 * a.steps / e0.elapsed_time(e1))
            rewind()
            for _ in range(3):
                tr.trainHost(hostcam, host["gt"], **hkw)
            tr.flushHost()
            rewind()
            e0.record()
            for _ in range(a.steps):
                tr.trainHost(hostcam, host["gt"], **hkw)
            tr.flushHost()
            e1.record()
            torch.cuda.synchronize()
            res[name]["e2e"].append(1000.0 * a.steps / e0.elapsed_time(e1))
            if a.dp == "slabs":
                continue
            rewind()
            tr.set_profiling(True)
            acc = {}
            for _ in range(a.steps):
                tr.trainForOneIteration(devcam, gt_dev, **dkw)
                tr.result()
                for k, v in tr.stage_times().items():
                    acc.setdefault(k, []).append(v)
            tr.set_profiling(False)
            res[name]["stages"].append({k: float(np.mean(v)) for k, v in acc.items()})
    rewind()
    out = {"config": a.config, "gaussians": a.points, "width": W, "height": H, "steps": a.steps, "rounds": a.rounds,
           "lambda_depth": a.lambda_depth, "valid_pixels": int(keep.sum().item()), "device": torch.cuda.get_device_name(dev),
           "step": a.dp or "fused", "unit": "iters/s (value, e2e), ms (stages)"}
    if a.dp:
        out["world"] = 1
        out["multi_gpu"] = "not measured: world 1 only"
    for name, r in res.items():
        out[name] = {"value": r["value"], "e2e": r["e2e"], "stages_per_round": r["stages"],
                     "stages": {k: float(np.mean([s[k] for s in r["stages"]])) for k in r["stages"][0]} if r["stages"] else {}}
    out["depth_stage_cost_ms"] = {k: out["depth"]["stages"][k] - out["plain"]["stages"][k] for k in out["plain"]["stages"]}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
