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

import torch

import harness


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="D", choices=["B", "C", "D"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--lambda-depth", type=float, default=0.1)
    ap.add_argument("--dp", choices=["p2p", "slabs"], default=None, help="time a data-parallel step at world 1 instead of the fused step")
    a = ap.parse_args()
    dev = harness.device()
    from photo_slam_b200 import trainer as T
    scene, cam, host, devcam, gt_dev = harness.workload(a.config, dev)
    model = T.GaussianModel.from_numpy(scene, dev)
    model.trainingSetup(T.GaussianOptimizationParams())
    if a.dp is None:
        tr = T.GaussianTrainer(model)
    else:
        tr = T.DataParallelTrainer(model, mode="p2p") if a.dp == "p2p" else T.DataParallelTrainer(model, mode="nccl", pipeline=True)
        assert tr.mode == ("p2p" if a.dp == "p2p" else "nccl"), getattr(tr, "_p2p_error", "")
    W, H = devcam["W"], devcam["H"]
    d0 = torch.empty((H, W), device=dev)
    tr.render(devcam, torch.empty((3, H, W), device=dev), out_depth=d0)
    keep = torch.rand((H, W), generator=torch.Generator().manual_seed(1)) >= 0.1
    gt_depth = (d0 * 1.02 * keep.to(dev)).contiguous()
    host_depth = gt_depth.cpu().pin_memory()
    kws = {"plain": (dict(), dict()),
           "depth": (dict(gt_depth=gt_depth, lambda_depth=a.lambda_depth), dict(host_depth=host_depth, lambda_depth=a.lambda_depth))}
    for _ in range(max(a.warmup, 3)):          # also grows the binning arena
        for dkw, _h in kws.values():
            tr.trainForOneIteration(devcam, gt_dev, **dkw)
            tr.result()
    rewind = harness.rewinder(model, tr)
    hostcam = dict(devcam, viewmatrix=host["viewmatrix"], projmatrix=host["projmatrix"], campos=host["campos"])

    def e2e(hkw):
        for _ in range(3):
            tr.trainHost(hostcam, host["gt"], **hkw)
        tr.flushHost()
        rewind()

        def window():
            for _ in range(a.steps):
                tr.trainHost(hostcam, host["gt"], **hkw)
            tr.flushHost()
        return 1000.0 * a.steps / harness.window_ms(window, 1)

    def leg(name):
        dkw, hkw = kws[name]
        value, _ = harness.step_leg(tr, devcam, gt_dev, a.steps, profile=False, **dkw)
        rewind()
        rate = e2e(hkw)
        stages = {}
        if a.dp != "slabs":
            rewind()
            stages = harness.stage_ms(tr, lambda: tr.trainForOneIteration(devcam, gt_dev, **dkw), a.steps)
        return value, rate, stages

    res = harness.alternate({k: (lambda k=k: leg(k)) for k in kws}, a.rounds, rewind)
    rewind()
    out = {"config": a.config, "gaussians": model.num_points(), "width": W, "height": H, "steps": a.steps, "rounds": a.rounds,
           "lambda_depth": a.lambda_depth, "valid_pixels": int(keep.sum().item()), "card": harness.card(),
           "step": a.dp or "fused", "unit": "iters/s (value, e2e), ms (stages)"}
    if a.dp:
        out["world"] = 1
        out["multi_gpu"] = "not measured: world 1 only"
    for name, r in res.items():
        stages = [x[2] for x in r if x[2]]
        out[name] = {"value": [x[0] for x in r], "e2e": [x[1] for x in r], "stages_per_round": stages, "stages": harness.mean_stages(stages)}
    out["depth_stage_cost_ms"] = {k: out["depth"]["stages"][k] - out["plain"]["stages"][k] for k in out["plain"]["stages"]}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
