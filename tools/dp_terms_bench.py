"""Cost of the normal, depth-normal consistency and distortion terms on the fused step and on the data-parallel steps at world 1, on
bench.py's workloads (default: configs B and D).

    python tools/dp_terms_bench.py [--configs B,D] [--steps K] [--warmup W] [--rounds R] [--lambda-normal L] [--lambda-dn L]
                                   [--lambda-dist L]

For each config and each step — the fused step (GaussianTrainer), the NVLink step (DataParallelTrainer(mode="p2p", geometry_terms=True),
psb_dp_step_dist) and the slab pipeline (mode="nccl", pipeline=True; psb_trainer_backward_begin_dist -> _slab) — three legs alternate R times in one
process, every leg restarting from the same training state: "plain" (colour only), "normal_dn" (the RGB-D normal term against the
sensor normals of the model's own rendered depth x 1.02, plus the consistency term) and "dist" (the distortion term). The order of
the legs rotates from round to round. Per leg: value (K device-input steps, CUDA events) and, except for the slab pipeline, which
reports none, the per-stage times of K profiled steps. The data-parallel steps run at world 1 on one GPU: they time the kernels of
the step (the 16-float push backward included), not the exchange between ranks. Prints one JSON line per config; writes nothing."""
import argparse
import json

import torch

import harness

STEPS = ("fused", "p2p", "slabs")


def make_trainer(T, model, step):
    if step == "fused":
        return T.GaussianTrainer(model)
    kw = dict(mode="p2p") if step == "p2p" else dict(mode="nccl", pipeline=True)
    tr = T.DataParallelTrainer(model, geometry_terms=True, **kw)
    assert tr.mode == ("p2p" if step == "p2p" else "nccl"), getattr(tr, "_p2p_error", "")
    return tr


def run_config(config, a, dev):
    from photo_slam_b200 import trainer as T
    scene, cam, host, devcam, gt_dev = harness.workload(config, dev)
    W, H = devcam["W"], devcam["H"]
    out = {"config": config, "gaussians": int(scene["xyz"].shape[0]), "width": W, "height": H, "steps": a.steps, "rounds": a.rounds,
           "lambda_normal": a.lambda_normal, "lambda_dn": a.lambda_dn, "lambda_dist": a.lambda_dist, "card": harness.card(), "world": 1,
           "multi_gpu": "not measured: world 1 only", "unit": "iters/s (value), ms (stages)"}
    gt_normal = None
    for step in STEPS:
        model = T.GaussianModel.from_numpy(scene, dev)
        model.trainingSetup(T.GaussianOptimizationParams())
        tr = make_trainer(T, model, step)
        if gt_normal is None:
            d0 = torch.empty((H, W), device=dev)
            tr.render(devcam, torch.empty((3, H, W), device=dev), out_depth=d0)
            gt_normal = T.normals_from_depth(devcam, (d0 * 1.02).contiguous())
            torch.cuda.synchronize()
            out["valid_normal_pixels"] = int((gt_normal != 0).any(0).sum().item())
        kws = {"plain": dict(),
               "normal_dn": dict(gt_normal=gt_normal, lambda_normal=a.lambda_normal, lambda_dn=a.lambda_dn),
               "dist": dict(lambda_dist=a.lambda_dist)}
        for _ in range(max(a.warmup, 3)):          # also grows the binning arena
            for kw in kws.values():
                tr.trainForOneIteration(devcam, gt_dev, **kw)
                tr.result()
        rewind = harness.rewinder(model, tr)

        def leg(name):
            value, _ = harness.step_leg(tr, devcam, gt_dev, a.steps, profile=False, **kws[name])
            stages = {}
            if step != "slabs":
                rewind()
                stages = harness.stage_ms(tr, lambda: tr.trainForOneIteration(devcam, gt_dev, **kws[name]), a.steps)
            return value, stages

        res = harness.alternate({k: (lambda k=k: leg(k)) for k in kws}, a.rounds, rewind)
        rewind()
        o = {}
        for name, r in res.items():
            stages = [x[1] for x in r if x[1]]
            o[name] = {"value": [x[0] for x in r], "stages": harness.mean_stages(stages)}
        for name in ("normal_dn", "dist"):
            o[name]["step_cost_ms"] = 1000.0 / (sum(o[name]["value"]) / len(o[name]["value"])) - 1000.0 / (sum(o["plain"]["value"]) / len(o["plain"]["value"]))
            if o["plain"]["stages"]:
                o[name]["stage_cost_ms"] = {k: o[name]["stages"][k] - o["plain"]["stages"][k] for k in o["plain"]["stages"]}
        out[step] = o
        if hasattr(tr, "close"):
            tr.close()
        del tr, model
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="B,D")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--lambda-normal", type=float, default=0.05)
    ap.add_argument("--lambda-dn", type=float, default=0.05)
    ap.add_argument("--lambda-dist", type=float, default=0.1)
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
