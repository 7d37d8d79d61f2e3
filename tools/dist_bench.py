"""Cost and payoff of the depth distortion term of the fused step (include/psb200.h, "Depth distortion").

    python tools/dist_bench.py [--configs B,D] [--steps K] [--warmup W] [--rounds R] [--payoff-steps N] [--skip-cost] [--skip-payoff]

Cost: on bench.py's workload at each config, four steps alternate R times in one process, every leg restarting from the same training
state: the colour-only step ("colour"), colour + the term ("colour_dist", psb_trainer_step_dist), the depth step against the rendered
depth of the start state ("depth") and depth + the term ("depth_dist"). Per leg: it/s of K device-input steps (CUDA events) and the
per-stage times of K profiled steps; "dist_stage_cost_ms" is the per-stage difference of each pair. The legs use --cost-lambda-dist
(default 1e-4): a weight that leaves the map's trajectory over K steps that of the leg without the term, so the difference is the cost
of the term's kernels and planes. With a weight that reshapes the map (lambda 1 on this random scene drives opacities down within a
few steps) the blend gets cheaper and the term's legs run faster than the legs without it.

Payoff: the planar scene (synthetic.planar_scene, 3 x per_wall rows, 160 x 120, 6 training and 3 held-out views as tools/dn_bench.py
poses them). The trainee is synthetic.distortion_trainee: the true rows moved along their plane's normal by N(0, 0.1 m) with opacity 0.3,
so several rows share each pixel. No densification; deterministic mode. It trains on colour alone, on colour + the term for each lambda
of the sweep, and (reported, not gated) on colour + depth-normal consistency with and without the term. On the held-out views, over
pixels with A > 0.9: PSNR, the mean depth spread sqrt(max(M / A - (D / A)^2, 0)) and the mean |D / A - D_true|. Prints one JSON line;
writes nothing."""
import argparse
import json

import numpy as np
import torch

import harness
from dn_bench import planar_views
from normal_bench import _model


def held_out_metrics(tr, held, targets, dev):
    """-> dict(psnr, spread, depth_err) over the held-out cameras (targets: planar_views' (image, true depth, N) of each)"""
    psnr, spread, err = [], [], []
    for c, (img_t, d_true, _) in zip(held, targets):
        H, W = c["H"], c["W"]
        img, D, A, M = (torch.empty((3, H, W), device=dev), torch.empty((H, W), device=dev), torch.empty((H, W), device=dev),
                        torch.empty((H, W), device=dev))
        tr.render(c, img, out_depth=D, out_alpha=A, out_depth2=M)
        sel = A > 0.9
        Db = D[sel] / A[sel]
        psnr.append(float(-10 * torch.log10(((img - img_t) ** 2).mean())))
        spread.append(float(torch.sqrt(torch.clamp_min(M[sel] / A[sel] - Db * Db, 0.0)).mean()))
        ok = d_true[sel] > 0
        err.append(float((Db[ok] - d_true[sel][ok]).abs().mean()))
    return dict(psnr=float(np.mean(psnr)), spread=float(np.mean(spread)), depth_err=float(np.mean(err)))


def distortion_payoff(dev, per_wall=3000, steps=300, W=160, H=120, lambdas=(0.1, 1.0, 10.0), lambda_dn=0.05, dn_lambda_dist=1.0, seed=0):
    """-> {"colour": metrics, "colour+dist@<lambda>": metrics for each lambda, "colour+dn": ..., "colour+dn+dist@<dn_lambda_dist>": ...}
    (see the module docstring)."""
    import photo_slam_b200.synthetic as syn
    from photo_slam_b200 import trainer
    sc, normals, train, held, targets = planar_views(dev, per_wall, W, H, seed)
    start = syn.distortion_trainee(sc, normals, seed=seed + 1)
    runs = [("colour", 0.0, 0.0)] + [(f"colour+dist@{lam:g}", lam, 0.0) for lam in lambdas]
    runs += [("colour+dn", 0.0, lambda_dn), (f"colour+dn+dist@{dn_lambda_dist:g}", dn_lambda_dist, lambda_dn)]
    res = {}
    for name, lam, lam_dn in runs:
        m = _model(start, dev)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        for it in range(steps):
            k = it % len(train)
            tr.trainForOneIteration(train[k], targets[k][0], densify_stats=False, lambda_dist=lam, lambda_dn=lam_dn)
            tr.result()
        res[name] = held_out_metrics(tr, held, targets[len(train):], dev)
    return res


def cost(config, steps, warmup, rounds, lambda_dist, dev):
    from photo_slam_b200 import trainer as T
    scene, cam, host, devcam, gt_dev = harness.workload(config, dev)
    model = T.GaussianModel.from_numpy(scene, dev)
    model.trainingSetup(T.GaussianOptimizationParams())
    tr = T.GaussianTrainer(model)
    W, H = devcam["W"], devcam["H"]
    # a depth target: the start state's own rendered depth, so the depth legs train against a plausible target
    D, A = torch.empty((H, W), device=dev), torch.empty((H, W), device=dev)
    tr.render(devcam, out_depth=D, out_alpha=A)
    gt_depth = torch.where(A > 0.5, D / A.clamp_min(1e-6), torch.zeros_like(D)).contiguous()
    dkw = dict(gt_depth=gt_depth, lambda_depth=0.1)
    kws = {"colour": {}, "colour_dist": dict(lambda_dist=lambda_dist), "depth": dkw, "depth_dist": dict(dkw, lambda_dist=lambda_dist)}
    for _ in range(max(warmup, 3)):          # also grows the binning arena and the planes of every leg
        for kw in kws.values():
            tr.trainForOneIteration(devcam, gt_dev, **kw)
            tr.result()
    rewind = harness.rewinder(model, tr)
    legs = {k: (lambda k=k: harness.step_leg(tr, devcam, gt_dev, steps, rewind=rewind, **kws[k])) for k in kws}
    res = harness.alternate(legs, rounds, rewind)
    rewind()
    out = {"gaussians": model.num_points(), "width": W, "height": H}
    for name, r in res.items():
        out[name] = {"value": [x[0] for x in r], "stages": harness.mean_stages([x[1] for x in r])}
    out["dist_stage_cost_ms"] = {
        base: {k: out[base + "_dist"]["stages"][k] - out[base]["stages"][k] for k in out[base]["stages"]} for base in ("colour", "depth")}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="B,D")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--cost-lambda-dist", type=float, default=1e-4)
    ap.add_argument("--payoff-steps", type=int, default=300)
    ap.add_argument("--skip-cost", action="store_true")
    ap.add_argument("--skip-payoff", action="store_true")
    a = ap.parse_args()
    dev = harness.device()
    out = {"card": harness.card(), "steps": a.steps, "rounds": a.rounds, "cost_lambda_dist": a.cost_lambda_dist,
           "unit": "iters/s (value), ms (stages), dB (psnr), metres (spread, depth_err)"}
    if not a.skip_cost:
        out["cost"] = {c: cost(c, a.steps, a.warmup, a.rounds, a.cost_lambda_dist, dev) for c in a.configs.split(",")}
    if not a.skip_payoff:
        out["payoff"] = distortion_payoff(dev, steps=a.payoff_steps)
        out["payoff"]["steps"] = a.payoff_steps
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
