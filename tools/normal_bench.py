"""Cost and payoff of the normal term of the fused step (include/psb200.h, "Rendered surface normals").

    python tools/normal_bench.py [--configs B,D] [--steps K] [--warmup W] [--rounds R] [--payoff-steps N] [--skip-cost] [--skip-payoff]

Cost: on bench.py's workload at each config, the step with the depth term and the step with the depth and normal terms alternate R
times in one process, every leg restarting from the same training state. The targets are the model's own rendered depth at the start
x 1.02 with ~10 % of the pixels zeroed, and the sensor normals of that depth (normals_from_depth). Per leg: it/s of K device-input
steps (CUDA events) and the per-stage times of K profiled steps; "render_fwd" and "render_bwd" are the tile kernels with and without
the normal plane.

Payoff: the planar scene (synthetic.planar_scene: a room corner of flat textured Gaussians with known normals) starts from random
rotations and near-isotropic scales and trains from 6 views with depth only, then with depth + normals; on 3 held-out views it reports
PSNR, depth L1 (metres, on pixels with a target) and the mean angle (degrees) between N / |N| and the true scene's normal plane on pixels
with A > 0.9. Prints one JSON line; writes nothing."""
import argparse
import json
import math

import numpy as np
import torch

import harness


def _model(sc, dev, sh=0):
    from photo_slam_b200 import trainer
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    m.setShDegree(sh)
    return m


def _angle_error(N, N_true, A):
    """mean angle (degrees) between N / |N| and the true plane's direction on pixels with A > 0.9"""
    sel = (A > 0.9) & (N_true.norm(dim=0) > 0.5)
    a = torch.nn.functional.normalize(N, dim=0)[:, sel]
    b = torch.nn.functional.normalize(N_true, dim=0)[:, sel]
    return float(torch.rad2deg(torch.acos((a * b).sum(0).clamp(-1, 1))).mean())


def planar_payoff(dev, per_wall=3000, steps=300, W=160, H=120, lambda_normal=0.05, lambda_depth=0.1, seed=0):
    """-> {"depth": dict(psnr, depth_l1, angle), "depth+normal": ...} (see the module docstring); deterministic mode."""
    import photo_slam_b200.synthetic as syn
    from photo_slam_b200 import trainer
    sc, _ = syn.planar_scene(per_wall, seed=seed)
    f = 0.7 * W
    cams = [syn.device_camera(syn.make_camera(W, H, f, f, *syn.random_pose(np.random.default_rng(100 + k), max_angle=0.12, max_trans=0.25)), dev)
            for k in range(9)]
    train, held = cams[:6], cams[6:]
    truth = trainer.GaussianTrainer(_model(sc, dev))
    targets = []
    for c in cams:
        img, D, A, N = (torch.empty((3, H, W), device=dev), torch.empty((H, W), device=dev), torch.empty((H, W), device=dev),
                        torch.empty((3, H, W), device=dev))
        truth.render(c, img, out_depth=D, out_alpha=A, out_normal=N)
        gd = torch.where(A > 0.5, D / A.clamp_min(1e-6), torch.zeros_like(D)).contiguous()
        targets.append((img, gd, trainer.normals_from_depth(c, gd), N))
    rng = np.random.default_rng(seed + 1)
    start = dict(sc, rotation=rng.normal(size=sc["rotation"].shape).astype(np.float32),
                 scaling=(np.full(sc["scaling"].shape, math.log(0.02)) + rng.normal(0, 0.1, sc["scaling"].shape)).astype(np.float32))
    res = {}
    for run, lam in (("depth", 0.0), ("depth+normal", lambda_normal)):
        m = _model(start, dev)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        for it in range(steps):
            k = it % len(train)
            img, gd, gn, _ = targets[k]
            kw = dict(gt_normal=gn, lambda_normal=lam) if lam > 0 else {}
            tr.trainForOneIteration(train[k], img, gt_depth=gd, lambda_depth=lambda_depth, densify_stats=False, **kw)
            tr.result()
        psnr, dl1, ang = [], [], []
        for j, c in enumerate(held):
            img_t, gd, _, N_true = targets[6 + j]
            img, D, A, N = (torch.empty((3, H, W), device=dev), torch.empty((H, W), device=dev), torch.empty((H, W), device=dev),
                            torch.empty((3, H, W), device=dev))
            tr.render(c, img, out_depth=D, out_alpha=A, out_normal=N)
            psnr.append(float(-10 * torch.log10(((img - img_t) ** 2).mean())))
            v = gd > 0
            dl1.append(float((D - gd).abs()[v].mean()))
            ang.append(_angle_error(N, N_true, A))
        res[run] = dict(psnr=float(np.mean(psnr)), depth_l1=float(np.mean(dl1)), angle=float(np.mean(ang)))
    return res


def cost(config, steps, warmup, rounds, lambda_depth, lambda_normal, dev):
    from photo_slam_b200 import trainer as T
    scene, cam, host, devcam, gt_dev = harness.workload(config, dev)
    model = T.GaussianModel.from_numpy(scene, dev)
    model.trainingSetup(T.GaussianOptimizationParams())
    tr = T.GaussianTrainer(model)
    W, H = devcam["W"], devcam["H"]
    d0 = torch.empty((H, W), device=dev)
    tr.render(devcam, torch.empty((3, H, W), device=dev), out_depth=d0)
    keep = torch.rand((H, W), generator=torch.Generator().manual_seed(1)) >= 0.1
    gt_depth = (d0 * 1.02 * keep.to(dev)).contiguous()
    gt_normal = T.normals_from_depth(devcam, gt_depth)
    kws = {"depth": dict(gt_depth=gt_depth, lambda_depth=lambda_depth),
           "depth+normal": dict(gt_depth=gt_depth, lambda_depth=lambda_depth, gt_normal=gt_normal, lambda_normal=lambda_normal)}
    for _ in range(max(warmup, 3)):          # also grows the binning arena and the normal planes
        for kw in kws.values():
            tr.trainForOneIteration(devcam, gt_dev, **kw)
            tr.result()
    rewind = harness.rewinder(model, tr)
    res = harness.alternate({k: (lambda k=k: harness.step_leg(tr, devcam, gt_dev, steps, rewind=rewind, **kws[k])) for k in kws}, rounds, rewind)
    rewind()
    out = {"gaussians": model.num_points(), "width": W, "height": H, "valid_normal_pixels": int((gt_normal != 0).any(0).sum().item())}
    for name, r in res.items():
        out[name] = {"value": [x[0] for x in r], "stages": harness.mean_stages([x[1] for x in r])}
    out["normal_stage_cost_ms"] = {k: out["depth+normal"]["stages"][k] - out["depth"]["stages"][k] for k in out["depth"]["stages"]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="B,D")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--lambda-depth", type=float, default=0.1)
    ap.add_argument("--lambda-normal", type=float, default=0.05)
    ap.add_argument("--payoff-steps", type=int, default=600)
    ap.add_argument("--skip-cost", action="store_true")
    ap.add_argument("--skip-payoff", action="store_true")
    a = ap.parse_args()
    dev = harness.device()
    out = {"card": harness.card(), "steps": a.steps, "rounds": a.rounds, "lambda_depth": a.lambda_depth, "lambda_normal": a.lambda_normal,
           "unit": "iters/s (value), ms (stages), dB (psnr), m (depth_l1), degrees (angle)"}
    if not a.skip_cost:
        out["cost"] = {c: cost(c, a.steps, a.warmup, a.rounds, a.lambda_depth, a.lambda_normal, dev) for c in a.configs.split(",")}
    if not a.skip_payoff:
        out["payoff"] = planar_payoff(dev, steps=a.payoff_steps, lambda_normal=a.lambda_normal, lambda_depth=a.lambda_depth)
        out["payoff"]["steps"] = a.payoff_steps
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
