"""Cost and payoff of the depth-normal consistency term of the fused step (include/psb200.h, "Depth-normal consistency").

    python tools/dn_bench.py [--configs B,D] [--steps K] [--warmup W] [--rounds R] [--payoff-steps N] [--skip-cost] [--skip-payoff]

Cost: on bench.py's workload at each config, three steps alternate R times in one process, every leg restarting from the same training
state: the colour-only step ("colour"), the built-in step with the term ("builtin_dn", psb_trainer_step_dn) and trainWithLoss computing
L1 + SSIM and the same term in torch float32 ("torch_dn": a caller's route without the built-in term). Per leg: it/s of K device-input
steps (CUDA events); for the two built-in legs also the per-stage times of K profiled steps.

Payoff: the planar scene (synthetic.planar_scene) starts from random rotations and near-isotropic scales and trains from 6 views on
colour alone (monocular: no depth or normal target), then on colour + the term; on 3 held-out views it reports PSNR, the mean angle
(degrees) between N / |N| and the true scene's normal plane on pixels with A > 0.9, and the scale-invariant depth error of D / A against
the true depth (the RMS of log(D / A) - log(D_true) about its mean, on pixels with A > 0.9). Prints one JSON line; writes nothing."""
import argparse
import json
import math

import numpy as np
import torch

import harness
from normal_bench import _angle_error, _model


def _si_depth_error(D, A, D_true):
    sel = (A > 0.9) & (D_true > 0) & (D > 0)
    d = torch.log(D[sel] / A[sel]) - torch.log(D_true[sel])
    return float(torch.sqrt((d * d).mean() - d.mean() ** 2))


def planar_views(dev, per_wall=3000, W=160, H=120, seed=0):
    """The planar payoff's setup: synthetic.planar_scene(per_wall) seen at W x H (f = 0.7 W) from 9 poses, the first 6 for training and
    the last 3 held out. -> (scene, normals, train cams, held-out cams, targets: per camera (image, true depth D / A where A > 0.5 else 0,
    normal plane N) rendered from the true scene)."""
    import photo_slam_b200.synthetic as syn
    from photo_slam_b200 import trainer
    sc, normals = syn.planar_scene(per_wall, seed=seed)
    f = 0.7 * W
    cams = [syn.device_camera(syn.make_camera(W, H, f, f, *syn.random_pose(np.random.default_rng(100 + k), max_angle=0.12, max_trans=0.25)), dev)
            for k in range(9)]
    truth = trainer.GaussianTrainer(_model(sc, dev))
    targets = []
    for c in cams:
        img, D, A, N = (torch.empty((3, H, W), device=dev), torch.empty((H, W), device=dev), torch.empty((H, W), device=dev),
                        torch.empty((3, H, W), device=dev))
        truth.render(c, img, out_depth=D, out_alpha=A, out_normal=N)
        targets.append((img, torch.where(A > 0.5, D / A.clamp_min(1e-6), torch.zeros_like(D)), N))
    return sc, normals, cams[:6], cams[6:], targets


def planar_payoff(dev, per_wall=3000, steps=300, W=160, H=120, lambda_dn=0.05, alpha_min=0.5, max_rel_jump=0.05, seed=0):
    """-> {"colour": dict(psnr, angle, si_depth), "colour+dn": ...} (see the module docstring); deterministic mode."""
    from photo_slam_b200 import trainer
    sc, _, train, held, targets = planar_views(dev, per_wall, W, H, seed)
    rng = np.random.default_rng(seed + 1)
    start = dict(sc, rotation=rng.normal(size=sc["rotation"].shape).astype(np.float32),
                 scaling=(np.full(sc["scaling"].shape, math.log(0.02)) + rng.normal(0, 0.1, sc["scaling"].shape)).astype(np.float32))
    res = {}
    for run, lam in (("colour", 0.0), ("colour+dn", lambda_dn)):
        m = _model(start, dev)
        tr = trainer.GaussianTrainer(m, deterministic=True)
        for it in range(steps):
            k = it % len(train)
            tr.trainForOneIteration(train[k], targets[k][0], densify_stats=False, lambda_dn=lam, dn_alpha_min=alpha_min, dn_max_rel_jump=max_rel_jump)
            tr.result()
        psnr, ang, si = [], [], []
        for j, c in enumerate(held):
            img_t, gd, N_true = targets[6 + j]
            img, D, A, N = (torch.empty((3, H, W), device=dev), torch.empty((H, W), device=dev), torch.empty((H, W), device=dev),
                            torch.empty((3, H, W), device=dev))
            tr.render(c, img, out_depth=D, out_alpha=A, out_normal=N)
            psnr.append(float(-10 * torch.log10(((img - img_t) ** 2).mean())))
            ang.append(_angle_error(N, N_true, A))
            si.append(_si_depth_error(D, A, gd))
        res[run] = dict(psnr=float(np.mean(psnr)), angle=float(np.mean(ang)), si_depth=float(np.mean(si)))
    return res


def _ssim_window(dev):
    g = torch.exp(-((torch.arange(11, dtype=torch.float32) - 5) ** 2) / (2 * 1.5 ** 2))
    g = g / g.sum()
    return (g[:, None] * g[None, :]).expand(3, 1, 11, 11).contiguous().to(dev)


def torch_loss(cam, gt, lambda_dssim, lambda_dn, alpha_min, max_rel_jump, dev):
    """loss_fn(image, D, A, N) for trainWithLoss: the built-in (1 - l) L1 + l (1 - SSIM) plus lambda_dn times the consistency term, in
    torch float32 (the term's definition as include/psb200.h states it; no host synchronisation)"""
    H, W = int(cam["H"]), int(cam["W"])
    fx, fy = W / (2.0 * float(cam["tanfovx"])), H / (2.0 * float(cam["tanfovy"]))
    v, u = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32), torch.arange(W, device=dev, dtype=torch.float32), indexing="ij")
    ray = torch.stack([(u + 0.5 - W / 2.0) / fx, (v + 0.5 - H / 2.0) / fy, torch.ones_like(u)], 0)
    win = _ssim_window(dev)
    C1, C2 = 0.01 ** 2, 0.03 ** 2

    def conv(x):
        return torch.nn.functional.conv2d(x[None], win, padding=5, groups=3)[0]

    def loss_fn(img, D, A, N):
        mu1, mu2 = conv(img), conv(gt)
        s11, s22, s12 = conv(img * img) - mu1 * mu1, conv(gt * gt) - mu2 * mu2, conv(img * gt) - mu1 * mu2
        ssim = ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 * mu1 + mu2 * mu2 + C1) * (s11 + s22 + C2))
        colour = (1 - lambda_dssim) * (img - gt).abs().mean() + lambda_dssim * (1 - ssim.mean())
        keep = A >= alpha_min
        Db = torch.where(keep, D / torch.where(keep, A, torch.ones_like(A)), torch.zeros_like(D))
        X = Db[None] * ray
        a = X[:, 1:-1, 2:] - X[:, 1:-1, :-2]
        b = X[:, 2:, 1:-1] - X[:, :-2, 1:-1]
        c = torch.linalg.cross(a, b, dim=0)
        z = Db.detach()
        zc = z[1:-1, 1:-1]
        ok = torch.isfinite(zc) & (zc > 0)
        for zn in (z[1:-1, :-2], z[1:-1, 2:], z[:-2, 1:-1], z[2:, 1:-1]):
            ok &= torch.isfinite(zn) & (zn > 0) & ~((zn - zc).abs() > max_rel_jump * zc)
        length = c.norm(dim=0)
        ok &= length.detach() > 0
        sign = torch.where((c * X[:, 1:-1, 1:-1]).sum(0).detach() < 0, 1.0, -1.0)
        n = c * (sign / torch.where(ok, length, torch.ones_like(length)))[None]
        term = torch.where(ok, 1.0 - (n * N[:, 1:-1, 1:-1]).sum(0), torch.zeros_like(zc))
        return colour + lambda_dn * term.sum() / ok.sum().clamp_min(1)

    return loss_fn


def cost(config, steps, warmup, rounds, lambda_dn, dev):
    from photo_slam_b200 import trainer as T
    scene, cam, host, devcam, gt_dev = harness.workload(config, dev)
    model = T.GaussianModel.from_numpy(scene, dev)
    model.trainingSetup(T.GaussianOptimizationParams())
    tr = T.GaussianTrainer(model)
    W, H = devcam["W"], devcam["H"]
    loss_fn = torch_loss(devcam, gt_dev, tr.opt.lambda_dssim, lambda_dn, 0.5, 0.05, dev)
    kws = {"colour": {}, "builtin_dn": dict(lambda_dn=lambda_dn)}

    def torch_leg():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            tr.trainWithLoss(devcam, loss_fn, depth=True, alpha=True, normal=True)
        e1.record()
        tr.result()
        torch.cuda.synchronize()
        return 1000.0 * steps / e0.elapsed_time(e1), {}

    for _ in range(max(warmup, 3)):          # also grows the binning arena and the planes of every leg
        for kw in kws.values():
            tr.trainForOneIteration(devcam, gt_dev, **kw)
            tr.result()
        tr.trainWithLoss(devcam, loss_fn, depth=True, alpha=True, normal=True)
        tr.result()
    rewind = harness.rewinder(model, tr)
    legs = {k: (lambda k=k: harness.step_leg(tr, devcam, gt_dev, steps, rewind=rewind, **kws[k])) for k in kws}
    legs["torch_dn"] = torch_leg
    res = harness.alternate(legs, rounds, rewind)
    rewind()
    out = {"gaussians": model.num_points(), "width": W, "height": H}
    for name, r in res.items():
        out[name] = {"value": [x[0] for x in r], "stages": harness.mean_stages([x[1] for x in r])}
    out["dn_stage_cost_ms"] = {k: out["builtin_dn"]["stages"][k] - out["colour"]["stages"][k] for k in out["colour"]["stages"]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="B,D")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--lambda-dn", type=float, default=0.05)
    ap.add_argument("--payoff-steps", type=int, default=300)
    ap.add_argument("--skip-cost", action="store_true")
    ap.add_argument("--skip-payoff", action="store_true")
    a = ap.parse_args()
    dev = harness.device()
    out = {"card": harness.card(), "steps": a.steps, "rounds": a.rounds, "lambda_dn": a.lambda_dn,
           "unit": "iters/s (value), ms (stages), dB (psnr), degrees (angle), log-depth RMS (si_depth)"}
    if not a.skip_cost:
        out["cost"] = {c: cost(c, a.steps, a.warmup, a.rounds, a.lambda_dn, dev) for c in a.configs.split(",")}
    if not a.skip_payoff:
        out["payoff"] = planar_payoff(dev, steps=a.payoff_steps, lambda_dn=a.lambda_dn)
        out["payoff"]["steps"] = a.payoff_steps
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
