"""What a loss of the caller's own costs on bench.py's workload: three legs alternating in one process.

    python tools/custom_loss_bench.py [--config B|C|D] [--steps K] [--warmup W] [--rounds R] [--lambda-depth L]

  (a) builtin  GaussianTrainer.trainForOneIteration (built-in L1 + D-SSIM loss, no depth target);
  (b) pixels   GaussianTrainer.trainWithLoss with a torch loss: masked colour L1 + lambda * L1 of the normalised depth D / A over the valid
               pixels (target > 0, A > 0.05), back-propagated through psb_trainer_backward_pixels into the fused Adam;
  (c) operator the same loss through renderer.render (the operator path; A from a second render with colours (1, 0, 0) on black) +
               torch autograd + torch.optim.Adam over the six parameter groups: what such a loss cost before (b) existed.

The target depth is the model's own normalised depth at the start x 1.02 with ~10 % of the pixels zeroed. Every leg restarts from the
same training state and times the same K iterations with CUDA events (one host synchronisation per K steps); the leg order rotates
from round to round. (a) and (b) also report the per-stage times of K profiled steps (GaussianTrainer.STAGES; for (b) "loss" is the
torch loss and its autograd between the two calls).

The opacity variants' own cost is then timed apart from any training: the same model state, K profiled render + backwardPixels
pairs in the gradient mode (the parameters do not move) on fixed random planes, with and without the opacity plane and its gradient,
alternating pair by pair; reported as the mean render_fwd / render_bwd stage times of each and their difference. Prints one JSON line;
writes nothing."""
import argparse
import json

import numpy as np
import torch

import harness


def make_loss(gt, mask, gt_depth, lam):
    def loss_fn(image, depth, alpha):
        l1 = ((image - gt).abs() * mask).mean()
        valid = (gt_depth > 0) & (alpha.detach() > 0.05)
        dn = depth / alpha.clamp_min(1e-3)
        return l1 + lam * ((dn - gt_depth).abs() * valid).sum() / valid.sum().clamp_min(1)
    return loss_fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="D", choices=["B", "C", "D"])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--lambda-depth", type=float, default=0.1)
    a = ap.parse_args()
    dev = harness.device()
    from photo_slam_b200 import renderer
    from photo_slam_b200 import trainer as T
    scene, cam, host, devcam, gt = harness.workload(a.config, dev)
    model = T.GaussianModel.from_numpy(scene, dev)
    model.trainingSetup(T.GaussianOptimizationParams())
    tr = T.GaussianTrainer(model)
    W, H = devcam["W"], devcam["H"]
    d0, a0 = torch.empty((H, W), device=dev), torch.empty((H, W), device=dev)
    tr.render(devcam, torch.empty((3, H, W), device=dev), out_depth=d0, out_alpha=a0)   # also grows the binning arena
    keep = torch.rand((H, W), generator=torch.Generator().manual_seed(1)) >= 0.1
    gt_depth = (d0 / a0.clamp_min(1e-3) * 1.02 * keep.to(dev)).contiguous()
    mask = torch.ones((3, H, W), device=dev)
    mask[:, : H // 10] = 0.0
    loss_fn = make_loss(gt, mask, gt_depth, a.lambda_depth)

    # leg (c): its own copy of the model as autograd leaves, and torch's Adam over the reference's six groups
    op = T.GaussianModel.from_numpy(scene, dev)
    op.active_sh_degree_ = model.active_sh_degree_
    leaves = [t.requires_grad_(True) for t in op.tensors()]
    red = torch.zeros((model.num_points(), 3), device=dev)
    red[:, 0] = 1.0
    black = torch.zeros(3, device=dev)

    def op_step(opt):
        img, _, _, _, depth = renderer.render(devcam, H, W, op, bg_color=tr.background, return_depth=True)
        alpha = renderer.render(devcam, H, W, op, bg_color=black, override_color=red, use_override_color=True)[0][0]
        loss = loss_fn(img, depth, alpha)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()

    def builtin():
        tr.trainForOneIteration(devcam, gt, mask)

    def pixels():
        tr.trainWithLoss(devcam, loss_fn, depth=True, alpha=True)

    for _ in range(max(a.warmup, 2)):
        builtin(); tr.result()
        pixels(); tr.result()
    model_rewind = harness.rewinder(model, tr)
    start = [t.detach().clone() for t in leaves]

    def rewind():
        model_rewind()
        with torch.no_grad():
            for t, s in zip(leaves, start):
                t.copy_(s)
        return torch.optim.Adam([{"params": [t], "lr": lr} for t, lr in zip(leaves, model.lr_)], betas=(0.9, 0.999), eps=1e-15)

    opt = rewind()
    for _ in range(max(a.warmup, 2)):
        op_step(opt)

    def leg(name):
        opt = rewind()
        step = {"builtin": builtin, "pixels": pixels, "operator": lambda: op_step(opt)}[name]
        ms = harness.window_ms(step, a.steps)
        if name == "operator":
            return ms, None
        tr.result()
        rewind()
        return ms, harness.stage_ms(tr, step, a.steps)

    res = harness.alternate({k: (lambda k=k: leg(k)) for k in ("builtin", "pixels", "operator")}, a.rounds)
    # the opacity variants against the same passes without them (gradient mode: no drift between the two)
    rewind()
    gen = torch.Generator().manual_seed(2)
    gc = (1e-4 * torch.randn((3, H, W), generator=gen)).to(dev)
    gd = (1e-5 * torch.randn((H, W), generator=gen)).to(dev)
    ga = (1e-4 * torch.randn((H, W), generator=gen)).to(dev)
    grads = [torch.zeros_like(t) for t in model.tensors()]
    D, A = torch.empty((H, W), device=dev), torch.empty((H, W), device=dev)
    variant = {True: {}, False: {}}
    tr.set_profiling(True)
    for i in range(2 * a.steps + 4):
        with_alpha = i % 2 == 0
        tr.render(devcam, torch.empty((3, H, W), device=dev), check=False, out_depth=D, out_alpha=A if with_alpha else None)
        tr.backwardPixels(gc, gd, ga if with_alpha else None, grads=grads)
        tr.result()
        if i >= 4:
            for k, v in tr.stage_times().items():
                variant[with_alpha].setdefault(k, []).append(v)
    tr.set_profiling(False)
    rewind()
    out = {"config": a.config, "gaussians": model.num_points(), "width": W, "height": H, "steps": a.steps, "rounds": a.rounds,
           "lambda_depth": a.lambda_depth, "card": harness.card(), "unit": "ms per step (CUDA events over K steps), ms per stage (K profiled steps)"}
    for name, r in res.items():
        ms = [x[0] for x in r]
        out[name] = {"ms_per_step": ms, "ms_per_step_mean": float(np.mean(ms))}
        if r[0][1] is not None:
            out[name]["stages"] = harness.mean_stages([x[1] for x in r])
    out["pixels_minus_builtin_stage_ms"] = {k: out["pixels"]["stages"][k] - out["builtin"]["stages"][k] for k in out["builtin"]["stages"]}
    out["opacity_variants"] = {"with_ms": {k: float(np.mean(variant[True][k])) for k in ("render_fwd", "render_bwd")},
                               "without_ms": {k: float(np.mean(variant[False][k])) for k in ("render_fwd", "render_bwd")}}
    out["opacity_variants"]["cost_ms"] = {k: out["opacity_variants"]["with_ms"][k] - out["opacity_variants"]["without_ms"][k]
                                          for k in ("render_fwd", "render_bwd")}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
