"""Cost and evidence of anti-aliasing (the 2D Mip filter, o' = o h): python tools/antialias_bench.py [--configs B D] [--steps 30]

Cost: at each config the fused step runs with AA off and on, legs alternating in one process and each leg starting from the same model
snapshot; it reports it/s, the per-stage times (psb_trainer_stage_times), the instance count (o' < o shortens the tight lists), and the
operator forward + backward per call. Evidence: a seeded synthetic scene is trained at full resolution with and without AA, then rendered
at 1/2 and 1/4 resolution and compared (PSNR) with area-downsampled full-resolution renders of the target scene.
Prints one JSON object. Writes nothing."""
import argparse
import json

import numpy as np
import torch

import harness
import photo_slam_b200.synthetic as syn
from photo_slam_b200 import rasterizer, trainer


def _operator(sc, c, dev, aa, reps=10):
    act = {k: torch.from_numpy(v).to(dev) for k, v in syn.activate(sc).items()}
    e = torch.empty(0, device=dev)
    bg = torch.zeros(3, device=dev)
    args = (bg, act["means3D"], e, act["opacities"], act["scales"], act["rotations"], 1.0, e, c["viewmatrix"], c["projmatrix"], c["tanfovx"],
            c["tanfovy"], c["H"], c["W"], act["shs"], 3, c["campos"], False)
    dpix = torch.full((3, c["H"], c["W"]), 1e-6, device=dev)

    def call():
        f = rasterizer.RasterizeGaussiansCUDA(*args, antialiasing=aa)
        rasterizer.RasterizeGaussiansBackwardCUDA(bg, act["means3D"], f[2], e, act["scales"], act["rotations"], 1.0, e, c["viewmatrix"],
                                                  c["projmatrix"], c["tanfovx"], c["tanfovy"], dpix, act["shs"], 3, c["campos"], f[3], f[0], f[4], f[5],
                                                  antialiasing=aa)
    return harness.cuda_ms(call, reps, warmup=2)


def cost(dev, config, steps, warmup, rounds):
    sc, _, _, c, gt = harness.workload(config, dev)
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    trs = {"off": trainer.GaussianTrainer(m, antialiasing=False), "on": trainer.GaussianTrainer(m, antialiasing=True)}
    rewind = harness.rewinder(m, *trs.values())   # every leg starts from the untrained model: the warm-up grows the arenas
    for _ in range(warmup):
        for tr in trs.values():
            tr.trainForOneIteration(c, gt)
            tr.result()
    res = harness.alternate({k: (lambda tr=tr: harness.step_leg(tr, c, gt, steps, rewind)) for k, tr in trs.items()}, rounds, rewind)
    instances = {}
    for k, tr in trs.items():      # read after as many steps as a leg used to take: its warm-up, timed and 5 profiled steps
        rewind()
        for _ in range(warmup + steps + 5):
            tr.trainForOneIteration(c, gt)
        instances[k] = int(tr.result()[3])
    rewind()
    out = {}
    for k, legs in res.items():
        stages = {s: round(v, 3) for s, v in harness.mean_stages([x[1] for x in legs]).items()}
        out[k] = {"it_s": [round(x[0], 1) for x in legs], "stage_ms": stages,
                  "instances": instances[k], "operator_fwd_bwd_ms": round(_operator(sc, c, dev, k == "on"), 3)}
    return out


def evidence(dev, steps=300):
    """train at 600x340 with and without AA; PSNR of 1/2 and 1/4 renders against the area-downsampled full-resolution target render"""
    W, H = 600, 340
    rng = np.random.default_rng(1)
    poses = [syn.random_pose(rng, max_angle=0.1, max_trans=0.1) for _ in range(8)]
    cams = [syn.make_camera(W, H, 300.0, 300.0, *p) for p in poses]
    cams = [(cam, syn.device_camera(cam, dev)) for cam in cams]
    target = syn.make_scene(40_000, cams[0][0], seed=11, scale_px=1.2)     # small splats: the case the filter is for
    tm = trainer.GaussianModel.from_numpy(target, dev)
    gts = [trainer.GaussianTrainer(tm).render(c) for _, c in cams]
    out = {}
    for aa in (False, True):
        m = trainer.GaussianModel.from_numpy(syn.make_scene(40_000, cams[0][0], seed=12, scale_px=1.2), dev)
        m.trainingSetup(trainer.GaussianOptimizationParams())
        tr = trainer.GaussianTrainer(m, antialiasing=aa)
        for it in range(steps):
            k = it % len(cams)
            tr.trainForOneIteration(cams[k][1], gts[k], densify_stats=False)
            tr.result()
        row = {}
        for f in (1, 2, 4):
            ps = []
            for (cam, c), (pose, gt) in zip(cams, zip(poses, gts)):
                cs = syn.device_camera(syn.make_camera(W // f, H // f, 300.0 / f, 300.0 / f, *pose), dev)
                img = tr.render(cs)
                ref = torch.nn.functional.avg_pool2d(gt[None], f)[0] if f > 1 else gt
                mse = ((img - ref[:, :img.shape[1], :img.shape[2]]) ** 2).mean().item()
                ps.append(10 * np.log10(1.0 / max(mse, 1e-12)))
            row[f"psnr_1/{f}"] = round(float(np.mean(ps)), 3)
        out["aa" if aa else "plain"] = row
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="*", default=["B", "D"])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--evidence-steps", type=int, default=300)
    a = ap.parse_args()
    dev = harness.device()
    res = {"card": harness.card(), "cost": {cfg: cost(dev, cfg, a.steps, a.warmup, a.rounds) for cfg in a.configs}}
    if a.evidence_steps > 0:
        res["evidence"] = evidence(dev, a.evidence_steps)
    print(json.dumps(res))
