"""Cost and evidence of per-keyframe exposure compensation: python tools/exposure_bench.py [--configs B D] [--steps 30]

Cost: at each config the fused step runs with exposure off (trainForOneIteration) and on (exposure_id=0), legs alternating in one process
and each leg starting from the same model snapshot; it reports it/s and the per-stage times (psb_trainer_stage_times; the exposure
kernels count in "loss"). Evidence: a seeded synthetic target scene is rendered from 8 poses and each render goes through a known affine
E*_k (per-channel gains 0.6-1.4, off-diagonal terms and biases within +-0.05; view 0 stays at identity and trains at lr 0, since only
exposures relative to it are identifiable). A model from another seed trains on those targets with and without compensation; reported
are the PSNR of its raw render against the untransformed renders and ||E - E*|| over views 1..7.
Prints one JSON object. Writes nothing."""
import argparse
import json
import math

import numpy as np
import torch

import harness
import photo_slam_b200.synthetic as syn
from photo_slam_b200 import trainer


def cost(dev, config, steps, warmup, rounds):
    sc, _, _, c, gt = harness.workload(config, dev)
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    m.ensureExposures(1)
    tr = trainer.GaussianTrainer(m)
    legs = {"off": None, "on": 0}
    rewind = harness.rewinder(m, tr)   # every leg starts from the untrained model: the warm-up grows the arenas
    for _ in range(warmup):
        for k in legs.values():
            tr.trainForOneIteration(c, gt, exposure_id=k)
            tr.result()
    res = harness.alternate({key: (lambda k=k: harness.step_leg(tr, c, gt, steps, rewind, exposure_id=k)) for key, k in legs.items()}, rounds, rewind)
    rewind()
    return {key: {"it_s": [round(x[0], 1) for x in r], "stage_ms": {s: round(v, 4) for s, v in harness.mean_stages([x[1] for x in r]).items()}}
            for key, r in res.items()}


def evidence(dev, steps, W=600, H=340, views=8, P=40_000):
    rng = np.random.default_rng(1)
    cams = [syn.make_camera(W, H, 300.0, 300.0, *syn.random_pose(rng, max_angle=0.1, max_trans=0.1)) for _ in range(views)]
    cams = [(cam, syn.device_camera(cam, dev)) for cam in cams]
    tm = trainer.GaussianModel.from_numpy(syn.make_scene(P, cams[0][0], seed=11, scale_px=2.0), dev)
    raw = [trainer.GaussianTrainer(tm).render(c) for _, c in cams]
    Es = torch.zeros(views, 3, 4)
    Es[:, :, :3] = torch.eye(3)
    for k in range(1, views):
        Es[k, :, :3] = torch.diag(torch.from_numpy(rng.uniform(0.6, 1.4, 3)).float()) + \
            torch.from_numpy(rng.uniform(-0.05, 0.05, (3, 3))).float() * (1 - torch.eye(3))
        Es[k, :, 3] = torch.from_numpy(rng.uniform(-0.05, 0.05, 3)).float()
    Es = Es.to(dev)
    em = trainer.GaussianModel(device=dev)
    em.ensureExposures(views)
    em.exposure_.copy_(Es)
    targets = [em.applyExposure(img, k).contiguous() for k, img in enumerate(raw)]
    out = {"identity_error": round((torch.eye(3, 4, device=dev) - Es[1:]).norm().item(), 4)}
    for compensate in (False, True):
        m = trainer.GaussianModel.from_numpy(syn.make_scene(P, cams[0][0], seed=12, scale_px=2.0), dev)
        m.trainingSetup(trainer.GaussianOptimizationParams())
        m.ensureExposures(views)
        tr = trainer.GaussianTrainer(m)
        lr = m.exposure_lr_
        for it in range(steps):
            k = it % views
            m.setExposureLearningRate(0.0 if k == 0 else lr)
            tr.trainForOneIteration(cams[k][1], targets[k], densify_stats=False, exposure_id=k if compensate else None)
            tr.result()
        psnr = [10 * math.log10(1.0 / max(((tr.render(c) - ref) ** 2).mean().item(), 1e-12)) for (_, c), ref in zip(cams, raw)]
        row = {"psnr_raw_vs_untransformed": round(float(np.mean(psnr)), 3)}
        if compensate:
            row["exposure_error"] = round((m.exposure_[1:] - Es[1:]).norm().item(), 4)
        out["compensated" if compensate else "plain"] = row
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="*", default=["B", "D"])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--evidence-steps", type=int, default=800)
    a = ap.parse_args()
    dev = harness.device()
    res = {"card": harness.card(), "cost": {cfg: cost(dev, cfg, a.steps, a.warmup, a.rounds) for cfg in a.configs}}
    if a.evidence_steps > 0:
        res["evidence"] = evidence(dev, a.evidence_steps)
    print(json.dumps(res))
