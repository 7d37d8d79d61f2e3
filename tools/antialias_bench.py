"""Cost and evidence of anti-aliasing (the 2D Mip filter, o' = o h): python tools/antialias_bench.py [--configs B D] [--steps 30]

Cost: at each config the fused step runs with AA off and on, legs alternating in one process and each leg starting from the same model
snapshot; it reports it/s, the per-stage times (psb_trainer_stage_times), the instance count (o' < o shortens the tight lists), and the
operator forward + backward per call. Evidence: a seeded synthetic scene is trained at full resolution with and without AA, then rendered
at 1/2 and 1/4 resolution and compared (PSNR) with area-downsampled full-resolution renders of the target scene.
Prints one JSON object. Writes nothing."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import photo_slam_b200.synthetic as syn  # noqa: E402
from photo_slam_b200 import rasterizer, trainer  # noqa: E402

CONFIGS = {"B": (500_000, "replica"), "D": (3_000_000, "replica")}


def _cam(dev, W, H, fx, fy, pose=None):
    cam = syn.make_camera(W, H, fx, fy, *(pose or (None, None)))
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return cam, dict(viewmatrix=T(cam["viewmatrix"]), projmatrix=T(cam["projmatrix"]), campos=T(cam["campos"]), tanfovx=float(cam["tanfovx"]),
                     tanfovy=float(cam["tanfovy"]), W=W, H=H)


def _leg(sc, c, gt, dev, aa, steps, warmup):
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    tr = trainer.GaussianTrainer(m, antialiasing=aa)
    tr.render(c)
    for _ in range(warmup):
        tr.trainForOneIteration(c, gt)
        tr.result()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        tr.trainForOneIteration(c, gt)
    tr.result()
    torch.cuda.synchronize()
    its = steps / (time.perf_counter() - t0)
    tr.set_profiling(True)
    st = {}
    for _ in range(5):
        tr.trainForOneIteration(c, gt)
        tr.result()
        for k, v in tr.stage_times().items():
            st[k] = st.get(k, 0.0) + v / 5
    n = tr.result()[3]
    return its, st, int(n)


def _operator(sc, c, dev, aa, reps=10):
    act = {k: torch.from_numpy(v).to(dev) for k, v in syn.activate(sc).items()}
    e = torch.empty(0, device=dev)
    bg = torch.zeros(3, device=dev)
    args = (bg, act["means3D"], e, act["opacities"], act["scales"], act["rotations"], 1.0, e, c["viewmatrix"], c["projmatrix"], c["tanfovx"],
            c["tanfovy"], c["H"], c["W"], act["shs"], 3, c["campos"], False)
    dpix = torch.full((3, c["H"], c["W"]), 1e-6, device=dev)
    times = []
    for i in range(reps + 2):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        f = rasterizer.RasterizeGaussiansCUDA(*args, antialiasing=aa)
        rasterizer.RasterizeGaussiansBackwardCUDA(bg, act["means3D"], f[2], e, act["scales"], act["rotations"], 1.0, e, c["viewmatrix"],
                                                  c["projmatrix"], c["tanfovx"], c["tanfovy"], dpix, act["shs"], 3, c["campos"], f[3], f[0], f[4], f[5],
                                                  antialiasing=aa)
        torch.cuda.synchronize()
        if i >= 2:
            times.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(times))


def cost(dev, config, steps, warmup, rounds):
    P, camname = CONFIGS[config]
    W, H, fx, fy = syn.CAMERAS[camname]
    cam, c = _cam(dev, W, H, fx, fy)
    sc = syn.make_scene(P, cam, seed=0)
    gt = torch.from_numpy(syn.target_image(H, W)).to(dev)
    res = {"off": [], "on": []}
    for _ in range(rounds):
        for aa in (False, True):
            res["on" if aa else "off"].append(_leg(sc, c, gt, dev, aa, steps, warmup))
    out = {}
    for k, legs in res.items():
        stages = {s: round(float(np.mean([x[1][s] for x in legs])), 3) for s in legs[0][1]}
        out[k] = {"it_s": [round(x[0], 1) for x in legs], "stage_ms": stages,
                  "instances": legs[-1][2], "operator_fwd_bwd_ms": round(_operator(sc, c, dev, k == "on"), 3)}
    return out


def evidence(dev, steps=300):
    """train at 600x340 with and without AA; PSNR of 1/2 and 1/4 renders against the area-downsampled full-resolution target render"""
    W, H = 600, 340
    rng = np.random.default_rng(1)
    poses = [syn.random_pose(rng, max_angle=0.1, max_trans=0.1) for _ in range(8)]
    cams = [_cam(dev, W, H, 300.0, 300.0, p) for p in poses]
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
                _, cs = _cam(dev, W // f, H // f, 300.0 / f, 300.0 / f, pose)
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
    dev = torch.device("cuda:0")
    props = torch.cuda.get_device_properties(dev)
    try:
        import subprocess
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True).stdout.strip()
    except Exception:  # noqa: BLE001
        pl = "unknown"
    res = {"gpu": props.name, "power_limit": pl, "cost": {cfg: cost(dev, cfg, a.steps, a.warmup, a.rounds) for cfg in a.configs}}
    if a.evidence_steps > 0:
        res["evidence"] = evidence(dev, a.evidence_steps)
    print(json.dumps(res))
