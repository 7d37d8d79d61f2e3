"""Cost of the deterministic backward on the rasterizer operator path (psb_rasterize_backward_deterministic through the B1 glue), on
bench.py's scenes at configs B and D (1200x680).

    python tools/operator_deterministic_bench.py [--configs B,D] [--calls K] [--warmup W] [--rounds R]

Per config, one forward with depth (RasterizeGaussiansDepthCUDA) provides the buffers every backward leg reads; the same seeded dL/dpix
and dL/dD feed every leg. Four backward legs (atomic / deterministic, colour only / with the depth gradient) alternate R times in one
process, their order rotating from round to round; each leg times K calls with CUDA events. The colour and depth forwards are timed the
same way in every round, so forward + backward is reported per leg. Prints one JSON line with the medians and ranges over the rounds,
the deterministic scratch size, the largest relative-norm difference between the atomic and deterministic gradients, the device name and
its power limit; writes nothing."""
import argparse
import json

import numpy as np
import torch
import torch.nn.functional as F

import harness

LEGS = ("atomic", "deterministic", "atomic_depth", "deterministic_depth")


def _stats(v):
    return {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v)), "range": float(np.max(v) - np.min(v))}


def run_config(config, a, dev):
    from photo_slam_b200 import _lib
    from photo_slam_b200 import rasterizer as R
    scene, cam, host, c, gt = harness.workload(config, dev)
    P = len(scene["xyz"])
    T = lambda k: torch.from_numpy(scene[k]).to(dev)
    means3D, opac = T("xyz"), torch.sigmoid(T("opacity"))
    scales, rots = torch.exp(T("scaling")), F.normalize(T("rotation"))
    shs = torch.cat((T("features_dc"), T("features_rest")), dim=1).contiguous()
    bg, e = torch.zeros(3, device=dev), torch.empty(0, device=dev)
    H, W = c["H"], c["W"]
    fwd_args = (bg, means3D, e, opac, scales, rots, 1.0, e, c["viewmatrix"], c["projmatrix"], c["tanfovx"], c["tanfovy"], H, W, shs, 3, c["campos"],
                False)
    gen = torch.Generator(device=dev).manual_seed(1)
    dpix = torch.randn((3, H, W), device=dev, generator=gen) / (3 * H * W)
    ddep = torch.randn((H, W), device=dev, generator=gen) / (H * W)
    nr, _, _, radii, gb, bb, ib = R.RasterizeGaussiansDepthCUDA(*fwd_args)
    head = (bg, means3D, radii, e, scales, rots, 1.0, e, c["viewmatrix"], c["projmatrix"], c["tanfovx"], c["tanfovy"], dpix)
    tail = (shs, 3, c["campos"], gb, nr, bb, ib)

    def backward(leg):
        det = leg.startswith("deterministic")
        if leg.endswith("depth"):
            return R.RasterizeGaussiansBackwardDepthCUDA(*head, ddep, *tail, deterministic=det)
        return R.RasterizeGaussiansBackwardCUDA(*head, *tail, deterministic=det)

    forwards = {"colour": lambda: R.RasterizeGaussiansCUDA(*fwd_args), "depth": lambda: R.RasterizeGaussiansDepthCUDA(*fwd_args)}
    for _ in range(a.warmup):
        for f in forwards.values():
            f()
        for leg in LEGS:
            backward(leg)
    fwd_ms = {k: [] for k in forwards}
    bwd_ms = {k: [] for k in LEGS}
    for rnd in range(a.rounds):
        for k in (("colour", "depth") if rnd % 2 == 0 else ("depth", "colour")):
            fwd_ms[k].append(harness.window_ms(forwards[k], a.calls))
        for leg in LEGS[rnd % len(LEGS):] + LEGS[:rnd % len(LEGS)]:
            bwd_ms[leg].append(harness.window_ms(lambda: backward(leg), a.calls))
    # the same gradients up to the order of the sums; the deterministic ones repeat bit for bit
    diff = {}
    for depth in (False, True):
        ga, gd = backward("atomic_depth" if depth else "atomic"), backward("deterministic_depth" if depth else "deterministic")
        gd2 = backward("deterministic_depth" if depth else "deterministic")
        diff["depth" if depth else "colour"] = {
            "max_relnorm_vs_atomic": max(((x - y).double().norm() / (y.double().norm() + 1e-30)).item() for x, y in zip(gd, ga) if y.numel()),
            "repeat_bit_identical": all(torch.equal(x, y) for x, y in zip(gd, gd2))}
    out = {"gaussians": P, "width": W, "height": H, "num_rendered": int(nr),
           "det_scratch_bytes": int(_lib.lib().psb_rasterize_backward_det_bytes(P, int(nr))),
           "forward_ms": {k: _stats(v) for k, v in fwd_ms.items()}, "backward_ms": {k: _stats(v) for k, v in bwd_ms.items()},
           "backward_rounds_ms": bwd_ms, "gradients": diff}
    out["forward_backward_ms"] = {leg: out["forward_ms"]["depth" if leg.endswith("depth") else "colour"]["median"] +
                                  out["backward_ms"][leg]["median"] for leg in LEGS}
    out["deterministic_cost_ms"] = {"colour": out["backward_ms"]["deterministic"]["median"] - out["backward_ms"]["atomic"]["median"],
                                    "depth": out["backward_ms"]["deterministic_depth"]["median"] - out["backward_ms"]["atomic_depth"]["median"]}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="B,D")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=4)
    a = ap.parse_args()
    dev = harness.device()
    out = {"card": harness.card(), "calls": a.calls, "rounds": a.rounds,
           "unit": "ms per call (CUDA events); median and range over the rounds"}
    for config in a.configs.split(","):
        out[config] = run_config(config, a, dev)
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
