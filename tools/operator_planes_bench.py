"""Cost of the opacity, normal and second-moment planes on the rasterizer operator path (psb_rasterize_forward_planes /
psb_rasterize_backward_planes through the B1 glue), on bench.py's scenes at configs B and D (1200x680).

    python tools/operator_planes_bench.py [--configs B,D] [--calls K] [--warmup W] [--rounds R]

Per config, five legs alternate R times in one process, their order rotating from round to round: plain (RasterizeGaussiansCUDA ->
RasterizeGaussiansBackwardCUDA) and +A, +N, +M and +A+N+M (RasterizeGaussiansPlanesCUDA -> RasterizeGaussiansBackwardPlanesCUDA with a
gradient on each requested plane). Each leg times K forward and K backward calls with CUDA events. Prints one JSON line with the
per-round times, the per-call cost of each leg over plain, the device name and its power limit; writes nothing."""
import argparse
import json

import numpy as np
import torch
import torch.nn.functional as F

import harness

LEGS = {"plain": (), "alpha": ("alpha",), "normal": ("normal",), "depth2": ("depth2",), "all": ("alpha", "normal", "depth2")}


def run_config(config, a, dev):
    from photo_slam_b200 import rasterizer as R
    scene, cam, host, c, gt = harness.workload(config, dev)
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
    grads = {p: torch.randn(((3, H, W) if p == "normal" else (H, W)), device=dev, generator=gen) / (H * W) for p in ("alpha", "normal", "depth2")}

    def leg(planes):
        last = {}
        if planes:
            kw = {p: True for p in planes}
            fwd = lambda: R.RasterizeGaussiansPlanesCUDA(*fwd_args, **kw)
        else:
            fwd = lambda: R.RasterizeGaussiansCUDA(*fwd_args)

        def forward():
            last["out"] = fwd()
        f_ms = harness.window_ms(forward, a.calls)
        out = last["out"]
        nr, radii, bufs = out[0], out[-4], out[-3:]
        bwd_args = (bg, means3D, radii, e, scales, rots, 1.0, e, c["viewmatrix"], c["projmatrix"], c["tanfovx"], c["tanfovy"], dpix)
        tail = (shs, 3, c["campos"], bufs[0], nr, bufs[1], bufs[2])
        if planes:
            g = [grads[p] if p in planes else None for p in ("alpha", "normal", "depth2")]
            bwd = lambda: R.RasterizeGaussiansBackwardPlanesCUDA(*bwd_args, None, *g, *tail)
        else:
            bwd = lambda: R.RasterizeGaussiansBackwardCUDA(*bwd_args, *tail)
        return f_ms, harness.window_ms(bwd, a.calls), nr

    for _ in range(a.warmup):
        for planes in LEGS.values():
            leg(planes)
    legs = harness.alternate({name: (lambda p=planes: leg(p)) for name, planes in LEGS.items()}, a.rounds)
    out = {"gaussians": len(scene["xyz"]), "width": W, "height": H, "num_rendered": int(legs["plain"][-1][2])}
    for name, r in legs.items():
        out[name] = {"forward_ms": [x[0] for x in r], "backward_ms": [x[1] for x in r]}
        for k in ("forward_ms", "backward_ms"):
            out[name][k + "_mean"] = float(np.mean(out[name][k]))
            out[name][k + "_spread"] = float(np.max(out[name][k]) - np.min(out[name][k]))
    out["cost_over_plain_ms"] = {name: {k: out[name][k + "_mean"] - out["plain"][k + "_mean"] for k in ("forward_ms", "backward_ms")}
                                 for name in LEGS if name != "plain"}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="B,D")
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=4)
    a = ap.parse_args()
    dev = harness.device()
    out = {"card": harness.card(), "calls": a.calls, "rounds": a.rounds, "unit": "ms per call (CUDA events)"}
    for config in a.configs.split(","):
        out[config] = run_config(config, a, dev)
        torch.cuda.empty_cache()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
