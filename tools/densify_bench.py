"""Time one densifyAndPrune at BASELINE sizes: the fused kernels (psb_densify_plan + psb_densify_apply) vs the reference's op chain restated
with ATen ops on the same GPU (oracle/ref_densify.py = src/gaussian_model.cpp:588-815 op for op). Usage: python tools/densify_bench.py [P ...]
Prints one JSON line per size."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import photo_slam_b200.synthetic as syn  # noqa: E402
from photo_slam_b200 import trainer  # noqa: E402
import ref_densify  # noqa: E402


def state(P, dev):
    sc = syn.make_scene(P, syn.make_camera(1200, 680, 600.0, 600.0), seed=0)
    m = trainer.GaussianModel.from_numpy(sc, dev)
    m.trainingSetup(trainer.GaussianOptimizationParams())
    gen = torch.Generator(device=dev).manual_seed(0)
    for t in m.exp_avg_ + m.exp_avg_sq_:
        t.copy_(torch.rand(t.shape, device=dev, generator=gen))
    m.xyz_gradient_accum_.copy_(torch.rand((P, 1), device=dev, generator=gen) * 0.004)
    m.denom_.fill_(2.0)
    m.max_radii2D_.copy_(torch.rand(P, device=dev, generator=gen) * 50)
    return m


def main():
    dev = torch.device("cuda:0")
    for P in [int(a) for a in sys.argv[1:]] or [500_000, 3_000_000]:
        extent, tau, min_op = 5.0, 0.0017, 0.05      # accum/denom is uniform in [0, 0.002): ~15 % of the rows clone or split
        times_psb, times_ref, counts = [], [], None
        # each arm runs on its own, warm (allocator blocks of the previous repetition are reused, as in a training loop)
        for rep in range(4):
            m = state(P, dev)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if os.environ.get("PSB_DENSIFY_BREAKDOWN"):
                import ctypes as C
                L = trainer._bind()
                stream = torch.cuda.current_stream().cuda_stream
                cfg = trainer._DensifyCfg(tau, min_op, extent, m.percent_dense_, 20, 1, rep)
                ws = torch.empty(L.psb_densify_workspace_bytes(P), dtype=torch.uint8, device=dev)
                cnt = (C.c_int * 5)()
                src = trainer._cmodel_of(**m._rows())
                ta = time.perf_counter()
                L.psb_densify_plan(P, C.byref(src), C.byref(cfg), ws.data_ptr(), cnt, stream)
                tb = tc = td = time.perf_counter()

                def apply(src, dst):   # runs after _out_of_place has allocated the new rows
                    nonlocal tc, td
                    torch.cuda.synchronize()
                    tc = time.perf_counter()
                    rc = L.psb_densify_apply(P, src, dst, cnt[0], C.byref(cfg), ws.data_ptr(), None, stream)
                    torch.cuda.synchronize()
                    td = time.perf_counter()
                    return rc
                m._out_of_place(cnt[0], apply, "psb_densify_apply")
                counts = tuple(cnt)
                print(f"  breakdown P={P}: setup {1e3*(ta-t0):.2f} plan {1e3*(tb-ta):.2f} alloc {1e3*(tc-tb):.2f} apply {1e3*(td-tc):.2f} ms", file=sys.stderr, flush=True)
            else:
                counts = m.densifyAndPrune(tau, min_op, extent, 20, seed=1, offset=rep)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            if rep:
                times_psb.append(1e3 * (t1 - t0))
            del m
        n_ref = None
        for rep in range(4):
            m = state(P, dev)
            st = dict(p=m.tensors(), m=m.exp_avg_, v=m.exp_avg_sq_, accum=m.xyz_gradient_accum_, denom=m.denom_, max_radii=m.max_radii2D_)
            del m
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            ref_densify.densify_and_prune(st, tau, min_op, extent, 20, 0.01, None)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if rep:
                times_ref.append(1e3 * (t2 - t1))
            n_ref = st["p"][0].size(0)
            del st
        assert counts[0] == n_ref, (counts, n_ref)
        row_bytes = 4 * (59 * 3 + 4)
        print(json.dumps({"op": "densifyAndPrune", "gaussians": P, "counts(P_new,kept,clones,children_per_copy,split)": list(counts),
                          "psb_ms": float(np.median(times_psb)), "aten_restatement_ms": float(np.median(times_ref)),
                          "psb_GBps_algorithmic": (counts[1] + counts[0]) * row_bytes / 1e6 / float(np.median(times_psb)),
                          "note": "wall time incl. the output allocation and the one host round trip (new row count); ATen = the reference's op chain on the same GPU"}), flush=True)


if __name__ == "__main__":
    main()
