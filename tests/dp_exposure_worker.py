"""Worker of tests/test_dp_exposure_gpu.py: one rank of a K-rank NVLink data-parallel step with exposure compensation
(DataParallelTrainer(mode="p2p", geometry_terms=True, exposure=True)), every rank on device 0 (tests/shared_device.py), checked against
float64 truth built from step64.grads64(...)["E"] and step64.adam64.

usage: dp_exposure_worker.py CASE[,CASE...]   (CASES below; every rank gets the same list)

Per case: rank 0 builds tests/dp64_worker.py's scene with a four-row exposure table (non-identity rows, seeded moments, different step
counts), settles it for every view and broadcasts it. Rank r trains camera r with dp64_worker's terms for rank r, through row ids[r] (None:
no exposure) with learning rate lrs[r]. Checked:
  - every rank's Gaussian replica and exposure table (rows, moments, step counts) equal rank 0's bit for bit;
  - rank 0's replica and moments against step64.dp_step64 of the views' float64 gradients, each view through its own row, with
    test_step64_gpu's gates;
  - every trained row against g_k = (1/world) sum of dL_r/dE_k over the non-dropped ranks with id k, one adam64 step at step count
    step_k + 1 with the lr of the lowest such rank: the step (in units of that lr) and the moments with test_step64_gpu's gates, the step
    count exactly; a row with lr 0 keeps its value bit for bit;
  - every row no non-dropped rank trained keeps its row, moments and step count bit for bit.
Rank 0 prints `MEASURED <case> <json>` and `OK <case>`; any failed check raises, and the launch fails."""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import shared_device  # noqa: E402
import step64  # noqa: E402
from dp64_worker import P_MAIN, View, _bcast, _same_as_rank0, _scene, _settle_views, _state  # noqa: E402
from test_dp64_gpu import _kw  # noqa: E402
from test_step64_gpu import BG, GATE_MOM, GATE_STEP, _compare, _model, _relnorm, _seed_moments, _step_err  # noqa: E402

K = 4
ROWS = [[[1.3, 0.1, -0.08, 0.05], [0.04, 0.7, 0.09, -0.06], [-0.07, 0.05, 1.2, 0.03]],
        [[0.8, -0.05, 0.06, -0.04], [0.07, 1.25, -0.03, 0.02], [0.05, -0.08, 0.9, -0.05]],
        [[1.1, 0.02, 0.03, 0.02], [-0.03, 0.95, 0.05, 0.04], [0.02, 0.06, 1.15, -0.02]],
        [[0.9, 0.06, -0.02, -0.03], [0.05, 1.05, -0.06, 0.01], [-0.04, 0.03, 0.85, 0.06]]]
STEPS = [3, 0, 7, 1]          # the rows' step counts before the case
LR = 0.01

# world, anti-aliasing, deterministic, ids (None: no exposure), lrs (default LR), overflow (the rank whose view overflows), twice
CASES = {
    "w2-distinct": dict(world=2, aa=False, det=True, ids=[0, 1]),
    "w4-distinct-aa": dict(world=4, aa=True, det=False, ids=[3, 2, 1, 0]),
    "w3-shared": dict(world=3, aa=False, det=False, ids=[1, 1, 2], lrs=[0.01, 0.03, 0.02]),
    "w3-none": dict(world=3, aa=True, det=True, ids=[0, None, 2]),
    "w4-lr0": dict(world=4, aa=False, det=True, ids=[0, 1, 2, 3], lrs=[0.01, 0.01, 0.0, 0.02]),
    "w3-drop-alone": dict(world=3, aa=False, det=True, ids=[0, 1, 3], overflow=2),
    "w3-drop-shared": dict(world=3, aa=False, det=False, ids=[1, 2, 1], overflow=2),
    "w3-det-twice": dict(world=3, aa=True, det=True, ids=[0, 0, 2], twice=True),
}


def _table(m):
    return [m.exposure_, m.exposure_exp_avg_, m.exposure_exp_avg_sq_, m.exposure_step_]


def _setup(cfg, rank, world, dev, seed):
    m = _model(_scene(P_MAIN, seed), dev, step64.Flags(), [])
    m.ensureExposures(K)
    gen = torch.Generator(device=dev).manual_seed(seed)
    for k in range(K):
        m.exposure_[k] = torch.tensor(ROWS[k], device=dev)
        m.exposure_exp_avg_[k] = 1e-3 * (2 * torch.rand((3, 4), generator=gen, device=dev) - 1)
        m.exposure_exp_avg_sq_[k] = 1e-6 * (0.5 + torch.rand((3, 4), generator=gen, device=dev))
    m.exposure_step_.copy_(torch.tensor(STEPS, dtype=torch.int32, device=dev))
    if rank == 0:
        views = [View(q, q, cfg["aa"], dev) for q in range(world) if q != cfg.get("overflow")]
        _settle_views(m, views, seed)
        st = _state(m)
        g = {k: sum(step64.grads64(st, *v.truth)["grads"][k] for v in views) for k in step64.GROUPS}
        _seed_moments(m, g, None)
    _bcast(m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + _table(m))
    m.invalidateAdamLive()
    return m


def _with_row(st, m, k):
    """step64's state with exposure row k of the table (None: no exposure)"""
    if k is None:
        return st
    d = lambda t: t.detach().double().clone()
    return dict(st, E=d(m.exposure_[k]), E_m=d(m.exposure_exp_avg_[k]), E_v=d(m.exposure_exp_avg_sq_[k]), E_step=int(m.exposure_step_[k]))


def _step(name, cfg, m, tr, rank, world, dev):
    ids, lrs, ovf = cfg["ids"], cfg.get("lrs", [LR] * world), cfg.get("overflow")
    views = [View(r, r, cfg["aa"], dev, big=(r == ovf)) for r in range(world)]
    mine = views[rank]
    m.exposure_lr_ = lrs[rank]
    before = [t.clone() for t in _table(m)]
    st = _state(m) if rank == 0 else None
    if not mine.big:
        tr.render(mine.c)                        # sizes the binning arena; the overflowing rank's stays fresh
    dist.barrier()
    tr.trainForOneIteration(mine.c, mine.tg["gt"], mine.tg["mask"], exposure_id=ids[rank], **_kw(mine.fl, mine.tg))
    tr.result_dist()
    tr.sync()
    torch.cuda.synchronize()
    assert tr.status() == 0, f"rank {rank}: status {tr.status()}"
    assert tr.dropped_views == int(mine.big), (rank, tr.dropped_views)
    dist.barrier()
    tr.gather_moments()
    torch.cuda.synchronize()
    _same_as_rank0(m.tensors(), "the parameter replica", rank)
    _same_as_rank0(m.exp_avg_ + m.exp_avg_sq_, "the gathered moments", rank)
    _same_as_rank0(_table(m), "the exposure table", rank)
    if rank != 0:
        return None
    dropped = tuple(r for r, v in enumerate(views) if v.big)
    E0 = [t.clone() for t in before]
    per_view = [None if v.big else step64.grads64(_with_row(st, _Table(E0), ids[r]), *v.truth) for r, v in enumerate(views)]
    r = step64.dp_step64(st, [v.truth for v in views], world, dropped, per_view=per_view)
    r0 = dict(r, state=dict(r["state"], **step64.stats64(st, per_view[0])), visible=per_view[0]["visible"],
              reached=torch.stack([pv["reached"] for pv in per_view if pv is not None]).any(0))
    errs, ex, nidle = _compare(m, st, r0, views[0].fl, exposure_id=None)
    # the table: every id a non-dropped rank trained takes one step from the mean gradient, with the lowest such rank's lr
    trained = {}
    for q, k in enumerate(ids):
        if k is not None and q not in dropped:
            trained.setdefault(k, []).append(q)
    d = lambda t: t.detach().double()
    for k in range(K):
        row, mm, vv, stp = (t[k] for t in _table(m))
        if k not in trained:
            assert all(torch.equal(t[k], b[k]) for t, b in zip(_table(m), before)), f"{name}: row {k} moved without a valid record"
            continue
        g = sum(per_view[q]["E"] for q in trained[k]) / world
        lr = lrs[trained[k][0]]
        t = int(before[3][k]) + 1
        p1, m1, v1 = step64.adam64(d(before[0][k]), g, d(before[1][k]), d(before[2][k]), lr, t)
        assert int(stp) == t, (name, k, int(stp), t)
        if lr > 0:
            errs[f"step-exposure{k}"] = _step_err(row, p1, lr)
        else:
            assert torch.equal(row, before[0][k]), f"{name}: row {k} with lr 0 moved"
        errs[f"mom-m-exposure{k}"] = _relnorm(mm, m1)
        errs[f"mom-v-exposure{k}"] = _relnorm(vv, v1)
    return dict(errs=errs, excluded=sum(ex.values()), trained={str(k): v for k, v in trained.items()}, dropped=list(dropped))


class _Table:
    """the exposure part of a model, from saved tensors (the state before the step)"""

    def __init__(self, t):
        self.exposure_, self.exposure_exp_avg_, self.exposure_exp_avg_sq_, self.exposure_step_ = t


def run(name, rank, world, dev, seed):
    from photo_slam_b200 import trainer
    cfg = CASES[name]
    assert cfg["world"] == world, (name, world)
    runs = []
    for rep in range(2 if cfg.get("twice") else 1):
        m = _setup(cfg, rank, world, dev, seed)
        if rep == 1:
            for t, s in zip(m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + _table(m), runs[0]["init"]):
                t.copy_(s)
            m.invalidateAdamLive()
        init = [t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + _table(m)]
        tr = trainer.DataParallelTrainer(m, background=torch.tensor(BG, device=dev), antialiasing=cfg["aa"], deterministic=cfg["det"],
                                         geometry_terms=True, exposure=True, mode="p2p")
        assert tr.mode == "p2p", f"rank {rank}: p2p did not connect ({getattr(tr, '_p2p_error', '')})"
        out = _step(name, cfg, m, tr, rank, world, dev)
        if rank == 0:
            print(f"MEASURED {name} run={rep} det={cfg['det']} " + json.dumps(out), flush=True)
        runs.append(dict(init=init, out=[t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + _table(m)]))
        tr.close()
    if len(runs) == 2:
        assert all(torch.equal(a, b) for a, b in zip(runs[0]["out"], runs[1]["out"])), f"rank {rank}: deterministic mode, two runs differ"
    dist.barrier()
    if rank == 0:
        print(f"OK {name}", flush=True)


def main():
    got = shared_device.init_rank()
    assert got, "launch through tests/shared_device.py"
    rank, world, dev = got
    for name in sys.argv[1].split(","):
        run(name, rank, world, dev, 700 + 41 * list(CASES).index(name))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
