"""Worker of tests/test_dp64_multirank_gpu.py: one rank of a K-rank NVLink data-parallel step (DataParallelTrainer(mode="p2p",
geometry_terms=True)) with every rank on device 0 (tests/shared_device.py), checked against the float64 step of step64.dp_step64.

usage: dp64_worker.py CASE[,CASE...]   (CASES below; every rank gets the same list)

Per case: rank 0 builds the scene, settles it for every view of the step (step64.margins of each view with its flags; the offenders of all
views are jittered together), seeds moments from the views' summed float64 gradient and broadcasts the state. Each rank trains its own
camera with its own terms (rank 0 normal + dn, 1 dist, 2 depth, 3 none), then sync(), status() == 0 and gather_moments(). Checked:
  - every rank's replica and gathered moments equal rank 0's bit for bit;
  - rank 0's replica and moments against dp_step64, with test_step64_gpu's gates and exact invariants (_compare);
  - each rank's densification statistics against its own view, and after sync_densify_stats() against the sum over the views (the max
    for the radii); each rank's result_dist() scalars against its own view's loss;
  - the scene: the rows and ranks each case exists for are there.
Rank 0 prints `MEASURED <case> <json>` per step, `PERTURBED <case> <what> <err>` per perturbed truth and `OK <case>` at the end of a
case; any failed check raises, and the launch fails."""
import dataclasses
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import photo_slam_b200.synthetic as syn  # noqa: E402
import shared_device  # noqa: E402
import splat64 as s64  # noqa: E402
import step64  # noqa: E402
from photo_slam_b200.parallel import CHUNK, owner_of_rows, sh_basis_weights  # noqa: E402
from test_dp64_gpu import _kw, _loss_errs, _tg64  # noqa: E402
from test_step64_gpu import (BG, GATE_ACCUM, H, W, _compare, _maxerr, _model, _pose, _random, _read, _seed_moments,  # noqa: E402
                             _settle, _step_err, _targets, _unseen)

TERMS = [step64.Flags(normal=True, dn=True), step64.Flags(dist=True), step64.Flags(depth=True), step64.Flags()]   # of rank 0..3
P_MAIN = 13 * CHUNK + 93    # 14 chunks: 14 % 3 and 14 % 4 != 0; the partial last chunk (93 rows) is owned by rank 1 at worlds 2, 3, 4
P_SMALL = CHUNK + 72        # 2 chunks: at world 3 rank 2 owns none

# world, P, anti-aliasing, deterministic; steps (cameras rotated by one rank between steps), overflow (the rank whose view is made to
# overflow a fresh binning arena), twice (the case is run twice from the same state: bit-identical), perturb (the perturbed truths)
CASES = {
    "w2-plain": dict(world=2, aa=False, det=True, perturb=True),
    "w2-aa": dict(world=2, aa=True, det=False),
    "w3-plain": dict(world=3, aa=False, det=False, perturb=True),
    "w3-aa": dict(world=3, aa=True, det=True),
    "w4-plain": dict(world=4, aa=False, det=True, perturb=True),
    "w4-aa": dict(world=4, aa=True, det=False),
    "w3-idle-rank": dict(world=3, P=P_SMALL, aa=True, det=False),
    "w4-rotate": dict(world=4, aa=False, det=False, steps=2),
    "w3-overflow": dict(world=3, aa=False, det=True, overflow=2),
    "w3-det-twice": dict(world=3, aa=True, det=True, twice=True),
}


# ---- scene and views ----------------------------------------------------------------------------------------------------------------
def _camera(q, scale=1):
    """view q: four poses whose camera centres lie 0.1 - 0.2 apart (the SH direction of a row at depth 1 turns by ~0.1 rad between
    them), rotated so that each sees rows at the edges the others do not; scale > 1: the same view at scale x the resolution"""
    f = 0.9 * W * scale
    R = [np.eye(3), _pose(1, 0.06)[0], _pose(0, -0.05)[0], _pose(1, -0.05)[0]][q]
    t = [(0.0, 0.0, 0.0), (0.12, -0.02, 0.03), (-0.10, 0.05, 0.0), (0.05, 0.10, -0.05)][q]
    return syn.make_camera(W * scale, H * scale, f, f, R, np.array(t))


def _scene(P, seed):
    """test_step64_gpu's "terminate" recipe at P rows, with the most opaque rows well inside view 0 (which every view sees) swapped into
    the partial last chunk"""
    cam = _camera(0)
    sc = _random(P, cam, seed=seed, scale_px=5.0)
    sc["opacity"][:] = np.abs(sc["opacity"]) + 0.5
    right = sc["xyz"][:, 0] / sc["xyz"][:, 2] > 0.6 * float(cam["tanfovx"])
    sc["xyz"][right, 2] *= -1.0
    _unseen(sc)
    fx = W / (2.0 * float(cam["tanfovx"]))
    x, y, z = sc["xyz"][:, 0], sc["xyz"][:, 1], sc["xyz"][:, 2]
    zs = np.where(z > 0, z, 1.0)
    u, v = x / zs * fx + 0.5 * (W - 1), y / zs * fx + 0.5 * (H - 1)
    inside = (z > 0.6) & (np.abs(u - 0.5 * W) < 0.3 * W) & (np.abs(v - 0.5 * H) < 0.3 * H)
    inside[P - P % CHUNK:] = False
    cand = np.nonzero(inside)[0]
    k = min(P % CHUNK, cand.size)
    src = cand[np.argsort(-sc["opacity"][cand, 0], kind="stable")[:k]]
    dst = np.arange(P - k, P)
    for a in sc.values():
        a[np.concatenate([src, dst])] = a[np.concatenate([dst, src])]
    return sc


class View:
    """what rank r trains on in one step: camera q, the rank's terms, the case's anti-aliasing; big: view q at 10x the resolution with no
    term (it overflows a fresh binning arena)"""

    def __init__(self, q, rank, aa, dev, big=False):
        self.q, self.big = q, big
        self.cam = _camera(q, 10 if big else 1)
        self.c = syn.device_camera(self.cam, dev)
        self.fl = dataclasses.replace(step64.Flags() if big else TERMS[rank], aa=aa)
        if big:
            gen = torch.Generator().manual_seed(40 + q)
            self.tg = dict(gt=torch.rand((3, 10 * H, 10 * W), generator=gen).to(dev), mask=None)
            self.cam64 = self.tg64 = None
        else:
            self.tg = _targets(dev, seed=3 + q)
            self.tg64 = _tg64(self.tg)
            self.cam64 = s64.camera64(self.cam, dev)

    def train(self, tr):
        tr.trainForOneIteration(self.c, self.tg["gt"], self.tg["mask"], **_kw(self.fl, self.tg))

    @property
    def truth(self):
        return self.cam64, self.tg64, self.fl


# ---- rank 0 -------------------------------------------------------------------------------------------------------------------------
def _state(m):
    st = _read(m, step64.Flags(), 0)
    st["E"] = None
    return st


def _settle_views(m, views, seed):
    """_settle with the margins of every view (its flags) at once: the union of their offenders is jittered -> the smallest margin. Four
    views' decisions take more rounds than one view's 60: a jitter that clears a row in one view can bring it near a threshold in another"""
    def margins():
        st, mg = _state(m), {}
        for i, vw in enumerate(views):
            for k, (val, ids) in step64.margins(st, *vw.truth).items():
                key = k if k == "axis" else f"{k}@{i}"      # the axis gap does not depend on the view
                mg[key] = (torch.cat([mg[key][0], val]), torch.cat([mg[key][1], ids])) if key in mg else (val, ids)
        return mg
    with torch.no_grad():
        return _settle(m, margins, seed, tries=300)


def _owner_centre_frest(st, per_view, views, own, world):
    """the f_rest gradient of each view rebuilt from the camera centre of the row's OWNER instead of the sender's -> (per-view results
    with it, [P] rows whose f_rest gradient comes from one sender only, a non-owner, and changes by more than 1e-3 of its norm)"""
    xyz, D = st["params"]["xyz"], st["D"]
    P = xyz.shape[0]
    W_of = torch.stack([sh_basis_weights(xyz, views[q].cam64["campos"], D)[:, 1:] for q in range(world)])   # [world, P, 15]
    W_own = W_of[own, torch.arange(P, device=xyz.device)]
    out, senders, changed = [], torch.zeros(P, dtype=torch.long, device=xyz.device), torch.zeros(P, dtype=torch.bool, device=xyz.device)
    for s, r in enumerate(per_view):
        gm = r["grads"]["features_dc"][:, 0, :] / s64.SH_C0          # the clamp-masked dL/dRGB the record carries
        true = r["grads"]["features_rest"]
        rebuilt = W_of[s][:, :, None] * gm[:, None, :]
        assert float((rebuilt - true).abs().max()) <= 1e-9 * max(float(true.abs().max()), 1e-30), "f_rest = w_k(sender's centre) x dL/dRGB"
        wrong = torch.where((own != s)[:, None, None], W_own[:, :, None] * gm[:, None, :], true)
        senders += (true != 0).reshape(P, -1).any(1).long()
        d = (wrong - true).reshape(P, -1).norm(dim=1) > 1e-3 * true.reshape(P, -1).norm(dim=1)
        changed |= d & (own != s)
        g = dict(r["grads"], features_rest=wrong)
        out.append(dict(r, grads=g))
    return out, changed & (senders == 1)


def _perturbed(name, m, st, views, per_view, world, own, P):
    """the perturbed truths: each must miss the step gate of the groups it changes"""
    nchunks = -(-P // CHUNK)
    last = torch.arange(P, device=own.device) >= (nchunks - 1) * CHUNK
    o_last = int(own[-1])
    s = next(q for q in range(world) if q != o_last and per_view[q]["reached"][last].any())
    cut = dict(per_view[s], grads={k: torch.where(last.reshape(-1, *[1] * (g.dim() - 1)), torch.zeros_like(g), g)
                                   for k, g in per_view[s]["grads"].items()})
    wrong, only = _owner_centre_frest(st, per_view, views, own, world)
    assert int(only.sum()) >= 10, f"{int(only.sum())} rows take their f_rest gradient from one non-owner sender whose centre matters"
    cases = {"owner-centre": (dict(per_view=wrong), ["features_rest"]),
             "grad-scale-1": (dict(per_view=per_view, scale=1.0), list(step64.GROUPS)),
             f"last-chunk-without-rank{s}": (dict(per_view=per_view[:s] + [cut] + per_view[s + 1:]), list(step64.GROUPS))}
    for what, (kw, groups) in cases.items():
        nx = step64.dp_step64(st, [v.truth for v in views], world, **kw)["state"]
        err = max(_step_err(t.detach(), nx["params"][q], st["lr"][i]) for i, (q, t) in enumerate(zip(step64.GROUPS, m.tensors())) if q in groups)
        print(f"PERTURBED {name} {what} {err:.3e} only-non-owner-rows={int(only.sum())}", flush=True)


# ---- every rank ---------------------------------------------------------------------------------------------------------------------
def _bcast(tensors):
    for t in tensors:
        dist.broadcast(t, src=0)


def _same_as_rank0(tensors, what, rank):
    for t in tensors:
        ref = t.clone()
        dist.broadcast(ref, src=0)
        assert torch.equal(ref, t), f"rank {rank}: {what} differs from rank 0's"


def _stats(m):
    return [t.detach().double().cpu() for t in (m.denom_, m.max_radii2D_, m.xyz_gradient_accum_)]


def _gather(obj, world):
    out = [None] * world
    dist.all_gather_object(out, obj)
    return out


def _setup(cfg, rank, world, dev, seed):
    """the case's model on every rank: built, settled and seeded on rank 0, broadcast"""
    P = cfg.get("P", P_MAIN)
    sc = _scene(P, seed)
    m = _model(sc, dev, step64.Flags(), [])
    mg = None
    if rank == 0:
        views = [View(q, q, cfg["aa"], dev) for q in range(world) if q != cfg.get("overflow")]
        mg = _settle_views(m, views, seed)
        st = _state(m)
        g = {k: sum(step64.grads64(st, *v.truth)["grads"][k] for v in views) for k in step64.GROUPS}
        _seed_moments(m, g, None)
    _bcast(m.tensors() + m.exp_avg_ + m.exp_avg_sq_)
    m.invalidateAdamLive()
    return m, mg


def _step(name, cfg, m, tr, k, rank, world, dev, seed, info):
    """step k of the case: rank r trains view (r + k) % world -> rank 0: the errors against the truth"""
    ovf = cfg.get("overflow")
    views = [View((r + k) % world, r, cfg["aa"], dev, big=(r == ovf and k == 0)) for r in range(world)]
    mine = views[rank]
    if rank == 0 and k > 0:                      # the kernels' own state after the last step, settled again for this step's views
        info["margin"] = _settle_views(m, [v for v in views if not v.big], seed + k)
    _bcast(m.tensors())
    before = _gather(_stats(m), world)
    st = _state(m) if rank == 0 else None
    if not mine.big:
        tr.render(mine.c)                        # sizes the binning arena; the overflowing rank's stays fresh
    dist.barrier()
    mine.train(tr)
    res = list(tr.result_dist()[:7])
    tr.sync()
    torch.cuda.synchronize()
    assert tr.status() == 0, f"rank {rank}: a cross-rank wait timed out"
    assert tr.dropped_views == int(mine.big), (rank, tr.dropped_views)
    dist.barrier()
    tr.gather_moments()
    torch.cuda.synchronize()
    _same_as_rank0(m.tensors(), "the parameter replica", rank)
    _same_as_rank0(m.exp_avg_ + m.exp_avg_sq_, "the gathered moments", rank)
    after = _gather(dict(res=res, stats=_stats(m)), world)
    if rank != 0:
        return None
    dropped = tuple(r for r, v in enumerate(views) if v.big)
    per_view = [None if v.big else step64.grads64(st, *v.truth) for v in views]
    r = step64.dp_step64(st, [v.truth for v in views], world, dropped, per_view=per_view)
    r0 = dict(r, state=dict(r["state"], **step64.stats64(st, per_view[0])), visible=per_view[0]["visible"],
              reached=torch.stack([pv["reached"] for pv in per_view if pv is not None]).any(0))
    errs, ex, nidle = _compare(m, st, r0, views[0].fl, exposure_id=None)
    assert nidle > 0
    stats_truth = []
    for q, (v, pv, b, a) in enumerate(zip(views, per_view, before, after)):
        den, rad, acc = a["stats"]
        if pv is None:                           # the dropped view: NaN scalars, and it drew nothing
            assert all(x != x for x in a["res"]) and all(torch.equal(x, y) for x, y in zip(b, a["stats"])), q
            stats_truth.append(dict(denom=b[0], max_radii=b[1], accum=b[2]))
            continue
        tru = step64.stats64(dict(denom=b[0].to(dev), max_radii=b[1].to(dev).reshape(-1), accum=b[2].to(dev)), pv)
        stats_truth.append({k_: t.cpu() for k_, t in tru.items()})
        assert torch.equal(den, stats_truth[-1]["denom"]) and torch.equal(rad.reshape(-1), stats_truth[-1]["max_radii"]), f"rank {q} statistics"
        errs[f"accum-r{q}"] = _maxerr(acc, stats_truth[-1]["accum"])
        errs.update({f"{k_}-r{q}": e for k_, e in _loss_errs(a["res"], pv, v.fl).items()})
    own = owner_of_rows(st["params"]["xyz"].shape[0], world, dev)
    info.update(excluded=sum(ex.values()), views=[v.q for v in views], terms=[step64.flag_name(v.fl) for v in views], dropped=list(dropped))
    return dict(errs=errs, per_view=per_view, st=st, views=views, own=own, stats_truth=stats_truth, r=r)


def _check_scene(name, cfg, out, world, P, prev):
    """the rows and ranks each case exists for"""
    own, per_view = out["own"], out["per_view"]
    nchunks = -(-P // CHUNK)
    last = torch.arange(P, device=own.device) >= (nchunks - 1) * CHUNK
    o_last = int(own[-1])
    if P % CHUNK == 0 or o_last == 0:
        raise AssertionError(f"{name}: the last chunk must be partial and owned by a rank other than 0 ({P}, owner {o_last})")
    if world > 2:
        assert nchunks % world != 0, f"{name}: the ranks must own different numbers of chunks"
    others = [q for q, pv in enumerate(per_view) if pv is not None and q != o_last and pv["reached"][last].any()]
    assert others, f"{name}: no rank other than the owner reaches a row of the partial last chunk"
    if "P" in cfg:
        assert nchunks < world, f"{name}: some rank must own no chunk"
    if prev is not None:                         # rows a non-owner reached in the last step but does not reach now: its record is stale
        stale = sum(int((pp["reached"] & ~pv["reached"] & (own != q)).sum()) for q, (pp, pv) in enumerate(zip(prev, per_view)))
        assert stale >= 10, f"{name}: {stale} rows carry a stale record of a non-owner"
        return dict(stale_rows=stale, others_in_last_chunk=others)
    return dict(others_in_last_chunk=others)


def run(name, rank, world, dev, seed):
    from photo_slam_b200 import trainer
    cfg = CASES[name]
    assert cfg["world"] == world, (name, world)
    P = cfg.get("P", P_MAIN)
    runs = []
    for rep in range(2 if cfg.get("twice") else 1):
        m, mg = _setup(cfg, rank, world, dev, seed)
        if rep == 1:                             # the first run's starting state, bit for bit
            for t, s in zip(m.tensors() + m.exp_avg_ + m.exp_avg_sq_, runs[0]["init"]):
                t.copy_(s)
            m.invalidateAdamLive()
        init = [t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_]
        tr = trainer.DataParallelTrainer(m, background=torch.tensor(BG, device=dev), antialiasing=cfg["aa"], deterministic=cfg["det"],
                                         geometry_terms=True, mode="p2p")
        assert tr.mode == "p2p", f"rank {rank}: p2p did not connect ({getattr(tr, '_p2p_error', '')}); the NCCL fallback is a failure here"
        prev = None
        for k in range(cfg.get("steps", 1)):
            info = dict(margin=mg)
            out = _step(name, cfg, m, tr, k, rank, world, dev, seed, info)
            if rank == 0:
                info.update(_check_scene(name, cfg, out, world, P, prev))
                print(f"MEASURED {name} step={k} run={rep} det={cfg['det']} " + json.dumps(dict(info, errs=out["errs"])), flush=True)
                if cfg.get("perturb"):
                    _perturbed(name, m, out["st"], out["views"], out["per_view"], world, out["own"], P)
                prev = out["per_view"]
        stats_local = _stats(m)
        tr.sync_densify_stats()
        torch.cuda.synchronize()
        summed = _gather(_stats(m), world)
        if rank == 0:
            assert all(all(torch.equal(a, b) for a, b in zip(summed[0], s)) for s in summed), "summed statistics differ between ranks"
            views_stats = out["stats_truth"]
            den = sum(s["denom"] for s in views_stats)
            rad = torch.stack([s["max_radii"].reshape(-1) for s in views_stats]).amax(0)
            acc = sum(s["accum"] for s in views_stats)
            assert torch.equal(summed[0][0], den) and torch.equal(summed[0][1].reshape(-1), rad), "summed denom / max radii"
            e = _maxerr(summed[0][2], acc)
            assert e < GATE_ACCUM, ("summed accum", e)
            print(f"MEASURED {name} summed-stats run={rep} " + json.dumps(dict(errs={"accum-summed": e})), flush=True)
        runs.append(dict(init=init, out=[t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_], stats=stats_local))
        tr.close()
    if len(runs) == 2:
        assert all(torch.equal(a, b) for a, b in zip(runs[0]["out"], runs[1]["out"])), f"rank {rank}: deterministic mode, two runs differ"
        assert all(torch.equal(a, b) for a, b in zip(runs[0]["stats"], runs[1]["stats"])), f"rank {rank}: statistics of two runs differ"
    dist.barrier()
    if rank == 0:
        print(f"OK {name}", flush=True)


def main():
    got = shared_device.init_rank()
    assert got, "launch through tests/shared_device.py"
    rank, world, dev = got
    for name in sys.argv[1].split(","):
        run(name, rank, world, dev, 500 + 37 * list(CASES).index(name))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
