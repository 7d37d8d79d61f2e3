"""-m gpu: exposure compensation on the data-parallel steps (DataParallelTrainer(exposure=True)) against float64 truth.

World 1, on every path (p2p: psb_dp_step_table; slabs: psb_trainer_backward_begin_table + _slab x 3 + psb_exposure_apply; flat:
psb_trainer_backward_table + psb_exposure_apply), plain and anti-aliased, colour alone and with a depth term: one step through exposure
row 0 from a settled state with seeded moments (tests/test_dp64_gpu.py's setup), against step64.step64 with that row. The Gaussians, their
moments and the row with its moments meet test_step64_gpu's gates, unchanged; the row's step count advances by one and row 1 keeps its
value, moments and count bit for bit.

Worlds 2, 3 and 4 with the ranks sharing one H100 (tests/dp_exposure_worker.py): distinct ids, two ranks on one id, a rank without
exposure, an id with lr 0, a dropped view whose id nobody else trained, a dropped view whose id another rank trained, and deterministic
mode run twice; every rank's table equals rank 0's bit for bit.

Also: at world 1 the p2p and flat paths leave bit-identical tables; psb_dp_step_table with a NULL table gives the bits of
psb_dp_step_dist in deterministic mode, and a table whose rank trains no row leaves the table untouched and the Gaussians as without it.

Largest values over all cases on an H100 80GB HBM3 (700 W power limit): step 7.0e-6 of the lr (features_rest, slabs, aa); the exposure
rows' steps 3.4e-6 of their lr (world 3, two ranks on one id), their second moments 6.8e-6; the whole file ran in about four minutes.
"""
import json
import os

import pytest
import torch

import photo_slam_b200.synthetic as syn
import shared_device
import step64
from test_dp64_gpu import PATHS, _scene_name, _setup
from test_step64_gpu import BG, LAMBDA_DEPTH, _assert_gates, _compare, _settled_state

pytestmark = pytest.mark.gpu
WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dp_exposure_worker.py")


def _trainer(m, path, fl, det, **kw):
    from photo_slam_b200 import trainer
    tr = trainer.DataParallelTrainer(m, background=torch.tensor(BG, device=m.xyz_.device), antialiasing=fl.aa, deterministic=det,
                                     geometry_terms=True, exposure=True, **PATHS[path], **kw)
    assert tr.mode == PATHS[path]["mode"]
    return tr


def _table(m):
    return [t.clone() for t in (m.exposure_, m.exposure_exp_avg_, m.exposure_exp_avg_sq_, m.exposure_step_)]


def _one_step(cuda, path, fl, scene, det, seed, exposure_id=0):
    """one DataParallelTrainer(exposure=True) step through row exposure_id -> (m, state before, table before, result)"""
    m, tg, tg64, cam = _setup(cuda, fl, scene, seed)
    # moments for the row from the truth's own gradient, as test_step64_gpu seeds them
    st, cam64, _ = _settled_state(m, fl, cam, tg64, seed, exposure_id=0)
    g = step64.grads64(st, cam64, tg64, fl)
    gen = torch.Generator(device=cuda).manual_seed(seed)
    m.exposure_exp_avg_[0] = (0.5 * g["E"] * (2 * torch.rand((3, 4), generator=gen, device=cuda, dtype=torch.float64) - 1)).float()
    m.exposure_exp_avg_sq_[0] = (g["E"] * g["E"] * 0.7 + 1e-12).float()
    m.exposure_step_[0] = 4
    tr = _trainer(m, path, fl, det)
    c = syn.device_camera(cam, cuda)
    tr.render(c)
    st, cam64, mg = _settled_state(m, fl, cam, tg64, seed + 1, exposure_id=0)
    before = _table(m)
    kw = dict(gt_depth=tg["depth"], lambda_depth=LAMBDA_DEPTH) if fl.depth else {}
    tr.trainForOneIteration(c, tg["gt"], tg["mask"], exposure_id=exposure_id, **kw)
    tr.result_dist()
    tr.sync()
    torch.cuda.synchronize()
    assert tr.dropped_views == 0 and tr.status() == 0
    if path == "p2p":
        tr.close()
    return m, st, cam64, tg64, before, mg


CASES = [(p, a, d) for p in PATHS for a in (False, True) for d in (False, True)]


@pytest.mark.parametrize("path,aa,depth", CASES, ids=[f"{p}-{'aa' if a else 'plain'}-{'depth' if d else 'colour'}" for p, a, d in CASES])
def test_world1(cuda, path, aa, depth):
    k = CASES.index((path, aa, depth))
    fl = step64.Flags(depth=depth, aa=aa)
    m, st, cam64, tg64, before, mg = _one_step(cuda, path, fl, _scene_name("normal", aa), k % 2 == 0, 3000 + 10 * k)
    r = step64.step64(st, cam64, tg64, fl)
    errs, ex, nidle = _compare(m, st, r, fl, exposure_id=0)
    assert "step-exposure" in errs and nidle > 0
    assert int(m.exposure_step_[0]) == int(before[3][0]) + 1 == r["state"]["E_step"]
    after = _table(m)
    assert all(torch.equal(a[1], b[1]) for a, b in zip(after, before)), "row 1 moved"
    print(f"MEASURED dp-exposure {path} {step64.flag_name(fl)} margin={mg:.1e} excluded={ex} {errs}")
    _assert_gates(errs)


def _state(m):
    """the model's training state: tensors, moments, table, statistics, then its Adam step count"""
    return [t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + _table(m) + [m.xyz_gradient_accum_, m.denom_, m.max_radii2D_]] + [m.step_]


def _restore(m, saved):
    for t, s in zip(m.tensors() + m.exp_avg_ + m.exp_avg_sq_ + [m.exposure_, m.exposure_exp_avg_, m.exposure_exp_avg_sq_, m.exposure_step_] +
                    [m.xyz_gradient_accum_, m.denom_, m.max_radii2D_], saved[:-1]):
        t.copy_(s)
    m.step_ = saved[-1]
    m.invalidateAdamLive()


def _legs(cuda, fl, scene, seed, legs):
    """one step per leg from the same starting state, bit for bit: legs = [(trainer kwargs, exposure_id, wrap the library or None)] ->
    [(Gaussians and moments, table, result_dist())]"""
    from photo_slam_b200 import trainer
    m, tg, tg64, cam = _setup(cuda, fl, scene, seed)
    c = syn.device_camera(cam, cuda)
    saved = _state(m)
    kw = dict(gt_depth=tg["depth"], lambda_depth=LAMBDA_DEPTH) if fl.depth else {}
    outs = []
    for tkw, eid, wrap in legs:
        _restore(m, saved)
        tr = trainer.DataParallelTrainer(m, background=torch.tensor(BG, device=cuda), antialiasing=fl.aa, deterministic=True, geometry_terms=True,
                                         **tkw)
        if wrap is not None:
            tr.L = wrap(tr.L)
        tr.render(c)
        tr.trainForOneIteration(c, tg["gt"], tg["mask"], exposure_id=eid, **kw)
        res = tr.result_dist()
        tr.sync()
        torch.cuda.synchronize()
        assert tr.status() == 0 and tr.dropped_views == 0
        if wrap is not None:
            assert tr.L.calls == 1
        outs.append(([t.clone() for t in m.tensors() + m.exp_avg_ + m.exp_avg_sq_], _table(m), res))
        tr.close()
    return outs, saved


def test_world1_paths_give_bit_identical_tables(cuda):
    fl = step64.Flags(depth=True)
    outs, saved = _legs(cuda, fl, "terminate", 3500, [(dict(exposure=True, **PATHS[p]), 1, None) for p in ("p2p", "flat", "slabs")])
    assert not torch.equal(outs[0][1][0][1], saved[18][1]), "row 1 did not move"
    for _, tab, _ in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(outs[0][1], tab)), "the paths' tables differ"


def test_null_table_is_dp_step_dist(cuda):
    """psb_dp_step_table(NULL) and a table without a row (id -1) give the Gaussians psb_dp_step_dist gives, bit for bit (deterministic),
    and leave the table as it was"""
    fl = step64.Flags(depth=True, aa=True)
    p2p = PATHS["p2p"]
    outs, saved = _legs(cuda, fl, "clamp", 3600, [(dict(p2p), None, None), (dict(p2p), None, _NullTable), (dict(exposure=True, **p2p), None, None)])
    table0 = saved[18:22]
    for leg, (g, tab, res) in zip(("null", "no-row"), outs[1:]):
        assert all(torch.equal(a, b) for a, b in zip(outs[0][0], g)), f"{leg}: the Gaussians differ from psb_dp_step_dist's"
        assert res == outs[0][2], leg
    for g, tab, res in outs:
        assert all(torch.equal(a, b) for a, b in zip(tab, table0)), "the table moved"


class _NullTable:
    """the library, with psb_dp_step_dist routed to psb_dp_step_table with a NULL table"""

    def __init__(self, L):
        self._L, self.calls = L, 0

    def __getattr__(self, n):
        return getattr(self._L, n)

    def psb_dp_step_dist(self, *a):
        self.calls += 1
        return self._L.psb_dp_step_table(*a[:-1], None, a[-1])


def _run(cases, world, timeout=900):
    why = shared_device.unavailable()
    if why:
        pytest.skip(why)
    codes, out, tails = shared_device.launch(WORKER, [",".join(cases)], world, timeout)
    assert codes == [0] * world, tails
    measured = {}
    for line in out.splitlines():
        print(line)
        if line.startswith("MEASURED "):
            measured.setdefault(line.split()[1], []).append(json.loads(line[line.index("{"):]))
    for c in cases:
        assert f"OK {c}" in out.splitlines() and c in measured, (c, tails)
    for recs in measured.values():
        for rec in recs:
            _assert_gates(rec["errs"])
    return measured


def test_world2(cuda):
    _run(["w2-distinct"], 2)


def test_world3(cuda):
    m = _run(["w3-shared", "w3-none", "w3-drop-alone", "w3-drop-shared", "w3-det-twice"], 3)
    assert m["w3-shared"][0]["trained"] == {"1": [0, 1], "2": [2]}
    assert m["w3-drop-alone"][0]["dropped"] == [2] and "3" not in m["w3-drop-alone"][0]["trained"]
    assert m["w3-drop-shared"][0]["trained"]["1"] == [0]


def test_world4(cuda):
    m = _run(["w4-distinct-aa", "w4-lr0"], 4)
    assert "step-exposure2" not in m["w4-lr0"][0]["errs"] and "mom-m-exposure2" in m["w4-lr0"][0]["errs"]
