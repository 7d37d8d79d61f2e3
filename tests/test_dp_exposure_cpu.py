"""CPU: exposure compensation on the data-parallel steps (psb_dp_step_table, psb_trainer_backward_begin_table, psb_trainer_backward_table,
psb_exposure_apply) rejects a malformed table with PSB_ERR_ARG before any CUDA call, naming the function; a well-formed one reaches the
ordinary checks; the header and the ctypes record agree; and DataParallelTrainer takes exposure_id only with exposure=True, refusing an id
outside the table it was built with."""
import ctypes as C
import math
import os
import re

import pytest
import torch

from photo_slam_b200 import _lib, trainer

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "psb200.h")
ONE = 4096  # fake non-null device pointer; never dereferenced because validation fails first
FNS = ["psb_dp_step_table", "psb_trainer_backward_begin_table", "psb_trainer_backward_table"]


def _table(**kw):
    f = dict(param=ONE, exp_avg=ONE, exp_avg_sq=ONE, step=ONE, K=4, id=1, lr=0.01, record=ONE)
    f.update(kw)
    return trainer._ExposureTable(f["param"], f["exp_avg"], f["exp_avg_sq"], f["step"], f["K"], f["id"], f["lr"], f["record"])


def _call(L, fn, h, table, depth=None):
    tb = C.byref(table) if table is not None else None
    if fn == "psb_dp_step_table":   # (t, dp, P, M, model, camera, background, gt, mask, step, out_color, radii, depth, normal, dn, dist, table, stream)
        return L.psb_dp_step_table(h, None, 10, 16, None, None, None, None, None, None, None, None, depth, None, None, None, tb, None)
    if fn == "psb_trainer_backward_begin_table":
        return L.psb_trainer_backward_begin_table(h, 10, 16, None, None, None, None, None, None, None, None, depth, None, None, None, tb, None)
    return L.psb_trainer_backward_table(h, 10, 16, None, None, None, None, None, None, None, None, (C.c_void_p * 6)(*[ONE] * 6), depth, None, None,
                                        None, tb, None)


BAD = [
    ("id past K", dict(id=4), b"exposure id must be -1 or lie in [0, K)"),
    ("id -2", dict(id=-2), b"exposure id must be -1 or lie in [0, K)"),
    ("K negative", dict(K=-1, id=-1), b"K >= 0"),
    ("K 0 with an id", dict(K=0, id=0), b"exposure id must be -1 or lie in [0, K)"),
    ("null param", dict(param=None), b"needs param, exp_avg, exp_avg_sq and step"),
    ("null exp_avg", dict(exp_avg=None), b"needs param, exp_avg, exp_avg_sq and step"),
    ("null exp_avg_sq", dict(exp_avg_sq=None), b"needs param, exp_avg, exp_avg_sq and step"),
    ("null step", dict(step=None), b"needs param, exp_avg, exp_avg_sq and step"),
    ("null step, no row", dict(step=None, id=-1), b"needs param, exp_avg, exp_avg_sq and step"),
    ("lr negative", dict(lr=-1e-3), b"exposure lr must be finite and >= 0"),
    ("lr nan", dict(lr=math.nan), b"exposure lr must be finite and >= 0"),
    ("lr inf", dict(lr=math.inf), b"exposure lr must be finite and >= 0"),
]


@pytest.mark.parametrize("what,fields,msg", BAD, ids=[b[0] for b in BAD])
@pytest.mark.parametrize("fn", FNS)
def test_bad_tables_are_rejected_naming_the_function(fn, what, fields, msg):
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        rc = _call(L, fn, h, _table(**fields))
        err = L.psb_last_error()
        assert rc == -1 and msg in err and fn.encode() in err, (fn, rc, err)
    finally:
        L.psb_trainer_destroy(h)


@pytest.mark.parametrize("fn", FNS[1:])
def test_gradient_modes_need_a_record(fn):
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        for k in (1, -1):
            assert _call(L, fn, h, _table(record=None, id=k)) == -1
            assert b"record output" in L.psb_last_error() and fn.encode() in L.psb_last_error()
    finally:
        L.psb_trainer_destroy(h)


@pytest.mark.parametrize("fn,what", [("psb_dp_step_table", b"context not connected"), ("psb_trainer_backward_begin_table", b"null argument"),
                                     ("psb_trainer_backward_table", b"null argument")])
def test_well_formed_tables_reach_the_ordinary_checks(fn, what):
    """A valid table (with a row, without one, an empty table, and no record on the NVLink step) stops at the call's own checks."""
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        goods = [_table(), _table(id=-1), _table(K=0, id=-1, param=None, exp_avg=None, exp_avg_sq=None, step=None), _table(lr=0.0, id=3)]
        if fn == "psb_dp_step_table":
            goods.append(_table(record=None))
        for tb in goods:
            rc = _call(L, fn, h, tb)
            assert rc == -1 and what in L.psb_last_error(), (fn, rc, L.psb_last_error())
    finally:
        L.psb_trainer_destroy(h)


def test_null_table_is_the_dist_call():
    """exposure == NULL: the _dist / _depth call's validation and messages."""
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        bad = trainer._Depth(None, -1.0, None)
        for fn, name in zip(FNS, (b"psb_dp_step_depth", b"psb_trainer_backward_begin_depth", b"psb_trainer_backward_table")):
            assert _call(L, fn, h, None, C.byref(bad)) == -1 and name + b": lambda_depth" in L.psb_last_error(), (fn, L.psb_last_error())
    finally:
        L.psb_trainer_destroy(h)


def test_exposure_apply_rejects_bad_arguments():
    L = trainer._bind()
    st = trainer._Step()
    cases = [(0, ONE, _table(), C.byref(st), 1.0, b"world"), (9, ONE, _table(), C.byref(st), 1.0, b"world"),
             (2, None, _table(), C.byref(st), 1.0, b"records"), (2, ONE, None, C.byref(st), 1.0, b"a table"),
             (2, ONE, _table(), None, 1.0, b"a step"), (2, ONE, _table(id=7), C.byref(st), 1.0, b"exposure id"),
             (2, ONE, _table(param=None), C.byref(st), 1.0, b"needs param"), (2, ONE, _table(lr=-1.0), C.byref(st), 1.0, b"lr"),
             (2, ONE, _table(), C.byref(st), math.nan, b"grad_scale")]
    for world, recs, tb, step, scale, msg in cases:
        rc = L.psb_exposure_apply(world, recs, C.byref(tb) if tb is not None else None, step, scale, None)
        assert rc == -1 and msg in L.psb_last_error() and b"psb_exposure_apply" in L.psb_last_error(), (world, L.psb_last_error())


def test_header_record_matches_ctypes():
    txt = open(HEADER).read()
    body = re.search(r"typedef struct psb_exposure_table \{(.*?)\} psb_exposure_table;", txt, re.S).group(1)
    names = re.findall(r"\b(\w+);", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f[0] for f in trainer._ExposureTable._fields_]
    assert re.search(r"#define PSB_EXPOSURE_RECORD (\d+)", txt).group(1) == str(trainer.EXPOSURE_RECORD) == "16"
    for n in FNS + ["psb_exposure_apply"]:
        assert n in _lib.exported_symbols()


def test_data_parallel_trainer_takes_exposure_only_when_asked():
    """Off by default exposure_id raises NotImplementedError naming the switch; exposure=True lets it through to the table checks."""
    import inspect
    assert inspect.signature(trainer.DataParallelTrainer.__init__).parameters["exposure"].default is False
    off = trainer.DataParallelTrainer.__new__(trainer.DataParallelTrainer)
    with pytest.raises(NotImplementedError, match=r"exposure=True"):
        off.trainForOneIteration(dict(W=4, H=4), None, exposure_id=0)
    on = trainer.DataParallelTrainer.__new__(trainer.DataParallelTrainer)
    on.exposure = True
    with pytest.raises(Exception) as e:    # (no model: the call stops at the trainer's state, past the refusal)
        on.trainForOneIteration(dict(W=4, H=4), None, exposure_id=0)
    assert not isinstance(e.value, NotImplementedError), e.value


class _M:
    """The exposure part of a GaussianModel, on the CPU."""

    def __init__(self, K):
        self.m = trainer.GaussianModel(device="cpu")
        self.m.ensureExposures(K)


def _table_trainer(K, checked=None):
    tr = trainer.DataParallelTrainer.__new__(trainer.DataParallelTrainer)
    tr.exposure = True
    tr.model = _M(K).m
    tr._exp_K = K if checked is None else checked
    tr._exp_rec = torch.zeros(trainer.EXPOSURE_RECORD)
    return tr


def test_exposure_id_outside_the_table_raises_value_error():
    tr = _table_trainer(3)
    for k in (3, 7, -1):
        with pytest.raises(ValueError, match="ensureExposures"):
            tr._exposure_table(k)
    t = tr._exposure_table(2)
    assert (t.K, t.id) == (3, 2) and abs(t.lr - tr.model.exposure_lr_) < 1e-9
    t = tr._exposure_table(None)
    assert (t.K, t.id) == (3, -1)


def test_table_grown_after_the_check_needs_a_rebuild():
    tr = _table_trainer(5, checked=3)
    with pytest.raises(ValueError, match="rebuild"):
        tr._exposure_table(1)
