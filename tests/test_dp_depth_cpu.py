"""CPU: the data-parallel depth entry points (psb_dp_step_depth, psb_trainer_backward_begin_depth) reject malformed depth arguments
with PSB_ERR_ARG before any CUDA call, and pass a well-formed one on to their ordinary argument checks."""
import ctypes as C
import math

import pytest

from photo_slam_b200 import trainer


def _call(L, fn, h, d):
    if fn == "psb_dp_step_depth":   # (t, dp, P, M, model, camera, background, gt, mask, step, out_color, radii, depth, stream)
        return L.psb_dp_step_depth(h, None, 10, 16, None, None, None, None, None, None, None, None, C.byref(d), None)
    return L.psb_trainer_backward_begin_depth(h, 10, 16, None, None, None, None, None, None, None, None, C.byref(d), None)


@pytest.mark.parametrize("gt,lam,what", [(None, -1.0, b"lambda_depth must be finite"), (4096, -0.5, b"lambda_depth must be finite"),
                                         (4096, math.nan, b"lambda_depth must be finite"), (4096, math.inf, b"lambda_depth must be finite"),
                                         (4096, 0.0, b"given together"), (None, 0.3, b"given together")])
@pytest.mark.parametrize("fn", ["psb_dp_step_depth", "psb_trainer_backward_begin_depth"])
def test_bad_depth_arguments_are_rejected(fn, gt, lam, what):
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        rc = _call(L, fn, h, trainer._Depth(gt, lam, None))
        assert rc == -1 and what in L.psb_last_error() and fn.encode() in L.psb_last_error(), (fn, rc, L.psb_last_error())
    finally:
        L.psb_trainer_destroy(h)


@pytest.mark.parametrize("fn,what", [("psb_dp_step_depth", b"context not connected"), ("psb_trainer_backward_begin_depth", b"null argument")])
def test_well_formed_depth_argument_reaches_the_ordinary_checks(fn, what):
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        for d in (trainer._Depth(4096, 0.1, None), trainer._Depth(None, 0.0, None)):
            rc = _call(L, fn, h, d)
            assert rc == -1 and what in L.psb_last_error(), (fn, rc, L.psb_last_error())
    finally:
        L.psb_trainer_destroy(h)
