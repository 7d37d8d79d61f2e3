"""CPU: the depth entry points reject malformed depth arguments with PSB_ERR_ARG before any CUDA call."""
import ctypes as C
import math

import pytest

from photo_slam_b200 import _lib, trainer


@pytest.mark.parametrize("gt,lam,what", [(None, -1.0, b"lambda_depth must be finite"), (4096, -0.5, b"lambda_depth must be finite"),
                                         (4096, math.nan, b"lambda_depth must be finite"), (4096, math.inf, b"lambda_depth must be finite"),
                                         (4096, 0.0, b"given together"), (None, 0.3, b"given together")])
def test_bad_depth_arguments_are_rejected(gt, lam, what):
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        d = trainer._Depth(gt, lam, None)
        for fn in ("psb_trainer_step_depth", "psb_trainer_backward_depth"):
            args = [h, 10, 16, None, None, None, None, None, None, None, None]
            if fn == "psb_trainer_backward_depth":
                args.append(None)
            rc = getattr(L, fn)(*args, C.byref(d), None)
            assert rc == -1 and what in L.psb_last_error(), (fn, rc, L.psb_last_error())
        # a well-formed depth argument passes on to the ordinary checks
        ok = trainer._Depth(4096, 0.1, None)
        rc = L.psb_trainer_step_depth(h, 10, 16, None, None, None, None, None, None, None, None, C.byref(ok), None)
        assert rc == -1 and b"null argument" in L.psb_last_error()
    finally:
        L.psb_trainer_destroy(h)
