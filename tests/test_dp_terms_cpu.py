"""CPU: the data-parallel entry points of the normal, depth-normal consistency and distortion terms (psb_dp_step_dist,
psb_trainer_backward_begin_dist, psb_trainer_backward_dist) reject malformed normal, dn and dist records with PSB_ERR_ARG before any
CUDA call, naming the function, and pass well-formed ones on to their ordinary argument checks."""
import ctypes as C
import math

import pytest
import torch

from photo_slam_b200 import trainer

FNS = ["psb_dp_step_dist", "psb_trainer_backward_begin_dist", "psb_trainer_backward_dist"]


def _call(L, fn, h, normal=None, dn=None, dist=None):
    r = lambda x: C.byref(x) if x is not None else None
    terms = (r(normal), r(dn), r(dist))
    if fn == "psb_dp_step_dist":   # (t, dp, P, M, model, camera, background, gt, mask, step, out_color, radii, depth, normal, dn, dist, stream)
        return L.psb_dp_step_dist(h, None, 10, 16, None, None, None, None, None, None, None, None, None, *terms, None)
    if fn == "psb_trainer_backward_begin_dist":
        return L.psb_trainer_backward_begin_dist(h, 10, 16, None, None, None, None, None, None, None, None, None, *terms, None)
    # (t, P, M, model, camera, background, gt, mask, step, out_color, radii, grads, depth, exposure, exposure_grad, normal, dn, dist, stream)
    return L.psb_trainer_backward_dist(h, 10, 16, None, None, None, None, None, None, None, None, None, None, None, None, *terms, None)


BAD = [
    (dict(normal=trainer._Normal(None, -1.0, None)), b"lambda_normal must be finite"),
    (dict(normal=trainer._Normal(4096, math.nan, None)), b"lambda_normal must be finite"),
    (dict(normal=trainer._Normal(4096, 0.0, None)), b"given together"),
    (dict(normal=trainer._Normal(None, 0.3, None)), b"given together"),
    (dict(dn=trainer._Dn(0.0, 0.5, 0.05, None)), b"lambda_dn must be finite and > 0"),
    (dict(dn=trainer._Dn(math.inf, 0.5, 0.05, None)), b"lambda_dn must be finite and > 0"),
    (dict(dn=trainer._Dn(0.1, 0.0, 0.05, None)), b"alpha_min must lie in (0, 1]"),
    (dict(dn=trainer._Dn(0.1, 1.5, 0.05, None)), b"alpha_min must lie in (0, 1]"),
    (dict(dn=trainer._Dn(0.1, 0.5, -1.0, None)), b"max_rel_jump must be finite and > 0"),
    (dict(dist=trainer._Dist(-0.1, None)), b"lambda_dist must be finite and >= 0"),
    (dict(dist=trainer._Dist(math.nan, None)), b"lambda_dist must be finite and >= 0"),
    # a malformed record behind a well-formed one is still found
    (dict(normal=trainer._Normal(4096, 0.1, None), dist=trainer._Dist(math.inf, None)), b"lambda_dist must be finite and >= 0"),
]


@pytest.mark.parametrize("kw,what", BAD, ids=[f"bad{i}" for i in range(len(BAD))])
@pytest.mark.parametrize("fn", FNS)
def test_bad_term_records_are_rejected_naming_the_function(fn, kw, what):
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        rc = _call(L, fn, h, **kw)
        err = L.psb_last_error()
        assert rc == -1 and what in err and fn.encode() in err, (fn, rc, err)
    finally:
        L.psb_trainer_destroy(h)


GOOD = [dict(normal=trainer._Normal(4096, 0.1, None)), dict(normal=trainer._Normal(None, 0.0, 4096)),
        dict(dn=trainer._Dn(0.05, 0.5, 0.05, None)), dict(dist=trainer._Dist(0.1, None)), dict(dist=trainer._Dist(0.0, 4096)),
        dict(normal=trainer._Normal(4096, 0.1, None), dn=trainer._Dn(0.05, 1.0, 0.05, None), dist=trainer._Dist(1.0, None))]


@pytest.mark.parametrize("fn,what", [("psb_dp_step_dist", b"context not connected"), ("psb_trainer_backward_begin_dist", b"null argument"),
                                     ("psb_trainer_backward_dist", b"grads required")])
def test_well_formed_term_records_reach_the_ordinary_checks(fn, what):
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        for kw in GOOD:
            rc = _call(L, fn, h, **kw)
            assert rc == -1 and what in L.psb_last_error(), (fn, kw, rc, L.psb_last_error())
    finally:
        L.psb_trainer_destroy(h)


def test_data_parallel_trainer_takes_the_terms_with_geometry_terms():
    """Off by default the three terms raise NotImplementedError as before; geometry_terms=True lets them through (the call then needs
    a built trainer). exposure_id raises either way, before any trainer state is needed."""
    import inspect
    sig = inspect.signature(trainer.DataParallelTrainer.trainForOneIteration)
    for k in ("gt_normal", "lambda_normal", "out_normal", "lambda_dn", "out_depth_normal", "lambda_dist", "out_depth2"):
        assert k in sig.parameters
    assert inspect.signature(trainer.DataParallelTrainer.__init__).parameters["geometry_terms"].default is False
    terms = (dict(gt_normal=torch.zeros(3, 2, 2), lambda_normal=0.1), dict(lambda_dn=0.05), dict(lambda_dist=1.0), dict(out_depth2=torch.zeros(2, 2)))
    off = trainer.DataParallelTrainer.__new__(trainer.DataParallelTrainer)
    on = trainer.DataParallelTrainer.__new__(trainer.DataParallelTrainer)
    on.geometry_terms = True
    for kw in terms:
        with pytest.raises(NotImplementedError, match="geometry_terms=True"):
            off.trainForOneIteration(dict(W=2, H=2), None, **kw)
        with pytest.raises(Exception) as e:     # (no model: the call stops at the trainer's state, past the refusal)
            on.trainForOneIteration(dict(W=2, H=2), None, **kw)
        assert not isinstance(e.value, NotImplementedError), e.value
    for tr in (off, on):
        with pytest.raises(NotImplementedError, match="exposure"):
            tr.trainForOneIteration(dict(W=4, H=4), None, exposure_id=0)
    assert "out_normal" in inspect.signature(trainer.DataParallelTrainer.render).parameters
    assert "dL_ddepth2" in inspect.signature(trainer.DataParallelTrainer.backwardPixels).parameters
