"""CPU: bounded-budget densification (3DGS-MCMC: psb_relocate, psb_grow, psb_trainer_inject_noise, psb_trainer_set_regularizers).

  * the relocation correction is what it claims: N copies of (o', s') have the alpha of the original at the centre, D equals the line
    integral it stands for, N = 1 is the identity;
  * the float64 restatement (tests/mcmc64.py) of sampling, multiplicity, relocate, grow and noise on small models;
  * the entry points reject bad arguments before any CUDA call; the Python surface: parameters, and the data-parallel trainer refuses.
"""
import ctypes as C
import math

import numpy as np
import pytest
from scipy import integrate

import mcmc64
from photo_slam_b200 import _lib, trainer

ONE = 4096  # fake non-null device pointer; never dereferenced because validation fails first


def _model(P, seed=0, dead=0.2):
    rng = np.random.default_rng(seed)
    r = lambda *s: rng.normal(0, 1, s)
    op = rng.normal(0.0, 1.5, (P, 1))
    op[rng.random(P) < dead] = -8.0        # sigmoid = 3.4e-4 <= 0.005: dead
    return dict(p=[r(P, 3), r(P, 1, 3), r(P, 15, 3), op, rng.normal(-3, 0.5, (P, 3)), r(P, 4)],
                m=[r(P, 3), r(P, 1, 3), r(P, 15, 3), r(P, 1), r(P, 3), r(P, 4)],
                v=[abs(r(P, 3)), abs(r(P, 1, 3)), abs(r(P, 15, 3)), abs(r(P, 1)), abs(r(P, 3)), abs(r(P, 4))],
                accum=abs(r(P, 1)), denom=np.full((P, 1), 2.0), max_radii=abs(r(P)), exist=np.arange(P, dtype=np.int32))


@pytest.mark.parametrize("N", [1, 2, 3, 7, 20, 51])
def test_correction_preserves_the_alpha_at_the_centre_and_D_is_the_line_integral(N):
    rng = np.random.default_rng(N)
    for o in list(rng.uniform(0.006, 0.999, 6)) + [0.9999999]:
        on, D = mcmc64.relocation(o, N)
        assert abs(1.0 - (1.0 - on) ** N - o) < 1e-12
        # 1 / sqrt(k + 1) = (1 / sqrt(pi)) int exp(-(k + 1) t^2) dt turns the double sum into the integral of the alpha of N copies
        # of opacity o' along a line through the centre: D = (1 / sqrt(pi)) int 1 - (1 - o' exp(-t^2))^N dt
        val, _ = integrate.quad(lambda t: 1.0 - (1.0 - on * math.exp(-t * t)) ** N, -12, 12, epsabs=1e-13, epsrel=1e-12, limit=400)
        assert abs(D - val / math.sqrt(math.pi)) < 2e-9 * max(D, 1.0), (o, N, D, val / math.sqrt(math.pi))
        if N == 1:
            assert abs(on - o) < 1e-15 and abs(D - o) < 1e-15       # s' = s o / D = s


def test_corrected_row_clamps_the_opacity_and_scales_all_axes_alike():
    lo, ls = mcmc64.corrected(0.3, np.array([-3.0, -2.5, -4.0]), 4, 0.005)
    o = float(mcmc64.sigmoid(0.3))
    on, D = mcmc64.relocation(o, 4)
    assert abs(float(mcmc64.sigmoid(lo)) - on) < 1e-12
    assert np.allclose(ls - np.array([-3.0, -2.5, -4.0]), math.log(o / D), atol=1e-12)
    # a barely alive row split 51 ways: o' falls below min_opacity and is clamped to it
    lo, _ = mcmc64.corrected(math.log(0.01 / 0.99), np.zeros(3), 51, 0.005)
    assert abs(float(mcmc64.sigmoid(lo)) - 0.005) < 1e-12


def test_sampling_picks_the_first_row_past_the_target_and_skips_zero_weights():
    w = np.array([0.0, 0.2, 0.0, 0.5, 0.3, 0.0])
    picks, margin = mcmc64.sample(w, [0.0, 0.1999, 0.2, 0.6999, 0.7, 0.999999])
    assert list(picks) == [1, 1, 3, 3, 4, 4]
    assert margin[0] == 0.0 and margin[2] < 1e-12 and abs(margin[1] - 1e-4) < 1e-9
    u = np.random.default_rng(0).random(200_000)
    freq = np.bincount(mcmc64.sample(w, u)[0], minlength=6) / len(u)
    assert np.abs(freq - w).max() < 5e-3 and freq[0] == freq[2] == freq[5] == 0


def test_relocate_restatement():
    P = 301
    src = _model(P, 1)
    u = np.random.default_rng(2).random(P)
    out, picks, dead, _ = mcmc64.relocate(src, u, 0.005, iteration=9)
    o = mcmc64.sigmoid(src["p"][3][:, 0])
    assert 30 < len(dead) < 100 and len(picks) == len(dead) and (o[dead] <= 0.005).all() and (o[picks] > 0.005).all()
    count = np.bincount(picks, minlength=P)
    for j, t in enumerate(dead):
        s = picks[j]
        assert all(np.array_equal(out["p"][q][t], out["p"][q][s]) for q in range(6))
        assert not any(out["m"][q][t].any() or out["v"][q][t].any() or out["m"][q][s].any() or out["v"][q][s].any() for q in range(6))
        assert out["exist"][t] == 9 and out["accum"][t] == 0 and out["denom"][t] == 0 and out["max_radii"][t] == 0
        N = 1 + count[s]
        assert abs(1.0 - (1.0 - mcmc64.sigmoid(out["p"][3][s, 0])) ** N - o[s]) < 1e-9
        assert np.array_equal(out["p"][0][s], src["p"][0][s]) and out["exist"][s] == s
    rest = np.setdiff1d(np.arange(P), np.concatenate([dead, picks]))
    for k in ("p", "m", "v"):
        assert all(np.array_equal(out[k][q][rest], src[k][q][rest]) for q in range(6))
    # nothing is written without a dead row, or without an alive one
    alive = _model(50, 3, dead=0.0)
    assert all(np.array_equal(a, b) for a, b in zip(mcmc64.relocate(alive, u)[0]["p"], alive["p"]))
    gone = _model(50, 3, dead=1.1)
    assert all(np.array_equal(a, b) for a, b in zip(mcmc64.relocate(gone, u)[0]["m"], gone["m"]))


def test_grow_restatement():
    P, P_new = 200, 210
    src = _model(P, 4)
    out, picks, _ = mcmc64.grow(src, P_new, np.random.default_rng(5).random(10), iteration=3)
    assert out["p"][0].shape == (P_new, 3) and len(picks) == 10
    for j, s in enumerate(picks):
        assert all(np.array_equal(out["p"][q][P + j], out["p"][q][s]) for q in range(6))
        assert not any(out["m"][q][P + j].any() or out["m"][q][s].any() for q in range(6)) and out["exist"][P + j] == 3
    rest = np.setdiff1d(np.arange(P), picks)
    assert all(np.array_equal(out["v"][q][rest], src["v"][q][rest]) for q in range(6))
    assert np.array_equal(out["denom"][:P], src["denom"]) and not out["denom"][P:].any()
    same, _, _ = mcmc64.grow(src, P, [])
    assert all(np.array_equal(a, b) for a, b in zip(same["p"], src["p"]))


def test_noise_restatement_moves_only_nearly_dead_rows_along_their_covariance():
    assert mcmc64.noise_gate(0.0) > 0.37 and mcmc64.noise_gate(0.005) == 0.5 and mcmc64.noise_gate(0.1) < 1e-4
    xi = np.array([mcmc64.normal3(i, 7, 3) for i in range(3000)])
    assert np.abs(xi.mean(0)).max() < 0.06 and np.abs(xi.var(0) - 1).max() < 0.1 and not np.array_equal(xi[0], mcmc64.normal3(0, 7, 4))
    P = 40
    m = _model(P, 6)
    m["p"][4][:] = np.log([0.3, 0.01, 0.01])       # a needle along its local x axis
    out = mcmc64.noise(m["p"][0], m["p"][3][:, 0], m["p"][4], m["p"][5], 1.6e-4, 5e5, seed=1, step=2)
    d = out - m["p"][0]
    o = mcmc64.sigmoid(m["p"][3][:, 0])
    assert np.abs(d[o > 0.1]).max() < 1e-3 * np.abs(d[o <= 0.005]).max()
    for i in np.nonzero(o <= 0.005)[0]:
        axis = mcmc64.rotation(m["p"][5][i])[:, 0]
        assert abs(d[i] @ axis) > 0.99 * np.linalg.norm(d[i])
    part = mcmc64.noise(m["p"][0], m["p"][3][:, 0], m["p"][4], m["p"][5], 1.6e-4, 5e5, seed=1, step=2, rows=[3, 5])
    assert np.array_equal(part[[3, 5]], out[[3, 5]]) and np.array_equal(np.delete(part, [3, 5], 0), np.delete(m["p"][0], [3, 5], 0))


# ---- the C entry points: validation before any CUDA call ---------------------------------------------------------------------------
def _cmodel(full=True):
    m = trainer._Model()
    for i in range(6):
        m.param[i] = ONE
        if full:
            m.exp_avg[i], m.exp_avg_sq[i] = ONE, ONE
    return m


def test_relocate_and_grow_reject_bad_arguments_without_a_device():
    L = trainer._bind()
    good, bad = trainer._RelocateCfg(0.005, 0, 0, 0), trainer._RelocateCfg(1.5, 0, 0, 0)
    nan = trainer._RelocateCfg(float("nan"), 0, 0, 0)
    m, nomom = _cmodel(), _cmodel(False)
    counts = (C.c_int * 2)()
    E = -1
    assert L.psb_relocate(-1, C.byref(m), C.byref(good), ONE, None, counts, None) == E
    assert L.psb_relocate(10, C.byref(m), None, ONE, None, counts, None) == E
    assert L.psb_relocate(10, C.byref(m), C.byref(bad), ONE, None, counts, None) == E
    assert L.psb_relocate(10, C.byref(m), C.byref(nan), ONE, None, counts, None) == E
    assert L.psb_relocate(10, None, C.byref(good), ONE, None, counts, None) == E
    assert L.psb_relocate(10, C.byref(nomom), C.byref(good), ONE, None, counts, None) == E
    assert L.psb_relocate(10, C.byref(m), C.byref(good), None, None, counts, None) == E
    assert L.psb_relocate(10, C.byref(m), C.byref(good), ONE + 4, None, counts, None) == E
    assert b"psb_relocate" in L.psb_last_error()
    assert L.psb_relocate(0, None, C.byref(good), None, None, counts, None) == 0 and list(counts) == [0, 0]
    assert L.psb_grow(10, C.byref(m), C.byref(m), 9, C.byref(good), ONE, None, None) == E
    assert L.psb_grow(10, C.byref(m), C.byref(m), 21, C.byref(good), ONE, None, None) == E
    assert L.psb_grow(10, C.byref(m), C.byref(nomom), 12, C.byref(good), ONE, None, None) == E
    assert L.psb_grow(10, C.byref(m), C.byref(m), 12, C.byref(bad), ONE, None, None) == E
    assert L.psb_grow(10, C.byref(m), C.byref(m), 12, C.byref(good), None, None, None) == E
    assert b"psb_grow" in L.psb_last_error()
    assert L.psb_grow(0, None, None, 0, C.byref(good), None, None, None) == 0
    assert L.psb_relocate_workspace_bytes(0) == 256 and L.psb_relocate_workspace_bytes(1000) >= 1000 * 17
    assert {"psb_relocate", "psb_grow", "psb_relocate_workspace_bytes", "psb_trainer_inject_noise",
            "psb_trainer_set_regularizers"} <= set(_lib.exported_symbols())


def test_trainer_entry_points_reject_bad_arguments_without_a_device():
    L = trainer._bind()
    h = C.c_void_p()
    assert L.psb_trainer_create(C.byref(h)) == 0
    try:
        assert L.psb_trainer_set_regularizers(None, 0.01, 0.01) == -1
        assert L.psb_trainer_set_regularizers(h, -0.01, 0.01) == -1
        assert L.psb_trainer_set_regularizers(h, 0.01, float("inf")) == -1
        assert L.psb_trainer_set_regularizers(h, 0.01, 0.01) == 0 and L.psb_trainer_set_regularizers(h, 0.0, 0.0) == 0
        m = _cmodel(False)
        assert L.psb_trainer_inject_noise(None, 10, C.byref(m), 1e-4, 5e5, 0, 1, 1, None) == -1
        assert L.psb_trainer_inject_noise(h, 10, None, 1e-4, 5e5, 0, 1, 1, None) == -1
        assert L.psb_trainer_inject_noise(h, 10, C.byref(m), -1e-4, 5e5, 0, 1, 1, None) == -1
        assert L.psb_trainer_inject_noise(h, 10, C.byref(m), 1e-4, float("nan"), 0, 1, 1, None) == -1
        assert L.psb_trainer_inject_noise(h, 10, C.byref(m), 1e-4, 5e5, 0, 1, 1, None) == -1       # the context has run no pass
        assert b"latest pass" in L.psb_last_error()
    finally:
        L.psb_trainer_destroy(h)


def test_python_surface_is_off_by_default_and_the_data_parallel_trainer_refuses():
    opt = trainer.GaussianOptimizationParams()
    assert opt.mcmc is False and opt.mcmc_noise_lr == 5e5 and opt.opacity_reg == opt.scale_reg == 0.01
    assert opt.mcmc_min_opacity == 0.005 and opt.mcmc_grow_factor == 1.05 and opt.cap_max > 0
    with pytest.raises(NotImplementedError, match="mcmc"):
        trainer.DataParallelTrainer(object(), trainer.GaussianOptimizationParams(mcmc=True))
