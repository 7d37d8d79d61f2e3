"""Float64 numpy restatement of the bounded-budget densification (3DGS-MCMC) as include/psb200.h defines it: the relocation correction, the
opacity-proportional sampling, psb_relocate, psb_grow and the position noise. Random words come from oracle/gs_oracle.c:orc_philox4x32_10
(pinned to the Random123 vectors in test_oracle_cpu.py); the word -> uniform and Box-Muller conventions are the header's. Models are dicts
p / m / v (lists of six arrays), accum, denom, max_radii, exist."""
import ctypes as C
import math

import numpy as np

N_MAX = 51
WIDTH = (3, 3, 45, 1, 3, 4)


def sigmoid(x):
    return 1.0 / (1.0 + np.exp(-np.asarray(x, np.float64)))


def relocation(o, N):
    """(o', D) of one row of opacity o standing for N copies: o' = 1 - (1 - o)^(1/N), D = sum_{a=1..N} sum_{k<a} C(a-1,k) (-1)^k o'^(k+1) / sqrt(k+1)."""
    on = 1.0 - (1.0 - o) ** (1.0 / N)
    D = 0.0
    for a in range(1, N + 1):
        for k in range(a):
            D += math.comb(a - 1, k) * (-1.0) ** k * on ** (k + 1) / math.sqrt(k + 1)
    return on, D


def corrected(opacity_raw, scaling_raw, N, min_opacity):
    """(logit(o'), log(s')) of a picked row with multiplicity N (o' clamped to [min_opacity, 1 - 1e-7], s' = s o / D with the unclamped o')."""
    o = float(sigmoid(opacity_raw))
    on, D = relocation(o, N)
    oc = min(max(on, min_opacity), 1.0 - 1e-7)
    return math.log(oc / (1.0 - oc)), np.log(np.exp(np.asarray(scaling_raw, np.float64)) * o / D)


def philox(ctr, key):
    import oracle_c
    c, k, o = (C.c_uint32 * 4)(*ctr), (C.c_uint32 * 2)(*key), (C.c_uint32 * 4)()
    oracle_c.lib().orc_philox4x32_10(c, k, o)
    return list(o)


def _words(j, sub, seed, offset):
    return philox([j, sub, offset & 0xffffffff, offset >> 32], [seed & 0xffffffff, seed >> 32])


def _u(word):
    """(float32(word) + 0.5) * 2^-32 in float32 arithmetic"""
    return np.float32(np.float32(np.float32(word) + np.float32(0.5)) * np.float32(2.3283064365386963e-10))


def uniform(j, sub, seed, offset):
    """u of draw j: sub = 1 relocate, 2 grow"""
    return min(_u(_words(j, sub, seed, offset)[0]), np.float32(0.99999994))


def normal3(row, seed, step):
    """xi of a row: Box-Muller on the four words of Philox(counter = (row, 0, step), key = seed)"""
    u = [float(_u(w)) for w in _words(row, 0, seed, step)]
    ra, rb = math.sqrt(-2.0 * math.log(min(u[0], 0.99999994))), math.sqrt(-2.0 * math.log(min(u[2], 0.99999994)))
    return np.array([ra * math.cos(2 * math.pi * u[1]), ra * math.sin(2 * math.pi * u[1]), rb * math.cos(2 * math.pi * u[3])])


def sample(weights, u):
    """picks[j] = first row whose inclusive cumulative weight exceeds u_j * total; also the margin |u_j total - nearest boundary| / total"""
    cum = np.cumsum(np.asarray(weights, np.float64))
    total = cum[-1]
    target = np.asarray(u, np.float64) * total
    picks = np.searchsorted(cum, target, side="right")
    picks = np.minimum(picks, len(cum) - 1)
    edges = np.concatenate([[0.0], cum])
    margin = np.minimum(np.abs(target - edges[picks]), np.abs(edges[picks + 1] - target)) / total
    return picks, margin


def _apply(model, picks, targets, min_opacity, iteration, P):
    """corrects the picked rows of model (first P rows) in place and writes each target as a copy of its corrected source"""
    count = np.bincount(picks, minlength=P)
    for i in np.nonzero(count)[0]:
        lo, ls = corrected(model["p"][3][i, 0], model["p"][4][i], min(1 + int(count[i]), N_MAX), min_opacity)
        model["p"][3][i, 0] = lo
        model["p"][4][i] = ls
        for q in range(6):
            model["m"][q][i] = 0
            model["v"][q][i] = 0
    for t, s in zip(targets, picks):
        for q in range(6):
            model["p"][q][t] = model["p"][q][s]
            model["m"][q][t] = 0
            model["v"][q][t] = 0
        model["accum"][t] = model["denom"][t] = 0
        model["max_radii"][t] = 0
        model["exist"][t] = iteration
    return count


def relocate(model, u, min_opacity=0.005, iteration=0):
    """psb_relocate on a float64 copy of the model. -> (model, picks, dead rows, margins); nothing changes without a dead or an alive row."""
    model = {k: ([np.array(a, np.float64) for a in v] if isinstance(v, list) else np.array(v)) for k, v in model.items()}
    o = sigmoid(model["p"][3][:, 0].astype(np.float32)).astype(np.float32)   # the kernel classifies on the float32 sigmoid
    dead = np.nonzero(o <= np.float32(min_opacity))[0]
    if len(dead) == 0 or len(dead) == len(o):
        return model, np.zeros(0, np.int64), dead, np.zeros(0)
    picks, margin = sample(np.where(o > np.float32(min_opacity), o.astype(np.float64), 0.0), np.asarray(u)[:len(dead)])
    _apply(model, picks, dead, min_opacity, iteration, len(o))
    return model, picks, dead, margin


def grow(model, P_new, u, min_opacity=0.005, iteration=0):
    """psb_grow: -> (model of P_new rows, picks, margins)"""
    P = model["p"][0].shape[0]
    n = P_new - P
    ext = lambda a: np.concatenate([np.array(a, np.float64 if a.dtype.kind == "f" else a.dtype), np.zeros((n,) + a.shape[1:], np.float64 if a.dtype.kind == "f" else a.dtype)])
    model = {k: ([ext(a) for a in v] if isinstance(v, list) else ext(np.asarray(v))) for k, v in model.items()}
    if n == 0:
        return model, np.zeros(0, np.int64), np.zeros(0)
    o = sigmoid(model["p"][3][:P, 0].astype(np.float32)).astype(np.float32)
    picks, margin = sample(o.astype(np.float64), np.asarray(u)[:n])
    _apply(model, picks, np.arange(P, P_new), min_opacity, iteration, P)
    return model, picks, margin


def rotation(q):
    q = np.asarray(q, np.float64)
    r, x, y, z = q / max(np.linalg.norm(q), 1e-12)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)],
                     [2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)],
                     [2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)]])


def noise_gate(o):
    return 1.0 / (1.0 + np.exp(-100.0 * ((1.0 - o) - 0.995)))


def noise(xyz, opacity_raw, scaling_raw, rotation_raw, lr_xyz, noise_lr, seed, step, rows=None):
    """xyz + Sigma xi lr_xyz noise_lr g(o) on `rows` (default all), Sigma = R diag(s^2) R^T"""
    out = np.array(xyz, np.float64)
    for i in (range(len(out)) if rows is None else rows):
        R = rotation(rotation_raw[i])
        S = R @ np.diag(np.exp(np.asarray(scaling_raw[i], np.float64)) ** 2) @ R.T
        out[i] += S @ normal3(i, seed, step) * (lr_xyz * noise_lr * noise_gate(float(sigmoid(opacity_raw[i]))))
    return out
