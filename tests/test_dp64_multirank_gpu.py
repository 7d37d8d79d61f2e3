"""-m gpu: the NVLink data-parallel step at worlds 2, 3 and 4 against the float64 step of tests/step64.py (dp_step64), with every rank a
process on the one GPU (tests/shared_device.py: CUDA IPC between processes on one device, gloo over loopback, contexts time-sliced).

At world 1 the sender of a record is the owner of its row, so the layer these cases exist for runs in its trivial form there:
  - gaussian_backward_kernel<MODE_PUSH | ...> routes chunk c to owner c % world, local chunk c / world, inbox slot rank * nlocal_max + lc;
  - shard_adam_small_kernel sums up to world records per row, skips stale epoch words, and rebuilds the f_rest gradient from the SENDER's
    camera centre and SH degree;
  - the all-gather of shard_adam_small_kernel and the scalar tail of shard_adam_frest_kernel write every replica; nlocal differs between
    ranks, and a rank may own no chunk; grad_scale = 1 / world, and a dropped view still signals.

Cases (tests/dp64_worker.py): rank r trains its own camera with its own terms (rank 0 normal + dn: MODE_PUSH | NORMAL | DEPTH; 1 dist and
2 depth: MODE_PUSH | DEPTH; 3 none: MODE_PUSH), plain and anti-aliased, deterministic mode alternating. P = 1757 (14 chunks, the last one
93 rows, owned by rank 1; 14 % 3 and 14 % 4 != 0; at world 2 the two cannot both hold, and the last chunk's owner is rank 1) with the rows
inside view 0 swapped into the partial last chunk, so that ranks other than its owner reach them.
  world 2 / 3 / 4    plain and aa; the perturbed truths on the plain case
  idle rank          world 3, P = 200: rank 2 owns no chunk
  rotated cameras    world 4, two steps, the cameras moved by one rank in between: rows a non-owner reached in step 1 and not in step 2
                     must not take its stale record
  dropped view       world 3, rank 2's view is its camera at 10x the resolution, which overflows its fresh binning arena (the other ranks
                     render first): the truth is the other views' sum x 1/3, rank 2's statistics do not move
  deterministic      world 3, the same step twice from the same state: replicas, moments and statistics bit-identical

Gates: test_step64_gpu's, unchanged, on rank 0's replica and moments (identical on every rank, bit for bit), each rank's statistics and
result_dist() scalars, and the statistics after sync_densify_stats(). Largest values measured over all cases on an H100 80GB HBM3 (700 W
power limit); the whole file ran in about four minutes there:
  GATE_STEP 1e-5      7.2e-6 (features_rest, second step of the rotated cameras)
  GATE_MOM 4e-5       3.7e-7 (first moment of the rotation, world 3, aa)
  GATE_LOSS 1e-5      4.8e-6 (ssim, world 4, aa)
  GATE_ACCUM 1e-5     2.3e-6 (the rank without a chunk)
The perturbed truths miss the step gate: the f_rest gradient rebuilt from the owner's camera centre and one sender's records dropped for
the last chunk by 2.0 (the step's sign flips), grad_scale = 1 by 3.0e-2 or more (world 3).
"""
import json
import os
import re

import pytest

import shared_device
from test_step64_gpu import GATE_STEP, _assert_gates

pytestmark = pytest.mark.gpu
WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dp64_worker.py")


def _run(cases, world, timeout=900):
    """launch the worker on `world` ranks of device 0 -> {case: [MEASURED records]}, {case: {what: err}}"""
    why = shared_device.unavailable()
    if why:
        pytest.skip(why)
    codes, out, tails = shared_device.launch(WORKER, [",".join(cases)], world, timeout)
    assert codes == [0] * world, tails
    measured, perturbed = {}, {}
    for line in out.splitlines():
        print(line)
        if line.startswith("MEASURED "):
            name = line.split()[1]
            measured.setdefault(name, []).append(json.loads(line[line.index("{"):]))
        elif line.startswith("PERTURBED "):
            _, name, what, err = line.split()[:4]
            perturbed.setdefault(name, {})[what] = float(err)
    for c in cases:
        assert f"OK {c}" in out.splitlines() and c in measured, (c, tails)
    return measured, perturbed


def _gates(measured):
    for name, recs in measured.items():
        for rec in recs:
            _assert_gates(rec["errs"])


@pytest.mark.parametrize("world", [2, 3, 4])
def test_world(cuda, world):
    """plain and anti-aliased steps at this world size; the perturbed truths of the plain step fail the step gate"""
    measured, perturbed = _run([f"w{world}-plain", f"w{world}-aa"], world)
    _gates(measured)
    p = perturbed[f"w{world}-plain"]
    assert {"owner-centre", "grad-scale-1"} <= set(p) and any(re.match(r"last-chunk-without-rank\d", k) for k in p), p
    for what, err in p.items():
        assert err > GATE_STEP, f"{what}: the gate does not see the perturbation ({err} <= {GATE_STEP})"


def test_rank_without_chunk(cuda):
    _gates(_run(["w3-idle-rank"], 3)[0])


def test_rotated_cameras(cuda):
    measured, _ = _run(["w4-rotate"], 4)
    _gates(measured)
    assert any(r.get("stale_rows", 0) >= 10 for r in measured["w4-rotate"])


def test_dropped_view(cuda):
    measured, _ = _run(["w3-overflow"], 3)
    _gates(measured)
    assert measured["w3-overflow"][0]["dropped"] == [2]


def test_deterministic_twice(cuda):
    _gates(_run(["w3-det-twice"], 3)[0])
