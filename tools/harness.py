"""What the A/B benchmarks under tools/ share: bench.py's workloads, the card header, CUDA-event timing and the alternating-leg protocol.

A benchmark compares legs (a feature off and on, two modes, two entry points) in one process. Every leg of a trainer comparison starts
from the same training state (rewinder), the legs take turns, and the order rotates from round to round so that a drift of the card
(clocks, temperature, other work on the host) does not favour one leg. Times come from CUDA events. There is no CPU fallback: without
a CUDA device, device() exits with a message."""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (os.path.join(ROOT, "oracle"), ROOT):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import bench  # noqa: E402  (its workload: make_inputs)

CONFIGS = {"B": (500_000, "replica"), "C": (1_000_000, "tum"), "D": (3_000_000, "replica")}   # as bench.py --config


def device():
    """cuda:0, or exit with a message."""
    if not torch.cuda.is_available():
        sys.exit(f"{os.path.basename(sys.argv[0])} needs a CUDA device")
    return torch.device("cuda", 0)


def workload(config, dev):
    """bench.py's workload at `config` (rank 0): -> (scene, cam, host, devcam, gt) as bench.make_inputs returns them."""
    a = argparse.Namespace(config=config)
    a.points, a.camera = CONFIGS[config]
    return bench.make_inputs(a, 0, dev)


def card():
    """The name, power limit (W) and max SM clock (MHz) of cuda:0, from NVML, else from `nvidia-smi --query-gpu`. Queries only.
    A value that could not be read is "not read: <why>"."""
    uuid = "GPU-" + str(torch.cuda.get_device_properties(0).uuid)
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByUUID(uuid.encode())
        name = pynvml.nvmlDeviceGetName(h)
        return {"name": name if isinstance(name, str) else name.decode(), "power_limit_w": pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0,
                "sm_max_mhz": float(pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)), "source": "nvml"}
    except Exception as e:  # noqa: BLE001
        why = f"nvml: {e}"
    try:
        q = subprocess.run(["nvidia-smi", f"--id={uuid}", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30, check=True).stdout
        name, pl, sm = [x.strip() for x in q.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit_w": float(pl), "sm_max_mhz": float(sm), "source": "nvidia-smi"}
    except Exception as e:  # noqa: BLE001
        why = f"not read: {why}; nvidia-smi: {e}"
    return {"name": torch.cuda.get_device_name(0), "power_limit_w": why, "sm_max_mhz": why, "source": None}


def cuda_ms(fn, reps, warmup=1):
    """Median over `reps` calls of fn() of the CUDA-event time around each call, after `warmup` untimed calls."""
    for _ in range(warmup):
        fn()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    torch.cuda.synchronize()
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def window_ms(fn, n):
    """CUDA-event time of n back-to-back calls of fn(), started on an idle device, divided by n: the mean cost of one call."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def rewinder(model, *trainers):
    """Snapshots `model` and the trainers' iteration counters now; the returned rewind() waits for the device, restores the snapshot
    and resets the counters, so that every leg trains the same iterations from the same state."""
    snap, its = model.snapshot(), [tr.iteration for tr in trainers]

    def rewind():
        torch.cuda.synchronize()
        model.restore(snap)
        for tr, it in zip(trainers, its):
            tr.iteration = it
    return rewind


def alternate(legs, rounds, rewind=None):
    """legs: {name: fn() -> measurement}. Runs every leg once per round, the order rotated by one leg each round (two legs: flipped),
    with rewind() before each leg. -> {name: [measurement of each round]}."""
    names = list(legs)
    out = {k: [] for k in names}
    for r in range(rounds):
        for k in names[r % len(names):] + names[:r % len(names)]:
            if rewind is not None:
                rewind()
            out[k].append(legs[k]())
    return out


def stage_ms(tr, step, n):
    """Mean per-stage times (tr.stage_times(), ms) over n profiled calls of step(), each followed by tr.result()."""
    acc = {}
    tr.set_profiling(True)
    for _ in range(n):
        step()
        tr.result()
        for k, v in tr.stage_times().items():
            acc.setdefault(k, []).append(v)
    tr.set_profiling(False)
    return {k: float(np.mean(v)) for k, v in acc.items()}


def step_leg(tr, cam, gt, steps, rewind=None, profile=True, **kw):
    """One leg of the training step: -> (it/s, {stage: ms}). it/s from CUDA events around `steps` device-input steps
    (trainForOneIteration(cam, gt, **kw); a data-parallel trainer's sync() inside the window), then result(); then, after rewind(),
    the mean stage times of the same `steps` steps profiled (none with profile=False)."""
    sync = getattr(tr, "sync", lambda: None)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        tr.trainForOneIteration(cam, gt, **kw)
    sync()
    e1.record()
    tr.result()
    torch.cuda.synchronize()
    its = 1000.0 * steps / e0.elapsed_time(e1)
    if not profile:
        return its, {}
    if rewind is not None:
        rewind()
    return its, stage_ms(tr, lambda: tr.trainForOneIteration(cam, gt, **kw), steps)


def mean_stages(per_round):
    """{stage: mean over rounds} of a list of {stage: ms}."""
    return {k: float(np.mean([s[k] for s in per_round])) for k in per_round[0]} if per_round else {}
