"""K ranks of the NVLink data-parallel step as K processes on ONE GPU.

The step's cross-rank traffic is CUDA IPC (psb_dp_connect -> cudaIpcOpenMemHandle), which also maps memory between two processes on the
same device; its waits are bounded (PSB_DP_TIMEOUT_MS) and sleep between polls, and contexts of different processes time-slice, so a rank
spinning in wait_flags_kernel is preempted and its peers' kernels run. NCCL refuses two ranks on one device: the ranks meet through gloo
over loopback, with a FileStore rendezvous in a temporary directory.

Launcher side: `unavailable()` (a read-only query of the compute mode and MIG) and `launch()`: every worker starts in its own session, and
any exit path of `launch` (timeout included) kills each worker's whole process group, so no worker outlives the call.
Worker side: `init_rank()`."""
import ctypes
import datetime
import os
import signal
import subprocess
import sys
import tempfile
import time

STORE_ENV = "PSB_DP_STORE"          # set by launch(): the FileStore path; its presence selects the shared-device mode of a worker
TIMEOUT_MS = "15000"                # each worker's bound on a cross-rank wait inside the step
CU_DEVICE_ATTRIBUTE_COMPUTE_MODE = 20
COMPUTE_MODES = {0: "Default", 1: "Exclusive Thread", 2: "Prohibited", 3: "Exclusive Process"}


def unavailable():
    """-> None if K processes can share device 0, else the reason they cannot: it is not in the Default compute mode (read with
    cuDeviceGetAttribute, nothing is changed) or it is a MIG instance."""
    import torch
    if not torch.cuda.is_available():
        return "no CUDA device"
    if "MIG-" in os.environ.get("CUDA_VISIBLE_DEVICES", "") or "MIG" in torch.cuda.get_device_name(0):
        return "device 0 is a MIG instance"
    try:
        cu = ctypes.CDLL("libcuda.so.1")
    except OSError as e:
        return f"libcuda not loadable: {e}"
    dev, mode = ctypes.c_int(), ctypes.c_int()
    if cu.cuInit(0) != 0 or cu.cuDeviceGet(ctypes.byref(dev), 0) != 0 or \
            cu.cuDeviceGetAttribute(ctypes.byref(mode), CU_DEVICE_ATTRIBUTE_COMPUTE_MODE, dev) != 0:
        return "the compute mode of device 0 could not be read"
    if mode.value != 0:
        return f"device 0 is in the {COMPUTE_MODES.get(mode.value, mode.value)} compute mode, not Default"
    return None


def launch(script, args, world, timeout):
    """Run `python script *args` as ranks 0..world-1 on device 0 -> (returncodes, rank 0's stdout, every rank's output tail).
    A worker still running after `timeout` seconds is killed with its process group; returncode None marks it."""
    with tempfile.TemporaryDirectory(prefix="psb_dp_") as tmp:
        env = dict(os.environ, WORLD_SIZE=str(world), LOCAL_RANK="0", GLOO_SOCKET_IFNAME="lo", PSB_DP_TIMEOUT_MS=TIMEOUT_MS,
                   **{STORE_ENV: os.path.join(tmp, "store")})
        env.pop("PSB_DP_MODE", None)
        procs, logs = [], []
        try:
            for r in range(world):
                log = open(os.path.join(tmp, f"rank{r}.log"), "w+")
                logs.append(log)
                procs.append(subprocess.Popen([sys.executable, script, *map(str, args)], env=dict(env, RANK=str(r)), stdout=log,
                                              stderr=subprocess.STDOUT, start_new_session=True, cwd=tmp))
            deadline = time.monotonic() + timeout
            codes = [None] * world
            while time.monotonic() < deadline and any(c is None for c in codes):
                codes = [p.poll() for p in procs]
                if any(c not in (None, 0) for c in codes):   # one rank failed: its peers would only wait for it
                    time.sleep(5.0)
                    codes = [p.poll() for p in procs]
                    break
                time.sleep(0.2)
        finally:
            for p in procs:
                if p.poll() is None:
                    try:
                        os.killpg(p.pid, signal.SIGKILL)
                    except ProcessLookupError:
                        pass
                p.wait()
        out = []
        for log in logs:
            log.seek(0)
            out.append(log.read())
            log.close()
        tails = "\n".join(f"---- rank {r} (exit {c}) ----\n{o[-4000:]}" for r, (c, o) in enumerate(zip(codes, out)))
        return codes, out[0] if out else "", tails


def init_rank(wall_s=600):
    """Worker side, when launched by launch(): device 0, gloo through the FileStore, and a wall-clock limit after which the worker
    prints its stacks and exits -> (rank, world, device). Otherwise None (a torch.distributed.run launch)."""
    if STORE_ENV not in os.environ:
        return None
    import faulthandler

    import torch
    import torch.distributed as dist
    faulthandler.dump_traceback_later(wall_s, exit=True)
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(0)
    store = dist.FileStore(os.environ[STORE_ENV], world)
    dist.init_process_group("gloo", store=store, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=wall_s))
    return rank, world, torch.device("cuda", 0)
