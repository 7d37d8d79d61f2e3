"""Resident blocks per SM of every tile backward variant on this GPU (cudaOccupancyMaxActiveBlocksPerMultiprocessor at the
dynamic shared memory the launch uses), with its registers per thread. Prints one JSON line; writes nothing.

    python tools/render_bwd_occupancy.py"""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from photo_slam_b200 import _lib  # noqa: E402

# variant v = depth | det << 1 | alpha << 2 is render_bwd_kernel<DEPTH, DET, ALPHA>
NAMES = ["render_bwd_kernel<%s, %s, %s>" % tuple("true" if v >> b & 1 else "false" for b in range(3)) for v in range(8)]


def main():
    import torch
    fn = _lib.lib().psb_debug_render_bwd_occupancy
    out = {"device": torch.cuda.get_device_name(0), "threads_per_block": 128, "kernels": {}}
    for v, name in enumerate(NAMES):
        blocks, smem, regs = C.c_int(), C.c_int(), C.c_int()
        _lib.check(fn(v, C.byref(blocks), C.byref(smem), C.byref(regs)), name)
        out["kernels"][name] = {"blocks_per_sm": blocks.value, "warps_per_sm": blocks.value * 4, "dynamic_smem_bytes": smem.value,
                                "registers": regs.value}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
