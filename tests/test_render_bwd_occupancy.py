"""Occupancy of the tile backward: every variant keeps 8 resident 128-thread blocks per SM (its shared memory and registers
allow it), and the diagnostic entry point rejects a variant it does not know before any CUDA call."""
import ctypes as C

import pytest

from photo_slam_b200 import _lib


def _query():
    return _lib.lib().psb_debug_render_bwd_occupancy


def test_unknown_variant_is_rejected():
    assert _query()(8, None, None, None) == -1
    assert b"variant" in _lib.lib().psb_last_error()


@pytest.mark.gpu
@pytest.mark.parametrize("variant", range(8))
def test_eight_blocks_per_sm(cuda, variant):
    blocks, smem, regs = C.c_int(), C.c_int(), C.c_int()
    _lib.check(_query()(variant, C.byref(blocks), C.byref(smem), C.byref(regs)), "psb_debug_render_bwd_occupancy")
    assert smem.value <= 25 * 1024, smem.value
    assert regs.value <= 64, regs.value
    assert blocks.value >= 8, (variant, blocks.value, smem.value, regs.value)
