"""The fused EASU->RCAS kernel's work split (FusedIter: each strip's CTAs take whole steps of it) on the CPU emulator, at CTA
counts and row slabs that put run boundaries everywhere they can fall: the output is the two-kernel path's, bit for bit, and
nothing outside the slab is written."""
import ctypes

import numpy as np
import pytest

import fsr1_b200 as F
import oracle_lib as ol
from test_emu import PROD, emu_easu, emu_lib, emu_rcas

IW, IH = 96, 64  # 192 x 128 output: 4 strips (the middle two with interior steps), 65 cell rows per strip


@pytest.fixture(scope="module")
def frame():
    src = F.to_half(F.uniform(IW, IH, 73))
    want = emu_rcas(emu_easu(PROD, src, 2 * IW, 2 * IH), 0.25).view(np.uint16)
    return np.ascontiguousarray(src.view(np.uint16)), want


def _fused(s16, y0, y1, ctas):
    ow, oh = 2 * IW, 2 * IH
    out = np.zeros((oh, ow, 4), np.uint16)
    con = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    rc = emu_lib().emu_fused_h(ctypes.c_void_p(s16.ctypes.data), IW, IH, ctypes.c_longlong(s16.strides[0]),
                               ctypes.c_void_p(out.ctypes.data), ow, oh, ctypes.c_longlong(out.strides[0]), con, y0, y1, ctas)
    assert rc == 0
    return out


@pytest.mark.parametrize("ctas", [3, 4, 8, 40, 44, 200],
                         ids=["fewer-ctas-than-strips", "one-run-per-strip", "two-runs-per-strip", "one-step-shares",
                              "uneven-one-step-shares", "more-ctas-than-steps"])
@pytest.mark.parametrize("rows", [(0, 128), (37, 100), (6, 121), (16, 127)],
                         ids=["frame", "odd-y0-odd-height", "y0-6", "y0-16-odd-height"])
def test_fused_shares_match_the_two_kernel_path(frame, ctas, rows):
    s16, want = frame
    y0, y1 = rows
    out = _fused(s16, y0, y1, ctas)
    assert np.array_equal(out[y0:y1], want[y0:y1]), (y0, y1, ctas)
    assert not out[:y0].any() and not out[y1:].any()
