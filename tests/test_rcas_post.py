"""fsr1_rcas_post without a GPU: the input-stage RCAS kernels (R11G11B10F decode, SRTM) run on the CPU emulator (tests/emu/emu_rcas_in.cpp)
against the chain the call replaces (decode, the oracle's FsrSrtmF rounded to half, then the emulated rcas_h_packed / rcas_h_packed_post),
bit for bit; and the ABI's refusals, which all return before any CUDA call.  The GPU side is tests/test_gpu_rcas_post.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import fsr1_b200 as F
import oracle_lib as ol
from fsr1_b200 import _lib
from test_emu import EMU_DIR, emu_lib
from test_r11g11b10 import decode, hdr_codes, raw_codes
from test_srtm_input import hdr_frame, srtm_half
from test_upscale_post import _emu_post, _out_buffer, _tiles, post_lib

R11 = 5
_rcas_in_lib = None


def rcas_in_lib():
    """tests/emu/emu_rcas_in.cpp: the input-stage RCAS kernels on CPU threads (a library of its own, tests/emu/rcas_in.mk)"""
    global _rcas_in_lib
    if _rcas_in_lib is None:
        subprocess.check_call(["make", "-s", "-C", EMU_DIR, "-f", "rcas_in.mk", "libfsr1_emu_rcas_in.so"])
        _rcas_in_lib = ctypes.CDLL(os.path.join(EMU_DIR, "libfsr1_emu_rcas_in.so"))
    return _rcas_in_lib


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def _pitch(a):
    return ctypes.c_longlong(a.strides[0])


# ---- the kernels on the emulator -------------------------------------------------------------------------------------------------
def _input(stage, w, h, seed):
    """(the call's input, r11, srtm, the RGBA16F image RCAS sees as uint16 bits [h, w, 4]) for an input stage"""
    if stage == "r11_raw":                              # every code: denormals, zeros, 65024, inf and NaN
        codes = raw_codes(w, h, seed)
        return codes, 1, 0, decode(codes)
    if stage == "r11_srtm":
        codes = hdr_codes(w, h, seed)
        return codes, 1, 1, np.ascontiguousarray(srtm_half(decode(codes).view(np.float16))).view(np.uint16)
    x = hdr_frame(w, h, seed)                           # "h16_srtm": RGBA16F with SRTM_INPUT
    x[..., 3] = np.random.default_rng(seed).random((h, w)).astype(np.float16)   # alpha passes through with PASSTHROUGH_ALPHA
    return np.ascontiguousarray(x).view(np.uint16), 0, 1, np.ascontiguousarray(srtm_half(x)).view(np.uint16)


STAGES = ["r11_raw", "r11_srtm", "h16_srtm"]
STORES = [(None, 1), (F.api.POST_SRTM_INVERSE | F.api.POST_LFGA, 1), (F.api.POST_LFGA | F.api.POST_TEPD8, 3),
          (F.api.POST_SRTM_INVERSE | F.api.POST_TEPD10, 4)]
OPTIONS = [(0, 0), (1, 0), (2, 0), (0, 1)]             # (opts, clamp): none, DENOISE, PASSTHROUGH_ALPHA, RCAS_CLAMP


def _reference(t16, w, h, out_format, con, clamp, y0, y1, opts, post):
    """the emulated rcas_h_packed (post None) or rcas_h_packed_post on the whole RGBA16F image t16"""
    want = _out_buffer(h, w, out_format)
    if post is None:
        assert emu_lib().emu_rcas_h_packed_opt(_ptr(t16), 0, h, _ptr(want), w, h, _pitch(t16), _pitch(want), con, clamp, y0, y1, opts) == 0
    else:
        assert post_lib().emu_rcas_h_packed_post(_ptr(t16), _ptr(want), w, h, _pitch(t16), _pitch(want), out_format, con, clamp, y0, y1,
                                                 opts, ctypes.byref(post)) == 0
    return want


@pytest.mark.parametrize("opts,clamp", OPTIONS)
@pytest.mark.parametrize("ops,out_format", STORES)
@pytest.mark.parametrize("stage", STAGES)
def test_emulated_input_stage_equals_decode_srtm_then_rcas(stage, ops, out_format, opts, clamp):
    """Odd widths (61: one border warp; 257: interior and border warps), whole images and row slabs read from windows that hold only
    rows [y0-1, y1+1): equal to decode -> srtm -> the emulated RCAS kernel, and nothing written outside [y0, y1)."""
    grains, dither_tile = _tiles(5)
    con = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    for k, (w, h, slabs) in enumerate([(61, 19, [(0, 19), (5, 14)]), (257, 67, [(0, 67), (17, 50)])]):
        inp, r11, srtm, t16 = _input(stage, w, h, 31 * k + len(stage) + opts)
        post = None if ops is None else _emu_post(ops, grains[k], 0.375, dither_tile if k == 1 else None, 9)
        for y0, y1 in slabs:
            want = _reference(t16, w, h, out_format, con, clamp, y0, y1, opts, post)
            r0, r1 = max(y0 - 1, 0), min(y1 + 1, h)
            win = np.ascontiguousarray(inp[r0:r1])
            got = _out_buffer(h, w, out_format)
            assert rcas_in_lib().emu_rcas_in(_ptr(win), r0, r1 - r0, _pitch(win), _ptr(got), _pitch(got), w, h, out_format, con, clamp,
                                             y0, y1, opts, ctypes.byref(post) if post is not None else None, r11, srtm) == 0
            assert np.array_equal(got[y0:y1], want[y0:y1]), (stage, w, h, y0, y1)
            assert not got[:y0].any() and not got[y1:].any()


def test_emulated_r11_without_srtm_is_rcas_of_the_decoded_image_with_output_square():
    """OUTPUT_SQUARE (option bit 2) and every option together on raw codes"""
    w, h = 131, 22
    codes = raw_codes(w, h, 77)
    t16 = decode(codes)
    con = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.5))
    for opts, clamp in ((4, 0), (7, 1)):
        want = _reference(t16, w, h, 1, con, clamp, 0, h, opts, None)
        got = _out_buffer(h, w, 1)
        assert rcas_in_lib().emu_rcas_in(_ptr(codes), 0, h, _pitch(codes), _ptr(got), _pitch(got), w, h, 1, con, clamp, 0, h, opts, None,
                                         1, 0) == 0
        assert np.array_equal(got, want)


# ---- the ABI's refusals ------------------------------------------------------------------------------------------------------------
def test_rcas_post_validation_without_gpu():
    """Every refusal of fsr1_rcas_post returns its code before any CUDA call: nothing is launched."""
    L = _lib.lib()
    api = F.api
    launches = L.fsr1_launch_count()   # the counter is process-wide: GPU tests may have run earlier in this process
    buf = (ctypes.c_uint8 * 65536)()
    addr = ctypes.addressof(buf)
    addr += (-addr) % 256
    rcon = (ctypes.c_uint32 * 4)(*api.rcas_con(0.25))
    BPP = {1: 8, 2: 16, 3: 4, 4: 4, R11: 4}

    def img(off, fmt, w=16, h=8, pitch=None, row0=0, rows=None):
        return _lib.Image(addr + off, pitch or 16 * ((w * BPP[fmt] + 15) // 16), w, h, row0, h if rows is None else rows, fmt, 0)

    h16, r11 = img(0, 1), img(0, R11)
    o16, o8, o10 = img(16384, 1), img(16384, 3), img(16384, 4)
    grain, grain_win, grain_u8 = img(32768, 1, 4, 4), img(32768, 1, 4, 4, row0=1, rows=2), img(32768, 3, 4, 4)

    def call(i=h16, o=o16, ops=api.POST_TEPD8, g=None, d=None, flags=0, y0=0, y1=0, con=rcon, post=True):
        p = _lib.Post(ops, 0.5, ctypes.pointer(g) if g is not None else None, ctypes.pointer(d) if d is not None else None, 0, 0)
        return L.fsr1_rcas_post(ctypes.byref(i) if i is not None else None, ctypes.byref(o) if o is not None else None, con,
                                ctypes.byref(p) if post else None, y0, y1, flags, None)

    INV, U, WIN = -1, -2, -3
    # FSR1_ERR_INVALID_ARGUMENT
    assert call(i=None, ops=0) == INV
    assert call(o=None, ops=0) == INV
    assert call(con=None, ops=0) == INV
    assert call(o=o8, flags=1 << 20) == INV                                  # flag 1 << 20 stays unknown
    assert call(o=o8, y0=5, y1=5) == INV                                     # bad row ranges
    assert call(o=o8, y0=0, y1=9) == INV
    assert call(o=img(16384, 3, 16, 9)) == INV                               # in and out of different sizes
    assert call(o=img(8, 3)) == INV                                          # linear storage that overlaps (8-byte aligned)
    assert call(i=r11, o=img(128, 1)) == INV
    assert call(o=o8, ops=1 << 4) == INV                                     # post_params: unknown ops bit
    assert call(o=o8, ops=api.POST_TEPD8 | api.POST_TEPD10) == INV           # both TEPD bits
    assert call(o=o16, ops=api.POST_LFGA) == INV                             # LFGA without a grain tile
    assert call(o=o16, ops=api.POST_LFGA, g=grain_win) == INV                # a tile that is a window
    assert call(o=o8, ops=api.POST_TEPD8, d=grain_win) == INV
    # FSR1_ERR_UNSUPPORTED: formats
    for fmt in (2, 3, 4):
        assert call(i=img(0, fmt), o=o16, ops=0) == U, fmt                   # input formats other than RGBA16F / R11G11B10F
    assert call(i=r11, o=img(16384, R11), ops=0) == U                        # R11G11B10F is never an output
    assert call(o=o8, ops=0) == U                                            # UNORM out needs TEPD
    assert call(o=o8, ops=api.POST_SRTM_INVERSE) == U
    assert call(o=o10, ops=api.POST_TEPD8) == U                              # TEPD8 writes RGBA8 codes, not RGB10A2
    assert call(o=o8, ops=api.POST_TEPD10) == U
    assert call(o=img(16384, 2), ops=0) == U                                 # RGBA32F out
    assert call(o=o16, ops=api.POST_LFGA, g=grain_u8) == U                   # grain is signed: float tiles only
    # flags
    for flag in (api.FLAG_EXACT, api.FLAG_FORCE_DIRECT, api.FLAG_H_REFERENCE, api.FLAG_PRECISE, api.FLAG_RCAS_HX2, api.FLAG_NO_RCAS,
                 api.FLAG_IN_SURFACE):
        for i in (h16, r11):
            assert call(i=i, o=o8, flags=flag) == U, flag
            assert call(i=i, o=o16, ops=0, flags=flag) == U, flag
    # layouts: one vector access per pixel pair
    assert call(i=img(8, 1), o=o8) == U                                      # RGBA16F in: 16-byte base and pitch
    assert call(i=img(0, 1, pitch=136), o=o8) == U
    assert call(i=img(4, R11), o=o8) == U                                    # R11G11B10F in: 8-byte base and pitch
    assert call(i=img(0, R11, pitch=68), o=o8) == U
    assert call(i=r11, o=img(16384 + 8, 1), ops=0) == U                      # RGBA16F out: 16-byte aligned
    assert call(i=r11, o=img(16384, 1, pitch=136), ops=0) == U
    assert call(o=img(16384 + 4, 3)) == U                                    # UNORM out: 8-byte aligned
    # FSR1_ERR_WINDOW: windows that do not hold the rows
    assert call(i=img(0, 1, row0=3, rows=5), o=o8, y0=3, y1=8) == WIN        # RCAS reads rows 2 .. 7: row 2 is not held
    assert call(i=img(0, R11, row0=0, rows=5), o=o8, y0=0, y1=5) == WIN      # row 5 is not held
    assert call(i=r11, o=img(16384, 3, row0=0, rows=4), y0=0, y1=5) == WIN
    # accepted flags, refused later for the layout: the flag checks let them through
    for flag in (api.FLAG_RCAS_CLAMP, api.FLAG_RCAS_DENOISE, api.FLAG_RCAS_PASSTHROUGH_ALPHA, api.FLAG_OUTPUT_SQUARE, api.FLAG_SRTM_INPUT,
                 api.FLAG_FUSED):
        assert call(i=img(4, R11), o=o8, flags=flag) == U, flag
    assert L.fsr1_launch_count() == launches                                 # nothing was launched
    assert L.fsr1_abi_version() == 3
