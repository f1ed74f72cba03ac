"""FSR1_FLAG_SRTM_INPUT without a GPU: the EASU kernels that apply FsrSrtmF as they load each texel, run on the CPU emulator
(tests/emu/emu_srtm_in.cpp), against the chain the flag replaces (the oracle's FsrSrtmF, rounded to half, then the flag-free emulated
kernel); and the ABI's refusals, which all return before any CUDA call.  The GPU side is tests/test_gpu_srtm_input.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import fsr1_b200 as F
import oracle_lib as ol
from fsr1_b200 import _lib
from test_emu import EMU_DIR, emu_lib
from test_upscale_post import CASES, _emu_post, _out_buffer, _tiles, post_lib

_srtm_lib = None


def srtm_lib():
    """tests/emu/emu_srtm_in.cpp: the kSrtmIn kernels on CPU threads (a library of its own, tests/emu/srtm_in.mk)"""
    global _srtm_lib
    if _srtm_lib is None:
        subprocess.check_call(["make", "-s", "-C", EMU_DIR, "-f", "srtm_in.mk", "libfsr1_emu_srtm_in.so"])
        _srtm_lib = ctypes.CDLL(os.path.join(EMU_DIR, "libfsr1_emu_srtm_in.so"))
    return _srtm_lib


def hdr_frame(w, h, seed):
    """Linear HDR half values over [0, 65504]: the LCG frame times 2^e (e drawn in [-8, 16) per texel and channel), quantised to half
    and clipped, with flat blocks of exactly 0, 1.0 and 65504 at the corners and in the middle (border tiles see them)."""
    f = F.uniform(w, h, seed).astype(np.float64)
    e = np.random.default_rng(seed).integers(-8, 16, size=f.shape)
    x = np.clip(f * np.exp2(e), 0.0, 65504.0).astype(np.float16)
    bw, bh = max(1, w // 5), max(1, h // 4)
    x[:bh, :bw] = 0.0
    x[h - bh:, w - bw:] = 65504.0
    x[h // 2 - bh // 2:h // 2 + (bh + 1) // 2, w // 2 - bw // 2:w // 2 + (bw + 1) // 2] = 1.0
    x[:bh, w - bw:] = 65504.0
    return x


def sdr_frame(w, h, seed):
    """The usual [0, 1) LCG frame (SRTM maps it into [0, 0.5])."""
    return F.to_half(F.uniform(w, h, seed))


FRAMES = {"hdr": hdr_frame, "sdr": sdr_frame}


def srtm_half(x16):
    """fsr1_srtm(in, I, 0) on an RGBA16F image: the oracle's FsrSrtmF in fp32, rounded once to half."""
    return ol.srtm(np.ascontiguousarray(x16.astype(np.float32)), inverse=False).astype(np.float16)


def _u16(a):
    return np.ascontiguousarray(a).view(np.uint16)


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def _pitch(a):
    return ctypes.c_longlong(a.strides[0])


def _easu_pair(flagged, plain, variant, src, ow, oh, con, y0, y1, ctas):
    """The kSrtmIn kernel on src and the flag-free kernel on srtm_half(src), both into sentinel-filled outputs."""
    ih, iw = src.shape[:2]
    c = (ctypes.c_uint32 * 16)(*con)
    s16, i16 = _u16(src), _u16(srtm_half(src))
    got = np.full((oh, ow, 4), 0x7E5A, np.uint16)
    want = got.copy()
    assert flagged(_ptr(s16), iw, ih, _pitch(s16), _ptr(got), ow, oh, _pitch(got), c, y0, y1, ctas) == 0
    assert plain(variant, _ptr(i16), iw, ih, _pitch(i16), _ptr(want), ow, oh, _pitch(want), c, y0, y1, ctas) == 0
    return got, want, s16


# ---- the two EASU kernels ----------------------------------------------------------------------------------------------------
# (iw, ih, ow, oh, row slabs): odd widths, border tiles on all four sides, more tiles than CTAs
QUAD_SHAPES = [(9, 5, 18, 10, [(0, 10)]), (37, 13, 74, 26, [(0, 26), (3, 21)]), (70, 21, 140, 42, [(0, 42), (7, 30), (1, 2)])]


@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("iw,ih,ow,oh,slabs", QUAD_SHAPES)
def test_emulated_quad2x_prologue_equals_srtm_then_easu(frame, iw, ih, ow, oh, slabs):
    src = FRAMES[frame](iw, ih, iw * 3 + ih)
    con = ol.easu_con(iw, ih, ow, oh)
    for y0, y1 in slabs:
        got, want, s16 = _easu_pair(srtm_lib().emu_easu_h_quad2x_srtm_in, emu_lib().emu_easu_h_quad2x, 12, src, ow, oh, con, y0, y1, 3)
        assert np.array_equal(got, want), (iw, ih, y0, y1)
        assert (got[:y0] == 0x7E5A).all() and (got[y1:] == 0x7E5A).all()
        assert np.array_equal(s16, _u16(src))                                  # the caller's input is never written


# (iw, ih, ow, oh): 2x through the any-scale kernel, 1.5x, 1.3x x 1.7x (anisotropic)
PAIRS_SHAPES = [(33, 17, 66, 34), (50, 27, 75, 40), (70, 19, 91, 33)]


@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("iw,ih,ow,oh", PAIRS_SHAPES)
def test_emulated_vpairs_prologue_equals_srtm_then_easu(frame, iw, ih, ow, oh):
    src = FRAMES[frame](iw, ih, iw + 5 * ih)
    con = ol.easu_con(iw, ih, ow, oh)
    for y0, y1 in ((0, oh), (5, oh - 2), (oh // 2, oh // 2 + 1)):
        got, want, s16 = _easu_pair(srtm_lib().emu_easu_h_pairs_srtm_in, emu_lib().emu_easu_h_pairs, 1, src, ow, oh, con, y0, y1, 2)
        assert np.array_equal(got, want), (iw, ih, ow, oh, y0, y1)
        assert (got[:y0] == 0x7E5A).all() and (got[y1:] == 0x7E5A).all()
        assert np.array_equal(s16, _u16(src))


# ---- the fused kernels -------------------------------------------------------------------------------------------------------
# (iw, ih, row slabs, CTAs): several steps per run (8 cell rows each), partial last steps, odd slab ends, 3 strips
FUSED_SHAPES = [(40, 37, [(0, 74), (5, 61)], 3), (70, 9, [(0, 18), (1, 16)], 2), (33, 52, [(0, 104), (17, 99)], 4)]


@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("iw,ih,slabs,ctas", FUSED_SHAPES)
def test_emulated_fused_prologue_equals_srtm_then_fused(frame, iw, ih, slabs, ctas):
    src = FRAMES[frame](iw, ih, 7 * iw + ih)
    ow, oh = 2 * iw - 1, 2 * ih                                                 # odd width: a partial last pair
    rcon = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    s16, i16 = _u16(src), _u16(srtm_half(src))
    for y0, y1 in slabs:
        got = np.full((oh, ow, 4), 0x7E5A, np.uint16)
        want = got.copy()
        assert srtm_lib().emu_fused_h_srtm_in(_ptr(s16), iw, ih, _pitch(s16), _ptr(got), ow, oh, _pitch(got), rcon, y0, y1, ctas) == 0
        assert emu_lib().emu_fused_h(_ptr(i16), iw, ih, _pitch(i16), _ptr(want), ow, oh, _pitch(want), rcon, y0, y1, ctas) == 0
        assert np.array_equal(got, want), (iw, ih, y0, y1)
        assert (got[:y0] == 0x7E5A).all() and (got[y1:] == 0x7E5A).all()
        assert np.array_equal(s16, _u16(src))


@pytest.mark.parametrize("ops,out_format", CASES)
def test_emulated_fused_post_prologue_equals_srtm_then_fused_post(ops, out_format):
    """Every op subset of the display epilogue, both UNORM outputs; odd widths, a row slab, grain and dither tiles."""
    grains, dither_tile = _tiles(13)
    rcon = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    for k, (iw, ih, ow, oh, frame) in enumerate([(40, 19, 79, 38, "hdr"), (70, 9, 139, 18, "sdr")]):
        src = FRAMES[frame](iw, ih, 11 + k)
        s16, i16 = _u16(src), _u16(srtm_half(src))
        post = _emu_post(ops, grains[k], 0.375, dither_tile if k == 0 else None, 5)
        for y0, y1 in ((0, oh), (oh // 3, 2 * oh // 3 + 1)):
            got, want = _out_buffer(oh, ow, out_format), _out_buffer(oh, ow, out_format)
            assert srtm_lib().emu_fused_h_post_srtm_in(_ptr(s16), iw, ih, _pitch(s16), _ptr(got), ow, oh, _pitch(got), out_format, rcon,
                                                       y0, y1, 3, ctypes.byref(post)) == 0
            assert post_lib().emu_fused_h_post(_ptr(i16), iw, ih, _pitch(i16), _ptr(want), ow, oh, _pitch(want), out_format, rcon,
                                               y0, y1, 3, ctypes.byref(post)) == 0
            assert np.array_equal(got, want), (iw, ih, y0, y1)
            assert not got[:y0].any() and not got[y1:].any()
            assert np.array_equal(s16, _u16(src))


# ---- the ABI's refusals ------------------------------------------------------------------------------------------------------
def test_srtm_input_validation_without_gpu():
    """Every refusal of the flag returns before any CUDA call: nothing is launched, no fallback kernel runs."""
    L = _lib.lib()
    api = F.api
    S = api.FLAG_SRTM_INPUT
    launches = L.fsr1_launch_count()   # the counter is process-wide: GPU tests may have run earlier in this process
    buf = (ctypes.c_uint8 * 65536)()
    addr = ctypes.addressof(buf)
    addr += (-addr) % 256
    econ = (ctypes.c_uint32 * 16)(*api.easu_con(8, 4, 8, 4, 16, 8))
    down = (ctypes.c_uint32 * 16)(*api.easu_con(16, 8, 16, 8, 8, 4))
    rcon = (ctypes.c_uint32 * 4)(*api.rcas_con(0.25))

    def img(off, pitch, w, h, fmt):
        return _lib.Image(addr + off, pitch, w, h, 0, h, fmt, 0)

    inp, tmp, out = img(0, 64, 8, 4, 1), img(4096, 128, 16, 8, 1), img(8192, 128, 16, 8, 1)

    def easu(i=inp, o=tmp, c=econ, flags=S):
        return L.fsr1_easu(ctypes.byref(i), ctypes.byref(o), c, 0, 0, flags, None)

    def upscale(i=inp, c=econ, flags=S):
        return L.fsr1_upscale(ctypes.byref(i), ctypes.byref(tmp), ctypes.byref(out), c, rcon, 0, 0, flags, None)

    def post(i=inp, c=econ, flags=S):
        p = _lib.Post(_lib.POST_SRTM_INVERSE | _lib.POST_TEPD10, 0.0, None, None, 0, 0)
        o10 = img(8192, 64, 16, 8, 4)
        return L.fsr1_upscale_post(ctypes.byref(i), ctypes.byref(tmp), ctypes.byref(o10), c, rcon, ctypes.byref(p), 0, 0, flags, None)

    # other input formats
    assert easu(img(0, 128, 8, 4, 2), img(4096, 256, 16, 8, 2)) == -2                # RGBA32F
    assert easu(img(0, 32, 8, 4, 3), img(4096, 64, 16, 8, 3)) == -2                  # RGBA8_UNORM
    assert easu(img(0, 32, 8, 4, 4), img(4096, 64, 16, 8, 4)) == -2                  # RGB10A2_UNORM
    for fmt, pin, pout in ((2, 128, 256), (3, 32, 64)):
        i, t, o = img(0, pin, 8, 4, fmt), img(4096, pout, 16, 8, fmt), img(8192, pout, 16, 8, fmt)
        for f in (S, S | api.FLAG_FUSED, S | api.FLAG_NO_RCAS):
            assert L.fsr1_upscale(ctypes.byref(i), ctypes.byref(t), ctypes.byref(o), econ, rcon, 0, 0, f, None) == -2, (fmt, f)
    assert post(img(0, 128, 8, 4, 2)) == -2
    # the paths that have no load prologue
    for flag in (api.FLAG_EXACT, api.FLAG_FORCE_DIRECT, api.FLAG_H_REFERENCE, api.FLAG_PRECISE):
        assert easu(flags=S | flag) == -2, flag
        assert upscale(flags=S | flag) == -2, flag
        assert upscale(flags=S | flag | api.FLAG_FUSED) == -2, flag
        assert upscale(flags=S | flag | api.FLAG_NO_RCAS) == -2, flag
        assert post(flags=S | flag | api.FLAG_FUSED) == -2, flag
    # inputs the tiled kernels decline: base or pitch not 16-byte aligned, constants that do not upscale
    unaligned, odd_pitch = img(8, 64, 8, 4, 1), img(0, 72, 8, 4, 1)
    for i in (unaligned, odd_pitch):
        assert easu(i) == -2
        assert upscale(i) == -2
        assert upscale(i, flags=S | api.FLAG_FUSED) == -2
        assert post(i, flags=S | api.FLAG_FUSED) == -2
    assert easu(o=img(4096 + 8, 128, 16, 8, 1)) == -2                                # EASU's output not 16-byte aligned
    big_in = img(0, 128, 16, 8, 1)
    assert easu(big_in, img(4096, 64, 8, 4, 1), down) == -2                          # downscaling constants
    assert upscale(big_in, down, S | api.FLAG_FUSED) == -2
    assert post(big_in, down, S | api.FLAG_FUSED) == -2
    # RCAS has no input stage
    assert L.fsr1_rcas(ctypes.byref(tmp), ctypes.byref(out), rcon, 0, 0, S, None) == -1
    assert L.fsr1_launch_count() == launches                                         # nothing was launched
