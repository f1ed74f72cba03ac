"""FSR1_FLAG_IN_SURFACE / FSR1_FLAG_OUT_SURFACE without a GPU: the flag, format and layout rules of the ABI, all of which return before
any CUDA call, and the surface twins of the RGBA16F kernels on the CPU emulator (tests/emu/emu_surf.cpp) against their linear twins, bit
for bit, with the logical image a poisoned array's top-left region.  The GPU side is tests/test_gpu_surface.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import fsr1_b200 as F
import oracle_lib as ol
from fsr1_b200 import _lib
from test_emu import EMU_DIR
from test_srtm_input import hdr_frame
from test_upscale_post import CASES, _emu_post, _tiles

IN, OUT = 1 << 12, 1 << 13
FLAGS = {"in": (1, 0), "out": (0, 1), "in_out": (1, 1)}
_surf_lib = None


def surf_lib():
    """tests/emu/emu_surf.cpp: the surface twins and their linear twins on CPU threads (a library of its own, tests/emu/surf.mk)"""
    global _surf_lib
    if _surf_lib is None:
        subprocess.check_call(["make", "-s", "-C", EMU_DIR, "-f", "surf.mk", "libfsr1_emu_surf.so"])
        _surf_lib = ctypes.CDLL(os.path.join(EMU_DIR, "libfsr1_emu_surf.so"))
        _surf_lib.emu_surface.restype = ctypes.c_ulonglong
        _surf_lib.emu_surface.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    return _surf_lib


# ---- the ABI's refusals ------------------------------------------------------------------------------------------------------------
def test_flag_values():
    assert _lib.FLAG_IN_SURFACE == IN and _lib.FLAG_OUT_SURFACE == OUT
    assert F.api.FLAG_IN_SURFACE == IN and F.api.FLAG_OUT_SURFACE == OUT
    img = F.api.surface_image(77, 10, 6, _lib.FORMAT_RGBA16F)
    assert (img.data, img.pitch_bytes, img.width, img.height, img.row0, img.rows, img.format) == (77, 0, 10, 6, 0, 6, 1)
    with pytest.raises(F.api.Fsr1Error):
        F.api.surface_image(0, 10, 6, _lib.FORMAT_RGBA16F)


def test_surface_validation_without_gpu():
    """Every flag, format and layout refusal returns its code before any CUDA call: nothing is launched."""
    L = _lib.lib()
    api = F.api
    launches = L.fsr1_launch_count()   # the counter is process-wide: GPU tests may have run earlier in this process
    buf = (ctypes.c_uint8 * 65536)()
    addr = ctypes.addressof(buf)
    addr += (-addr) % 256
    econ = (ctypes.c_uint32 * 16)(*api.easu_con(8, 4, 8, 4, 16, 8))
    down = (ctypes.c_uint32 * 16)(*api.easu_con(16, 8, 16, 8, 8, 4))
    rcon = (ctypes.c_uint32 * 4)(*api.rcas_con(0.25))
    BPP = {1: 8, 2: 16, 3: 4, 4: 4, 5: 4}
    I, U = -1, -2

    def img(off, w, h, fmt):
        return _lib.Image(addr + off, 16 * ((w * BPP[fmt] + 15) // 16), w, h, 0, h, fmt, 0)

    def surf(w, h, fmt, handle=0x51, pitch=0, row0=0, rows=None):
        return _lib.Image(handle, pitch, w, h, row0, h if rows is None else rows, fmt, 0)

    def easu(i, o, flags, con=econ):
        return L.fsr1_easu(ctypes.byref(i), ctypes.byref(o), con, 0, 0, flags, None)

    def rcas(i, o, flags):
        return L.fsr1_rcas(ctypes.byref(i), ctypes.byref(o), rcon, 0, 0, flags, None)

    def upscale(i, t, o, flags, con=econ):
        return L.fsr1_upscale(ctypes.byref(i), ctypes.byref(t) if t is not None else None, ctypes.byref(o), con, rcon, 0, 0, flags, None)

    def post(i, t, o, ops, flags, con=econ):
        p = _lib.Post(ops, 0.0, None, None, 0, 0)
        return L.fsr1_upscale_post(ctypes.byref(i), ctypes.byref(t) if t is not None else None, ctypes.byref(o), con, rcon,
                                   ctypes.byref(p), 0, 0, flags, None)

    s_in, h16, tmp16 = surf(8, 4, 1), img(8192, 16, 8, 1), img(16384, 16, 8, 1)
    lin_in, s_out = img(0, 8, 4, 1), surf(16, 8, 1, handle=0x52)
    refused = (api.FLAG_EXACT, api.FLAG_FORCE_DIRECT, api.FLAG_H_REFERENCE, api.FLAG_PRECISE, api.FLAG_RCAS_HX2)
    # the layout of a surface image: a handle, pitch 0, never a window
    bad_layouts = (surf(8, 4, 1, handle=0), surf(8, 4, 1, pitch=64), surf(8, 4, 1, row0=1, rows=3), surf(8, 4, 1, rows=3), surf(8, 4, 9),
                   surf(0, 4, 1))
    for b in bad_layouts:
        assert easu(b, h16, IN) == I
        assert upscale(b, tmp16, h16, IN | api.FLAG_FUSED) == I
        assert post(b, tmp16, h16, api.POST_SRTM_INVERSE, IN | api.FLAG_FUSED) == I
    for b in (surf(16, 8, 1, handle=0), surf(16, 8, 1, pitch=128), surf(16, 8, 1, row0=2, rows=6)):
        assert rcas(tmp16, b, OUT) == I
        assert upscale(lin_in, tmp16, b, OUT) == I
        assert post(lin_in, tmp16, b, api.POST_SRTM_INVERSE, OUT) == I
    # fsr1_easu: IN only; RGBA16F input; no other path; constants that upscale
    assert easu(lin_in, h16, OUT) == U
    assert easu(s_in, h16, IN | OUT) == U
    for fmt in (2, 3, 4, 5):
        assert easu(surf(8, 4, fmt), img(8192, 16, 8, fmt if fmt != 5 else 1), IN) == U, fmt
    for r in refused:
        assert easu(s_in, h16, IN | r) == U, r
        assert easu(s_in, h16, IN | api.FLAG_SRTM_INPUT | r) == U, r
    assert easu(surf(16, 8, 1), img(8192, 8, 4, 1), IN, down) == U
    # fsr1_rcas: OUT only, RGBA16F, the packed kernel only
    assert rcas(tmp16, h16, IN) == U
    assert rcas(tmp16, s_out, IN | OUT) == U
    assert rcas(img(0, 16, 8, 3), surf(16, 8, 3), OUT) == U
    assert rcas(img(0, 16, 8, 2), surf(16, 8, 2), OUT) == U
    for r in refused:
        assert rcas(tmp16, s_out, OUT | r) == U, r
    # fsr1_upscale: both; never OUT with NO_RCAS; RGBA16F input; the RGBA16F kernels' outputs
    for f in (0, api.FLAG_FUSED, api.FLAG_FUSED | api.FLAG_RCAS_DENOISE):
        assert upscale(lin_in, None, s_out, f | OUT | api.FLAG_NO_RCAS) == U, f
        assert upscale(s_in, None, s_out, f | IN | OUT | api.FLAG_NO_RCAS) == U, f
        for r in refused:
            for fl in (IN, OUT, IN | OUT):
                assert upscale(s_in if fl & IN else lin_in, tmp16, s_out if fl & OUT else h16, f | fl | r) == U, (f, fl, r)
        assert upscale(surf(16, 8, 1), tmp16, h16, f | IN, down) == U
        assert upscale(surf(8, 4, 2), img(16384, 16, 8, 2), img(8192, 16, 8, 2), f | IN) == U
        assert upscale(img(0, 8, 4, 2), img(16384, 16, 8, 2), surf(16, 8, 2), f | OUT) == U
        assert upscale(img(0, 8, 4, 5), tmp16, s_out, f | OUT) == U
        assert upscale(lin_in, tmp16, surf(16, 8, 3), f | OUT) == U
    # fsr1_upscale_post: its own format rules (TEPD's UNORM outputs) and the surface rules
    for r in refused:
        assert post(s_in, tmp16, s_out, api.POST_SRTM_INVERSE, IN | OUT | api.FLAG_FUSED | r) == U, r
    assert post(s_in, tmp16, s_out, api.POST_SRTM_INVERSE, IN | OUT | api.FLAG_NO_RCAS) == U
    assert post(surf(16, 8, 1), tmp16, h16, api.POST_SRTM_INVERSE, IN | api.FLAG_FUSED, down) == U
    assert post(img(0, 8, 4, 5), tmp16, s_out, api.POST_SRTM_INVERSE, OUT | api.FLAG_FUSED) == U
    assert post(lin_in, tmp16, surf(16, 8, 4), api.POST_TEPD8, OUT | api.FLAG_FUSED) == U   # TEPD8 writes RGBA8
    assert post(lin_in, tmp16, surf(16, 8, 2), api.POST_SRTM_INVERSE, OUT | api.FLAG_FUSED) == U
    # shards: windows and slabs are linear memory
    h = ctypes.c_void_p()
    for fl in (IN, OUT, IN | OUT):
        assert L.fsr1_shard_create(ctypes.byref(h), 8, 4, 16, 8, 1, 1, 0, 1, ctypes.c_float(0.25), fl) == U
        p = _lib.Post(api.POST_SRTM_INVERSE, 0.0, None, None, 0, 0)
        assert L.fsr1_shard_create_post(ctypes.byref(h), 8, 4, 16, 8, 1, 1, ctypes.byref(p), 1, 0, 1, ctypes.c_float(0.25), fl) == U
    # flag 1 << 20 stays unknown
    assert easu(s_in, h16, IN | (1 << 20)) == I
    assert L.fsr1_launch_count() == launches                                         # nothing was launched


# ---- the kernels on the emulator -------------------------------------------------------------------------------------------------
POISON16 = np.array([0x7E00, 0x7C00, 0x7BFF, 0xFC00], np.uint16)   # NaN, inf, 65504, -inf


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def _pitch(a):
    return ctypes.c_longlong(a.strides[0])


class Arr:
    """An emulated 2D CUDA array holding a logical image in its top-left region; the rest is poison.  .h: its surface handle."""

    def __init__(self, slot, logical, extra=(3, 5), poison=None):
        lh, lw = logical.shape[:2]
        shape = (lh + extra[0], lw + extra[1]) + logical.shape[2:]
        if poison is None:
            poison = np.resize(POISON16, shape) if logical.dtype == np.uint16 else np.full(shape, 0xA5C3E1F0, np.uint32)
        self.a = np.ascontiguousarray(poison.reshape(shape).astype(logical.dtype))
        self.a[:lh, :lw] = logical
        self.before = self.a.copy()
        elem = 8 if logical.dtype == np.uint16 else 4
        self.h = surf_lib().emu_surface(slot, self.a.ctypes.data, self.a.strides[0], shape[1], shape[0], elem)
        self.lh, self.lw = lh, lw

    def logical(self):
        return self.a[:self.lh, :self.lw]

    def outside_unchanged(self):
        return np.array_equal(self.a[self.lh:], self.before[self.lh:]) and np.array_equal(self.a[:, self.lw:], self.before[:, self.lw:])


def _frame(w, h, seed, hdr):
    return hdr_frame(w, h, seed).view(np.uint16) if hdr else np.ascontiguousarray(F.uniform(w, h, seed).astype(np.float16).view(np.uint16))


def _out(oh, ow, out_format, fill):
    return np.full((oh, ow, 4), fill, np.uint16) if out_format == 1 else np.full((oh, ow), fill, np.uint32)


QUAD_SHAPES = [(9, 5, 18, 10, [(0, 10)]), (37, 13, 74, 26, [(0, 26), (3, 21)]), (70, 21, 140, 42, [(0, 42), (7, 30), (1, 2)])]


@pytest.mark.parametrize("srtm", [0, 1])
@pytest.mark.parametrize("iw,ih,ow,oh,slabs", QUAD_SHAPES)
def test_emulated_quad2x_surface_input_equals_linear(srtm, iw, ih, ow, oh, slabs):
    L = surf_lib()
    x = _frame(iw, ih, iw + ih + srtm, srtm)
    src = Arr(0, x)
    con = (ctypes.c_uint32 * 16)(*ol.easu_con(iw, ih, ow, oh))
    for y0, y1 in slabs:
        got, want = _out(oh, ow, 1, 0x7E5A), _out(oh, ow, 1, 0x7E5A)
        assert L.emu_easu_quad2x_surf(ctypes.c_void_p(src.h), 0, iw, ih, _ptr(got), ow, oh, _pitch(got), con, y0, y1, 3, srtm, 1) == 0
        assert L.emu_easu_quad2x_surf(_ptr(x), _pitch(x), iw, ih, _ptr(want), ow, oh, _pitch(want), con, y0, y1, 3, srtm, 0) == 0
        assert np.array_equal(got, want), (iw, ih, y0, y1)
        assert (got[:y0] == 0x7E5A).all() and (got[y1:] == 0x7E5A).all()
        assert np.array_equal(src.a, src.before)


# 2x through the any-scale kernel, 1.5x, 1.3x x 1.7x (anisotropic), 1.0x x 1.1x, 41 -> 82 (almost 2x)
PAIRS_SHAPES = [(33, 17, 66, 34), (50, 27, 75, 40), (70, 19, 91, 33), (69, 37, 69, 41), (41, 23, 82, 46)]


@pytest.mark.parametrize("srtm", [0, 1])
@pytest.mark.parametrize("iw,ih,ow,oh", PAIRS_SHAPES)
def test_emulated_vpairs_surface_input_equals_linear(srtm, iw, ih, ow, oh):
    L = surf_lib()
    x = _frame(iw, ih, 3 * iw + ih + srtm, srtm)
    src = Arr(0, x, extra=(2, 9))
    con = (ctypes.c_uint32 * 16)(*ol.easu_con(iw, ih, ow, oh))
    for y0, y1 in ((0, oh), (5, oh - 2), (oh // 2, oh // 2 + 1)):
        got, want = _out(oh, ow, 1, 0x7E5A), _out(oh, ow, 1, 0x7E5A)
        assert L.emu_easu_pairs_surf(ctypes.c_void_p(src.h), 0, iw, ih, _ptr(got), ow, oh, _pitch(got), con, y0, y1, 2, srtm, 1) == 0
        assert L.emu_easu_pairs_surf(_ptr(x), _pitch(x), iw, ih, _ptr(want), ow, oh, _pitch(want), con, y0, y1, 2, srtm, 0) == 0
        assert np.array_equal(got, want), (iw, ih, ow, oh, y0, y1)


def _fused_pair(x, iw, ih, ow, oh, out_format, rcon, y0, y1, ctas, post, srtm, surf_in, surf_out):
    """the fused kernel's surface twin (flags surf_in / surf_out) and the linear kernel on the same pixels; (got, want, arrays)"""
    L = surf_lib()
    src = Arr(0, x) if surf_in else None
    fill = 0x7E5A if out_format == 1 else 0xA5C3E1F0
    dst = Arr(1, _out(oh, ow, out_format, fill), extra=(2, 3)) if surf_out else None
    got, want = _out(oh, ow, out_format, fill), _out(oh, ow, out_format, fill)
    a_in = (ctypes.c_void_p(src.h), 0) if surf_in else (_ptr(x), _pitch(x))
    a_out = (ctypes.c_void_p(dst.h), 0) if surf_out else (_ptr(got), _pitch(got))
    pp = ctypes.byref(post) if post is not None else None
    assert L.emu_fused_surf(*a_in, iw, ih, *a_out, ow, oh, out_format, rcon, y0, y1, ctas, pp, srtm, surf_in, surf_out) == 0
    assert L.emu_fused_surf(_ptr(x), _pitch(x), iw, ih, _ptr(want), _pitch(want), ow, oh, out_format, rcon, y0, y1, ctas, pp, srtm, 0, 0) == 0
    if surf_out:
        assert dst.outside_unchanged()
        got = dst.logical()
    if surf_in:
        assert np.array_equal(src.a, src.before)
    return got, want


# (iw, ih, row slabs, CTAs): several steps per run, partial last steps, odd slab ends, 3 strips; odd strip origins
FUSED_SHAPES = [(40, 37, [(0, 74), (5, 61)], 3), (70, 9, [(0, 18), (1, 16)], 2), (33, 52, [(0, 104), (17, 99)], 4), (95, 11, [(0, 22)], 5)]


@pytest.mark.parametrize("flags", list(FLAGS))
@pytest.mark.parametrize("srtm", [0, 1])
@pytest.mark.parametrize("iw,ih,slabs,ctas", FUSED_SHAPES)
def test_emulated_fused_surface_equals_linear(flags, srtm, iw, ih, slabs, ctas):
    x = _frame(iw, ih, 7 * iw + ih + srtm, srtm)
    ow, oh = 2 * iw - 1, 2 * ih                                                 # odd width: a partial last pair
    rcon = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    for y0, y1 in slabs:
        got, want = _fused_pair(x, iw, ih, ow, oh, 1, rcon, y0, y1, ctas, None, srtm, *FLAGS[flags])
        assert np.array_equal(got, want), (iw, ih, y0, y1)
        assert (got[:y0] == 0x7E5A).all() and (got[y1:] == 0x7E5A).all()


@pytest.mark.parametrize("flags", list(FLAGS))
@pytest.mark.parametrize("srtm", [0, 1])
@pytest.mark.parametrize("ops,out_format", CASES)
def test_emulated_fused_post_surface_equals_linear(flags, srtm, ops, out_format):
    """Every op subset of the display epilogue into RGBA16F, RGBA8 and RGB10A2; an odd width, a row slab, grain and dither tiles."""
    grains, dither_tile = _tiles(17)
    rcon = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    iw, ih, ow, oh = 40, 19, 79, 38
    x = _frame(iw, ih, 11 + ops, srtm)
    post = _emu_post(ops, grains[srtm], 0.375, dither_tile if srtm == 0 else None, 5)
    for y0, y1 in ((0, oh), (oh // 3, 2 * oh // 3 + 1)):
        got, want = _fused_pair(x, iw, ih, ow, oh, out_format, rcon, y0, y1, 3, post, srtm, *FLAGS[flags])
        assert np.array_equal(got, want), (ops, out_format, y0, y1)


@pytest.mark.parametrize("post_case", [None] + CASES[::2])
@pytest.mark.parametrize("opts", [0, 1, 2, 3, 4, 7])
@pytest.mark.parametrize("clamp", [0, 1])
def test_emulated_rcas_surface_output_equals_linear(post_case, opts, clamp):
    """rcas_surf_out_kernel: RCAS_CLAMP, DENOISE (opts bit 0), PASSTHROUGH_ALPHA (bit 1), OUTPUT_SQUARE (bit 2), with and without the
    display epilogue; an odd width over three CTAs, row slabs."""
    L = surf_lib()
    w, h = 127, 23
    x = _frame(w, h, 31 + opts, 0).copy()
    x[..., 3] = np.random.default_rng(opts).integers(0x3000, 0x3C00, size=(h, w), dtype=np.uint16)   # alpha for PASSTHROUGH_ALPHA
    con = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.5))
    ops, out_format = post_case if post_case is not None else (0, 1)
    grains, dither_tile = _tiles(3)
    post = _emu_post(ops, grains[0], 0.25, dither_tile, 9) if post_case is not None else None
    pp = ctypes.byref(post) if post is not None else None
    fill = 0x7E5A if out_format == 1 else 0xA5C3E1F0
    for y0, y1 in ((0, h), (3, 17)):
        dst = Arr(1, _out(h, w, out_format, fill), extra=(3, 2))
        want = _out(h, w, out_format, fill)
        assert L.emu_rcas_surf(_ptr(x), _pitch(x), ctypes.c_void_p(dst.h), 0, w, h, out_format, con, clamp, y0, y1, opts, pp, 1) == 0
        assert L.emu_rcas_surf(_ptr(x), _pitch(x), _ptr(want), _pitch(want), w, h, out_format, con, clamp, y0, y1, opts, pp, 0) == 0
        assert np.array_equal(dst.logical(), want), (y0, y1)
        assert dst.outside_unchanged()
