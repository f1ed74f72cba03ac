"""FSR1_FLAG_IN_TEXTURE without a GPU: the flag, format and layout rules of the ABI, all of which return before any CUDA call, and the
texture twins of the RGBA16F and R11G11B10F kernels on the CPU emulator (tests/emu/emu_tex.cpp) against their linear twins, bit for bit,
with the logical image a poisoned array's top-left region.  The GPU side is tests/test_gpu_texture.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import fsr1_b200 as F
import oracle_lib as ol
from fsr1_b200 import _lib
from test_emu import EMU_DIR
from test_r11g11b10 import hdr_codes, raw_codes
from test_srtm_input import hdr_frame
from test_upscale_post import CASES, _emu_post, _tiles

TEX, SURF_IN, SURF_OUT = 1 << 14, 1 << 12, 1 << 13
_tex_lib = None


def tex_lib():
    """tests/emu/emu_tex.cpp: the texture twins and their linear twins on CPU threads (a library of its own, tests/emu/tex.mk)"""
    global _tex_lib
    if _tex_lib is None:
        subprocess.check_call(["make", "-s", "-C", EMU_DIR, "-f", "tex.mk", "libfsr1_emu_tex.so"])
        _tex_lib = ctypes.CDLL(os.path.join(EMU_DIR, "libfsr1_emu_tex.so"))
        for fn in (_tex_lib.emu_texture, _tex_lib.emu_tex_surface):
            fn.restype = ctypes.c_ulonglong
            fn.argtypes = [ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_int, ctypes.c_int]
        _tex_lib.emu_tex_faults.restype = ctypes.c_longlong
    return _tex_lib


# ---- the ABI's refusals ------------------------------------------------------------------------------------------------------------
def test_flag_values():
    assert _lib.FLAG_IN_TEXTURE == TEX and F.api.FLAG_IN_TEXTURE == TEX
    img = F.api.texture_image(91, 10, 6, _lib.FORMAT_R11G11B10_FLOAT)
    assert (img.data, img.pitch_bytes, img.width, img.height, img.row0, img.rows, img.format) == (91, 0, 10, 6, 0, 6, 5)
    for bad in (0, -3, 1.5):
        with pytest.raises(F.api.Fsr1Error):
            F.api.texture_image(bad, 10, 6, _lib.FORMAT_RGBA16F)


def test_texture_validation_without_gpu():
    """Every flag, format and layout refusal of FSR1_FLAG_IN_TEXTURE returns its code before any CUDA call: nothing is launched."""
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

    def arr(w, h, fmt, handle=0x61, pitch=0, row0=0, rows=None):
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

    def rcas_post(i, o, flags):
        return L.fsr1_rcas_post(ctypes.byref(i), ctypes.byref(o), rcon, None, 0, 0, flags, None)

    h16, tmp16 = img(8192, 16, 8, 1), img(16384, 16, 8, 1)
    lin_in, s_out = img(0, 8, 4, 1), arr(16, 8, 1, handle=0x62)
    refused = (api.FLAG_EXACT, api.FLAG_FORCE_DIRECT, api.FLAG_H_REFERENCE, api.FLAG_PRECISE, api.FLAG_RCAS_HX2)
    for fmt in (1, 5):
        t_in = arr(8, 4, fmt)
        # the layout of a texture image: a handle, pitch 0, never a window
        for b in (arr(8, 4, fmt, handle=0), arr(8, 4, fmt, pitch=64), arr(8, 4, fmt, row0=1, rows=3), arr(8, 4, fmt, rows=3),
                  arr(0, 4, fmt), arr(8, 4, 9)):
            assert easu(b, h16, TEX) == I
            assert upscale(b, tmp16, h16, TEX | api.FLAG_FUSED) == I
            assert upscale(b, tmp16, h16, TEX) == I
            assert post(b, tmp16, h16, api.POST_SRTM_INVERSE, TEX | api.FLAG_FUSED) == I
        # IN_TEXTURE with IN_SURFACE: one input cannot be both
        assert easu(t_in, h16, TEX | SURF_IN) == I
        for f in (0, api.FLAG_FUSED):
            assert upscale(t_in, tmp16, h16, f | TEX | SURF_IN) == I, f
            assert post(t_in, tmp16, h16, api.POST_SRTM_INVERSE, f | TEX | SURF_IN) == I, f
        assert rcas(tmp16, h16, TEX | SURF_IN) == I
        assert rcas_post(lin_in, h16, TEX | SURF_IN) == I
        # the other arithmetic paths
        for r in refused:
            assert easu(t_in, h16, TEX | r) == U, r
            assert easu(t_in, h16, TEX | api.FLAG_SRTM_INPUT | r) == U, r
            for f in (0, api.FLAG_FUSED):
                assert upscale(t_in, tmp16, h16, f | TEX | r) == U, (f, r)
                assert upscale(t_in, tmp16, s_out, f | TEX | SURF_OUT | r) == U, (f, r)
                assert post(t_in, tmp16, h16, api.POST_SRTM_INVERSE, f | TEX | r) == U, (f, r)
        # constants that do not upscale: no kernel reads an array for a downscale
        assert easu(arr(16, 8, fmt), img(8192, 8, 4, 1), TEX, down) == U
        for f in (0, api.FLAG_FUSED):
            assert upscale(arr(16, 8, fmt), tmp16, h16, f | TEX, down) == U, f
            assert post(arr(16, 8, fmt), tmp16, h16, api.POST_SRTM_INVERSE, f | TEX, down) == U, f
            # EASU stores to linear images only
            assert upscale(t_in, None, s_out, f | TEX | SURF_OUT | api.FLAG_NO_RCAS) == U, f
        assert easu(t_in, h16, TEX | SURF_OUT) == U
    # RGBA16F and R11G11B10F only
    for fmt in (2, 3, 4):
        assert easu(arr(8, 4, fmt), img(8192, 16, 8, fmt), TEX) == U, fmt
        assert upscale(arr(8, 4, fmt), img(16384, 16, 8, fmt), img(8192, 16, 8, fmt), TEX) == U, fmt
        assert upscale(arr(8, 4, fmt), img(16384, 16, 8, fmt), img(8192, 16, 8, fmt), TEX | api.FLAG_FUSED) == U, fmt
    # RCAS reads the linear intermediate: fsr1_rcas and fsr1_rcas_post refuse the flag
    assert rcas(tmp16, h16, TEX) == U
    assert rcas(tmp16, s_out, TEX | SURF_OUT) == U
    assert rcas_post(img(0, 16, 8, 1), h16, TEX) == U
    assert rcas_post(img(0, 16, 8, 5), h16, TEX) == U
    # shards: windows and slabs are linear memory
    h = ctypes.c_void_p()
    for fl in (TEX, TEX | SURF_OUT, TEX | api.FLAG_SRTM_INPUT):
        assert L.fsr1_shard_create(ctypes.byref(h), 8, 4, 16, 8, 1, 1, 0, 1, ctypes.c_float(0.25), fl) == U
        assert L.fsr1_shard_create(ctypes.byref(h), 8, 4, 16, 8, 5, 1, 0, 1, ctypes.c_float(0.25), fl) == U
        p = _lib.Post(api.POST_SRTM_INVERSE, 0.0, None, None, 0, 0)
        assert L.fsr1_shard_create_post(ctypes.byref(h), 8, 4, 16, 8, 1, 1, ctypes.byref(p), 1, 0, 1, ctypes.c_float(0.25), fl) == U
    # flag 1 << 20 stays unknown
    assert easu(arr(8, 4, 1), h16, TEX | (1 << 20)) == I
    assert upscale(arr(8, 4, 1), tmp16, h16, TEX | api.FLAG_FUSED | (1 << 20)) == I
    assert L.fsr1_launch_count() == launches                                         # nothing was launched


# ---- the kernels on the emulator -------------------------------------------------------------------------------------------------
POISON16 = np.array([0x7E00, 0x7C00, 0x7BFF, 0xFC00], np.uint16)   # NaN, inf, 65504, -inf
POISON_R11 = np.array([0xFFFFFFFF, 0x7BFEF7BF, 0xF83E0FC0], np.uint32)   # NaN, 65024, inf in every channel


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def _pitch(a):
    return ctypes.c_longlong(a.strides[0])


class Tex:
    """An emulated 2D CUDA array read through a texture: the logical image in its top-left region, poison around it.  .h: the handle."""

    def __init__(self, slot, logical, extra=(3, 5)):
        lh, lw = logical.shape[:2]
        shape = (lh + extra[0], lw + extra[1]) + logical.shape[2:]
        self.a = np.ascontiguousarray(np.resize(POISON16 if logical.dtype == np.uint16 else POISON_R11, shape))
        self.a[:lh, :lw] = logical
        self.before = self.a.copy()
        self.h = tex_lib().emu_texture(slot, self.a.ctypes.data, self.a.strides[0], shape[1], shape[0], 8 if logical.dtype == np.uint16 else 4)


class Surf:
    """An emulated 2D CUDA array the fused kernels store into (FSR1_FLAG_OUT_SURFACE), poison around the logical image."""

    def __init__(self, slot, logical, extra=(2, 3)):
        lh, lw = logical.shape[:2]
        self.a = np.full((lh + extra[0], lw + extra[1]) + logical.shape[2:], 0x5A5A if logical.dtype == np.uint16 else 0x5A5A5A5A,
                         logical.dtype)
        self.a[:lh, :lw] = logical
        self.before = self.a.copy()
        self.lh, self.lw = lh, lw
        self.h = tex_lib().emu_tex_surface(slot, self.a.ctypes.data, self.a.strides[0], self.a.shape[1], self.a.shape[0],
                                           8 if logical.dtype == np.uint16 else 4)

    def logical(self):
        return self.a[:self.lh, :self.lw]

    def outside_unchanged(self):
        return np.array_equal(self.a[self.lh:], self.before[self.lh:]) and np.array_equal(self.a[:, self.lw:], self.before[:, self.lw:])


def raw_half(w, h, seed):
    """Random RGBA16F bits: NaNs with payloads, +-inf, -0, denormals and every exponent, with flat blocks at two corners."""
    x = np.random.default_rng(seed).integers(0, 1 << 16, size=(h, w, 4), dtype=np.uint32).astype(np.uint16)
    bw, bh = max(1, w // 5), max(1, h // 4)
    x[:bh, :bw] = 0x8000                 # -0
    x[h - bh:, w - bw:] = 0x0001         # the smallest denormal
    x[0, -1], x[-1, 0] = 0x7C00, 0xFC00  # +inf, -inf
    x[1 % h, 1 % w] = 0x7D23             # a NaN with a payload
    return x


def frame(fmt, w, h, seed, srtm):
    """The input in format fmt ("f16" RGBA16F bits, "r11" R11G11B10F codes): linear HDR content with SRTM_INPUT, raw bits without."""
    if fmt == "r11":
        return hdr_codes(w, h, seed) if srtm else raw_codes(w, h, seed)
    return np.ascontiguousarray(hdr_frame(w, h, seed).view(np.uint16)) if srtm else raw_half(w, h, seed)


def _out(oh, ow, out_format, fill):
    return np.full((oh, ow, 4), fill, np.uint16) if out_format == 1 else np.full((oh, ow), fill, np.uint32)


def _check_no_faults(before):
    assert tex_lib().emu_tex_faults() == before, "a texture fetch left the array or read the wrong element size"


QUAD_SHAPES = [(9, 5, 18, 10, [(0, 10)]), (37, 13, 74, 26, [(0, 26), (3, 21)]), (70, 21, 140, 42, [(0, 42), (7, 30), (1, 2)])]


@pytest.mark.parametrize("srtm", [0, 1])
@pytest.mark.parametrize("fmt", ["f16", "r11"])
@pytest.mark.parametrize("iw,ih,ow,oh,slabs", QUAD_SHAPES)
def test_emulated_quad2x_texture_input_equals_linear(srtm, fmt, iw, ih, ow, oh, slabs):
    L = tex_lib()
    faults = L.emu_tex_faults()
    x = frame(fmt, iw, ih, iw + 3 * ih + srtm, srtm)
    src = Tex(0, x)
    con = (ctypes.c_uint32 * 16)(*ol.easu_con(iw, ih, ow, oh))
    r11 = int(fmt == "r11")
    for y0, y1 in slabs:
        got, want = _out(oh, ow, 1, 0x7E5A), _out(oh, ow, 1, 0x7E5A)
        assert L.emu_easu_quad2x_tex(ctypes.c_void_p(src.h), 0, iw, ih, _ptr(got), ow, oh, _pitch(got), con, y0, y1, 3, srtm, r11, 1) == 0
        assert L.emu_easu_quad2x_tex(_ptr(x), _pitch(x), iw, ih, _ptr(want), ow, oh, _pitch(want), con, y0, y1, 3, srtm, r11, 0) == 0
        assert np.array_equal(got, want), (iw, ih, y0, y1)
        assert (got[:y0] == 0x7E5A).all() and (got[y1:] == 0x7E5A).all()
    assert np.array_equal(src.a, src.before)
    _check_no_faults(faults)


# 2x through the any-scale kernel, 1.5x, 1.3x x 1.7x (anisotropic), 1.0x x 1.1x, 41 -> 82 (almost 2x), 1.3x
PAIRS_SHAPES = [(33, 17, 66, 34), (50, 27, 75, 40), (70, 19, 91, 33), (69, 37, 69, 41), (41, 23, 82, 46), (77, 45, 100, 58)]


@pytest.mark.parametrize("srtm", [0, 1])
@pytest.mark.parametrize("fmt", ["f16", "r11"])
@pytest.mark.parametrize("iw,ih,ow,oh", PAIRS_SHAPES)
def test_emulated_vpairs_texture_input_equals_linear(srtm, fmt, iw, ih, ow, oh):
    L = tex_lib()
    faults = L.emu_tex_faults()
    x = frame(fmt, iw, ih, 3 * iw + ih + srtm, srtm)
    src = Tex(0, x, extra=(2, 9))
    con = (ctypes.c_uint32 * 16)(*ol.easu_con(iw, ih, ow, oh))
    r11 = int(fmt == "r11")
    for y0, y1 in ((0, oh), (5, oh - 2), (oh // 2, oh // 2 + 1)):
        got, want = _out(oh, ow, 1, 0x7E5A), _out(oh, ow, 1, 0x7E5A)
        assert L.emu_easu_pairs_tex(ctypes.c_void_p(src.h), 0, iw, ih, _ptr(got), ow, oh, _pitch(got), con, y0, y1, 2, srtm, r11, 1) == 0
        assert L.emu_easu_pairs_tex(_ptr(x), _pitch(x), iw, ih, _ptr(want), ow, oh, _pitch(want), con, y0, y1, 2, srtm, r11, 0) == 0
        assert np.array_equal(got, want), (iw, ih, ow, oh, y0, y1)
    _check_no_faults(faults)


def _fused_pair(x, iw, ih, ow, oh, out_format, rcon, y0, y1, ctas, post, srtm, r11, surf_out):
    """the fused kernel's texture twin (storing through a surface with surf_out) and the linear kernel on the same pixels: (got, want)"""
    L = tex_lib()
    faults = L.emu_tex_faults()
    src = Tex(0, x)
    fill = 0x7E5A if out_format == 1 else 0xA5C3E1F0
    dst = Surf(1, _out(oh, ow, out_format, fill)) if surf_out else None
    got, want = _out(oh, ow, out_format, fill), _out(oh, ow, out_format, fill)
    a_out = (ctypes.c_void_p(dst.h), 0) if surf_out else (_ptr(got), _pitch(got))
    pp = ctypes.byref(post) if post is not None else None
    assert L.emu_fused_tex(ctypes.c_void_p(src.h), 0, iw, ih, *a_out, ow, oh, out_format, rcon, y0, y1, ctas, pp, srtm, r11, 1, surf_out) == 0
    assert L.emu_fused_tex(_ptr(x), _pitch(x), iw, ih, _ptr(want), _pitch(want), ow, oh, out_format, rcon, y0, y1, ctas, pp, srtm, r11, 0,
                           0) == 0
    if surf_out:
        assert dst.outside_unchanged()
        got = dst.logical()
    assert np.array_equal(src.a, src.before)
    _check_no_faults(faults)
    return got, want


# (iw, ih, row slabs, CTAs): several steps per run, partial last steps, odd slab ends, 3 strips; odd strip origins
FUSED_SHAPES = [(40, 37, [(0, 74), (5, 61)], 3), (70, 9, [(0, 18), (1, 16)], 2), (33, 52, [(0, 104), (17, 99)], 4), (95, 11, [(0, 22)], 5)]


@pytest.mark.parametrize("surf_out", [0, 1])
@pytest.mark.parametrize("srtm", [0, 1])
@pytest.mark.parametrize("fmt", ["f16", "r11"])
@pytest.mark.parametrize("iw,ih,slabs,ctas", FUSED_SHAPES)
def test_emulated_fused_texture_input_equals_linear(surf_out, srtm, fmt, iw, ih, slabs, ctas):
    x = frame(fmt, iw, ih, 7 * iw + ih + srtm, srtm)
    ow, oh = 2 * iw - 1, 2 * ih                                                 # odd width: a partial last pair
    rcon = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    for y0, y1 in slabs:
        got, want = _fused_pair(x, iw, ih, ow, oh, 1, rcon, y0, y1, ctas, None, srtm, int(fmt == "r11"), surf_out)
        assert np.array_equal(got, want), (iw, ih, y0, y1)
        assert (got[:y0] == 0x7E5A).all() and (got[y1:] == 0x7E5A).all()


@pytest.mark.parametrize("surf_out", [0, 1])
@pytest.mark.parametrize("srtm", [0, 1])
@pytest.mark.parametrize("fmt", ["f16", "r11"])
@pytest.mark.parametrize("ops,out_format", CASES)
def test_emulated_fused_post_texture_input_equals_linear(surf_out, srtm, fmt, ops, out_format):
    """Every op subset of the display epilogue into RGBA16F, RGBA8 and RGB10A2; an odd width, a row slab, grain and dither tiles."""
    grains, dither_tile = _tiles(17)
    rcon = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    iw, ih, ow, oh = 40, 19, 79, 38
    x = frame(fmt, iw, ih, 11 + ops, srtm)
    post = _emu_post(ops, grains[srtm], 0.375, dither_tile if srtm == 0 else None, 5)
    for y0, y1 in ((0, oh), (oh // 3, 2 * oh // 3 + 1)):
        got, want = _fused_pair(x, iw, ih, ow, oh, out_format, rcon, y0, y1, 3, post, srtm, int(fmt == "r11"), surf_out)
        assert np.array_equal(got, want), (ops, out_format, y0, y1)
