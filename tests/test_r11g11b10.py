"""FSR1_FORMAT_R11G11B10_FLOAT input without a GPU: the test-side decoder against the format's definition, the R11G11B10F variants of the
EASU kernels run on the CPU emulator (tests/emu/emu_r11.cpp) against their RGBA16F twins on the decoded image, and the ABI's refusals, which
all return before any CUDA call.  The GPU side is tests/test_gpu_r11g11b10.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import fsr1_b200 as F
import oracle_lib as ol
from fsr1_b200 import _lib
from test_emu import EMU_DIR, emu_lib
from test_srtm_input import hdr_frame, srtm_lib
from test_upscale_post import CASES, _emu_post, _out_buffer, _tiles, post_lib

R11 = 5
_r11_lib = None


def r11_lib():
    """tests/emu/emu_r11.cpp: the R11G11B10F-input kernels on CPU threads (a library of its own, tests/emu/r11.mk)"""
    global _r11_lib
    if _r11_lib is None:
        subprocess.check_call(["make", "-s", "-C", EMU_DIR, "-f", "r11.mk", "libfsr1_emu_r11.so"])
        _r11_lib = ctypes.CDLL(os.path.join(EMU_DIR, "libfsr1_emu_r11.so"))
    return _r11_lib


# ---- the format ----------------------------------------------------------------------------------------------------------------
def decode(codes):
    """uint32 [H, W] R11G11B10F codes -> the RGBA16F image of their values, as uint16 bits [H, W, 4] (alpha 1.0): each channel's
    5-bit exponent and 6- (R, G) or 5-bit (B) mantissa are a half's exponent and the top of its mantissa."""
    c = np.asarray(codes, np.uint32)
    r, g, b = (c & 0x7FF) << 4, ((c >> 11) & 0x7FF) << 4, ((c >> 22) & 0x3FF) << 5
    return np.stack([r, g, b, np.full_like(r, 0x3C00)], axis=-1).astype(np.uint16)


def raw_codes(w, h, seed):
    """Raw random 32-bit codes: every exponent of every channel, denormals, zeros, 65024, inf and NaN all appear; plus flat blocks
    of all-zero and all-max-finite codes at two corners (border tiles see them)."""
    c = np.random.default_rng(seed).integers(0, 1 << 32, size=(h, w), dtype=np.uint64).astype(np.uint32)
    bw, bh = max(1, w // 5), max(1, h // 4)
    c[:bh, :bw] = 0
    c[h - bh:, w - bw:] = (0x3DF << 22) | (0x7BF << 11) | 0x7BF       # 65024 in every channel
    return c


def hdr_codes(w, h, seed):
    """A linear HDR image (tests/test_srtm_input.hdr_frame: values up to 65504, flat 0 / 1 / max blocks) in R11G11B10F, every half
    truncated to the format's mantissa (65504 becomes 65024)."""
    x = hdr_frame(w, h, seed).view(np.uint16).astype(np.uint32) & 0x7FFF
    return ((x[..., 0] >> 4) | ((x[..., 1] >> 4) << 11) | ((x[..., 2] >> 5) << 22)).astype(np.uint32)


FRAMES = {"raw": raw_codes, "hdr": hdr_codes}


def _definition(code, k):
    """value of one unsigned small float with a 5-bit exponent (bias 15) and a k-bit mantissa"""
    e, m = code >> k, code & ((1 << k) - 1)
    if e == 0:
        return m / 2.0 ** k * 2.0 ** -14
    if e == 31:
        return np.inf if m == 0 else np.nan
    return (1.0 + m / 2.0 ** k) * 2.0 ** (e - 15)


@pytest.mark.parametrize("channel,k,shift", [("R", 6, 0), ("G", 6, 11), ("B", 5, 22)])
def test_decoder_matches_the_format_definition_for_every_code(channel, k, shift):
    n = 1 << (k + 5)
    codes = np.arange(n, dtype=np.uint32) << shift
    got = decode(codes[None, :])[0, :, "RGB".index(channel)].view(np.float16).astype(np.float64)
    want = np.array([_definition(int(x), k) for x in range(n)])
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    assert np.array_equal(got[ok], want[ok])
    assert (decode(codes[None, :])[0, :, 3] == 0x3C00).all()
    if channel == "R":
        assert _definition(0x7BF, 6) == 65024.0 and _definition(1, 6) == 2.0 ** -20


# ---- the kernels on the emulator -------------------------------------------------------------------------------------------------
def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def _pitch(a):
    return ctypes.c_longlong(a.strides[0])


def _run_pair(r11_fn, twin_fn, twin_pre, codes, ow, oh, con, y0, y1, ctas, srtm, extra=()):
    """the R11G11B10F kernel on `codes` and its RGBA16F twin on decode(codes), both into sentinel-filled outputs"""
    ih, iw = codes.shape
    dec = decode(codes)
    got = np.full((oh, ow, 4), 0x7E5A, np.uint16)
    want = got.copy()
    assert r11_fn(_ptr(codes), iw, ih, _pitch(codes), _ptr(got), ow, oh, _pitch(got), *extra[:1], con, y0, y1, ctas, *extra[1:], srtm) == 0
    assert twin_fn(*twin_pre, _ptr(dec), iw, ih, _pitch(dec), _ptr(want), ow, oh, _pitch(want), *extra[:1], con, y0, y1, ctas,
                   *extra[1:]) == 0
    return got, want


QUAD_SHAPES = [(9, 5, 18, 10, [(0, 10)]), (37, 13, 74, 26, [(0, 26), (3, 21)]), (70, 21, 140, 42, [(0, 42), (7, 30), (1, 2)])]


@pytest.mark.parametrize("srtm", [0, 1])
@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("iw,ih,ow,oh,slabs", QUAD_SHAPES)
def test_emulated_quad2x_equals_rgba16f_twin(srtm, frame, iw, ih, ow, oh, slabs):
    codes = FRAMES[frame](iw, ih, iw * 3 + ih + srtm)
    con = (ctypes.c_uint32 * 16)(*ol.easu_con(iw, ih, ow, oh))
    twin, pre = (srtm_lib().emu_easu_h_quad2x_srtm_in, ()) if srtm else (emu_lib().emu_easu_h_quad2x, (12,))
    for y0, y1 in slabs:
        before = codes.copy()
        got, want = _run_pair(r11_lib().emu_easu_r11_quad2x, twin, pre, codes, ow, oh, con, y0, y1, 3, srtm)
        assert np.array_equal(got, want), (iw, ih, y0, y1)
        assert (got[:y0] == 0x7E5A).all() and (got[y1:] == 0x7E5A).all()
        assert np.array_equal(codes, before)


# 2x through the any-scale kernel, 1.5x, 1.3x x 1.7x (anisotropic), 1.0x x 1.1x (the largest boxes)
PAIRS_SHAPES = [(33, 17, 66, 34), (50, 27, 75, 40), (70, 19, 91, 33), (69, 37, 69, 41)]


@pytest.mark.parametrize("srtm", [0, 1])
@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("iw,ih,ow,oh", PAIRS_SHAPES)
def test_emulated_vpairs_equals_rgba16f_twin(srtm, frame, iw, ih, ow, oh):
    codes = FRAMES[frame](iw, ih, iw + 5 * ih + srtm)
    con = (ctypes.c_uint32 * 16)(*ol.easu_con(iw, ih, ow, oh))
    twin, pre = (srtm_lib().emu_easu_h_pairs_srtm_in, ()) if srtm else (emu_lib().emu_easu_h_pairs, (1,))
    for y0, y1 in ((0, oh), (5, oh - 2), (oh // 2, oh // 2 + 1)):
        got, want = _run_pair(r11_lib().emu_easu_r11_pairs, twin, pre, codes, ow, oh, con, y0, y1, 2, srtm)
        assert np.array_equal(got, want), (iw, ih, ow, oh, y0, y1)
        assert (got[:y0] == 0x7E5A).all() and (got[y1:] == 0x7E5A).all()


# (iw, ih, row slabs, CTAs): several steps per run, partial last steps, odd slab ends, 3 strips; odd strip origins (box shift 0 and 2)
FUSED_SHAPES = [(40, 37, [(0, 74), (5, 61)], 3), (70, 9, [(0, 18), (1, 16)], 2), (33, 52, [(0, 104), (17, 99)], 4), (95, 11, [(0, 22)], 5)]


@pytest.mark.parametrize("srtm", [0, 1])
@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("iw,ih,slabs,ctas", FUSED_SHAPES)
def test_emulated_fused_equals_rgba16f_twin(srtm, frame, iw, ih, slabs, ctas):
    codes = FRAMES[frame](iw, ih, 7 * iw + ih + srtm)
    ow, oh = 2 * iw - 1, 2 * ih                                                 # odd width: a partial last pair
    rcon = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    twin = srtm_lib().emu_fused_h_srtm_in if srtm else emu_lib().emu_fused_h
    for y0, y1 in slabs:
        got, want = _run_pair(r11_lib().emu_fused_r11, twin, (), codes, ow, oh, rcon, y0, y1, ctas, srtm)
        assert np.array_equal(got, want), (iw, ih, y0, y1)
        assert (got[:y0] == 0x7E5A).all() and (got[y1:] == 0x7E5A).all()


@pytest.mark.parametrize("srtm", [0, 1])
@pytest.mark.parametrize("ops,out_format", CASES)
def test_emulated_fused_post_equals_rgba16f_twin(srtm, ops, out_format):
    """Every op subset of the display epilogue, both UNORM outputs; odd widths, a row slab, grain and dither tiles."""
    grains, dither_tile = _tiles(17)
    rcon = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    twin = srtm_lib().emu_fused_h_post_srtm_in if srtm else post_lib().emu_fused_h_post
    for k, (iw, ih, ow, oh, frame) in enumerate([(40, 19, 79, 38, "hdr"), (70, 9, 139, 18, "raw")]):
        codes = FRAMES[frame](iw, ih, 11 + k)
        dec = decode(codes)
        post = _emu_post(ops, grains[k], 0.375, dither_tile if k == 0 else None, 5)
        for y0, y1 in ((0, oh), (oh // 3, 2 * oh // 3 + 1)):
            got, want = _out_buffer(oh, ow, out_format), _out_buffer(oh, ow, out_format)
            assert r11_lib().emu_fused_r11_post(_ptr(codes), iw, ih, _pitch(codes), _ptr(got), ow, oh, _pitch(got), out_format, rcon,
                                                y0, y1, 3, ctypes.byref(post), srtm) == 0
            assert twin(_ptr(dec), iw, ih, _pitch(dec), _ptr(want), ow, oh, _pitch(want), out_format, rcon, y0, y1, 3,
                        ctypes.byref(post)) == 0
            assert np.array_equal(got, want), (iw, ih, y0, y1)
            assert not got[:y0].any() and not got[y1:].any()


# ---- the ABI's refusals ------------------------------------------------------------------------------------------------------------
def test_r11g11b10_validation_without_gpu():
    """Every refusal of the format returns before any CUDA call: nothing is launched."""
    L = _lib.lib()
    api = F.api
    assert _lib.FORMAT_R11G11B10_FLOAT == R11 and api.FORMAT_R11G11B10_FLOAT == R11
    launches = L.fsr1_launch_count()   # the counter is process-wide: GPU tests may have run earlier in this process
    buf = (ctypes.c_uint8 * 65536)()
    addr = ctypes.addressof(buf)
    addr += (-addr) % 256
    econ = (ctypes.c_uint32 * 16)(*api.easu_con(8, 4, 8, 4, 16, 8))
    rcon = (ctypes.c_uint32 * 4)(*api.rcas_con(0.25))
    BPP = {1: 8, 2: 16, 3: 4, 4: 4, R11: 4}

    def img(off, w, h, fmt, pitch=None):
        return _lib.Image(addr + off, pitch or 16 * ((w * BPP[fmt] + 15) // 16), w, h, 0, h, fmt, 0)

    inp = img(0, 8, 4, R11)
    h16, h32, u8, u10, r11o = img(8192, 16, 8, 1), img(8192, 16, 8, 2), img(8192, 16, 8, 3), img(8192, 16, 8, 4), img(8192, 16, 8, R11)
    tmp16 = img(16384, 16, 8, 1)
    U = -2

    def easu(i, o, flags=0):
        return L.fsr1_easu(ctypes.byref(i), ctypes.byref(o), econ, 0, 0, flags, None)

    def upscale(i, t, o, flags=0):
        return L.fsr1_upscale(ctypes.byref(i), ctypes.byref(t) if t is not None else None, ctypes.byref(o), econ, rcon, 0, 0, flags, None)

    def post(i, t, o, ops, flags=api.FLAG_FUSED, dither=None):
        p = _lib.Post(ops, 0.0, None, ctypes.pointer(dither) if dither is not None else None, 0, 0)
        return L.fsr1_upscale_post(ctypes.byref(i), ctypes.byref(t) if t is not None else None, ctypes.byref(o), econ, rcon,
                                   ctypes.byref(p), 0, 0, flags, None)

    # EASU: R11G11B10F in, RGBA16F out is the one mixed pair; it is never an output
    for o in (r11o, h32, u8, u10):
        assert easu(inp, o) == U
    assert easu(img(0, 8, 4, 1), r11o) == U
    assert easu(img(0, 8, 4, 1), h32) == U                                          # RGBA16F -> RGBA32F stays refused
    refused = (api.FLAG_EXACT, api.FLAG_H_REFERENCE, api.FLAG_PRECISE, api.FLAG_RCAS_HX2)
    for f in refused:
        assert easu(inp, h16, f) == U, f
    # RCAS never takes it
    for a, b in ((r11o, r11o), (img(0, 16, 8, R11), h16), (h16, r11o)):
        assert L.fsr1_rcas(ctypes.byref(a), ctypes.byref(b), rcon, 0, 0, 0, None) == U
    # upscale: tmp and out are RGBA16F; nothing runs before a refusal
    for f in (0, api.FLAG_FUSED, api.FLAG_RCAS_CLAMP, api.FLAG_FUSED | api.FLAG_RCAS_DENOISE):
        for t, o in ((tmp16, r11o), (tmp16, h32), (tmp16, u8), (img(16384, 16, 8, R11), h16), (img(16384, 16, 8, 2), h16)):
            assert upscale(inp, t, o, f) == U, (f, t.format, o.format)
        for r in refused:
            assert upscale(inp, tmp16, h16, f | r) == U, (f, r)
    for o in (r11o, u8, u10):
        assert upscale(inp, None, o, api.FLAG_NO_RCAS) == U
    # upscale_post: as fsr1_upscale_post's rules, plus PRECISE and RCAS_HX2
    for ops, o in ((api.POST_SRTM_INVERSE, r11o), (api.POST_TEPD8, u10), (api.POST_TEPD10, u8), (api.POST_TEPD8, r11o)):
        assert post(inp, tmp16, o, ops) == U
    for r in refused + (api.FLAG_FORCE_DIRECT, api.FLAG_NO_RCAS):
        assert post(inp, tmp16, h16, api.POST_SRTM_INVERSE, api.FLAG_FUSED | r) == U, r
    assert post(inp, img(16384, 16, 8, R11), h16, api.POST_SRTM_INVERSE) == U                   # tmp
    assert post(img(0, 8, 4, 1), tmp16, u10, api.POST_TEPD10, dither=img(32768, 4, 4, R11)) == U  # a dither tile
    # the pointwise passes, both forms
    a, b = img(0, 16, 8, R11), img(8192, 16, 8, R11)
    assert L.fsr1_srtm(ctypes.byref(a), ctypes.byref(b), 0, 0, 0, None) == U
    assert L.fsr1_srtm(ctypes.byref(a), ctypes.byref(h16), 1, 0, 0, None) == U
    assert L.fsr1_srtm(ctypes.byref(h16), ctypes.byref(a), 0, 0, 0, None) == U
    assert L.fsr1_tepd(ctypes.byref(a), None, ctypes.byref(u8), 8, 0, 0, 0, None) == U
    assert L.fsr1_tepd(ctypes.byref(tmp16), ctypes.byref(img(32768, 4, 4, R11)), ctypes.byref(u10), 10, 0, 0, 0, None) == U
    assert L.fsr1_lfga(ctypes.byref(tmp16), ctypes.byref(img(32768, 4, 4, R11)), ctypes.byref(h16), 0.5, 0, 0, None) == U
    assert L.fsr1_lfga(ctypes.byref(a), ctypes.byref(img(32768, 4, 4, 1)), ctypes.byref(b), 0.5, 0, 0, None) == U
    assert L.fsr1_srtm_h(ctypes.byref(a), ctypes.byref(h16), 0, 0, 0, None) == U
    assert L.fsr1_tepd_h(ctypes.byref(a), None, ctypes.byref(h16), 8, 0, 0, 0, None) == U
    assert L.fsr1_lfga_h(ctypes.byref(a), ctypes.byref(img(32768, 4, 4, 1)), ctypes.byref(h16), 0.5, 0, 0, None) == U
    # SRTM_INPUT keeps its own rules: a direct kernel or an unaligned layout is refused
    S = api.FLAG_SRTM_INPUT
    assert easu(inp, h16, S | api.FLAG_FORCE_DIRECT) == U
    assert easu(img(0, 8, 4, R11, pitch=36), h16, S) == U
    assert easu(img(4, 8, 4, R11), h16, S) == U
    assert upscale(img(0, 8, 4, R11, pitch=36), tmp16, h16, S | api.FLAG_FUSED) == U
    # shards: slabs are RGBA16F (or the TEPD format); the format is never an output
    h = ctypes.c_void_p()
    assert L.fsr1_shard_create_post(ctypes.byref(h), 8, 4, 16, 8, R11, R11, None, 1, 0, 1, ctypes.c_float(0.25), 0) == U
    assert L.fsr1_shard_create_post(ctypes.byref(h), 8, 4, 16, 8, R11, 3, None, 1, 0, 1, ctypes.c_float(0.25), 0) == U
    p = _lib.Post(api.POST_TEPD8, 0.0, None, None, 0, 0)
    assert L.fsr1_shard_create_post(ctypes.byref(h), 8, 4, 16, 8, R11, 3, ctypes.byref(p), 1, 0, 1, ctypes.c_float(0.25),
                                    api.FLAG_PRECISE) == U
    assert L.fsr1_shard_create_post(ctypes.byref(h), 8, 4, 16, 8, R11, 4, ctypes.byref(p), 1, 0, 1, ctypes.c_float(0.25), 0) == U
    # format 9 and flag 1 << 20 stay unknown
    assert easu(_lib.Image(addr, 64, 8, 4, 0, 4, 9, 0), h16) == -1
    assert easu(inp, h16, 1 << 20) == -1
    assert L.fsr1_launch_count() == launches                                         # nothing was launched


def test_image_descriptor_of_an_r11g11b10_tensor():
    """api.image: int32 [H, W] is RGB10A2 unless format=FORMAT_R11G11B10_FLOAT says otherwise (checked on a CPU tensor's refusal:
    descriptors are built for CUDA tensors only)."""
    torch = pytest.importorskip("torch")
    api = F.api
    t = torch.zeros((4, 8), dtype=torch.int32)
    with pytest.raises(api.Fsr1Error, match="CUDA"):
        api.image(t, format=api.FORMAT_R11G11B10_FLOAT)
    if torch.cuda.is_available():
        assert api.image(t.cuda()).format == api.FORMAT_RGB10A2_UNORM
        assert api.image(t.cuda(), format=api.FORMAT_R11G11B10_FLOAT).format == R11
        with pytest.raises(api.Fsr1Error):
            api.image(torch.zeros((4, 8, 4), dtype=torch.float16, device="cuda"), format=api.FORMAT_R11G11B10_FLOAT)
