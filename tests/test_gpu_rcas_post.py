"""fsr1_rcas_post on the H100: one RCAS kernel with the input stage (R11G11B10F decode, SRTM) and the display epilogue is bit-identical to
the composition of existing entry points it replaces: decode (bit operations in torch) -> srtm -> rcas -> srtm(inverse) -> lfga -> tepd,
through RGBA16F images.  Also: row slabs read from windows, every RCAS option, surface outputs, guard bytes around every linear image, and
which kernel runs."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

from fsr1_b200 import _lib, api

pytestmark = pytest.mark.gpu

CLAMP, DENOISE, ALPHA, SQUARE = api.FLAG_RCAS_CLAMP, api.FLAG_RCAS_DENOISE, api.FLAG_RCAS_PASSTHROUGH_ALPHA, api.FLAG_OUTPUT_SQUARE
S, OUT = api.FLAG_SRTM_INPUT, api.FLAG_OUT_SURFACE
RCAS_FLAGS = CLAMP | DENOISE | ALPHA | SQUARE
STAGES = ["r11", "r11_srtm", "h16_srtm", "h16"]


# ---- images ------------------------------------------------------------------------------------------------------------------------
def padded(h, w, dtype, channels=4, fill=None):
    """an [h, w, channels] ([h, w] with channels 0) tensor whose rows are padded to an even number of pixels: the 16-byte (RGBA16F) or
    8-byte (4-byte texels) aligned pitch the packed kernels take, on both sides of every comparison"""
    t = torch.empty((h, w + (w & 1), channels) if channels else (h, w + (w & 1)), dtype=dtype, device="cuda")[:, :w]
    if fill is not None:
        t.fill_(fill)
    return t


def padded_copy(x):
    t = padded(x.shape[0], x.shape[1], x.dtype, x.shape[2] if x.dim() == 3 else 0)
    t.copy_(x)
    return t


def r11_codes(w, h, seed, hdr):
    """R11G11B10F codes, int32 [h, w]: raw random codes (denormals, inf and NaN included) or an HDR image (finite values up to 65024)"""
    g = torch.Generator().manual_seed(seed)
    if not hdr:
        return padded_copy(torch.randint(-2 ** 31, 2 ** 31, (h, w), generator=g, dtype=torch.int64).to(torch.int32).cuda())
    e = torch.randint(0, 31, (h, w, 3), generator=g)                         # exponents 0..30: denormals to 65024, no inf / NaN
    m = torch.randint(0, 64, (h, w, 3), generator=g)
    ch = (e << 6 | m)
    ch[..., 2] >>= 1                                                           # B: 5 exponent bits over 5 mantissa bits
    return padded_copy((ch[..., 0] | ch[..., 1] << 11 | ch[..., 2] << 22).to(torch.int32).cuda())


def decode(codes):
    """the RGBA16F image (R, G, B, 1.0) of R11G11B10F codes: each channel is a half without its sign and low mantissa bits"""
    c = codes.to(torch.int64) & 0xFFFFFFFF
    r, g, b = (c & 0x7FF) << 4, ((c >> 11) & 0x7FF) << 4, ((c >> 22) & 0x3FF) << 5
    return torch.stack([r, g, b, torch.full_like(r, 0x3C00)], dim=-1).to(torch.int16).view(torch.float16)


def h16_frame(w, h, seed):
    """linear HDR RGBA16F with a random alpha (PASSTHROUGH_ALPHA carries it)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((h, w, 4), generator=g) * torch.exp2(torch.randint(-8, 12, (h, w, 4), generator=g).float())
    x[..., 3] = torch.rand((h, w), generator=g)
    return padded_copy(x.to(torch.float16).cuda())


def stage_input(stage, w, h, seed):
    """(the call's input tensor, its fsr1_image, the flag of the stage, the RGBA16F image the reference starts from)"""
    if stage.startswith("r11"):
        codes = r11_codes(w, h, seed, hdr=stage == "r11_srtm")
        return codes, api.image(codes, format=api.FORMAT_R11G11B10_FLOAT), S if stage == "r11_srtm" else 0, decode(codes)
    x = h16_frame(w, h, seed)
    return x, api.image(x), S if stage == "h16_srtm" else 0, x


def out_tensor(h, w, bits, fill=0):
    if bits == 8:
        return padded(h, w, torch.uint8, fill=fill)
    if bits == 10:
        return padded(h, w, torch.int32, 0, fill=fill)
    return padded(h, w, torch.float16, fill=fill)


def tile(seed, shape, dtype=torch.float16, shift=-0.5):
    g = torch.Generator().manual_seed(seed)
    return (torch.rand(shape, generator=g) + shift).to(dtype).cuda()


def reference(src16, flags, rcon, srtm_inverse, grain, amount, tepd_bits, dither, frame, want, y0=0, y1=0):
    """the separate passes: srtm (SRTM_INPUT) -> rcas -> srtm(inverse) -> lfga -> tepd through RGBA16F images, into `want`"""
    h, w = src16.shape[:2]
    i16 = padded_copy(src16)
    if flags & S:
        api.srtm(src16, i16)
    t = padded(h, w, torch.float16, fill=0)
    api.rcas(i16, t, rcon, y0, y1, flags & RCAS_FLAGS)
    if srtm_inverse:
        api.srtm(t, t, inverse=True, y0=y0, y1=y1)
    if grain is not None:
        api.lfga(t, grain, t, amount, y0=y0, y1=y1)
    if tepd_bits:
        api.tepd(t, want, tepd_bits, frame=frame, dither=dither, y0=y0, y1=y1)
    else:
        want[y0:y1 or h].copy_(t[y0:y1 or h])


def check(stage, w, h, seed, flags=0, srtm_inverse=False, grain=None, tepd_bits=0, dither=None, frame=0, y0=0, y1=0, sharpness=0.25):
    """fsr1_rcas_post against the separate passes, bit for bit, in one launch; returns the kernel name"""
    x, img, sflag, src16 = stage_input(stage, w, h, seed)
    rcon = api.rcas_con(sharpness)
    want = out_tensor(h, w, tepd_bits, fill=0x55)
    reference(src16, flags | sflag, rcon, srtm_inverse, grain, 0.3, tepd_bits, dither, frame, want, y0, y1)
    got = out_tensor(h, w, tepd_bits, fill=0x55)
    n0 = api.launch_count()
    api.rcas_post(img, got, rcon, srtm_inverse=srtm_inverse, grain=grain, amount=0.3, tepd_bits=tepd_bits, dither=dither, frame=frame,
                  y0=y0, y1=y1, flags=flags | sflag)
    torch.cuda.synchronize()
    n, name = api.launch_count() - n0, api.last_kernel()
    assert torch.equal(got.view(torch.uint8), want.view(torch.uint8)), (stage, w, h, flags, srtm_inverse, grain is not None, tepd_bits,
                                                                       y0, y1, name)
    assert n == 1, name
    return name


def expected_name(stage, post, store, surf=False):
    tags = {"r11": ",r11g11b10f_in", "r11_srtm": ",r11g11b10f_in,srtm_in", "h16_srtm": ",srtm_in", "h16": ""}[stage]
    return "rcas_h_packed%s<2px,4rows,shfl60%s%s%s>" % ("_post" if post else "", tags, ("," + store) if post else "",
                                                         ",surf_out" if surf else "")


# ---- the composition, bit for bit --------------------------------------------------------------------------------------------------
SIZES = [(3840, 2160), (2560, 1440), (61, 19), (257, 67)]
ENDINGS = [(False, False, 0), (False, True, 8), (True, False, 10)]   # (srtm_inverse, lfga, tepd_bits): none, SDR, HDR10-style


@pytest.mark.parametrize("ending", ENDINGS)
@pytest.mark.parametrize("stage", STAGES)
@pytest.mark.parametrize("size", SIZES)
def test_equals_the_separate_passes(size, stage, ending):
    w, h = size
    srtm_inverse, lfga, bits = ending
    name = check(stage, w, h, w + h, srtm_inverse=srtm_inverse, grain=tile(1, (64, 64, 4)) if lfga else None, tepd_bits=bits, frame=3)
    post = srtm_inverse or lfga or bits
    assert name == expected_name(stage, post, {0: "rgba16f", 8: "rgba8", 10: "rgb10a2"}[bits]), name


@pytest.mark.parametrize("flags", [CLAMP, DENOISE, ALPHA, SQUARE, CLAMP | DENOISE | ALPHA | SQUARE, DENOISE | SQUARE, api.FLAG_FUSED])
@pytest.mark.parametrize("stage", STAGES)
def test_every_rcas_option(stage, flags):
    for bits in (0, 8):
        for w, h in ((257, 67), (61, 19)):
            check(stage, w, h, 5 + bits, flags=flags, srtm_inverse=True, tepd_bits=bits, frame=1)
    check(stage, 257, 67, 9, flags=flags)


@pytest.mark.parametrize("srtm_inverse,lfga,bits", list(itertools.product((False, True), (False, True), (0, 8, 10))))
@pytest.mark.parametrize("stage", ["r11", "r11_srtm", "h16_srtm"])
def test_every_ops_set_with_tiles(stage, srtm_inverse, lfga, bits):
    """grain tiles RGBA16F and RGBA32F, a dither tile and the positional dither with frame != 0"""
    for k, (w, h) in enumerate(((257, 67), (131, 40))):
        grain = tile(2 + k, (5, 12, 4) if k == 0 else (7, 9, 4), torch.float16 if k == 0 else torch.float32) if lfga else None
        dither = tile(4, (3, 7, 4), torch.float32, shift=0.0) if bits and k == 1 else None
        check(stage, w, h, 11 + k, srtm_inverse=srtm_inverse, grain=grain, tepd_bits=bits, dither=dither, frame=7 + k)


@pytest.mark.parametrize("stage", STAGES)
def test_row_slabs_on_windows(stage):
    """each slab reads a window holding only rows [y0-1, y1+1) and writes nothing outside [y0, y1)"""
    for w, h, y0, y1, bits, flags in ((257, 67, 17, 50, 8, 0), (640, 360, 0, 101, 10, CLAMP), (640, 360, 101, 360, 0, DENOISE | ALPHA),
                                      (61, 19, 5, 6, 8, CLAMP | SQUARE)):
        x, _, sflag, src16 = stage_input(stage, w, h, y0 + w)
        rcon = api.rcas_con(0.5)
        want = out_tensor(h, w, bits, fill=77)
        reference(src16, flags | sflag, rcon, bits == 10, None, 0.0, bits, None, 2, want, y0, y1)
        r0, r1 = max(y0 - 1, 0), min(y1 + 1, h)
        win = x[r0:r1]
        img = api.image(win, height=h, row0=r0, format=api.FORMAT_R11G11B10_FLOAT if stage.startswith("r11") else None)
        got = out_tensor(h, w, bits, fill=77)
        api.rcas_post(img, got, rcon, srtm_inverse=bits == 10, tepd_bits=bits, frame=2, y0=y0, y1=y1, flags=flags | sflag)
        torch.cuda.synchronize()
        assert torch.equal(got.view(torch.uint8), want.view(torch.uint8)), (stage, w, h, y0, y1)


def test_no_post_on_rgba16f_is_rcas():
    """post == None (or ops == 0) on RGBA16F input without SRTM_INPUT runs fsr1_rcas's kernel and writes its bits"""
    x = h16_frame(640, 360, 3)
    rcon = api.rcas_con(0.25)
    for flags in (0, CLAMP | DENOISE | ALPHA | SQUARE):
        want = torch.zeros_like(x)
        api.rcas(x, want, rcon, flags=flags)
        torch.cuda.synchronize()
        rcas_name = api.last_kernel()
        got = torch.zeros_like(x)
        post = _lib.Post(0, 0.0, None, None, 0, 0)
        for p in (None, ctypes.byref(post)):
            got.zero_()
            _lib.check(_lib.lib().fsr1_rcas_post(ctypes.byref(api.image(x)), ctypes.byref(api.image(got)), (ctypes.c_uint32 * 4)(*rcon), p,
                                                 0, 0, flags, None))
            torch.cuda.synchronize()
            assert api.last_kernel() == rcas_name == "rcas_h_packed<2px,4rows,shfl60>"
            assert torch.equal(got.view(torch.int16), want.view(torch.int16))


# ---- surface outputs ---------------------------------------------------------------------------------------------------------------
class _Desc3D(ctypes.Structure):
    _fields_ = [("Width", ctypes.c_size_t), ("Height", ctypes.c_size_t), ("Depth", ctypes.c_size_t), ("Format", ctypes.c_int),
                ("NumChannels", ctypes.c_uint), ("Flags", ctypes.c_uint)]


class _ResDesc(ctypes.Structure):  # CUDA_RESOURCE_DESC with the array member of its union
    _fields_ = [("resType", ctypes.c_int), ("hArray", ctypes.c_void_p), ("reserved", ctypes.c_int * 30), ("flags", ctypes.c_uint)]


class _Copy2D(ctypes.Structure):  # CUDA_MEMCPY2D
    _fields_ = [("srcXInBytes", ctypes.c_size_t), ("srcY", ctypes.c_size_t), ("srcMemoryType", ctypes.c_int), ("srcHost", ctypes.c_void_p),
                ("srcDevice", ctypes.c_uint64), ("srcArray", ctypes.c_void_p), ("srcPitch", ctypes.c_size_t),
                ("dstXInBytes", ctypes.c_size_t), ("dstY", ctypes.c_size_t), ("dstMemoryType", ctypes.c_int), ("dstHost", ctypes.c_void_p),
                ("dstDevice", ctypes.c_uint64), ("dstArray", ctypes.c_void_p), ("dstPitch", ctypes.c_size_t),
                ("WidthInBytes", ctypes.c_size_t), ("Height", ctypes.c_size_t)]


_cu = None


def cu():
    global _cu
    if _cu is None:
        torch.zeros(1, device="cuda")          # torch's primary context is current on this thread
        _cu = ctypes.CDLL("libcuda.so.1")
    return _cu


def _ok(rc):
    assert rc == 0, "CUDA driver error %d" % rc


KINDS = {"rgba16f": (0x10, 4, 8), "rgba8": (0x01, 4, 4), "u32": (0x03, 1, 4)}   # (CUarray_format, channels, bytes)


class CudaArray:
    """A 2D CUDA array with surface load/store and a surface object on it."""

    def __init__(self, w, h, kind):
        fmt, ch, self.elem = KINDS[kind]
        self.w, self.h = w, h
        self.arr = ctypes.c_void_p()
        _ok(cu().cuArray3DCreate_v2(ctypes.byref(self.arr), ctypes.byref(_Desc3D(w, h, 0, fmt, ch, 0x02))))
        self.surf = ctypes.c_uint64()
        _ok(cu().cuSurfObjectCreate(ctypes.byref(self.surf), ctypes.byref(_ResDesc(0, self.arr))))
        self.handle = self.surf.value

    def _copy(self, t, to_array):
        c = _Copy2D()
        if to_array:
            c.srcMemoryType, c.srcDevice, c.srcPitch, c.dstMemoryType, c.dstArray = 2, t.data_ptr(), t.stride(0) * t.element_size(), 3, self.arr
        else:
            c.srcMemoryType, c.srcArray, c.dstMemoryType, c.dstDevice, c.dstPitch = 3, self.arr, 2, t.data_ptr(), t.stride(0) * t.element_size()
        c.WidthInBytes, c.Height = t.shape[1] * self.elem, t.shape[0]
        torch.cuda.synchronize()
        _ok(cu().cuMemcpy2D_v2(ctypes.byref(c)))

    def upload(self, t):
        self._copy(t, True)

    def download(self):
        """the whole array as raw bits: int16 [h, w, 4] for 8-byte elements, int32 [h, w] for 4-byte ones"""
        t = torch.empty((self.h, self.w, 4) if self.elem == 8 else (self.h, self.w), dtype=torch.int16 if self.elem == 8 else torch.int32,
                        device="cuda")
        self._copy(t, False)
        return t

    def close(self):
        cu().cuSurfObjectDestroy(ctypes.c_uint64(self.handle))
        cu().cuArrayDestroy(self.arr)


@pytest.mark.parametrize("bits,kind,fmt", [(0, "rgba16f", api.FORMAT_RGBA16F), (8, "rgba8", api.FORMAT_RGBA8_UNORM),
                                           (10, "u32", api.FORMAT_RGB10A2_UNORM)])
@pytest.mark.parametrize("stage", STAGES)
def test_surface_output_equals_linear_output(stage, bits, kind, fmt):
    """OUT_SURFACE into an array larger than the logical image: the linear call's bits inside, every texel outside unchanged"""
    w, h, aw, ah = 257, 67, 300, 80
    arr = CudaArray(aw, ah, kind)
    try:
        for flags, y0, y1, post in ((0, 0, 0, bits != 0), (CLAMP | ALPHA, 9, 40, True), (DENOISE | SQUARE, 0, 0, True)):
            x, img, sflag, _ = stage_input(stage, w, h, 21 + y0)
            rcon = api.rcas_con(0.5)
            fill = torch.full((ah, aw, 4) if kind != "u32" else (ah, aw), 0x3A, dtype=torch.int16 if kind == "rgba16f" else
                              torch.uint8 if kind == "rgba8" else torch.int32, device="cuda")
            arr.upload(fill)
            before = arr.download()
            want = out_tensor(h, w, bits)
            kw = dict(srtm_inverse=post and bits != 8, tepd_bits=bits, frame=5, y0=y0, y1=y1)
            api.rcas_post(img, want, rcon, flags=flags | sflag, **kw)
            api.rcas_post(img, api.surface_image(arr.handle, w, h, fmt), rcon, flags=flags | sflag | OUT, **kw)
            torch.cuda.synchronize()
            got = arr.download()
            r1 = y1 or h
            if kind == "rgba16f":
                inside = want.view(torch.int16)[y0:r1]
            else:
                inside = want.view(torch.int32).reshape(h, w)[y0:r1]
            assert torch.equal(got[y0:r1, :w], inside), (stage, kind, flags)
            mask = torch.ones(got.shape[:2], dtype=torch.bool, device="cuda")
            mask[y0:r1, :w] = False
            assert torch.equal(got[mask], before[mask]), (stage, kind, flags)
            want_name = expected_name(stage, kw["srtm_inverse"] or bits, {0: "rgba16f", 8: "rgba8", 10: "rgb10a2"}[bits], surf=True)
            assert api.last_kernel() == want_name, api.last_kernel()
    finally:
        torch.cuda.synchronize()
        arr.close()


# ---- guard bytes: the call reads and writes only its own pixels --------------------------------------------------------------------
GR, GC = 3, 32   # guard rows above and below, guard bytes left and right of every row


class Guarded:
    """rows x row_bytes bytes at byte offset GC of row GR in a poisoned buffer (NaN halves, or 0xFF bytes)"""

    def __init__(self, rows, row_bytes, poison):
        pitch = (row_bytes + 2 * GC + 127) // 128 * 128
        self.buf = torch.full((rows + 2 * GR, pitch), poison, dtype=torch.uint8, device="cuda")
        self.rows, self.row_bytes = rows, row_bytes
        self.inner = self.buf[GR:GR + rows, GC:GC + row_bytes]

    def outside(self):
        m = torch.ones_like(self.buf, dtype=torch.bool)
        m[GR:GR + self.rows, GC:GC + self.row_bytes] = False
        return self.buf[m].clone()


@pytest.mark.parametrize("poison", [0x7E, 0xFF])
@pytest.mark.parametrize("stage", STAGES)
def test_stays_inside_its_images(stage, poison):
    for w, h, y0, y1, bits, flags in ((257, 67, 0, 67, 8, 0), (61, 19, 0, 19, 0, CLAMP), (131, 40, 9, 30, 10, ALPHA | DENOISE),
                                      (63, 33, 3, 20, 0, CLAMP | SQUARE)):
        x, _, sflag, src16 = stage_input(stage, w, h, w + poison)
        r0, r1 = max(y0 - 1, 0), min(y1 + 1, h)
        r11 = stage.startswith("r11")
        bpp = 4 if r11 else 8
        gin = Guarded(r1 - r0, w * bpp, poison)
        gin.inner.copy_(x[r0:r1].contiguous().view(torch.uint8).reshape(r1 - r0, w * bpp))
        obpp = 8 if bits == 0 else 4
        gout = Guarded(h, w * obpp, poison)
        gin_out, gout_out = gin.outside(), gout.outside()
        fmt = api.FORMAT_R11G11B10_FLOAT if r11 else api.FORMAT_RGBA16F
        img_in = _lib.Image(gin.inner.data_ptr(), gin.buf.stride(0), w, h, r0, r1 - r0, fmt, 0)
        ofmt = {0: api.FORMAT_RGBA16F, 8: api.FORMAT_RGBA8_UNORM, 10: api.FORMAT_RGB10A2_UNORM}[bits]
        img_out = _lib.Image(gout.inner.data_ptr(), gout.buf.stride(0), w, h, 0, h, ofmt, 0)
        rcon = api.rcas_con(0.25)
        api.rcas_post(img_in, img_out, rcon, srtm_inverse=bits == 10, tepd_bits=bits, frame=1, y0=y0, y1=y1, flags=flags | sflag)
        want = out_tensor(h, w, bits)
        reference(src16, flags | sflag, rcon, bits == 10, None, 0.0, bits, None, 1, want, y0, y1)
        torch.cuda.synchronize()
        assert torch.equal(gin.outside(), gin_out) and torch.equal(gout.outside(), gout_out), (stage, w, h, y0, y1)
        got = gout.inner[y0:y1]
        assert torch.equal(got, want.view(torch.uint8).reshape(h, w * obpp)[y0:y1]), (stage, w, h, y0, y1)
        assert (gout.inner[:y0] == poison).all() and (gout.inner[y1:] == poison).all()
