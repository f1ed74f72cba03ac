"""FSR1_FLAG_IN_SURFACE / FSR1_FLAG_OUT_SURFACE on the H100: every call that reads its input from, or writes its output to, a CUDA array
through a surface object is bit-identical to the same call on linear tensors holding the same pixels, and runs the surface twin of the
kernel the linear call runs.  torch has no CUDA arrays: they are made with the driver API through ctypes (libcuda.so.1, torch's primary
context), as an engine's interop would hand them over."""
import ctypes
import fnmatch

import numpy as np
import pytest
import torch

from fsr1_b200 import _lib, api

pytestmark = pytest.mark.gpu

IN, OUT, S, FUSED = api.FLAG_IN_SURFACE, api.FLAG_OUT_SURFACE, api.FLAG_SRTM_INPUT, api.FLAG_FUSED
RGBA16F, RGBA8, RGB10A2 = api.FORMAT_RGBA16F, api.FORMAT_RGBA8_UNORM, api.FORMAT_RGB10A2_UNORM


# ---- CUDA arrays and surface objects through the driver API --------------------------------------------------------------------------
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


# element kinds: (CUarray_format, channels, bytes)
KINDS = {"rgba16f": (0x10, 4, 8), "rgba8": (0x01, 4, 4), "u32": (0x03, 1, 4)}
KIND_OF = {RGBA16F: "rgba16f", RGBA8: "rgba8", RGB10A2: "u32"}


class CudaArray:
    """A 2D CUDA array with surface load/store (layered: one layer of a layered array) and a surface object on it."""

    def __init__(self, w, h, kind, layered=False):
        fmt, ch, self.elem = KINDS[kind]
        self.w, self.h = w, h
        self.arr = ctypes.c_void_p()
        _ok(cu().cuArray3DCreate_v2(ctypes.byref(self.arr), ctypes.byref(_Desc3D(w, h, 1 if layered else 0, fmt, ch, 0x02 | (0x01 if layered else 0)))))
        self.surf = ctypes.c_uint64()
        _ok(cu().cuSurfObjectCreate(ctypes.byref(self.surf), ctypes.byref(_ResDesc(0, self.arr))))
        self.handle = self.surf.value

    def _copy(self, t, to_array):
        rows, row_bytes = t.shape[0], t.shape[1] * self.elem
        c = _Copy2D()
        if to_array:
            c.srcMemoryType, c.srcDevice, c.srcPitch, c.dstMemoryType, c.dstArray = 2, t.data_ptr(), t.stride(0) * t.element_size(), 3, self.arr
        else:
            c.srcMemoryType, c.srcArray, c.dstMemoryType, c.dstDevice, c.dstPitch = 3, self.arr, 2, t.data_ptr(), t.stride(0) * t.element_size()
        c.WidthInBytes, c.Height = row_bytes, rows
        torch.cuda.synchronize()
        _ok(cu().cuMemcpy2D_v2(ctypes.byref(c)))

    def upload(self, t):
        """t (a device tensor of whole texels, rows x cols <= the array) into the array's top-left region"""
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


@pytest.fixture
def arrays():
    made = []

    def make(*a, **k):
        made.append(CudaArray(*a, **k))
        return made[-1]
    yield make
    torch.cuda.synchronize()
    for a in made:
        a.close()


# ---- images ------------------------------------------------------------------------------------------------------------------------
def plain(t):
    """a copy of t whose rows are padded to 16 bytes: the layout the linear call's tiled kernels take (an unaligned pitch would send it
    to another kernel)"""
    h, w = t.shape[:2]
    out = torch.empty((h, w + (w & 1)) + tuple(t.shape[2:]), dtype=t.dtype, device="cuda")[:, :w]
    out.copy_(t)
    return out


def frame(w, h, seed, hdr=False):
    """float16 [h, w, 4] in rows padded to 16 bytes: [0, 1) values, or linear HDR up to 65504 for SRTM_INPUT"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand((h, w, 4), generator=g, device="cuda")
    if hdr:
        x = torch.clamp(x * torch.exp2(torch.randint(-8, 16, (h, w, 4), generator=g, device="cuda").float()), max=65504.0)
    return plain(x.half())


def bits(t):
    """raw bits of a linear image or an array download: int16 [h, w, 4] (RGBA16F) or int32 [h, w] (4-byte texels)"""
    if t.dtype == torch.float16:
        return t.view(torch.int16)
    if t.dtype == torch.uint8:
        return t.contiguous().view(torch.int32)[..., 0]
    if t.dtype == torch.int16:
        return t
    return t


def linear_out(oh, ow, fmt):
    if fmt == RGBA16F:
        return plain(torch.full((oh, ow, 4), 3.0, dtype=torch.float16, device="cuda"))
    if fmt == RGBA8:
        return torch.zeros((oh, ow + (-ow & 1), 4), dtype=torch.uint8, device="cuda")[:, :ow]
    return torch.zeros((oh, ow + (-ow & 1)), dtype=torch.int32, device="cuda")[:, :ow]


def poison_like(a, seed):
    """NaN, inf, 65504 and random bits, as the array's elements"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if a.elem == 8:
        p = torch.randint(-32768, 32767, (a.h, a.w, 4), generator=g, device="cuda", dtype=torch.int32).to(torch.int16)
        p[::3] = 0x7E00
        p[1::3, ::2] = 0x7C00
        p[2::3, 1::2] = 0x7BFF
    else:
        p = torch.randint(-2 ** 31, 2 ** 31 - 1, (a.h, a.w), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)
    return p


def in_array(arrays, x, extra=(0, 0), seed=1):
    """an RGBA16F array holding x in its top-left region, poisoned outside it"""
    h, w = x.shape[:2]
    a = arrays(w + extra[0], h + extra[1], "rgba16f")
    if extra != (0, 0):
        a.upload(poison_like(a, seed))
    a.upload(x)
    return a


def out_array(arrays, oh, ow, fmt, extra=(0, 0), seed=2):
    """a poisoned array of the output format, at least ow x oh; (array, its contents before the call)"""
    a = arrays(ow + extra[0], oh + extra[1], KIND_OF[fmt])
    a.upload(poison_like(a, seed))
    return a, a.download()


def surf(a, w, h, fmt=RGBA16F):
    return api.surface_image(a.handle, w, h, fmt)


def ran(pattern):
    k = api.last_kernel()
    assert fnmatch.fnmatchcase(k, pattern), k
    return k


def check(got_array, before, want, w, y0, y1):
    """the array's [0, w) x [y0, y1) equals the linear call's rows; every other element is what it was"""
    got = got_array.download()
    assert torch.equal(got[y0:y1, :w], bits(want)[y0:y1]), "surface output differs from the linear call"
    mask = torch.ones(got.shape[:2], dtype=torch.bool, device="cuda")
    mask[y0:y1, :w] = False
    assert torch.equal(got[mask], before[mask]), "texels outside the written region changed"


def exact2x(iw, ih, ow, oh):
    c = np.array(api.easu_con(iw, ih, iw, ih, ow, oh)[:4], np.uint32).view(np.float32)
    return tuple(c) == (0.5, 0.5, -0.25, -0.25)


FLAG_SETS = {"in": IN, "out": OUT, "in_out": IN | OUT}


def run_pair(arrays, iw, ih, ow, oh, flags, call, out_fmt=RGBA16F, hdr=False, seed=0, extra=(0, 0)):
    """call(inp, out, flags) on surfaces for the flags given and on linear tensors; compares the whole output as bits"""
    x = frame(iw, ih, seed, hdr)
    want = linear_out(oh, ow, out_fmt)
    call(x, want, flags & ~(IN | OUT))
    k_lin = api.last_kernel()
    inp = surf(in_array(arrays, x, extra), iw, ih) if flags & IN else x
    if flags & OUT:
        oa, before = out_array(arrays, oh, ow, out_fmt, extra)
        out = surf(oa, ow, oh, out_fmt)
    else:
        out = linear_out(oh, ow, out_fmt)
    n0 = api.launch_count()
    call(inp, out, flags)
    n = api.launch_count() - n0
    k = api.last_kernel()
    if flags & OUT:
        check(oa, before, want, ow, 0, oh)
    else:
        assert torch.equal(bits(out), bits(want))
    return k_lin, k, n


# ---- fsr1_upscale ------------------------------------------------------------------------------------------------------------------
FUSED_SIZES = [(1920, 1080, 3840, 2160), (125, 67, 250, 134), (127, 33, 254, 66), (95, 53, 190, 106)]


@pytest.mark.parametrize("srtm", [0, S])
@pytest.mark.parametrize("flags", list(FLAG_SETS))
@pytest.mark.parametrize("size", FUSED_SIZES)
def test_fused_upscale_equals_the_linear_call(arrays, size, flags, srtm):
    iw, ih, ow, oh = size
    assert exact2x(*size)
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)

    def call(i, o, f):
        api.upscale(i, linear_out(oh, ow, RGBA16F), o, econ, rcon, flags=f | FUSED | srtm)
    k_lin, k, n = run_pair(arrays, iw, ih, ow, oh, FLAG_SETS[flags], call, hdr=bool(srtm), seed=iw, extra=(3, 2))
    assert n == 1
    assert k_lin.startswith("fused_easu_rcas_h_quad2x<4w,7/sm,tma2,strips")
    for f in ("in", "out"):
        assert ((",surf_%s" % f) in k) == (f in flags.split("_")), k
    # the twin that takes its input by TMA and stores through a surface runs at 6 CTAs per SM (no spills), the others at 7
    per_sm = "6/sm" if flags == "out" else "7/sm"
    assert k.startswith("fused_easu_rcas_h_quad2x<4w,%s," % per_sm) and ((",srtm_in" in k) == bool(srtm)), k


TWO_KERNEL = [(1477, 831, 1920, 1080), (1280, 720, 1920, 1080), (1129, 635, 1920, 1080), (41, 23, 82, 46)]
RCAS_OPTS = [FUSED, FUSED | api.FLAG_RCAS_CLAMP, api.FLAG_RCAS_DENOISE, api.FLAG_RCAS_PASSTHROUGH_ALPHA, api.FLAG_OUTPUT_SQUARE]


@pytest.mark.parametrize("opts", RCAS_OPTS)
@pytest.mark.parametrize("flags", list(FLAG_SETS))
@pytest.mark.parametrize("size", TWO_KERNEL)
def test_two_kernel_upscale_equals_the_linear_call(arrays, size, flags, opts):
    iw, ih, ow, oh = size
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.5)

    def call(i, o, f):
        api.upscale(i, linear_out(oh, ow, RGBA16F), o, econ, rcon, flags=f | opts)
    k_lin, k, n = run_pair(arrays, iw, ih, ow, oh, FLAG_SETS[flags], call, seed=ih, extra=(1, 3))
    assert n == 2 and k_lin == "rcas_h_packed<2px,4rows,shfl60>"
    assert k == ("rcas_h_packed<2px,4rows,shfl60,surf_out>" if FLAG_SETS[flags] & OUT else k_lin)


def test_surface_input_takes_the_surface_easu_kernels(arrays):
    for size, kernel in (((640, 360, 1280, 720), "easu_h_quad2x<4w,7/sm,surf_in>"), ((1280, 720, 1920, 1080), "easu_h_vpairs<*,surf_in>")):
        iw, ih, ow, oh = size
        con = api.easu_con(iw, ih, iw, ih, ow, oh)

        def call(i, o, f):
            api.easu(i, o, con, flags=f)
        k_lin, k, n = run_pair(arrays, iw, ih, ow, oh, IN, call, seed=5, extra=(2, 2))
        assert n == 1 and fnmatch.fnmatchcase(k, kernel), k
        assert ",tma2" in k_lin and "surf" not in k_lin


# ---- fsr1_upscale_post -------------------------------------------------------------------------------------------------------------
POST_OPS = [(s, g, t) for s in (False, True) for g in (False, True) for t in (0, 8, 10)]


@pytest.mark.parametrize("srtm_inverse,lfga,tepd_bits", POST_OPS)
@pytest.mark.parametrize("size", [(960, 540, 1920, 1080), (960, 540, 1440, 810)])
@pytest.mark.parametrize("flags", list(FLAG_SETS))
def test_upscale_post_equals_the_linear_call(arrays, srtm_inverse, lfga, tepd_bits, size, flags):
    iw, ih, ow, oh = size
    fmt = {0: RGBA16F, 8: RGBA8, 10: RGB10A2}[tepd_bits]
    grain = (torch.rand((5, 12, 4), device="cuda") - 0.5).half() if lfga else None
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    kw = dict(srtm_inverse=srtm_inverse, grain=grain, amount=0.375, tepd_bits=tepd_bits, frame=3)

    def call(i, o, f):
        api.upscale_post(i, linear_out(oh, ow, RGBA16F), o, econ, rcon, flags=f | FUSED, **kw)
    k_lin, k, n = run_pair(arrays, iw, ih, ow, oh, FLAG_SETS[flags], call, out_fmt=fmt, seed=tepd_bits + iw, extra=(2, 1))
    fused = exact2x(*size)
    ops = srtm_inverse or lfga or tepd_bits
    assert n == (1 if fused else 2)
    if fused:
        per_sm = "6/sm" if ops or flags == "out" else "7/sm"   # the post kernels, and the plain twin fed by TMA that stores to a surface
        assert k.startswith("fused_easu_rcas_h_quad2x<4w,%s," % per_sm) and (",post," in k) == bool(ops), k
    elif FLAG_SETS[flags] & OUT:
        assert k.startswith("rcas_h_packed_post<" if ops else "rcas_h_packed<") and k.endswith(",surf_out>"), k
    else:
        assert k == k_lin


@pytest.mark.parametrize("flags", list(FLAG_SETS))
def test_hdr_round_trip_into_rgb10a2(arrays, flags):
    iw, ih, ow, oh = 1920, 1080, 3840, 2160
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)

    def call(i, o, f):
        api.upscale_post(i, None, o, econ, rcon, srtm_inverse=True, tepd_bits=10, frame=1, flags=f | FUSED | S)
    k_lin, k, n = run_pair(arrays, iw, ih, ow, oh, FLAG_SETS[flags], call, out_fmt=RGB10A2, hdr=True, seed=77)
    assert n == 1 and ",post,rgb10a2,srtm_in" in k, k


# ---- row slabs, and texels the call must not touch ------------------------------------------------------------------------------
def test_easu_and_rcas_on_row_slabs(arrays):
    iw, ih, ow, oh = 320, 180, 640, 360
    x = frame(iw, ih, 9)
    ina = in_array(arrays, x, extra=(6, 4))
    con, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    y0, y1 = 101, 233
    got, want = linear_out(oh, ow, RGBA16F), linear_out(oh, ow, RGBA16F)
    api.easu(surf(ina, iw, ih), got, con, y0, y1, flags=IN)
    ran("easu_h_quad2x<4w,7/sm,surf_in>")
    api.easu(x, want, con, y0, y1)
    assert torch.equal(bits(got), bits(want))
    # fsr1_rcas into a larger, poisoned array: only [0, ow) x [y0, y1) is written
    t = frame(ow, oh, 10)
    oa, before = out_array(arrays, oh, ow, RGBA16F, extra=(5, 7))
    for opts in (0, api.FLAG_RCAS_CLAMP | api.FLAG_RCAS_DENOISE):
        want = linear_out(oh, ow, RGBA16F)
        api.rcas(t, want, rcon, y0, y1, flags=opts)
        api.rcas(t, surf(oa, ow, oh), rcon, y0, y1, flags=opts | OUT)
        ran("rcas_h_packed<2px,4rows,shfl60,surf_out>")
        check(oa, before, want, ow, y0, y1)


@pytest.mark.parametrize("post", [False, True])
def test_fused_slab_leaves_every_other_texel_untouched(arrays, post):
    iw, ih, ow, oh = 640, 360, 1280, 720
    x = frame(iw, ih, 12)
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    y0, y1 = 77, 501
    fmt = RGBA8 if post else RGBA16F
    oa, before = out_array(arrays, oh, ow, fmt, extra=(9, 5))
    want = linear_out(oh, ow, fmt)
    if post:
        api.upscale_post(x, None, want, econ, rcon, tepd_bits=8, frame=4, y0=y0, y1=y1, flags=FUSED)
        api.upscale_post(x, None, surf(oa, ow, oh, fmt), econ, rcon, tepd_bits=8, frame=4, y0=y0, y1=y1, flags=FUSED | OUT)
    else:
        api.upscale(x, linear_out(oh, ow, RGBA16F), want, econ, rcon, y0, y1, flags=FUSED)
        api.upscale(x, linear_out(oh, ow, RGBA16F), surf(oa, ow, oh), econ, rcon, y0, y1, flags=FUSED | OUT)
    ran("fused_easu_rcas_h_quad2x<*,surf_out>")
    check(oa, before, want, ow, y0, y1)


# ---- contexts ----------------------------------------------------------------------------------------------------------------------
def test_context_calls_clamp_at_the_render_region(arrays):
    """The input array is larger than the render region and holds NaN, inf and 65504 beyond it; the result equals the linear call on a
    buffer of the render region only."""
    iw, ih, ow, oh = 1280, 720, 2560, 1440
    x = frame(iw, ih, 21, hdr=True)
    ina = arrays(iw + 16, ih + 8, "rgba16f")
    ina.upload(poison_like(ina, 3))
    ina.upload(x)
    ctx = api.HostContext(iw, ih, ow, oh)
    try:
        for rw, rh in ((iw, ih), (960, 540), (1111, 607)):
            region = plain(x[:rh, :rw])
            for flags in (IN, IN | OUT, IN | S):
                want = linear_out(oh, ow, RGBA16F)
                ctx.upscale_render(region, rw, rh, want, flags=flags & S)
                if flags & OUT:
                    oa, before = out_array(arrays, oh, ow, RGBA16F, extra=(1, 1))
                    ctx.upscale_render(ina.handle, rw, rh, oa.handle, flags=flags)
                    check(oa, before, want, ow, 0, oh)
                else:
                    got = linear_out(oh, ow, RGBA16F)
                    ctx.upscale_render(ina.handle, rw, rh, got, flags=flags)
                    assert torch.equal(bits(got), bits(want)), (rw, rh, flags)
            for bits_, fmt in ((10, RGB10A2), (8, RGBA8)):
                want = linear_out(oh, ow, fmt)
                ctx.upscale_post(region, want, rw, rh, srtm_inverse=True, tepd_bits=bits_, frame=2, flags=S)
                oa, before = out_array(arrays, oh, ow, fmt)
                ctx.upscale_post(ina.handle, oa.handle, rw, rh, srtm_inverse=True, tepd_bits=bits_, frame=2, flags=S | IN | OUT)
                check(oa, before, want, ow, 0, oh)
        want, got = linear_out(oh, ow, RGBA16F), linear_out(oh, ow, RGBA16F)
        ctx.upscale(x, want)
        ctx.upscale(ina.handle, got, flags=IN)
        ran("fused_easu_rcas_h_quad2x<4w,7/sm,strips,surf_in>")
        assert torch.equal(bits(got), bits(want))
    finally:
        ctx.close()


# ---- refusals of the handles -------------------------------------------------------------------------------------------------------
def test_handle_refusals_launch_nothing(arrays):
    L = _lib.lib()
    iw, ih, ow, oh = 64, 36, 128, 72
    econ, rcon = (ctypes.c_uint32 * 16)(*api.easu_con(iw, ih, iw, ih, ow, oh)), (ctypes.c_uint32 * 4)(*api.rcas_con(0.25))
    x, tmp, out = frame(iw, ih, 1), linear_out(oh, ow, RGBA16F), linear_out(oh, ow, RGBA16F)
    good_in, good_out = arrays(iw, ih, "rgba16f"), arrays(ow, oh, "rgba16f")
    cases = [  # (in image, out image, flags, expected)
        (_lib.Image(0, 0, iw, ih, 0, ih, RGBA16F, 0), api.image(out), IN, -1),                      # handle 0
        (surf(arrays(iw, ih, "u32"), iw, ih), api.image(out), IN, -2),                             # 4-byte elements for RGBA16F
        (surf(arrays(iw - 1, ih, "rgba16f"), iw, ih), api.image(out), IN, -1),                     # extent too small
        (surf(arrays(iw, ih - 1, "rgba16f"), iw, ih), api.image(out), IN, -1),
        (surf(arrays(iw, ih, "rgba16f", layered=True), iw, ih), api.image(out), IN, -2),           # layered
        (api.image(x), surf(arrays(ow, oh, "rgba8"), ow, oh), OUT, -2),                            # 4-byte elements for RGBA16F
        (api.image(x), surf(arrays(ow, oh - 3, "rgba16f"), ow, oh), OUT, -1),
        (api.image(x), surf(arrays(ow, oh, "rgba16f", layered=True), ow, oh), OUT, -2),
        (surf(good_in, iw, ih), surf(good_out, ow, oh), IN | OUT | api.FLAG_PRECISE, -2),
    ]
    t = api.image(tmp)
    n0 = api.launch_count()
    for i, o, flags, rc in cases:
        for f in (flags, flags | FUSED):
            assert L.fsr1_upscale(ctypes.byref(i), ctypes.byref(t), ctypes.byref(o), econ, rcon, 0, 0, f, None) == rc, (f, rc)
        p = _lib.Post(api.POST_SRTM_INVERSE, 0.0, None, None, 0, 0)
        assert L.fsr1_upscale_post(ctypes.byref(i), ctypes.byref(t), ctypes.byref(o), econ, rcon, ctypes.byref(p), 0, 0, flags | FUSED,
                                   None) == rc
    # fsr1_easu / fsr1_rcas
    assert L.fsr1_easu(ctypes.byref(cases[1][0]), ctypes.byref(api.image(out)), econ, 0, 0, IN, None) == -2
    assert L.fsr1_rcas(ctypes.byref(t), ctypes.byref(cases[5][1]), rcon, 0, 0, OUT, None) == -2
    # the context calls: the handle with pitch 0; never the host-frame call
    ctx = api.HostContext(iw, ih, ow, oh)
    try:
        assert L.fsr1_context_upscale(ctx._h, ctypes.c_void_p(good_in.handle), 64, ctypes.c_void_p(out.data_ptr()), ow * 8,
                                      ctypes.c_float(0.25), IN, None) == -1
        hin, hout = torch.zeros((ih, iw, 4), dtype=torch.float16), torch.zeros((oh, ow, 4), dtype=torch.float16)
        for f in (IN, OUT):
            assert L.fsr1_context_upscale_host(ctx._h, ctypes.c_void_p(hin.data_ptr()), iw * 8, ctypes.c_void_p(hout.data_ptr()), ow * 8,
                                               ctypes.c_float(0.25), f, None) == -2
    finally:
        ctx.close()
    assert api.launch_count() == n0
