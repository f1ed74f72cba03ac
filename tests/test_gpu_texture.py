"""FSR1_FLAG_IN_TEXTURE on the H100: every call that reads its input from a CUDA array through a texture object is bit-identical to the
same call on a linear tensor holding the same texels, and runs the texture twin of the kernel the linear call runs.  The arrays are made
with the driver API through ctypes (libcuda.so.1, torch's primary context) WITHOUT surface load/store, as a render target mapped for
sampling only is, and the texture path reads them in place.  RGBA16F arrays have 16,16,16,16 unsigned-integer channels, R11G11B10F arrays
one 32-bit unsigned channel."""
import ctypes

import pytest
import torch

from fsr1_b200 import _lib, api
from test_gpu_surface import CudaArray, _Desc3D, _ResDesc, _ok, bits, cu, linear_out, out_array, plain, poison_like, surf

pytestmark = pytest.mark.gpu

TEX, SURF_IN, OUT, S, FUSED = api.FLAG_IN_TEXTURE, api.FLAG_IN_SURFACE, api.FLAG_OUT_SURFACE, api.FLAG_SRTM_INPUT, api.FLAG_FUSED
RGBA16F, RGBA8, RGB10A2, R11 = api.FORMAT_RGBA16F, api.FORMAT_RGBA8_UNORM, api.FORMAT_RGB10A2_UNORM, api.FORMAT_R11G11B10_FLOAT
CU_AD_FORMAT_UNSIGNED_INT16, CU_AD_FORMAT_UNSIGNED_INT32, CU_AD_FORMAT_HALF = 0x02, 0x03, 0x10
CU_TRSF_READ_AS_INTEGER, CU_TRSF_NORMALIZED_COORDINATES, CU_TRSF_SRGB = 0x01, 0x02, 0x10


# ---- CUDA arrays and texture objects through the driver API --------------------------------------------------------------------------
class _TexDesc(ctypes.Structure):  # CUDA_TEXTURE_DESC
    _fields_ = [("addressMode", ctypes.c_int * 3), ("filterMode", ctypes.c_int), ("flags", ctypes.c_uint), ("maxAnisotropy", ctypes.c_uint),
                ("mipmapFilterMode", ctypes.c_int), ("mipmapLevelBias", ctypes.c_float), ("minMipmapLevelClamp", ctypes.c_float),
                ("maxMipmapLevelClamp", ctypes.c_float), ("borderColor", ctypes.c_float * 4), ("reserved", ctypes.c_int * 12)]


class _ResDescPitch(ctypes.Structure):  # CUDA_RESOURCE_DESC with the pitch2D member of its union
    _fields_ = [("resType", ctypes.c_int), ("devPtr", ctypes.c_uint64), ("format", ctypes.c_int), ("numChannels", ctypes.c_uint),
                ("width", ctypes.c_size_t), ("height", ctypes.c_size_t), ("pitchInBytes", ctypes.c_size_t), ("reserved", ctypes.c_int * 22),
                ("flags", ctypes.c_uint)]


def tex_desc(filter_mode=0, flags=CU_TRSF_READ_AS_INTEGER, address=1):
    """point filtering (0), element reads (READ_AS_INTEGER), unnormalized coordinates; address mode clamp (1) by default"""
    d = _TexDesc()
    d.addressMode[0] = d.addressMode[1] = d.addressMode[2] = address
    d.filterMode, d.flags = filter_mode, flags
    return d


def make_tex(res, desc):
    t = ctypes.c_uint64()
    rc = cu().cuTexObjectCreate(ctypes.byref(t), ctypes.byref(res), ctypes.byref(desc), None)
    return rc, t.value


class TexArray(CudaArray):
    """A 2D CUDA array made WITHOUT surface load/store (layered: one layer of a layered array) and a texture object on it.  `fmt`:
    RGBA16F (16,16,16,16 unsigned; or with `ad_format` another channel format) or R11G11B10F (32 unsigned)."""

    def __init__(self, w, h, fmt=RGBA16F, layered=False, ad_format=None, desc=None):
        ch = 4 if fmt == RGBA16F else 1
        ad = ad_format if ad_format is not None else (CU_AD_FORMAT_UNSIGNED_INT16 if fmt == RGBA16F else CU_AD_FORMAT_UNSIGNED_INT32)
        self.w, self.h, self.elem = w, h, 8 if fmt == RGBA16F else 4
        self.arr = ctypes.c_void_p()
        _ok(cu().cuArray3DCreate_v2(ctypes.byref(self.arr), ctypes.byref(_Desc3D(w, h, 1 if layered else 0, ad, ch, 0x01 if layered else 0))))
        rc, self.handle = make_tex(_ResDesc(0, self.arr), desc if desc is not None else tex_desc())
        self.tex_rc = rc

    def close(self):
        if self.tex_rc == 0:
            cu().cuTexObjectDestroy(ctypes.c_uint64(self.handle))
        cu().cuArrayDestroy(self.arr)


@pytest.fixture
def textures():
    made = []

    def make(*a, **k):
        made.append(TexArray(*a, **k))
        return made[-1]
    yield make
    torch.cuda.synchronize()
    for a in made:
        a.close()


@pytest.fixture
def surfaces():
    made = []

    def make(*a, **k):
        made.append(CudaArray(*a, **k))
        return made[-1]
    yield make
    torch.cuda.synchronize()
    for a in made:
        a.close()


# ---- content -------------------------------------------------------------------------------------------------------------------------
def specials16(x, seed):
    """sprinkle RGBA16F special values over ~4 % of the texels and fill a band of rows with raw random bits: NaNs with payloads, +-inf,
    -0, denormals"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    v = x.view(torch.int16)
    h, w = v.shape[:2]
    vals = torch.tensor([0x7E00, 0x7D23, -0x0201, 0x7C00, -0x0400, -0x8000, 0x0001, 0x03FF, -0x7C01], dtype=torch.int16, device="cuda")
    pick = torch.randint(0, 25, (h, w, 4), generator=g, device="cuda")
    v[pick < vals.numel()] = vals[pick[pick < vals.numel()]]
    band = slice(h // 3, h // 3 + max(1, h // 16))
    v[band] = torch.randint(-32768, 32767, v[band].shape, generator=g, device="cuda", dtype=torch.int32).to(torch.int16)
    return x


def frame16(w, h, seed, hdr):
    """float16 [h, w, 4] in rows padded to 16 bytes: [0, 1) values, or linear HDR up to 65504 for SRTM_INPUT, with special values"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.rand((h, w, 4), generator=g, device="cuda")
    if hdr:
        x = torch.clamp(x * torch.exp2(torch.randint(-8, 16, (h, w, 4), generator=g, device="cuda").float()), max=65504.0)
    return specials16(plain(x.half()), seed + 1)


def frame_r11(w, h, seed):
    """int32 [h, w] R11G11B10F codes in rows padded to 16 bytes: random codes (every exponent, denormals, inf, NaN)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    c = torch.randint(-2 ** 31, 2 ** 31 - 1, (h, w), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)
    out = torch.empty((h, w + (-w & 3)), dtype=torch.int32, device="cuda")[:, :w]
    out.copy_(c)
    return out


def frame(fmt, w, h, seed, hdr=False):
    return frame16(w, h, seed, hdr) if fmt == RGBA16F else frame_r11(w, h, seed)


def lin(x, fmt):
    return api.image(x, format=R11) if fmt == R11 else api.image(x)


def tex_in(textures, x, fmt, extra=(0, 0), seed=1):
    """a texture image on an array made without surface load/store, holding x in its top-left region and poison outside it"""
    h, w = x.shape[:2]
    a = textures(w + extra[0], h + extra[1], fmt)
    assert a.tex_rc == 0
    if extra != (0, 0):
        a.upload(poison_like(a, seed))
    a.upload(x)
    return a, api.texture_image(a.handle, w, h, fmt)


def ran_tex(k):
    assert ",tex_in" in k and "tma2" not in k, k


FORMATS = {"rgba16f": RGBA16F, "r11": R11}
FULL = [(1920, 1080, 3840, 2160), (2560, 1440, 3840, 2160)]  # 2x (fused), BASELINE's 1440p -> 4K (1.5x, two kernels)


# ---- fsr1_easu and fsr1_upscale --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("srtm", [0, S])
@pytest.mark.parametrize("fmt", list(FORMATS))
@pytest.mark.parametrize("size", FULL + [(125, 67, 250, 134), (97, 55, 126, 71)])
def test_easu_and_upscale_equal_the_linear_call(textures, size, fmt, srtm):
    iw, ih, ow, oh = size
    f = FORMATS[fmt]
    x = frame(f, iw, ih, iw + ih + srtm, hdr=bool(srtm))
    a, t = tex_in(textures, x, f, extra=(3, 2))
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    want, got = linear_out(oh, ow, RGBA16F), linear_out(oh, ow, RGBA16F)
    api.easu(lin(x, f), want, econ, flags=srtm)
    k_lin = api.last_kernel()
    n0 = api.launch_count()
    api.easu(t, got, econ, flags=srtm | TEX)
    assert api.launch_count() - n0 == 1
    ran_tex(api.last_kernel())
    assert api.last_kernel().split("<")[0] == k_lin.split("<")[0]
    assert torch.equal(bits(got), bits(want)), "fsr1_easu"
    for opts in (FUSED, 0):
        want, got = linear_out(oh, ow, RGBA16F), linear_out(oh, ow, RGBA16F)
        api.upscale(lin(x, f), linear_out(oh, ow, RGBA16F), want, econ, rcon, flags=opts | srtm)
        n0 = api.launch_count()
        api.upscale(t, linear_out(oh, ow, RGBA16F), got, econ, rcon, flags=opts | srtm | TEX)
        fused = opts and 2 * iw == ow and 2 * ih == oh
        assert api.launch_count() - n0 == (1 if fused else 2)
        if fused:
            ran_tex(api.last_kernel())
            assert api.last_kernel().startswith("fused_easu_rcas_h_quad2x<4w,7/sm,strips,")
        assert torch.equal(bits(got), bits(want)), ("fsr1_upscale", opts)


def test_upscale_into_an_output_surface(textures, surfaces):
    for f in (RGBA16F, R11):
        iw, ih, ow, oh = 640, 360, 1280, 720
        x = frame(f, iw, ih, 4)
        _, t = tex_in(textures, x, f, extra=(2, 5))
        econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
        want = linear_out(oh, ow, RGBA16F)
        api.upscale(lin(x, f), linear_out(oh, ow, RGBA16F), want, econ, rcon, flags=FUSED)
        oa, before = out_array(surfaces, oh, ow, RGBA16F, extra=(3, 1))
        api.upscale(t, linear_out(oh, ow, RGBA16F), surf(oa, ow, oh), econ, rcon, flags=FUSED | TEX | OUT)
        ran_tex(api.last_kernel())
        assert api.last_kernel().endswith(",tex_in,surf_out>")
        got = oa.download()
        assert torch.equal(got[:oh, :ow], bits(want))
        mask = torch.ones(got.shape[:2], dtype=torch.bool, device="cuda")
        mask[:oh, :ow] = False
        assert torch.equal(got[mask], before[mask])


# ---- fsr1_upscale_post ---------------------------------------------------------------------------------------------------------------
POST_OPS = [(s, g, t) for s in (False, True) for g in (False, True) for t in (0, 8, 10)]


@pytest.mark.parametrize("out_surface", [False, True])
@pytest.mark.parametrize("srtm_inverse,lfga,tepd_bits", POST_OPS)
@pytest.mark.parametrize("fmt", list(FORMATS))
def test_upscale_post_equals_the_linear_call(textures, surfaces, fmt, srtm_inverse, lfga, tepd_bits, out_surface):
    f = FORMATS[fmt]
    ofmt = {0: RGBA16F, 8: RGBA8, 10: RGB10A2}[tepd_bits]
    grain = (torch.rand((5, 12, 4), device="cuda") - 0.5).half() if lfga else None
    kw = dict(srtm_inverse=srtm_inverse, grain=grain, amount=0.375, tepd_bits=tepd_bits, frame=3)
    for iw, ih, ow, oh in ((960, 540, 1920, 1080), (960, 540, 1440, 810)):
        srtm = S if srtm_inverse else 0
        x = frame(f, iw, ih, tepd_bits + iw, hdr=bool(srtm))
        _, t = tex_in(textures, x, f, extra=(2, 1))
        econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
        want = linear_out(oh, ow, ofmt)
        api.upscale_post(lin(x, f), linear_out(oh, ow, RGBA16F), want, econ, rcon, flags=FUSED | srtm, **kw)
        if out_surface:
            oa, before = out_array(surfaces, oh, ow, ofmt, extra=(1, 2))
            out = surf(oa, ow, oh, ofmt)
        else:
            out = linear_out(oh, ow, ofmt)
        api.upscale_post(t, linear_out(oh, ow, RGBA16F), out, econ, rcon, flags=FUSED | srtm | TEX | (OUT if out_surface else 0), **kw)
        k = api.last_kernel()
        if 2 * iw == ow:
            ran_tex(k)
            assert k.endswith(",surf_out>") == out_surface, k
        if out_surface:
            got = oa.download()
            assert torch.equal(got[:oh, :ow], bits(want)), (iw, ow)
            mask = torch.ones(got.shape[:2], dtype=torch.bool, device="cuda")
            mask[:oh, :ow] = False
            assert torch.equal(got[mask], before[mask])
        else:
            assert torch.equal(bits(out), bits(want)), (iw, ow)


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_hdr_round_trip_into_rgb10a2(textures, surfaces, fmt):
    f = FORMATS[fmt]
    for iw, ih, ow, oh in FULL:
        x = frame(f, iw, ih, 77, hdr=True)
        _, t = tex_in(textures, x, f)
        econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
        kw = dict(srtm_inverse=True, tepd_bits=10, frame=1)
        want = linear_out(oh, ow, RGB10A2)
        api.upscale_post(lin(x, f), linear_out(oh, ow, RGBA16F), want, econ, rcon, flags=FUSED | S, **kw)
        oa, _ = out_array(surfaces, oh, ow, RGB10A2)
        api.upscale_post(t, linear_out(oh, ow, RGBA16F), surf(oa, ow, oh, RGB10A2), econ, rcon, flags=FUSED | S | TEX | OUT, **kw)
        assert torch.equal(oa.download(), bits(want)), (iw, ow)


# ---- row slabs and contexts ------------------------------------------------------------------------------------------------------------
def test_row_slabs(textures):
    for f in (RGBA16F, R11):
        for iw, ih, ow, oh in ((320, 180, 640, 360), (320, 180, 480, 270)):
            x = frame(f, iw, ih, 9)
            _, t = tex_in(textures, x, f, extra=(6, 4))
            econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
            for y0, y1 in ((101, 233), (0, 7), (oh - 5, oh)):
                got, want = linear_out(oh, ow, RGBA16F), linear_out(oh, ow, RGBA16F)
                api.easu(t, got, econ, y0, y1, flags=TEX)
                api.easu(lin(x, f), want, econ, y0, y1)
                assert torch.equal(bits(got), bits(want)), (f, ow, y0, y1)
                got, want = linear_out(oh, ow, RGBA16F), linear_out(oh, ow, RGBA16F)
                api.upscale(t, linear_out(oh, ow, RGBA16F), got, econ, rcon, y0, y1, flags=FUSED | TEX)
                api.upscale(lin(x, f), linear_out(oh, ow, RGBA16F), want, econ, rcon, y0, y1, flags=FUSED)
                assert torch.equal(bits(got), bits(want)), (f, ow, y0, y1)


@pytest.mark.parametrize("fmt", list(FORMATS))
def test_context_calls_clamp_at_the_render_region(textures, surfaces, fmt):
    """The input array is larger than the render region and holds poison beyond it; the result equals the linear call on a buffer of the
    render region only."""
    f = FORMATS[fmt]
    iw, ih, ow, oh = 1280, 720, 2560, 1440
    x = frame(f, iw, ih, 21, hdr=True)
    ina, _ = tex_in(textures, x, f, extra=(16, 8), seed=3)
    ctx = api.HostContext(iw, ih, ow, oh, f)
    try:
        for rw, rh in ((iw, ih), (960, 540), (1111, 607)):
            region = plain(x[:rh, :rw]) if f == RGBA16F else frame_r11(rw, rh, 0).copy_(x[:rh, :rw])
            for flags in (TEX, TEX | S):
                want, got = linear_out(oh, ow, RGBA16F), linear_out(oh, ow, RGBA16F)
                ctx.upscale_render(region, rw, rh, want, flags=flags & S)
                ctx.upscale_render(ina.handle, rw, rh, got, flags=flags)
                assert torch.equal(bits(got), bits(want)), (rw, rh, flags)
            want = linear_out(oh, ow, RGB10A2)
            ctx.upscale_post(region, want, rw, rh, srtm_inverse=True, tepd_bits=10, frame=2, flags=S)
            oa, _ = out_array(surfaces, oh, ow, RGB10A2)
            ctx.upscale_post(ina.handle, oa.handle, rw, rh, srtm_inverse=True, tepd_bits=10, frame=2, flags=S | TEX | OUT)
            assert torch.equal(oa.download()[:oh, :ow], bits(want)), (rw, rh)
        want, got = linear_out(oh, ow, RGBA16F), linear_out(oh, ow, RGBA16F)
        ctx.upscale(x, want)
        ctx.upscale(ina.handle, got, flags=TEX)
        ran_tex(api.last_kernel())
        assert torch.equal(bits(got), bits(want))
    finally:
        ctx.close()


# ---- refusals of the handles -------------------------------------------------------------------------------------------------------
def test_handle_refusals_launch_nothing(textures):
    L = _lib.lib()
    iw, ih, ow, oh = 64, 36, 128, 72
    econ, rcon = (ctypes.c_uint32 * 16)(*api.easu_con(iw, ih, iw, ih, ow, oh)), (ctypes.c_uint32 * 4)(*api.rcas_con(0.25))
    tmp, out = linear_out(oh, ow, RGBA16F), linear_out(oh, ow, RGBA16F)

    def timg(a, fmt=RGBA16F, w=iw, h=ih):
        return api.texture_image(a.handle, w, h, fmt)
    pitched = torch.zeros((ih, iw, 4), dtype=torch.float16, device="cuda")
    res = _ResDescPitch(3, pitched.data_ptr(), CU_AD_FORMAT_UNSIGNED_INT16, 4, iw, ih, iw * 8)
    rc, pitch_tex = make_tex(res, tex_desc())
    _ok(rc)
    linear_filter = textures(iw, ih, desc=tex_desc(filter_mode=1))
    cases = [  # (texture image, expected)
        (timg(textures(iw, ih, ad_format=CU_AD_FORMAT_HALF)), -2),                                        # float channels: converted
        (timg(textures(iw, ih, R11, ad_format=CU_AD_FORMAT_UNSIGNED_INT16)), -2),                         # wrong channel size
        (timg(textures(iw, ih), R11), -2),                                                                # 8-byte texels for R11
        (timg(textures(iw, ih, desc=tex_desc(flags=CU_TRSF_READ_AS_INTEGER | CU_TRSF_NORMALIZED_COORDINATES))), -2),
        (timg(textures(iw, ih, desc=tex_desc(flags=0))), -2),                                             # normalized-float reads
        (timg(textures(iw, ih, layered=True)), -2),
        (api.texture_image(pitch_tex, iw, ih, RGBA16F), -2),                                             # a pitch2D resource
        (timg(textures(iw - 1, ih)), -1),                                                                 # extent too small
        (timg(textures(iw, ih - 1, R11), R11), -1),
    ]
    if linear_filter.tex_rc == 0:   # linear filtering of integer texels, where the driver creates such a texture
        cases.append((timg(linear_filter), -2))
    t, o = api.image(tmp), api.image(out)
    n0 = api.launch_count()
    try:
        for i, rc in cases:
            assert L.fsr1_easu(ctypes.byref(i), ctypes.byref(o), econ, 0, 0, TEX, None) == rc
            for f in (TEX, TEX | FUSED, TEX | S):
                assert L.fsr1_upscale(ctypes.byref(i), ctypes.byref(t), ctypes.byref(o), econ, rcon, 0, 0, f, None) == rc, (f, rc)
            p = _lib.Post(api.POST_SRTM_INVERSE, 0.0, None, None, 0, 0)
            assert L.fsr1_upscale_post(ctypes.byref(i), ctypes.byref(t), ctypes.byref(o), econ, rcon, ctypes.byref(p), 0, 0, TEX | FUSED,
                                       None) == rc
        # the context calls: never the host-frame call
        ctx = api.HostContext(iw, ih, ow, oh)
        try:
            hin, hout = torch.zeros((ih, iw, 4), dtype=torch.float16), torch.zeros((oh, ow, 4), dtype=torch.float16)
            assert L.fsr1_context_upscale_host(ctx._h, ctypes.c_void_p(hin.data_ptr()), iw * 8, ctypes.c_void_p(hout.data_ptr()), ow * 8,
                                               ctypes.c_float(0.25), TEX, None) == -2
        finally:
            ctx.close()
        # fsr1_rcas / fsr1_rcas_post refuse the flag
        good = timg(textures(iw, ih))
        assert L.fsr1_rcas(ctypes.byref(t), ctypes.byref(o), rcon, 0, 0, TEX, None) == -2
        assert L.fsr1_rcas_post(ctypes.byref(t), ctypes.byref(o), rcon, None, 0, 0, TEX, None) == -2
        assert L.fsr1_easu(ctypes.byref(good), ctypes.byref(o), econ, 0, 0, TEX | SURF_IN, None) == -1
        assert api.launch_count() == n0
    finally:
        torch.cuda.synchronize()
        cu().cuTexObjectDestroy(ctypes.c_uint64(pitch_tex))

