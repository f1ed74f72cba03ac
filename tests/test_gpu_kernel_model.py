"""The production half-storage kernels against the per-pixel model of their arithmetic (tests/model/fsr1_kernel_model.c), bit for
bit: easu_h_quad2x, easu_h_vpairs, rcas_h_packed (every option set, both out-of-image rules), the fused EASU -> RCAS kernel,
easu_u8_quad2x and rcas_u8_packed.  Every case checks the kernel family that ran and reports the number of differing values, the
first (y, x, channel) and both bit patterns.

Shapes straddle the tiles: output widths 1-3, 61-66 and 119-130 and heights 1-2, 15-17 and 31-33 cross the 64x16 quad tile, the
64x32 pair tile, the 60-pixel RCAS span and the 62-pixel fused strip; odd row slabs read input row windows; the geometry table of
test_gpu_parity.py; full frames are multi-wave persistent launches.  Content: see kernel_model.CONTENT and CODES."""
import numpy as np
import pytest
import torch

import fsr1_b200 as F
import kernel_model as km
from easu_checks import expected_easu_kernel
from test_gpu_parity import GEOMETRY, dev, empty_like_image, geometry_con

pytestmark = pytest.mark.gpu
api = F.api
WIDTHS = [1, 2, 3] + list(range(61, 67)) + list(range(119, 131))
HEIGHTS = [1, 2, 15, 16, 17, 31, 32, 33]
SHAPES = [(w, h) for w in WIDTHS for h in HEIGHTS]
KINDS = list(km.CONTENT)


def _bits(t):
    torch.cuda.synchronize()
    return t.cpu().numpy().view(np.uint16) if t.dtype == torch.float16 else t.cpu().numpy()


def gpu_easu(src, ow, oh, con, y0=0, y1=0):
    out = empty_like_image(oh, ow, torch.from_numpy(src[:0]).dtype)
    api.easu(dev(src), out, con, y0=y0, y1=y1)
    assert api.last_kernel().startswith(expected_easu_kernel(con, api.FORMAT_RGBA16F if src.dtype == np.float16 else api.FORMAT_RGBA8_UNORM)), api.last_kernel()
    return _bits(out)


def gpu_rcas(src, con, flags=0, family="rcas_h_packed"):
    out = empty_like_image(src.shape[0], src.shape[1], torch.from_numpy(src[:0]).dtype)
    api.rcas(dev(src), out, con, flags=flags)
    assert api.last_kernel().startswith(family), api.last_kernel()
    return _bits(out)


def flags_of(opts, clamp):
    return ((api.FLAG_RCAS_DENOISE if opts & 1 else 0) | (api.FLAG_RCAS_PASSTHROUGH_ALPHA if opts & 2 else 0) |
            (api.FLAG_OUTPUT_SQUARE if opts & 4 else 0) | (api.FLAG_RCAS_CLAMP if clamp else 0))


def con_2x_for(ow, oh):
    iw, ih = (ow + 1) // 2, (oh + 1) // 2
    return iw, ih, km.con_2x(api.easu_con(iw, ih, iw, ih, 2 * iw, 2 * ih))


@pytest.mark.parametrize("kind", KINDS)
def test_easu_h_quad2x_tile_edges(kind):
    for ow, oh in SHAPES:
        iw, ih, con = con_2x_for(ow, oh)
        src = km.content(kind, iw, ih, ow * 1000 + oh)
        km.assert_same_bits(gpu_easu(src, ow, oh, con), km.easu_h(src, ow, oh, con), ("easu_h_quad2x", kind, ow, oh))


@pytest.mark.parametrize("kind", KINDS)
def test_easu_h_vpairs_tile_edges(kind):
    """1.5x and 1.3x: output pixel pairs that share an input cell row and pairs that do not."""
    for i, (ow, oh) in enumerate(SHAPES):
        s = 1.5 if i % 2 else 1.3
        iw, ih = max(1, int(np.ceil(ow / s))), max(1, int(np.ceil(oh / s)))
        con = api.easu_con(iw, ih, iw, ih, ow, oh)
        if con[:4] == km.QUAD_2X:
            continue
        src = km.content(kind, iw, ih, ow * 1000 + oh)
        km.assert_same_bits(gpu_easu(src, ow, oh, con), km.easu_h(src, ow, oh, con), ("easu_h_vpairs", kind, ow, oh, s))


RCAS_SHAPES = [(w, h) for w in WIDTHS for h in (1, 17, 33)] + [(w, h) for w in (2, 64, 125) for h in HEIGHTS]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("clamp", [False, True])
def test_rcas_h_packed_every_option_set(kind, clamp):
    con = api.rcas_con(0.25)
    for i, (w, h) in enumerate(RCAS_SHAPES):
        src = km.content(kind, w, h, w * 1000 + h)
        for opts in range(8) if i % 4 == 0 else (i % 8,):
            km.assert_same_bits(gpu_rcas(src, con, flags_of(opts, clamp)), km.rcas_h(src, con, clamp, opts), ("rcas_h_packed", kind, w, h, opts, clamp))
    src = km.content(kind, 259, 141, 3)
    for sharp in (0.0, 1.0, 2.0):                                        # other sharpness values on every option set
        c = api.rcas_con(sharp)
        for opts in range(8):
            km.assert_same_bits(gpu_rcas(src, c, flags_of(opts, clamp)), km.rcas_h(src, c, clamp, opts), ("rcas_h_packed", kind, sharp, opts, clamp))


@pytest.mark.parametrize("kind", KINDS)
def test_fused_equals_model_easu_then_rcas(kind):
    rcon = api.rcas_con(0.25)
    for ow, oh in [(w, h) for w in WIDTHS for h in (1, 2, 17, 33)] + [(w, h) for w in (3, 62, 63, 124, 125) for h in HEIGHTS]:
        iw, ih, con = con_2x_for(ow, oh)
        src = km.content(kind, iw, ih, ow * 1000 + oh)
        tmp, out = empty_like_image(oh, ow, torch.float16), empty_like_image(oh, ow, torch.float16)
        api.upscale(dev(src), tmp, out, con, rcon, flags=api.FLAG_FUSED)
        assert api.last_kernel().startswith("fused_easu_rcas_h"), api.last_kernel()
        km.assert_same_bits(_bits(out), km.rcas_h(km.easu_h(src, ow, oh, con), rcon), ("fused", kind, ow, oh))


@pytest.mark.parametrize("codes", list(km.CODES))
def test_u8_kernels(codes):
    rcon = api.rcas_con(0.25)
    for i, (ow, oh) in enumerate(SHAPES):
        iw, ih, con = con_2x_for(ow, oh)
        raw = km.CODES[codes](iw, ih, ow * 1000 + oh)
        km.assert_same_bits(gpu_easu(raw, ow, oh, con), km.easu_u8(raw, ow, oh, con), ("easu_u8_quad2x", codes, ow, oh))
        raw = km.CODES[codes](ow, oh, ow * 1000 + oh + 1)
        for clamp in (False, True):
            opts = i % 8
            km.assert_same_bits(gpu_rcas(raw, rcon, flags_of(opts, clamp), "rcas_u8_packed"), km.rcas_u8(raw, rcon, clamp, opts),
                                ("rcas_u8_packed", codes, ow, oh, opts, clamp))


# ---- row slabs: odd row ranges, each reading only the input rows it needs -------------------------------------------------
SLABS = [(0, 7), (7, 30), (30, 31), (31, 64), (64, 97)]


@pytest.mark.parametrize("kind", ["uniform", "structured", "hdr", "signed_zero"])
def test_odd_row_slabs_with_input_windows(kind):
    ow, oh = 125, 97
    rcon = api.rcas_con(0.25)
    for con_kind in ("2x", "1.5x"):
        if con_kind == "2x":
            iw, ih, con = con_2x_for(ow, oh)
        else:
            iw, ih = 84, 65
            con = api.easu_con(iw, ih, iw, ih, ow, oh)
        src = km.content(kind, iw, ih, 21)
        want = km.easu_h(src, ow, oh, con)
        full_in = dev(src)
        for (y0, y1) in SLABS:
            n0, n1 = api.easu_input_rows(con, ih, y0, y1)                  # first and last input row read
            o = empty_like_image(y1 - y0, ow, torch.float16)
            api.easu(api.image(full_in[n0:n1 + 1], height=ih, row0=n0), api.image(o, height=oh, row0=y0), con, y0=y0, y1=y1)
            assert api.last_kernel().startswith(expected_easu_kernel(con, api.FORMAT_RGBA16F)), api.last_kernel()
            km.assert_same_bits(_bits(o), want[y0:y1], ("easu slab", con_kind, kind, y0, y1))
    mid = km.content(kind, ow, oh, 22)
    full_mid = dev(mid)
    for opts in (0, 1, 7):
        for clamp in (False, True):
            want = km.rcas_h(mid, rcon, clamp, opts)
            for (y0, y1) in SLABS:
                r0, r1 = max(y0 - 1, 0), min(y1 + 1, oh)
                o = empty_like_image(y1 - y0, ow, torch.float16)
                api.rcas(api.image(full_mid[r0:r1], height=oh, row0=r0), api.image(o, height=oh, row0=y0), rcon, y0=y0, y1=y1,
                         flags=flags_of(opts, clamp))
                assert api.last_kernel().startswith("rcas_h_packed"), api.last_kernel()
                km.assert_same_bits(_bits(o), want[y0:y1], ("rcas slab", kind, opts, clamp, y0, y1))
    iw, ih, con = con_2x_for(ow, oh)
    src = km.content(kind, iw, ih, 23)
    want = km.rcas_h(km.easu_h(src, ow, oh, con), rcon)
    din, sentinel, out = dev(src), empty_like_image(oh, ow, torch.float16), empty_like_image(oh, ow, torch.float16)
    for (y0, y1) in SLABS:
        api.upscale(din, sentinel, out, con, rcon, y0=y0, y1=y1, flags=api.FLAG_FUSED)
        assert api.last_kernel().startswith("fused_easu_rcas_h"), api.last_kernel()
    km.assert_same_bits(_bits(out), want, ("fused slabs", kind))


# ---- the geometry table and full frames (persistent, multi-wave) ----------------------------------------------------------
@pytest.mark.parametrize("case", [c for c in GEOMETRY if c != "y_downscaled"])
def test_geometry(case):
    iw, ih, vw, vh, off, ow, oh = GEOMETRY[case]
    con = geometry_con(iw, ih, vw, vh, off, ow, oh)
    for kind in ("structured", "near_flat"):
        src = km.content(kind, iw, ih, 31)
        km.assert_same_bits(gpu_easu(src, ow, oh, con), km.easu_h(src, ow, oh, con), (case, kind))


@pytest.mark.parametrize("size", [(1920, 1080, 3840, 2160), (2560, 1440, 3840, 2160), (2953, 1661, 3840, 2160)], ids=["1080p", "1440p", "2953x1661"])
def test_full_frames_f16(size):
    iw, ih, ow, oh = size
    con = api.easu_con(iw, ih, iw, ih, ow, oh)
    src = km.content("uniform" if iw != 2560 else "hdr", iw, ih, 41)
    e = km.easu_h(src, ow, oh, con)
    km.assert_same_bits(gpu_easu(src, ow, oh, con), e, ("full frame easu", size))
    if iw == 1920:
        rcon = api.rcas_con(0.25)
        r = km.rcas_h(e, rcon)
        km.assert_same_bits(gpu_rcas(e.view(np.float16), rcon), r, ("full frame rcas", size))
        tmp, out = empty_like_image(oh, ow, torch.float16), empty_like_image(oh, ow, torch.float16)
        api.upscale(dev(src), tmp, out, con, rcon, flags=api.FLAG_FUSED)
        assert api.last_kernel().startswith("fused_easu_rcas_h"), api.last_kernel()
        km.assert_same_bits(_bits(out), r, ("full frame fused", size))


def test_full_frame_u8_1080p_to_4k():
    iw, ih, ow, oh = 1920, 1080, 3840, 2160
    con = api.easu_con(iw, ih, iw, ih, ow, oh)
    raw = km.CODES["uniform"](iw, ih, 42)
    e = km.easu_u8(raw, ow, oh, con)
    km.assert_same_bits(gpu_easu(raw, ow, oh, con), e, "full frame easu_u8")
    rcon = api.rcas_con(0.25)
    km.assert_same_bits(gpu_rcas(e, rcon, 0, "rcas_u8_packed"), km.rcas_u8(e, rcon), "full frame rcas_u8")
