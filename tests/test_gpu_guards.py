"""Every kernel family reads and writes only its own pixels.

Each test image sits inside a larger allocation whose other bytes are poison: GR guard rows above and below, guard columns on the
right (through the pitch) and a 16-byte left offset (so the production kernels still take the image: TMA and 128-bit access need
16-byte alignment).  The poison is
  * "nan": float NaNs with a payload (UNORM: a distinctive code pattern),
  * "big": large finite values (65504 / 3e38; UNORM: all ones).  HLSL min/max (minNum/maxNum) drop a NaN, so a stray NaN read into
    the de-ringing bounds or the RCAS lobe can vanish where a large value cannot,
  * "atlas": a different valid frame, as in a texture atlas; the result must be bit-identical to the same frame allocated alone.
Out-of-image taps are defined (EASU clamps to the edge, RCAS reads 0 or clamps), so a kernel that loads the pitch padding or the
row after the image instead gets a different answer than the oracle; a store one pixel or one row too far changes a guard byte.
Row windows hold exactly the rows fsr1_easu_input_rows (or RCAS's one-row apron) requires; the buffer rows around them are guard.

Each case checks: the kernel family the launchers pick, the family's oracle contract (the tolerances of tests/test_gpu_parity.py,
tests/test_upscale_post.py and tests/test_gpu_pointwise.py), every guard byte, and every output row outside [y0, y1)."""
import numpy as np
import pytest
import torch

import fsr1_b200 as F
import oracle_lib as ol
from easu_checks import expected_easu_kernel, viewport_2x

pytestmark = pytest.mark.gpu
api = F.api
GR = 8            # guard rows above and below (RCAS requests kRows + 2 = 6 rows up front)
RIGHT = 64        # guard bytes right of the image, before rounding the pitch to 16 bytes
POISONS = ["nan", "big", "atlas"]

# (element dtype, elements per pixel, integer view for bit comparisons)
KINDS = {"f16": (torch.float16, 4, torch.int16), "f32": (torch.float32, 4, torch.int32), "u8": (torch.uint8, 4, torch.uint8),
         "u10": (torch.int32, 1, torch.int32)}
POISON_BITS = {"nan": {"f16": 0x7E5A, "f32": 0x7FC0BEEF, "u8": 0xA5, "u10": 0x5A5A5A5A},
               "big": {"f16": 0x7BFF, "f32": 0x7F61BF3F, "u8": 0xFF, "u10": -1}}    # 65504, 3.0e38, all ones


def _bpp(kind):
    dt, per, _ = KINDS[kind]
    return per * torch.empty(0, dtype=dt).element_size()


def _random_frame(kind, rows, w, seed):
    """A valid frame of this storage kind: [rows, w, 4] (u10: [rows, w] packed words)."""
    f = F.uniform(w, rows, seed)
    if kind == "f16":
        return F.to_half(f)
    if kind == "f32":
        return f
    if kind == "u8":
        return np.floor(f * 255.0 + 0.5).astype(np.uint8)
    q = np.floor(f * 1023.0 + 0.5).astype(np.uint32)
    q[..., 3] &= 3
    return (q[..., 0] | (q[..., 1] << 10) | (q[..., 2] << 20) | (q[..., 3] << 30)).view(np.int32)


class Guarded:
    """An image of `rows` x `w` pixels at byte offset `left` of row GR of a poisoned buffer; `img` is the tensor view."""

    def __init__(self, kind, rows, w, poison, left=16, seed=0):
        dt, per, self.ivt = KINDS[kind]
        es = torch.empty(0, dtype=dt).element_size()
        pitch = -(-(left + w * _bpp(kind) + RIGHT) // 16) * 16
        self.buf = torch.empty((rows + 2 * GR, pitch // es), dtype=dt, device="cuda")
        if poison == "atlas":
            nb = _random_frame(kind, rows + 2 * GR, pitch // _bpp(kind), 900 + seed + rows + w)
            self.buf.view(self.ivt).copy_(torch.from_numpy(np.ascontiguousarray(nb).reshape(rows + 2 * GR, -1)).view(self.ivt))
        else:
            self.buf.view(self.ivt).fill_(POISON_BITS[poison][kind])
        self.rows, self.w, self.kind = rows, w, kind
        self.c0, self.c1 = left // es, left // es + w * per
        # explicit strides: a view of one row would otherwise report a compact row stride, which is not the buffer's pitch
        shape, strides = ((rows, w, 4), (self.buf.stride(0), 4, 1)) if per == 4 else ((rows, w), (self.buf.stride(0), 1))
        self.img = self.buf.as_strided(shape, strides, self.buf.storage_offset() + GR * self.buf.stride(0) + self.c0)
        self.snap()

    def snap(self):
        self.before = self.buf.clone()

    def set(self, a):
        self.img.copy_(torch.from_numpy(np.ascontiguousarray(a)).to(self.img.device))
        self.snap()

    def image(self, height=None, row0=0):
        return api.image(self.img, height=height, row0=row0)

    def numpy(self):
        return self.img.cpu().numpy()

    def assert_untouched(self, what, r0=0, r1=0):
        """Every byte of the buffer outside image rows [r0, r1) (window rows) still holds what it held before the launch."""
        diff = self.buf.view(self.ivt) != self.before.view(self.ivt)
        diff[GR + r0:GR + r1, self.c0:self.c1] = False
        if diff.any():
            y, x = (int(v) for v in torch.nonzero(diff)[0])
            raise AssertionError("%s: %d guard elements changed, first at buffer row %d element %d (image rows %d..%d at row %d, "
                                 "elements %d..%d)" % (what, int(diff.sum()), y, x, r0, r1, GR, self.c0, self.c1))


def plain(a, left=16):
    """The frame allocated alone: rows padded to 16 bytes with zeros, the [H, W, ...] view; left = 8 starts it 8 bytes into
    the allocation (the layout of the unaligned cases)."""
    a = np.ascontiguousarray(a)
    h, w = a.shape[:2]
    per = 16 // (a.itemsize * (4 if a.ndim == 3 else 1))
    x0 = 0 if left == 16 else left // (16 // per)
    t = torch.zeros((h, -(-(w + x0) // per) * per) + a.shape[2:], dtype=torch.from_numpy(a[:0]).dtype, device="cuda")
    t[:, x0:x0 + w] = torch.from_numpy(a).cuda()
    return t[:, x0:x0 + w]


def _q(x, n):
    s = np.float32((1 << n) - 1)
    return (np.nan_to_num(np.clip(x, 0.0, 1.0), nan=0.0).astype(np.float32) * s + np.float32(0.5)).astype(np.uint32)


def _codes(a, kind):
    """[H, W, 4] code values of a UNORM image (u8 array or packed u10 words)."""
    if kind == "u8":
        return a.astype(np.int64)
    u = a.view(np.uint32).astype(np.int64)
    return np.stack([u & 1023, (u >> 10) & 1023, (u >> 20) & 1023, u >> 30], axis=-1)


def _float_of(src, kind):
    """What the F-path arithmetic reads from this storage (c / (2^n - 1) for UNORM, alpha over 3 for RGB10A2)."""
    if kind in ("f16", "f32"):
        return src.astype(np.float32)
    c = _codes(src, kind).astype(np.float32)
    s = np.float32(255.0 if kind == "u8" else 1023.0)
    f = (c / s).astype(np.float32)
    f[..., 3] = c[..., 3] / np.float32(255.0 if kind == "u8" else 3.0)
    return f


def check_contract(got, want, contract, kind, what):
    """got / want: rows [y0, y1) of the stored result and of the oracle (float32 oracle values; UNORM: the oracle's float values)."""
    if contract == "bits":                               # bit-identical (half oracle, EXACT, Hx2, the two-kernel path)
        g, w_ = np.ascontiguousarray(got), np.ascontiguousarray(want)
        assert np.array_equal(g.view(np.uint8), w_.view(np.uint8)), what
        return
    if kind in ("u8", "u10"):                            # code values: "exact" or within `contract` codes
        bits = 8 if kind == "u8" else 10
        c = _codes(got, kind)
        d = np.abs(c[..., :3] - _q(want[..., :3], bits).astype(np.int64))
        assert d.max() <= contract, (what, int(d.max()))
        return
    d = np.abs(got.astype(np.float32) - want)[..., :3]
    assert not np.isnan(d).any() and d.max() <= contract, (what, float(np.nanmax(d)) if d.size else 0.0)


# ---- shapes ----------------------------------------------------------------------------------------------------------------
# Output widths around the 60-pixel RCAS span, the 62-pixel fused strip, the 64-pixel EASU tile and odd pair ends; heights around
# the 16-row steps.  Widths and heights are paired cyclically so that every width and every height occurs.
WIDTHS = [1, 2, 61, 62, 63, 64, 65, 120, 121, 122, 123, 124, 125, 126, 127, 128, 129]
HEIGHTS = [1, 2, 15, 16, 17, 33]
SHAPES = [(w, HEIGHTS[i % len(HEIGHTS)]) for i, w in enumerate(WIDTHS)] + [(63, 33), (125, 17), (2, 15), (1, 33)]
SLABS = [(125, 33, 3, 20), (64, 33, 7, 25), (121, 17, 1, 16), (63, 16, 5, 6)]     # (w, h, y0, y1): odd y0 / y1
BIG = (1920, 1080)                                                               # multi-wave: interior copies next to the guards


# ---- EASU ------------------------------------------------------------------------------------------------------------------
# id: (storage, flags, output/viewport scale, contract, kernel-name prefix or None = expected_easu_kernel, left offset)
EASU = {
    "h_quad2x": ("f16", 0, 2.0, 1e-2, None, 16),
    "h_vpairs_1.5x": ("f16", 0, 1.5, 1e-2, None, 16),
    "h_vpairs_1.3x": ("f16", 0, 1.3, 1e-2, None, 16),
    "h_vpairs_3x": ("f16", 0, 3.0, 1e-2, None, 16),
    "h_vpairs_1x_box_over_48KB": ("f16", 0, 1.0, 1e-2, None, 16),      # a 64x32 tile at 1x needs a ~67x35 box: ~85 KB of smem
    "f32_quad2x": ("f32", 0, 2.0, 1e-5, None, 16),
    "f32_vpairs_1.5x": ("f32", 0, 1.5, 1e-5, None, 16),
    "h_precise_2x": ("f16", api.FLAG_PRECISE, 2.0, 6e-4, None, 16),
    "h_precise_1.5x": ("f16", api.FLAG_PRECISE, 1.5, 6e-4, None, 16),
    "u8_quad2x": ("u8", 0, 2.0, 1, None, 16),
    "direct_f16_unaligned": ("f16", 0, 2.0, 1e-2, "easu_direct<f16io", 8),
    "direct_f32_exact": ("f32", api.FLAG_EXACT, 1.5, "bits", None, 16),
    "direct_u8_exact": ("u8", api.FLAG_EXACT, 2.0, 0, None, 16),
    "direct_u10": ("u10", 0, 2.0, 1, "easu_direct<unorm10", 16),
    "direct_u10_exact": ("u10", api.FLAG_EXACT, 1.5, 0, None, 16),
    "href": ("f16", api.FLAG_H_REFERENCE, 2.0, "bits", None, 16),
}
FMT = {"f16": api.FORMAT_RGBA16F, "f32": api.FORMAT_RGBA32F, "u8": api.FORMAT_RGBA8_UNORM, "u10": api.FORMAT_RGB10A2_UNORM}


QUAD_2X = [0x3F000000, 0x3F000000, 0xBE800000, 0xBE800000]        # con0 = {0.5, 0.5, -0.25, -0.25}


def easu_geometry(ow, oh, scale):
    """Constants for an output of ow x oh at `scale`: the viewport is ow / scale (at 2x exactly the 2x constants, odd outputs
    included), the resource the whole texels it touches."""
    if scale == 2.0:
        con_of = lambda v, n: api.easu_con(v, v, n, n, n, n)
        vw, vh = viewport_2x(ow, con_of), viewport_2x(oh, con_of)
    else:
        vw, vh = ow / scale, oh / scale
    iw, ih = max(1, int(np.ceil(vw))), max(1, int(np.ceil(vh)))
    con = api.easu_con(vw, vh, iw, ih, ow, oh)
    assert scale != 2.0 or con[:4] == QUAD_2X, (ow, oh, con[:4])
    return iw, ih, con


def run_easu(case, ow, oh, poison, y0=0, y1=None):
    kind, flags, scale, contract, prefix, left = EASU[case]
    y1 = oh if y1 is None else y1
    iw, ih, con = easu_geometry(ow, oh, scale)
    src = _random_frame(kind, ih, iw, ow * 7 + oh)
    r0, r1 = api.easu_input_rows(con, ih, y0, y1)
    gin = Guarded(kind, r1 - r0 + 1, iw, poison, left, seed=1)
    gin.set(src[r0:r1 + 1])
    gout = Guarded(kind, oh, ow, poison, left, seed=2)
    api.easu(gin.image(height=ih, row0=r0), gout.image(), con, y0=y0, y1=y1, flags=flags)
    torch.cuda.synchronize()
    what = (case, ow, oh, poison, y0, y1, api.last_kernel())
    want_prefix = prefix or expected_easu_kernel(con, FMT[kind], flags)
    assert api.last_kernel().startswith(want_prefix), (what, want_prefix)
    got = gout.numpy()
    if contract == "bits" and kind == "f16":
        want = ol.easu(src, ow, oh, con, y0=y0, y1=y1)                     # the H-path model on the half input
    else:
        want = ol.easu(_float_of(src, kind), ow, oh, con, y0=y0, y1=y1)
        if contract == "bits":
            want = want.astype(np.float32)
    check_contract(got[y0:y1], want[y0:y1], contract, kind, what)
    if kind in ("f16", "f32"):
        assert np.all(got[y0:y1, :, 3] == 1.0), what
    gin.assert_untouched(what + ("input",))
    gout.assert_untouched(what + ("output",), y0, y1)
    if poison == "atlas":                                                  # == the frame allocated alone
        alone = plain(np.zeros(got.shape, got.dtype), left)
        api.easu(plain(src, left), alone, con, y0=y0, y1=y1, flags=flags)
        torch.cuda.synchronize()
        assert np.array_equal(np.ascontiguousarray(got[y0:y1]).view(np.uint8), np.ascontiguousarray(alone.cpu().numpy()[y0:y1]).view(np.uint8)), what


@pytest.mark.parametrize("poison", POISONS)
@pytest.mark.parametrize("case", list(EASU))
def test_easu_stays_inside_its_images(case, poison):
    for ow, oh in SHAPES:
        run_easu(case, ow, oh, poison)
    for ow, oh, y0, y1 in SLABS:
        run_easu(case, ow, oh, poison, y0, y1)


@pytest.mark.parametrize("case", list(EASU))
def test_easu_stays_inside_its_images_multi_wave(case):
    run_easu(case, BIG[0] - 1, BIG[1] - 1, "nan")                          # odd sizes: partial pairs on both edges
    run_easu(case, BIG[0], BIG[1], "big", 301, 777)


# ---- RCAS ------------------------------------------------------------------------------------------------------------------
# id: (storage, flags, contract, kernel-name prefix, left offset)
RCAS = {"h_packed": ("f16", 0, 1e-2, "rcas_h_packed<", 16),
        "f32_packed": ("f32", 0, 1e-5, "rcas_f32_packed", 16),
        "u8_packed": ("u8", 0, 1, "rcas_u8_packed", 16),
        "direct_u10_exact": ("u10", api.FLAG_EXACT, 0, "rcas_direct<unorm10,exact", 16),
        "direct_f32_exact": ("f32", api.FLAG_EXACT, "bits", "rcas_direct<f32,exact", 16),
        "direct_f16_unaligned": ("f16", 0, 1e-2, "rcas_direct<f16io", 8),
        "href": ("f16", api.FLAG_H_REFERENCE, "bits", "rcas_href", 16),
        "hx2": ("f16", api.FLAG_RCAS_HX2, "bits", "rcas_hx2", 16)}
RCAS_OPTS = {1: api.FLAG_RCAS_DENOISE, 2: api.FLAG_RCAS_PASSTHROUGH_ALPHA, 4: api.FLAG_OUTPUT_SQUARE}


def run_rcas(case, w, h, poison, clamp=0, opts=0, y0=0, y1=None):
    kind, flags, contract, prefix, left = RCAS[case]
    y1 = h if y1 is None else y1
    for bit, f in RCAS_OPTS.items():
        if opts & bit:
            flags |= f
    flags |= api.FLAG_RCAS_CLAMP if clamp else 0
    src = _random_frame(kind, h, w, w * 5 + h + opts)
    n0, n1 = max(y0 - 1, 0), min(y1, h - 1)                                 # the rows RCAS reads: one-row apron
    gin = Guarded(kind, n1 - n0 + 1, w, poison, left, seed=3)
    gin.set(src[n0:n1 + 1])
    gout = Guarded(kind, h, w, poison, left, seed=4)
    api.rcas(gin.image(height=h, row0=n0), gout.image(), api.rcas_con(0.25), y0=y0, y1=y1, flags=flags)
    torch.cuda.synchronize()
    what = (case, w, h, poison, clamp, opts, y0, y1, api.last_kernel())
    if not (opts & 4 and prefix.startswith(("rcas_direct", "rcas_href", "rcas_hx2"))):   # those square in a second pass
        assert api.last_kernel().startswith(prefix), what
    got = gout.numpy()
    half_model = contract == "bits" and kind == "f16"
    fin = src if half_model else _float_of(src, kind)
    want = ol.rcas(fin, ol.rcas_con(0.25), bool(clamp), y0=y0, y1=y1, denoise=bool(opts & 1), alpha=bool(opts & 2))
    if opts & 4:
        if half_model:
            want = want.astype(np.float32)
            want[..., :3] = (want[..., :3] * want[..., :3]).astype(np.float16).astype(np.float32)
            want = want.astype(np.float16)
        else:
            want[..., :3] = want[..., :3] * want[..., :3]
    tol = contract
    if opts & 4 and kind == "f32" and contract != "bits":
        tol = 2e-5
    check_contract(got[y0:y1], want[y0:y1], tol, kind, what)
    if kind in ("f16", "f32"):
        a = got[y0:y1, :, 3]
        assert np.array_equal(a, src[y0:y1, :, 3]) if opts & 2 else np.all(a == 1.0), what
    gin.assert_untouched(what + ("input",))
    gout.assert_untouched(what + ("output",), y0, y1)
    if poison == "atlas":
        alone = plain(np.zeros(got.shape, got.dtype), left)
        api.rcas(plain(src, left), alone, api.rcas_con(0.25), y0=y0, y1=y1, flags=flags)
        torch.cuda.synchronize()
        assert np.array_equal(np.ascontiguousarray(got[y0:y1]).view(np.uint8), np.ascontiguousarray(alone.cpu().numpy()[y0:y1]).view(np.uint8)), what


@pytest.mark.parametrize("poison", POISONS)
@pytest.mark.parametrize("case", list(RCAS))
def test_rcas_stays_inside_its_images(case, poison):
    for clamp in (0, 1):
        if clamp and case == "u8_packed":
            continue                      # the packed UNORM kernel is held to the oracle without the clamp (test_gpu_parity.py)
        for w, h in SHAPES:
            run_rcas(case, w, h, poison, clamp)
        for w, h, y0, y1 in SLABS:
            run_rcas(case, w, h, poison, clamp, 0, y0, y1)


@pytest.mark.parametrize("opts", range(8))
@pytest.mark.parametrize("clamp", [0, 1])
def test_rcas_h_packed_options_stay_inside_their_images(opts, clamp):
    for poison in ("nan", "big"):
        for w, h in SHAPES[::2]:
            run_rcas("h_packed", w, h, poison, clamp, opts)
        run_rcas("h_packed", 63, 33, poison, clamp, opts, 3, 20)


@pytest.mark.parametrize("case", list(RCAS))
def test_rcas_stays_inside_its_images_multi_wave(case):
    run_rcas(case, BIG[0] - 1, BIG[1] - 1, "nan")
    run_rcas(case, BIG[0], BIG[1], "big", 0, 0, 301, 777)


# ---- fsr1_upscale with FSR1_FLAG_FUSED -------------------------------------------------------------------------------------
def run_fused(ow, oh, poison, y0=0, y1=None):
    y1 = oh if y1 is None else y1
    iw, ih, econ = easu_geometry(ow, oh, 2.0)
    rcon = api.rcas_con(0.25)
    src = _random_frame("f16", ih, iw, ow * 3 + oh)
    # the two-kernel path on frames allocated alone: what the fused kernel must reproduce bit for bit
    want = plain(np.zeros((oh, ow, 4), np.float16))
    api.upscale(plain(src), plain(np.zeros((oh, ow, 4), np.float16)), want, econ, rcon)
    e0, e1 = max(y0 - 1, 0), min(y1 + 1, oh)
    r0, r1 = api.easu_input_rows(econ, ih, e0, e1)
    gin = Guarded("f16", r1 - r0 + 1, iw, poison, seed=5)
    gin.set(src[r0:r1 + 1])
    gtmp = Guarded("f16", oh, ow, poison, seed=6)
    gout = Guarded("f16", oh, ow, poison, seed=7)
    api.upscale(gin.image(height=ih, row0=r0), gtmp.image(), gout.image(), econ, rcon, y0=y0, y1=y1, flags=api.FLAG_FUSED)
    torch.cuda.synchronize()
    what = ("fused", ow, oh, poison, y0, y1, api.last_kernel())
    assert api.last_kernel().startswith("fused_easu_rcas_h_quad2x"), what
    check_contract(gout.numpy()[y0:y1], want.cpu().numpy()[y0:y1], "bits", "f16", what)
    gin.assert_untouched(what + ("input",))
    gtmp.assert_untouched(what + ("tmp",))                                   # no intermediate image
    gout.assert_untouched(what + ("output",), y0, y1)


@pytest.mark.parametrize("poison", POISONS)
def test_fused_upscale_stays_inside_its_images(poison):
    for ow, oh in SHAPES:
        run_fused(ow, oh, poison)
    for ow, oh, y0, y1 in SLABS:
        run_fused(ow, oh, poison, y0, y1)
    run_fused(BIG[0] * 2 - 1, BIG[1] * 2 - 1, poison)
    run_fused(BIG[0] * 2, BIG[1] * 2, poison, 301, 777)


# ---- fsr1_upscale_post ---------------------------------------------------------------------------------------------------
# id: (TEPD bits, SRTM inverse, LFGA, dither tile).  Output: RGBA16F without TEPD, RGBA8 with TEPD 8, RGB10A2 with TEPD 10.
POST = {"rgba16f": (0, True, True, False), "rgba8": (8, False, True, True), "rgb10a2": (10, True, True, True)}
OUT_KIND = {0: "f16", 8: "u8", 10: "u10"}


def run_post(case, scale, ow, oh, poison, y0=0, y1=None):
    tepd_bits, srtm_inv, lfga, use_dither = POST[case]
    y1 = oh if y1 is None else y1
    iw, ih, econ = easu_geometry(ow, oh, scale)
    rcon = api.rcas_con(0.25)
    src = _random_frame("f16", ih, iw, ow + oh * 3)
    rng = np.random.default_rng(ow * 31 + oh)
    grain = (rng.random((3, 5, 4), np.float32) - 0.5).astype(np.float16)          # odd tile widths: pairs wrap inside the tile
    dither = (rng.random((3, 7, 4), np.float32) * 1.2 - 0.1).astype(np.float32)
    kind = OUT_KIND[tepd_bits]
    # the sequence of separate calls on frames allocated alone (the contract of fsr1_upscale_post)
    t = plain(np.zeros((oh, ow, 4), np.float16))
    api.upscale(plain(src), plain(np.zeros((oh, ow, 4), np.float16)), t, econ, rcon, y0, y1, api.FLAG_FUSED)
    pg, pd = plain(grain), plain(dither) if use_dither else None
    if srtm_inv:
        api.srtm(t, t, inverse=True, y0=y0, y1=y1)
    if lfga:
        api.lfga(t, pg, t, 0.3, y0=y0, y1=y1)
    if tepd_bits:
        want = plain(np.zeros((oh, ow, 4), np.uint8) if tepd_bits == 8 else np.zeros((oh, ow), np.int32))
        api.tepd(t, want, tepd_bits, frame=7, dither=pd, y0=y0, y1=y1)
    else:
        want = t
    e0, e1 = max(y0 - 1, 0), min(y1 + 1, oh)
    r0, r1 = api.easu_input_rows(econ, ih, e0, e1)
    gin = Guarded("f16", r1 - r0 + 1, iw, poison, seed=8)
    gin.set(src[r0:r1 + 1])
    gtmp = Guarded("f16", oh, ow, poison, seed=9)
    gout = Guarded(kind, oh, ow, poison, seed=10)
    gg = Guarded("f16", 3, 5, poison, seed=11)
    gg.set(grain)
    gd = Guarded("f32", 3, 7, poison, seed=12)
    gd.set(dither)
    api.upscale_post(gin.image(height=ih, row0=r0), gtmp.image(), gout.image(), econ, rcon, srtm_inverse=srtm_inv,
                     grain=gg.image() if lfga else None, amount=0.3, tepd_bits=tepd_bits, dither=gd.image() if use_dither else None,
                     frame=7, y0=y0, y1=y1, flags=api.FLAG_FUSED)
    torch.cuda.synchronize()
    what = ("post", case, scale, ow, oh, poison, y0, y1, api.last_kernel())
    fused = scale == 2.0
    assert api.last_kernel().startswith("fused_easu_rcas_h_quad2x" if fused else "rcas_h_packed_post"), what
    check_contract(gout.numpy()[y0:y1], want.cpu().numpy()[y0:y1], "bits", kind, what)
    gin.assert_untouched(what + ("input",))
    if fused:
        gtmp.assert_untouched(what + ("tmp",))
    else:
        gtmp.assert_untouched(what + ("tmp",), e0, e1)                         # EASU wrote the slab and its apron rows
    gout.assert_untouched(what + ("output",), y0, y1)
    gg.assert_untouched(what + ("grain",))
    gd.assert_untouched(what + ("dither",))


@pytest.mark.parametrize("poison", POISONS)
@pytest.mark.parametrize("scale", [2.0, 1.5], ids=["fused_2x", "rcas_epilogue_1.5x"])
@pytest.mark.parametrize("case", list(POST))
def test_upscale_post_stays_inside_its_images(case, scale, poison):
    for ow, oh in SHAPES:
        run_post(case, scale, ow, oh, poison)
    for ow, oh, y0, y1 in SLABS:
        run_post(case, scale, ow, oh, poison, y0, y1)
    if poison == "nan":
        run_post(case, scale, BIG[0] - 1, BIG[1] - 1, poison)
        run_post(case, scale, BIG[0], BIG[1], poison, 301, 777)


# ---- pointwise passes ------------------------------------------------------------------------------------------------------
def _to_half(a):
    with np.errstate(over="ignore"):
        return a.astype(np.float16)


def pointwise_want(op, src, kind, grain, dither, y0, y1):
    """The oracle of one pointwise pass on rows [y0, y1): fp32 passes bit-exact on RGBA32F, rounded once on RGBA16F; _h passes
    bit-exact to the half oracle."""
    if op.endswith("_h"):
        if op == "srtm_h":
            return ol.srtm_h(src)
        if op == "lfga_h":
            return ol.lfga_h(src, grain, 0.35)
        return ol.tepd_h(src, 8, dither=dither)
    f = src.astype(np.float32)
    if op == "srtm":
        r = ol.srtm(f, inverse=False)
    elif op == "lfga":
        r = ol.lfga(f, np.ascontiguousarray(grain.astype(np.float32)), 0.35)
    else:
        r = ol.tepd(f, 10, frame=3, dither=None if dither is None else np.ascontiguousarray(dither.astype(np.float32)))
    return r if kind == "f32" else _to_half(r)


def run_pointwise(op, kind, w, h, poison, in_place, y0=0, y1=None):
    y1 = h if y1 is None else y1
    src = _random_frame(kind, h, w, w + 11 * h)
    rng = np.random.default_rng(w + h)
    gdt = np.float16 if kind == "f16" else np.float32
    grain = (rng.random((3, 5, 4), np.float32) - 0.5).astype(gdt)
    dither = (rng.random((3, 7, 4), np.float32)).astype(gdt) if op.startswith("tepd") else None
    gin = Guarded(kind, h, w, poison, seed=13)
    gin.set(src)
    gout = gin if in_place else Guarded(kind, h, w, poison, seed=14)
    gaux = None
    if op.startswith("lfga"):
        gaux = Guarded(kind, 3, 5, poison, seed=15)
        gaux.set(grain)
    elif dither is not None:
        gaux = Guarded(kind, 3, 7, poison, seed=15)
        gaux.set(dither)
    a, b, x = gin.image(), gout.image(), gaux.image() if gaux else None
    {"srtm": lambda: api.srtm(a, b, y0=y0, y1=y1), "lfga": lambda: api.lfga(a, x, b, 0.35, y0=y0, y1=y1),
     "tepd": lambda: api.tepd(a, b, 10, frame=3, dither=x, y0=y0, y1=y1), "srtm_h": lambda: api.srtm_h(a, b, y0=y0, y1=y1),
     "lfga_h": lambda: api.lfga_h(a, x, b, 0.35, y0=y0, y1=y1), "tepd_h": lambda: api.tepd_h(a, b, 8, dither=x, y0=y0, y1=y1)}[op]()
    torch.cuda.synchronize()
    what = (op, kind, w, h, poison, in_place, y0, y1, api.last_kernel())
    assert api.last_kernel().startswith("pointwise_hx2" if op.endswith("_h") else "pointwise<"), what
    got = gout.numpy()
    want = pointwise_want(op, src, kind, grain, dither, y0, y1)
    check_contract(got[y0:y1], want[y0:y1], "bits", kind, what)
    if in_place:
        assert np.array_equal(got[:y0].view(np.uint8), src[:y0].view(np.uint8)), what
        assert np.array_equal(got[y1:].view(np.uint8), src[y1:].view(np.uint8)), what
    gin.assert_untouched(what + ("input",), y0 if in_place else 0, y1 if in_place else 0)
    gout.assert_untouched(what + ("output",), y0, y1)
    if gaux:
        gaux.assert_untouched(what + ("aux",))


@pytest.mark.parametrize("poison", ["nan", "big"])
@pytest.mark.parametrize("op,kind", [("srtm", "f32"), ("lfga", "f32"), ("tepd", "f16"), ("srtm_h", "f16"), ("lfga_h", "f16"),
                                     ("tepd_h", "f16")])
def test_pointwise_passes_stay_inside_their_images(op, kind, poison):
    for in_place in (False, True):
        for w, h in SHAPES[::3] + [(1025, 3), (2049, 2)]:                   # 1024-pixel row stretches per CTA
            run_pointwise(op, kind, w, h, poison, in_place)
        run_pointwise(op, kind, 125, 33, poison, in_place, 3, 20)
