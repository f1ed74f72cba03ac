"""The per-pixel model of the half-storage kernels (tests/model/fsr1_kernel_model.c) against the emulator running their device code,
bit for bit, and against the fp32 oracle at the tolerances the other tests use.

Why bit-exact is possible: every operation of these kernels is correctly rounded (fp32 and half IEEE operations, integer bit tricks)
except the two reciprocals, rcp.approx.ftz.f32 of a half operand whose result is rounded to half at once.  The first test shows,
exactly, that 1/x lies at least 2 fp32 ulps from every half rounding boundary for every finite half x, so any fp32 value within the
1 ulp PTX documents for rcp.approx rounds to the correctly rounded half of 1/x.  The GPU side of the same comparison is
tests/test_gpu_kernel_model.py."""
from fractions import Fraction

import ctypes

import numpy as np
import pytest

import kernel_model as km
import oracle_lib as ol
from test_emu import EMU_GEOMETRY, PROD, emu_easu, emu_easu_pairs, emu_lib

KINDS = list(km.CONTENT)


def _half_values():
    """Every finite half as (bits, exact Fraction), ascending."""
    bits = np.arange(0, 0x7c00, dtype=np.uint16)
    return bits, [Fraction(float(v)) for v in bits.view(np.float16).astype(np.float64)]


def test_half_reciprocal_is_correctly_rounded_with_two_ulp_margin():
    """For every positive finite half x: 1/x lies at least 2 fp32 ulps from every half rounding boundary (the midpoints between
    neighbouring halves, and 65520 where rounding overflows), and the model's reciprocal is the correctly rounded half of 1/x.
    Negative halves are the mirror image; 0 gives inf in the kernels and the model alike."""
    _, vals = _half_values()
    lib = km.lib()
    worst = None
    for b in range(1, 0x7c00):
        v = 1 / vals[b]
        r = lib.fkm_h_recip(b)
        e = v.numerator.bit_length() - v.denominator.bit_length()
        if Fraction(2) ** e > v:
            e -= 1
        ulp = Fraction(2) ** (e - 23)                                   # fp32 ulp at v (v is in the normal fp32 range)
        if v >= 65520:
            assert r == 0x7c00, (b, hex(r))
            margin = (v - 65520) / ulp
        else:
            assert r < 0x7c00, (b, hex(r))
            lo = (vals[r - 1] + vals[r]) / 2 if r > 0 else Fraction(0)
            hi = (vals[r] + vals[r + 1]) / 2 if r + 1 < 0x7c00 else Fraction(65520)
            assert lo < v < hi, (b, hex(r))                               # correctly rounded (no ties: margins below)
            margin = min(v - lo, hi - v) / ulp
        worst = margin if worst is None or margin < worst else worst
    print("smallest distance of 1/x from a half rounding boundary: %.5f fp32 ulps" % float(worst))
    assert worst >= 2


def _round_half_exact(x, vals, keys):
    """Correctly rounded half (bits) of the exact rational x, round to nearest even, overflow to inf."""
    s = 0x8000 if x < 0 else 0
    a = -x if x < 0 else x
    if a >= 65520:
        return s | 0x7c00
    i = int(np.searchsorted(keys, float(a)))
    i = min(max(i, 1), 0x7bff)
    for j in (i - 1, i, i + 1):                                           # the float key can be off by one
        if j + 1 <= 0x7bff and vals[j] <= a <= vals[j + 1]:
            lo, hi = j, j + 1
            break
    else:
        lo = hi = 0x7bff
    mid = (vals[lo] + vals[hi]) / 2
    r = lo if a < mid else hi if a > mid else (lo if lo % 2 == 0 else hi)
    return s | r


def test_model_half_fma_rounds_once():
    """hfma is the one place where double arithmetic is not exact (a b + c spans up to 64 bits): against exact rational arithmetic
    on random operands and on ones built to put a b + c next to a half rounding boundary, subnormals and signs included."""
    bits, vals = _half_values()
    keys = bits.view(np.float16).astype(np.float64)
    lib = km.lib()
    rng = np.random.default_rng(5)
    cases = []
    for _ in range(6000):
        a, b = rng.integers(0, 0x7c00, size=2)
        c = rng.integers(0, 0x7c00)
        if rng.random() < 0.5:                                             # c large, a b tiny: the sum needs more than 53 bits
            a, b = rng.integers(0, 0x1800, size=2)
            c = rng.integers(0x5800, 0x7c00)
        sa, sb, sc = rng.integers(0, 2, size=3)
        cases.append((int(a) | int(sa) << 15, int(b) | int(sb) << 15, int(c) | int(sc) << 15))
    for c in (0x7bff, 0x7bfe, 0x3c00, 0x3c01, 0x0400, 0x0001):             # c at a half ulp's midpoint +- the smallest products
        for a in (0x0001, 0x0002, 0x0003, 0x03ff):
            for sgn in (0, 0x8000):
                cases.append((a | sgn, 0x0001, c))
                cases.append((a | sgn, 0x3800, c))
    for a, b, c in cases:
        va, vb, vc = vals[a & 0x7fff], vals[b & 0x7fff], vals[c & 0x7fff]
        exact = (-va if a & 0x8000 else va) * (-vb if b & 0x8000 else vb) + (-vc if c & 0x8000 else vc)
        want = _round_half_exact(exact, vals, keys)
        got = lib.fkm_hfma(a, b, c)
        if exact == 0:                                                     # the sign of an exact zero follows IEEE's sum rule
            continue
        assert got == want, (hex(a), hex(b), hex(c), hex(got), hex(want))


# ---- model == emulator, bit for bit ----------------------------------------------------------------------------------------
EMU_SIZES = [(64, 36), (70, 23), (33, 17), (5, 3)]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size", EMU_SIZES)
def test_model_equals_emulated_easu_h_quad2x(size, kind):
    iw, ih = size
    ow, oh = 2 * iw, 2 * ih
    src = km.content(kind, iw, ih, 11)
    con = km.con_2x(ol.easu_con(iw, ih, ow, oh))
    got = emu_easu(PROD, src, ow, oh, con=con)
    km.assert_same_bits(got, km.easu_h(src, ow, oh, con), ("easu_h_quad2x", size, kind))


ANY_SCALE = [(96, 54, 144, 81), (96, 54, 125, 70), (64, 64, 64, 64), (50, 20, 65, 26), (33, 17, 57, 31), (64, 36, 128, 72),
             (96, 54, 192, 81)]


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("shape", ANY_SCALE)
def test_model_equals_emulated_easu_h_vpairs(shape, kind):
    iw, ih, ow, oh = shape
    src = km.content(kind, iw, ih, 12)
    con = ol.easu_con(iw, ih, ow, oh)
    got = emu_easu_pairs(src, ow, oh, con=con)
    km.assert_same_bits(got, km.easu_h(src, ow, oh, con, any_scale=True), ("easu_h_vpairs", shape, kind))


@pytest.mark.parametrize("case", list(EMU_GEOMETRY))
def test_model_equals_emulated_easu_geometry(case):
    """Viewports, offsets, anisotropic and extreme scales: the kernel the constants select, on every content class."""
    iw, ih, vw, vh, off, ow, oh = EMU_GEOMETRY[case]
    con = ol.easu_con(iw, ih, ow, oh, vw, vh, off=off)
    quad = con[:4] == km.QUAD_2X
    y0, y1 = oh // 3, 2 * oh // 3 + 1
    for kind in KINDS:
        src = km.content(kind, iw, ih, 13)
        run = (lambda **kw: emu_easu(PROD, src, ow, oh, con=con, **kw)) if quad else (lambda **kw: emu_easu_pairs(src, ow, oh, con=con, **kw))
        want = km.easu_h(src, ow, oh, con)
        km.assert_same_bits(run(ctas=2), want, (case, kind))
        km.assert_same_bits(run(y0=y0, y1=y1, ctas=1)[y0:y1], want[y0:y1], (case, kind, "rows"))


def emu_rcas_opt(src, con, clamp, opts, y0=0, y1=None):
    h, w = src.shape[:2]
    y1 = h if y1 is None else y1
    s = np.ascontiguousarray(src.view(np.uint16))
    out = np.zeros((h, w, 4), np.uint16)
    rc = emu_lib().emu_rcas_h_packed_opt(ctypes.c_void_p(s.ctypes.data), 0, h, ctypes.c_void_p(out.ctypes.data), w, h,
                                         ctypes.c_longlong(s.strides[0]), ctypes.c_longlong(out.strides[0]), (ctypes.c_uint32 * 4)(*con),
                                         1 if clamp else 0, y0, y1, opts)
    assert rc == 0
    return out


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("clamp", [False, True])
@pytest.mark.parametrize("size", [(128, 72), (61, 19), (6, 5)])
def test_model_equals_emulated_rcas_h_packed(size, clamp, kind):
    """All eight option sets (DENOISE, PASSTHROUGH_ALPHA, OUTPUT_SQUARE) and both out-of-image rules, two sharpness values."""
    w, h = size
    src = km.content(kind, w, h, 14)
    for sharp in (0.25, 0.0):
        con = ol.rcas_con(sharp)
        for opts in range(8) if sharp == 0.25 else (0, 1):
            km.assert_same_bits(emu_rcas_opt(src, con, clamp, opts), km.rcas_h(src, con, clamp, opts), ("rcas_h_packed", size, clamp, kind, opts, sharp))


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("size", [(64, 36), (33, 17), (5, 3)])
def test_model_equals_emulated_fused(size, kind):
    """fused_h_quad2x_kernel == model EASU -> half intermediate -> model RCAS, whole frame and a row range."""
    iw, ih = size
    ow, oh = 2 * iw, 2 * ih
    src = km.content(kind, iw, ih, 15)
    con = km.con_2x(ol.easu_con(iw, ih, ow, oh))
    rcon = ol.rcas_con(0.25)
    want = km.rcas_h(km.easu_h(src, ow, oh, con), rcon)
    s16 = np.ascontiguousarray(src.view(np.uint16))
    for (y0, y1, ctas) in ((0, oh, 3), (oh // 3, 2 * oh // 3 + 1, 1)):
        out = np.zeros((oh, ow, 4), np.uint16)
        rc = emu_lib().emu_fused_h(ctypes.c_void_p(s16.ctypes.data), iw, ih, ctypes.c_longlong(s16.strides[0]), ctypes.c_void_p(out.ctypes.data),
                                   ow, oh, ctypes.c_longlong(out.strides[0]), (ctypes.c_uint32 * 4)(*rcon), y0, y1, ctas)
        assert rc == 0
        km.assert_same_bits(out[y0:y1], want[y0:y1], ("fused", size, kind, y0, y1))


@pytest.mark.parametrize("codes", list(km.CODES))
@pytest.mark.parametrize("size", [(64, 36), (70, 23), (33, 17)])
def test_model_equals_emulated_u8(size, codes):
    """easu_u_quad2x_kernel<8> and rcas_u_packed_kernel<8> (every option set, both out-of-image rules)."""
    iw, ih = size
    ow, oh = 2 * iw, 2 * ih
    raw = km.CODES[codes](iw, ih, 16)
    src = km._pack8(raw)
    con = km.con_2x(ol.easu_con(iw, ih, ow, oh))
    out = np.zeros((oh, ow), np.uint32)
    rc = emu_lib().emu_easu_u_quad2x(8, ctypes.c_void_p(src.ctypes.data), iw, ih, ctypes.c_longlong(src.strides[0]),
                                     ctypes.c_void_p(out.ctypes.data), ow, oh, ctypes.c_longlong(out.strides[0]), (ctypes.c_uint32 * 16)(*con), 0, oh, 3)
    assert rc == 0
    km.assert_same_bits(out.view(np.uint8).reshape(oh, ow, 4), km.easu_u8(raw, ow, oh, con), ("easu_u8", size, codes))
    rcon = ol.rcas_con(0.25)
    for clamp in (0, 1):
        for opts in range(8):
            o = np.zeros((ih, iw), np.uint32)
            rc = emu_lib().emu_rcas_u_packed_opt(8, ctypes.c_void_p(src.ctypes.data), ctypes.c_void_p(o.ctypes.data), iw, ih,
                                                 ctypes.c_longlong(src.strides[0]), ctypes.c_longlong(o.strides[0]), (ctypes.c_uint32 * 4)(*rcon),
                                                 clamp, 0, ih, opts)
            assert rc == 0
            km.assert_same_bits(o.view(np.uint8).reshape(ih, iw, 4), km.rcas_u8(raw, rcon, clamp, opts), ("rcas_u8", size, codes, clamp, opts))


# ---- the model is FSR: against the fp32 oracle ------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_model_against_oracle(kind):
    """On the content the other tests use (uniform, structured), the model is held to their tolerances against the fp32 oracle
    reading the same half input: EASU 5e-3 (2x and any scale), RCAS 4e-3.  On the other classes the error is printed only."""
    rows = []
    for (iw, ih, ow, oh) in ((64, 36, 128, 72), (96, 54, 144, 81), (33, 17, 57, 31)):
        src = km.content(kind, iw, ih, 17)
        con = ol.easu_con(iw, ih, ow, oh)
        want = ol.easu(src.astype(np.float32), ow, oh, con)
        got = km.easu_h(src, ow, oh, con).view(np.float16).astype(np.float32)
        rows.append(("easu", (iw, ih, ow, oh), np.nanmax(np.abs(got - want)[..., :3])))
        for clamp in (False, True):
            r_want = ol.rcas(src.astype(np.float32), ol.rcas_con(0.25), clamp)
            r_got = km.rcas_h(src, ol.rcas_con(0.25), clamp).view(np.float16).astype(np.float32)
            rows.append(("rcas", (iw, ih, clamp), np.nanmax(np.abs(r_got - r_want)[..., :3])))
    for what, shape, err in rows:
        print("model vs oracle %-12s %-5s %-22s max abs %.3g" % (kind, what, shape, err))
        if kind in ("uniform", "structured"):
            assert err <= (5e-3 if what == "easu" else 4e-3), (what, shape, err)
