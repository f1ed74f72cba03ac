"""ctypes access to the per-pixel model of the half-storage kernels (tests/model/fsr1_kernel_model.c), the content classes the
bit-exact tests run it on, and the comparison they use.  TEST INFRASTRUCTURE ONLY.

The model restates the arithmetic of easu_h_quad2x, easu_h_vpairs, easu_u8_quad2x, rcas_h_packed and rcas_u8_packed one output
pixel at a time; each of those kernels, and the emulator running their device code, must give the model's bits exactly."""
import ctypes
import os
import subprocess

import numpy as np

import fsr1_b200 as F

MODEL_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "model")
QUAD_2X = [0x3F000000, 0x3F000000, 0xBE800000, 0xBE800000]        # con0 = {0.5, 0.5, -0.25, -0.25}
P, LL = ctypes.c_void_p, ctypes.c_longlong
_lib = None


def lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "-C", MODEL_DIR, "libfsr1_kernel_model.so"])
        _lib = ctypes.CDLL(os.path.join(MODEL_DIR, "libfsr1_kernel_model.so"))
        for f in ("fkm_h_recip", "fkm_hfma"):
            getattr(_lib, f).restype = ctypes.c_uint16
        _lib.fkm_h_recip.argtypes = [ctypes.c_uint16]
        _lib.fkm_hfma.argtypes = [ctypes.c_uint16] * 3
    return _lib


def _u32(con):
    return (ctypes.c_uint32 * len(con))(*con)


def con_2x(con):
    """The constant block with con0 replaced by the exactly-2x constants (the kernels read only con0)."""
    return QUAD_2X + list(con[4:])


def easu_h(src, ow, oh, con, y0=0, y1=None, any_scale=False):
    """[H,W,4] float16 -> [oh,ow,4] uint16 bits of rows [y0, y1) (other rows 0).  The constants select the 2x or the any-scale
    form as the launcher does; any_scale forces the any-scale form (easu_h_vpairs run at exactly 2x)."""
    y1 = oh if y1 is None else y1
    s = np.ascontiguousarray(src.view(np.uint16))
    out = np.zeros((oh, ow, 4), np.uint16)
    rc = lib().fkm_easu_h(P(s.ctypes.data), s.shape[1], s.shape[0], LL(s.shape[1] * 4), P(out.ctypes.data), ow, oh, LL(ow * 4),
                          _u32(con), y0, y1, 1 if any_scale else 0)
    assert rc == 0, rc
    return out


def _pack8(raw):
    return np.ascontiguousarray(np.ascontiguousarray(raw, np.uint8).view(np.uint32)[..., 0])


def easu_u8(raw, ow, oh, con, y0=0, y1=None):
    """[H,W,4] uint8 codes -> [oh,ow,4] uint8, exactly 2x."""
    y1 = oh if y1 is None else y1
    s = _pack8(raw)
    out = np.zeros((oh, ow), np.uint32)
    rc = lib().fkm_easu_u8(P(s.ctypes.data), s.shape[1], s.shape[0], LL(s.shape[1]), P(out.ctypes.data), ow, oh, LL(ow), _u32(con), y0, y1)
    assert rc == 0, rc
    return out.view(np.uint8).reshape(oh, ow, 4)


def rcas_h(src, con, clamp=False, opts=0, y0=0, y1=None):
    """[H,W,4] float16 (or uint16 bits) -> [H,W,4] uint16 bits; opts: bit 0 DENOISE, 1 PASSTHROUGH_ALPHA, 2 OUTPUT_SQUARE."""
    h, w = src.shape[:2]
    y1 = h if y1 is None else y1
    s = np.ascontiguousarray(src.view(np.uint16))
    out = np.zeros((h, w, 4), np.uint16)
    rc = lib().fkm_rcas_h(P(s.ctypes.data), w, h, LL(w * 4), P(out.ctypes.data), LL(w * 4), _u32(con), 1 if clamp else 0, y0, y1, opts)
    assert rc == 0, rc
    return out


def rcas_u8(raw, con, clamp=False, opts=0, y0=0, y1=None):
    h, w = raw.shape[:2]
    y1 = h if y1 is None else y1
    s = _pack8(raw)
    out = np.zeros((h, w), np.uint32)
    rc = lib().fkm_rcas_u8(P(s.ctypes.data), w, h, LL(w), P(out.ctypes.data), LL(w), _u32(con), 1 if clamp else 0, y0, y1, opts)
    assert rc == 0, rc
    return out.view(np.uint8).reshape(h, w, 4)


def assert_same_bits(got, want, what=""):
    """Equal bits, or a report of how many values differ, the first (y, x, channel) and both bit patterns there."""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if got.dtype != want.dtype or got.dtype.kind == "f":
        got, want = got.view(np.uint16 if got.itemsize == 2 else np.uint8), want.view(np.uint16 if want.itemsize == 2 else np.uint8)
    bad = got != want
    if bad.any():
        y, x, c = np.argwhere(bad)[0]
        fmt = "0x%04x" if got.itemsize == 2 else "%d"
        raise AssertionError("%s: %d values differ; first at (y=%d, x=%d, channel %d): got %s, model %s"
                             % (what, int(bad.sum()), y, x, c, fmt % got[y, x, c], fmt % want[y, x, c]))


# ---- content classes ------------------------------------------------------------------------------------------------------
# Each returns a [h, w, 4] float16 image (alpha = random halves, so PASSTHROUGH_ALPHA is visible); seeded.
def _rng(seed, tag):
    return np.random.default_rng([seed, sum(map(ord, tag))])


def _with_alpha(rgb, rng):
    h, w = rgb.shape[:2]
    a = rng.random((h, w, 1), np.float32)
    return np.concatenate([rgb.astype(np.float32), a], axis=2).astype(np.float16)


def content_uniform(w, h, seed):
    return F.to_half(F.uniform(w, h, seed))


def content_structured(w, h, seed):
    return F.to_half(F.structured(w, h, seed))


def content_flat(w, h, seed):
    """Flat 3x3 and 4x4 blocks of one colour, many of them grey or sharing a luma with a neighbour: exact luma ties, the 0/0
    of the length term (ffx_fsr1.h:298)."""
    rng = _rng(seed, "flat")
    pal = rng.integers(0, 5, size=(16, 3)) / np.float32(4.0)
    pal[:4] = pal[:4, :1]                                            # greys
    y, x = np.mgrid[0:h, 0:w]
    idx = ((x // 3) * 7 + (y // 4) * 3 + ((x // 3 + y // 4) % 2) * 5) % 16
    idx[(x // 8 + y // 8) % 3 == 0] = 1                              # larger flat regions
    return _with_alpha(pal[idx], rng)


def content_near_flat(w, h, seed):
    """Gradients of one or two half ulps around a flat level: the blended direction lands on both sides of dirR < 1/32768."""
    rng = _rng(seed, "nearflat")
    base = np.float16(rng.choice([0.25, 0.5, 0.75, 1.0]))
    bits = np.full((h, w, 3), base.view(np.uint16), np.int32)
    y, x = np.mgrid[0:h, 0:w]
    step = rng.integers(0, 3, size=(h, w))
    ramp = ((x * step[0, 0] + y) // 3) % 3 + ((x // 5 + y // 7) % 2)  # 0..3 ulps, piecewise
    bits += ramp[..., None] * np.array([1, 1, 1]) + rng.integers(-1, 2, size=(h, w, 3)) * (rng.random((h, w, 1)) < 0.2)
    rgb = bits.astype(np.uint16).view(np.float16).astype(np.float32)
    return _with_alpha(rgb, rng)


def content_subnormal(w, h, seed):
    """Half subnormals of either sign, +0 and -0."""
    rng = _rng(seed, "subnormal")
    bits = rng.integers(0, 0x400, size=(h, w, 3)).astype(np.uint16)
    bits[rng.random((h, w, 3)) < 0.3] = 0
    bits |= (rng.random((h, w, 3)) < 0.5).astype(np.uint16) << 15
    out = _with_alpha(np.zeros((h, w, 3), np.float32), rng)
    out.view(np.uint16)[..., :3] = bits
    return out


def content_signed_zero(w, h, seed):
    """Blocks of +0 and -0 beside small positive and negative values: which zero min / max and the products return."""
    rng = _rng(seed, "zero")
    y, x = np.mgrid[0:h, 0:w]
    bits = np.where(((x // 2 + y // 3) % 3 == 0)[..., None], 0x8000, 0).astype(np.uint16) * np.ones(3, np.uint16)
    pick = rng.random((h, w, 3))
    bits[pick < 0.1] = np.float16(0.25).view(np.uint16)
    bits[(pick >= 0.1) & (pick < 0.2)] = np.float16(-0.25).view(np.uint16)
    out = _with_alpha(np.zeros((h, w, 3), np.float32), rng)
    out.view(np.uint16)[..., :3] = bits
    return out


def content_negative(w, h, seed):
    rng = _rng(seed, "negative")
    return _with_alpha(rng.uniform(-1.0, 1.0, size=(h, w, 3)).astype(np.float32), rng)


def content_hdr(w, h, seed):
    """Linear HDR up to 1024, and 4x4 blocks of 65504 where the half accumulators overflow (inf, inf - inf = NaN) and the
    de-ringing min / max resolve them."""
    rng = _rng(seed, "hdr")
    v = np.exp2(rng.uniform(-8.0, 10.0, size=(h, w, 3))).astype(np.float32)
    y, x = np.mgrid[0:h, 0:w]
    v[((x // 4) * 3 + (y // 4) * 5) % 11 == 0] = 65504.0
    return _with_alpha(v, rng)


def content_luma_rounding(w, h, seed):
    """G = 2048 and R, B below the fp32 ulp there (2^-12), swapped between neighbours: each luma 0.5 B + (0.5 R + G) rounds twice,
    so neighbours whose exact lumas tie differ by an ulp one way or the other, and the order of the two FMAs decides the
    direction EASU sees."""
    rng = _rng(seed, "luma")
    small = rng.integers(1, 16, size=(h, w, 2)) * np.float32(2.0 ** -15)
    swap = rng.random((h, w)) < 0.5
    r, b = np.where(swap, small[..., 1], small[..., 0]), np.where(swap, small[..., 0], small[..., 1])
    return _with_alpha(np.stack([r, np.full((h, w), 2048.0, np.float32), b], axis=2), rng)


def content_bright_spikes(w, h, seed):
    """Values in [0, 1] with single texels of 16000 (2 luma = 32000, still finite) in odd columns: the RCAS noise-measure range of
    the even pixel to a spike's right exceeds 0x778d as half bits, while that of the odd pixel next to it stays small.  The two
    pixels share a lane of the packed kernels, so a magic subtract that borrowed across lanes would change the odd pixel."""
    rng = _rng(seed, "spikes")
    v = rng.random((h, w, 3), np.float32)
    y, x = np.mgrid[0:h, 0:w]
    v[(x % 4 == 1) & ((y + x // 4) % 3 == 0)] = 16000.0
    return _with_alpha(v, rng)


CONTENT = {"uniform": content_uniform, "structured": content_structured, "flat": content_flat, "near_flat": content_near_flat,
           "subnormal": content_subnormal, "signed_zero": content_signed_zero, "negative": content_negative, "hdr": content_hdr,
           "luma_rounding": content_luma_rounding, "bright_spikes": content_bright_spikes}


def content(kind, w, h, seed=1):
    return CONTENT[kind](w, h, seed)


def codes_all(w, h, seed):
    """R8G8B8A8: every code 0..255 in every channel, shuffled in 2x2 blocks."""
    rng = _rng(seed, "codes")
    n = w * h
    c = np.stack([rng.permutation(np.resize(np.arange(256), n)) for _ in range(4)], axis=1).reshape(h, w, 4)
    return c.astype(np.uint8)


def codes_alternating(w, h, seed):
    """R8G8B8A8: 0 / 255 alternating per pixel (one channel per row offset), the strongest edges the format has."""
    y, x = np.mgrid[0:h, 0:w]
    c = np.stack([((x + y) % 2) * 255, ((x // 2 + y) % 2) * 255, (x % 2) * 255, ((x + y) % 3) * 120], axis=2)
    return c.astype(np.uint8)


CODES = {"uniform": lambda w, h, s: np.floor(F.uniform(w, h, s) * 255.0 + 0.5).astype(np.uint8), "all_codes": codes_all,
         "alternating": codes_alternating}
