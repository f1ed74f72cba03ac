"""Checks of EASU results that hold for every kernel family, at any scale, viewport or offset.

expected_easu_kernel(): which kernel family the launchers pick (csrc/fsr1_capi.cu fsr1_easu), stated from the constant block
and the flags alone, so that a test does not guess it from image sizes ("twice the width" is not always exactly 2x in fp32).

assert_within_cell_bounds(): the de-ringing clamp.  Every EASU output lies within [min, max] of the 2x2 texels f, g, j, k of
its cell, because every kernel clamps its result to the min/max of the stored texel values.  The bound has no tolerance: a
wrong cell, a wrong clamp at the image border or a read outside the image fails it."""
import numpy as np

from fsr1_b200 import _lib as L

_QUAD_2X = [0x3F000000, 0x3F000000, 0xBE800000, 0xBE800000]        # con0 = {0.5, 0.5, -0.25, -0.25}


def _f(word):
    return np.array([word], np.uint32).view(np.float32)[0]


def expected_easu_kernel(con, fmt, flags=0):
    """Name prefix of the EASU kernel for a 16-byte aligned image of format `fmt` with these constants and flags."""
    if flags & L.FLAG_H_REFERENCE:
        return "easu_href"
    if flags & (L.FLAG_EXACT | L.FLAG_FORCE_DIRECT):
        return "easu_direct"
    quad = list(con[:4]) == _QUAD_2X
    c0x, c0y = _f(con[0]), _f(con[1])
    any_scale = 0.0 < c0x <= 1.0 and 0.0 < c0y <= 1.0
    if fmt == L.FORMAT_RGBA16F:
        if flags & L.FLAG_PRECISE and (quad or any_scale):
            return "easu_h16io_f32math_quad2x" if quad else "easu_h16io_f32math_vpairs"
        return "easu_h_quad2x" if quad else "easu_h_vpairs" if any_scale else "easu_direct"
    if fmt == L.FORMAT_RGBA32F:
        return "easu_f32_quad2x" if quad else "easu_f32_vpairs" if any_scale else "easu_direct"
    if fmt == L.FORMAT_RGBA8_UNORM and quad and not flags & L.FLAG_PRECISE:
        return "easu_u8_quad2x"
    return "easu_direct"


def viewport_2x(n, con_of):
    """A viewport for an output n pixels long whose constants are exactly 2x: n / 2, or the float32 nearest to it for which
    FsrEasuCon's n / 2 * rcp(n) rounds to 0.5 (for n = 61 it gives 0.49999997), so that odd outputs take the 2x kernels.
    con_of(v, n): the constant block of a v x v viewport scaled to n x n."""
    up = dn = np.float32(n / 2.0)
    for _ in range(16):
        for v in (up, dn):
            if con_of(float(v), n)[:4:2] == _QUAD_2X[:4:2]:
                return float(v)
        up, dn = np.nextafter(up, np.float32(np.inf)), np.nextafter(dn, np.float32(0))
    raise AssertionError("no exact 2x viewport for %d" % n)


def cells(n_out, scale_word, offset_word):
    """Cell index of each output pixel along one axis, in the fp32 arithmetic of host_cell (csrc/fsr1_capi.cu): one rounding
    per operation, no fused multiply-add."""
    m = np.arange(n_out).astype(np.float32) * _f(scale_word)
    return np.floor(m + _f(offset_word)).astype(np.int64)


def assert_within_cell_bounds(out, src, con, y0=0, y1=None, what=""):
    """Every RGB value of output rows [y0, y1) lies within [min, max] of its cell's texels f, g, j, k (clamped to `src`).
    `out` and `src` are [H, W, 4] arrays of the stored type: float16, float32, or uint8 code values for R8G8B8A8."""
    ih, iw = src.shape[:2]
    oh, ow = out.shape[:2]
    y1 = oh if y1 is None else y1
    fx = cells(ow, con[0], con[2])
    fy = cells(oh, con[1], con[3])[y0:y1]
    x0, x1 = np.clip(fx, 0, iw - 1), np.clip(fx + 1, 0, iw - 1)
    r0, r1 = np.clip(fy, 0, ih - 1), np.clip(fy + 1, 0, ih - 1)
    rgb = src[..., :3]
    lo = hi = None
    for r in (r0, r1):
        rows = rgb[r]
        for c in (x0, x1):
            t = rows[:, c]
            lo = t if lo is None else np.minimum(lo, t)
            hi = t if hi is None else np.maximum(hi, t)
    g = out[y0:y1, :, :3]
    bad = (g < lo) | (g > hi)
    if bad.any():
        y, x, ch = np.argwhere(bad)[0]
        raise AssertionError("%s: %d values outside their cell's texel range; first at output (%d, %d) channel %d: %r not in [%r, %r]"
                             % (what, int(bad.sum()), y0 + y, x, ch, g[y, x, ch], lo[y, x, ch], hi[y, x, ch]))
