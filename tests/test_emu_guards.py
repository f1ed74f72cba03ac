"""The guard checks of tests/test_gpu_guards.py without a GPU: the device code on the CPU emulator (tests/emu) reading from and
writing into views of larger poisoned buffers.  Each image sits GR rows below the top of its buffer, 16 bytes from the row start,
with guard columns on the right (through the pitch) and guard rows below; every byte outside the image (and every output row outside
[y0, y1)) must keep its poison, and the result must equal the one on a frame allocated alone.  The emulator's TMA zero-fills outside
the tensor, so it cannot see a load from the padding through TMA; its direct loads and all of its stores can."""
import ctypes

import numpy as np
import pytest

import fsr1_b200 as F
import oracle_lib as ol
from test_emu import PROD, emu_easu, emu_easu_pairs, emu_lib, emu_rcas
from easu_checks import viewport_2x
from test_upscale_post import EmuPost, post_lib, reference_chain

P, LL = ctypes.c_void_p, ctypes.c_longlong
GR = 8
POISON = {"nan": 0x7E5A, "big": 0x7BFF}        # RGBA16F: a NaN with a payload, 65504
POISON32 = {"nan": 0x5A5A5A5A, "big": 0xFFFFFFFF}


class Buf:
    """rows x w pixels of `per` elements (uint16: RGBA16F; uint32: one UNORM word) at row GR, byte offset 16 of a poisoned buffer."""

    def __init__(self, rows, w, poison, per=4, dtype=np.uint16, left=16, right=48):
        es = np.dtype(dtype).itemsize
        pitch = -(-(left + w * per * es + right) // 16) * 16
        self.buf = np.full((rows + 2 * GR, pitch // es), (POISON if dtype == np.uint16 else POISON32)[poison], dtype)
        self.rows, self.w, self.per = rows, w, per
        self.c0, self.c1 = left // es, left // es + w * per
        self.before = self.buf.copy()

    def set(self, a):
        self.buf[GR:GR + self.rows, self.c0:self.c1] = np.ascontiguousarray(a).reshape(self.rows, -1)
        self.before = self.buf.copy()

    @property
    def ptr(self):
        return P(self.buf.ctypes.data + GR * self.buf.strides[0] + self.c0 * self.buf.itemsize)

    @property
    def pitch(self):
        return LL(self.buf.strides[0])

    def get(self):
        a = self.buf[GR:GR + self.rows, self.c0:self.c1]
        return a.reshape(self.rows, self.w, self.per) if self.per > 1 else a.copy()

    def assert_untouched(self, what, r0=0, r1=0):
        diff = self.buf != self.before
        diff[GR + r0:GR + r1, self.c0:self.c1] = False
        assert not diff.any(), (what, int(diff.sum()), np.argwhere(diff)[0].tolist())


RCAS_SHAPES = [(61, 17), (63, 15), (65, 5), (125, 9), (2, 3), (1, 2)]


@pytest.mark.parametrize("poison", ["nan", "big"])
@pytest.mark.parametrize("clamp", [0, 1])
def test_emulated_rcas_reads_and_writes_only_its_image(clamp, poison):
    """rcas_packed_kernel (RGBA16F): the checked border path with a right edge inside a pair, in a 60-pixel span, and a row slab whose
    input window holds exactly the apron rows."""
    con = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    for (w, h) in RCAS_SHAPES:
        src = F.to_half(F.uniform(w, h, w + h))
        for (y0, y1) in ((0, h), (1, h - 1) if h > 2 else (0, 1)):
            n0, n1 = max(y0 - 1, 0), min(y1, h - 1)
            gi, go = Buf(n1 - n0 + 1, w, poison), Buf(h, w, poison)
            gi.set(src.view(np.uint16)[n0:n1 + 1])
            assert emu_lib().emu_rcas_h_packed_opt(gi.ptr, n0, n1 - n0 + 1, go.ptr, w, h, gi.pitch, go.pitch, con, clamp, y0, y1, 0) == 0
            what = (w, h, y0, y1, clamp, poison)
            got = go.get()[y0:y1].view(np.float16)
            want = ol.rcas(src.astype(np.float32), ol.rcas_con(0.25), bool(clamp), y0=y0, y1=y1)[y0:y1]
            d = np.abs(got.astype(np.float32) - want)[..., :3]
            assert not np.isnan(d).any() and d.max() <= 4e-3, what
            gi.assert_untouched(what + ("input",))
            go.assert_untouched(what + ("output",), y0, y1)


@pytest.mark.parametrize("poison", ["nan", "big"])
def test_emulated_unorm_and_fp32_rcas_write_only_their_image(poison):
    """rcas_u_packed_kernel (4-byte pixel pairs) and rcas_f32_packed_kernel (two 16-byte stores) at odd widths."""
    con = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    for (w, h) in ((61, 17), (65, 5), (1, 2)):
        raw = np.floor(F.uniform(w, h, 3) * 255.0 + 0.5).astype(np.uint32)
        words = raw[..., 0] | (raw[..., 1] << 8) | (raw[..., 2] << 16) | (raw[..., 3] << 24)
        gi, go = Buf(h, w, poison, 1, np.uint32), Buf(h, w, poison, 1, np.uint32)
        gi.set(words)
        assert emu_lib().emu_rcas_u_packed(8, gi.ptr, go.ptr, w, h, gi.pitch, go.pitch, con, 0, 0, h) == 0
        plain_out = np.zeros((h, w), np.uint32)
        emu_lib().emu_rcas_u_packed(8, P(words.ctypes.data), P(plain_out.ctypes.data), w, h, LL(w * 4), LL(w * 4), con, 0, 0, h)
        assert np.array_equal(go.get(), plain_out), (w, h)
        gi.assert_untouched((w, h, "u8 input"))
        go.assert_untouched((w, h, "u8 output"), 0, h)
        src = np.ascontiguousarray(F.uniform(w, h, 4))
        gi, go = Buf(h, w, poison, 8), Buf(h, w, poison, 8)              # float32 pixels as pairs of uint16 words
        gi.set(src.view(np.uint16))
        assert emu_lib().emu_rcas_f32_packed(1, gi.ptr, go.ptr, w, h, gi.pitch, go.pitch, con, 0, 0, h) == 0
        got = np.ascontiguousarray(go.get()).view(np.float32)
        assert np.abs(got - ol.rcas(src, ol.rcas_con(0.25)))[..., :3].max() <= 1e-5, (w, h)
        gi.assert_untouched((w, h, "f32 input"))
        go.assert_untouched((w, h, "f32 output"), 0, h)


def _quad_con(iw, ih, ow, oh):
    """The 2x constants for odd outputs too: a viewport of (about) half the output."""
    con_of = lambda v, n: ol.easu_con(n, n, n, n, vw=v, vh=v)
    return ol.easu_con(iw, ih, ow, oh, vw=viewport_2x(ow, con_of), vh=viewport_2x(oh, con_of))


FUSED_SHAPES = [(61, 17), (63, 15), (125, 9), (124, 33), (2, 2), (1, 1)]


@pytest.mark.parametrize("poison", ["nan", "big"])
def test_emulated_fused_kernel_writes_only_its_image(poison):
    """fused_h_quad2x_kernel at odd output widths (the last pair of a strip half outside), 62-pixel strip ends and a row slab: the
    two-kernel result, bit for bit, and nothing outside the output rows [y0, y1)."""
    rcon = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    for (ow, oh) in FUSED_SHAPES:
        iw, ih = (ow + 1) // 2, (oh + 1) // 2
        src = F.to_half(F.uniform(iw, ih, ow + oh))
        want = emu_rcas(emu_easu(PROD, src, ow, oh, con=_quad_con(iw, ih, ow, oh)), 0.25).view(np.uint16)
        for (y0, y1) in ((0, oh), (1, oh - 1) if oh > 2 else (0, 1)):
            gi, go = Buf(ih, iw, poison), Buf(oh, ow, poison)
            gi.set(src.view(np.uint16))
            assert emu_lib().emu_fused_h(gi.ptr, iw, ih, gi.pitch, go.ptr, ow, oh, go.pitch, rcon, y0, y1, 3) == 0
            what = (ow, oh, y0, y1, poison)
            assert np.array_equal(go.get()[y0:y1], want[y0:y1]), what
            gi.assert_untouched(what + ("input",))
            go.assert_untouched(what + ("output",), y0, y1)


@pytest.mark.parametrize("poison", ["nan", "big"])
def test_emulated_vertical_pair_easu_writes_only_its_image(poison):
    """easu_h_pairs_kernel: a lane stores the vertical pair (oy, oy + 1); the second row of the last pair of an odd row range is not
    the caller's."""
    for (iw, ih, ow, oh) in ((40, 11, 61, 17), (50, 10, 65, 15), (2, 1, 3, 1)):
        con = ol.easu_con(iw, ih, ow, oh)
        src = F.to_half(F.uniform(iw, ih, 6))
        full = emu_easu_pairs(src, ow, oh).view(np.uint16)
        for (y0, y1) in ((0, oh), (1, oh) if oh > 1 else (0, 1)):
            gi, go = Buf(ih, iw, poison), Buf(oh, ow, poison)
            gi.set(src.view(np.uint16))
            assert emu_lib().emu_easu_h_pairs(1, gi.ptr, iw, ih, gi.pitch, go.ptr, ow, oh, go.pitch, (ctypes.c_uint32 * 16)(*con),
                                              y0, y1, 2) == 0
            what = (ow, oh, y0, y1, poison)
            assert np.array_equal(go.get()[y0:y1], full[y0:y1]), what
            gi.assert_untouched(what + ("input",))
            go.assert_untouched(what + ("output",), y0, y1)


def _post_tiles(poison):
    """A 5 x 3 RGBA16F grain tile and a 7 x 3 RGBA16F dither tile (odd widths: a pixel pair wraps inside the tile), guarded."""
    rng = np.random.default_rng(5)
    grain = (rng.random((3, 5, 4), np.float32) - 0.5).astype(np.float16)
    dither = (rng.random((3, 7, 4), np.float32) * 1.2 - 0.1).astype(np.float16)
    gg, gd = Buf(3, 5, poison), Buf(3, 7, poison)
    gg.set(grain.view(np.uint16))
    gd.set(dither.view(np.uint16))
    return grain, dither, gg, gd


def _emu_post(ops, gg, gd):
    return EmuPost(ops, 0.375, 5, gg.ptr.value, 5, 3, gg.pitch.value, 1, gd.ptr.value if gd else None, 7, 3,
                   gd.pitch.value if gd else 0, 1)


POST_CASES = [(1 | 2, 1), (2 | 4, 3), (1 | 2 | 8, 4)]      # (FSR1_POST_* ops, output format: 1 RGBA16F, 3 RGBA8, 4 RGB10A2)


@pytest.mark.parametrize("poison", ["nan", "big"])
@pytest.mark.parametrize("ops,out_format", POST_CASES)
def test_emulated_post_epilogues_read_only_their_tiles_and_write_only_their_image(ops, out_format, poison):
    """Both epilogues of fsr1_upscale_post (fused_h_quad2x_post_kernel, rcas_post_kernel) with guarded grain and dither tiles: the pass
    sequence on the same RCAS output, bit for bit, and no byte of a tile's padding or of the output's guards used or written."""
    grain, dither, gg, gd = _post_tiles(poison)
    use_dither = bool(ops & (4 | 8))
    per, dt = (4, np.uint16) if out_format == 1 else (1, np.uint32)
    rcon = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    for (ow, oh) in ((61, 17), (63, 9), (1, 2)):
        iw, ih = (ow + 1) // 2, (oh + 1) // 2
        src = F.to_half(F.structured(iw, ih, ow))
        y0, y1 = (1, oh - 1) if oh > 2 else (0, oh)
        # the fused epilogue
        plain = emu_rcas(emu_easu(PROD, src, ow, oh, con=_quad_con(iw, ih, ow, oh)), 0.25)
        want = reference_chain(plain, ops, grain, 0.375, dither if use_dither else None, 5, out_format)
        gi, go = Buf(ih, iw, poison), Buf(oh, ow, poison, per, dt)
        gi.set(src.view(np.uint16))
        post = _emu_post(ops, gg, gd if use_dither else None)
        assert post_lib().emu_fused_h_post(gi.ptr, iw, ih, gi.pitch, go.ptr, ow, oh, go.pitch, out_format, rcon, y0, y1, 3,
                                           ctypes.byref(post)) == 0
        what = ("fused", ow, oh, ops, out_format, poison)
        assert np.array_equal(go.get()[y0:y1], want[y0:y1]), what
        for g, name in ((gi, "input"), (gg, "grain"), (gd, "dither")):
            g.assert_untouched(what + (name,))
        go.assert_untouched(what + ("output",), y0, y1)
        # the RCAS epilogue, on an RGBA16F image of the output size
        img = F.to_half(F.structured(ow, oh, oh))
        want = reference_chain(emu_rcas(img, 0.25, False, y0, y1), ops, grain, 0.375, dither if use_dither else None, 5, out_format)
        n0, n1 = max(y0 - 1, 0), min(y1, oh - 1)
        gi, go = Buf(oh, ow, poison), Buf(oh, ow, poison, per, dt)
        gi.set(img.view(np.uint16))
        assert post_lib().emu_rcas_h_packed_post(gi.ptr, go.ptr, ow, oh, gi.pitch, go.pitch, out_format, rcon, 0, y0, y1, 0,
                                                 ctypes.byref(post)) == 0
        what = ("rcas", ow, oh, ops, out_format, poison, n0, n1)
        assert np.array_equal(go.get()[y0:y1], want[y0:y1]), what
        for g, name in ((gi, "input"), (gg, "grain"), (gd, "dither")):
            g.assert_untouched(what + (name,))
        go.assert_untouched(what + ("output",), y0, y1)


@pytest.mark.parametrize("poison", ["nan", "big"])
def test_emulated_hx2_kernels_read_and_write_only_their_images(poison):
    """rcas_hx2_kernel (both out-of-image rules, a row-slab window) and pointwise_hx2_kernel (LFGA with a guarded 5-wide grain tile,
    TEPD with a guarded dither tile) at widths that end inside a 16-pixel lane strip: bit for bit the half oracle."""
    con = ol.rcas_con(0.25)
    grain, dither, gg, gd = _post_tiles(poison)
    for (w, h) in ((37, 9), (5, 4), (1, 2)):
        img = F.to_half(F.uniform(w, h, 9 + w))
        for clamp in (0, 1):
            y0, y1 = (1, h - 1) if h > 2 else (0, h)
            n0, n1 = max(y0 - 1, 0), min(y1, h - 1)
            gi, go = Buf(n1 - n0 + 1, w, poison), Buf(h, w, poison)
            gi.set(img.view(np.uint16)[n0:n1 + 1])
            assert emu_lib().emu_rcas_hx2(gi.ptr, n0, n1 - n0 + 1, go.ptr, w, h, gi.pitch, go.pitch, (ctypes.c_uint32 * 4)(*con), clamp,
                                          y0, y1, 0) == 0
            what = ("rcas_hx2", w, h, clamp, poison)
            assert np.array_equal(go.get()[y0:y1], ol.rcas(img, con, bool(clamp), y0=y0, y1=y1).view(np.uint16)[y0:y1]), what
            gi.assert_untouched(what + ("input",))
            go.assert_untouched(what + ("output",), y0, y1)
        for op, aux, want in ((3, gg, ol.lfga_h(img, grain, 0.375)), (4, gd, ol.tepd_h(img, 8, dither=dither)), (2, None, None)):
            gi, go = Buf(h, w, poison), Buf(h, w, poison)
            gi.set(img.view(np.uint16))
            args = (aux.ptr, aux.w, aux.rows, aux.pitch) if aux else (P(0), 0, 0, LL(0))
            assert emu_lib().emu_pointwise_hx2(op, gi.ptr, gi.pitch, go.ptr, go.pitch, w, h, *args, ctypes.c_float(0.375),
                                               ctypes.c_uint32(0), 0, h) == 0
            what = ("pointwise_hx2", op, w, h, poison)
            if want is not None:
                assert np.array_equal(go.get(), want.view(np.uint16)), what
            gi.assert_untouched(what + ("input",))
            go.assert_untouched(what + ("output",), 0, h)
            gg.assert_untouched(what + ("grain",))
            gd.assert_untouched(what + ("dither",))
