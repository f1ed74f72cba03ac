"""The device code of csrc/fsr1_easu_tiled.cu, csrc/fsr1_rcas_packed.cu and csrc/fsr1_rcas_f32.cu compiled for the HOST (tests/emu: one OS
thread per CUDA thread, emulated TMA / mbarrier / half arithmetic) and checked against the oracle — kernel logic can be debugged
without a GPU: tiling, clamp-to-edge fix-up, persistent tile loop, row ranges, image borders, both out-of-image rules.
The GPU remains the authority on the hardware (tests/test_gpu_parity.py); this is a second, cheaper net."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import fsr1_b200 as F
import oracle_lib as ol
from easu_checks import assert_within_cell_bounds

PROD = 12   # the production 2x kernel's number in the emulator harness (emu_easu.cpp)
EMU_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu")
_lib = None


def emu_lib():
    global _lib
    if _lib is None:
        subprocess.check_call(["make", "-s", "-C", EMU_DIR, "libfsr1_emu.so"])
        _lib = ctypes.CDLL(os.path.join(EMU_DIR, "libfsr1_emu.so"))
    return _lib


def emu_easu(variant, src_h, ow, oh, y0=0, y1=None, ctas=3, con=None):
    ih, iw = src_h.shape[:2]
    y1 = oh if y1 is None else y1
    con = (ctypes.c_uint32 * 16)(*(con or ol.easu_con(iw, ih, ow, oh)))
    src = np.ascontiguousarray(src_h.view(np.uint16))
    out = np.zeros((oh, ow, 4), np.uint16)
    rc = emu_lib().emu_easu_h_quad2x(variant, ctypes.c_void_p(src.ctypes.data), iw, ih, ctypes.c_longlong(src.strides[0]),
                                     ctypes.c_void_p(out.ctypes.data), ow, oh, ctypes.c_longlong(out.strides[0]), con, y0, y1, ctas)
    assert rc == 0
    return out.view(np.float16)


@pytest.mark.parametrize("size", [(64, 36), (70, 23), (33, 17), (5, 3)])
@pytest.mark.parametrize("gen", ["uniform", "structured"])
def test_emulated_production_kernel_within_fp16_tolerance(size, gen):
    iw, ih = size
    ow, oh = 2 * iw, 2 * ih
    src = F.to_half(getattr(F, gen)(iw, ih, 31))
    want = ol.easu(src.astype(np.float32), ow, oh)
    got = emu_easu(PROD, src, ow, oh)
    assert np.abs(got.astype(np.float32) - want)[..., :3].max() <= 5e-3       # GPU tolerance is 1e-2; measured there <= 2.8e-3
    assert (got[..., 3] == np.float16(1.0)).all()
    # one CTA or many, same result (persistent tile loop, double buffering)
    assert np.array_equal(emu_easu(PROD, src, ow, oh, ctas=1).view(np.uint16), got.view(np.uint16))


def test_emulated_row_range_only_touches_its_rows():
    iw, ih, ow, oh = 64, 36, 128, 72
    src = F.to_half(F.uniform(iw, ih, 5))
    full = emu_easu(PROD, src, ow, oh)
    part = emu_easu(PROD, src, ow, oh, y0=19, y1=53)
    assert np.array_equal(part[19:53].view(np.uint16), full[19:53].view(np.uint16))
    assert not part[:19].view(np.uint16).any() and not part[53:].view(np.uint16).any()


def emu_easu_pairs(src_h, ow, oh, y0=0, y1=None, ctas=2, variant=1, con=None):
    ih, iw = src_h.shape[:2]
    y1 = oh if y1 is None else y1
    con = (ctypes.c_uint32 * 16)(*(con or ol.easu_con(iw, ih, ow, oh)))
    src = np.ascontiguousarray(src_h.view(np.uint16))
    out = np.zeros((oh, ow, 4), np.uint16)
    rc = emu_lib().emu_easu_h_pairs(variant, ctypes.c_void_p(src.ctypes.data), iw, ih, ctypes.c_longlong(src.strides[0]),
                                    ctypes.c_void_p(out.ctypes.data), ow, oh, ctypes.c_longlong(out.strides[0]), con, y0, y1, ctas)
    assert rc == 0
    return out.view(np.float16)


@pytest.mark.parametrize("shape", [(96, 54, 144, 81), (96, 54, 125, 70), (64, 64, 64, 64), (50, 20, 65, 26), (33, 17, 57, 31),
                                   (64, 36, 128, 72), (96, 54, 192, 81)])
@pytest.mark.parametrize("gen", ["uniform", "structured"])
def test_emulated_any_scale_kernel_within_fp16_tolerance(shape, gen, variant=1):
    """easu_h_pairs_kernel (1.5x, 1.3x, 1x, ragged sizes, 2x through the generic path, x2.0/y1.5): vertical pixel pairs
    sharing or not sharing an input cell row, box footprints computed per launch, even-aligned box origins."""
    iw, ih, ow, oh = shape
    src = F.to_half(getattr(F, gen)(iw, ih, 31))
    want = ol.easu(src.astype(np.float32), ow, oh)
    got = emu_easu_pairs(src, ow, oh, variant=variant)
    assert np.abs(got.astype(np.float32) - want)[..., :3].max() <= 5e-3
    y0, y1 = oh // 3, 2 * oh // 3 + 1
    part = emu_easu_pairs(src, ow, oh, y0=y0, y1=y1, ctas=1, variant=variant)
    assert np.array_equal(part[y0:y1].view(np.uint16), got[y0:y1].view(np.uint16))
    assert not part[:y0].view(np.uint16).any() and not part[y1:].view(np.uint16).any()


def emu_rcas(src_h, sharp, clamp=False, y0=0, y1=None):
    h, w = src_h.shape[:2]
    y1 = h if y1 is None else y1
    con = (ctypes.c_uint32 * 4)(*ol.rcas_con(sharp))
    src = np.ascontiguousarray(src_h.view(np.uint16))
    out = np.zeros((h, w, 4), np.uint16)
    rc = emu_lib().emu_rcas_h_packed(ctypes.c_void_p(src.ctypes.data), ctypes.c_void_p(out.ctypes.data), w, h,
                                     ctypes.c_longlong(src.strides[0]), ctypes.c_longlong(out.strides[0]), con, 1 if clamp else 0, y0, y1)
    assert rc == 0
    return out.view(np.float16)


@pytest.mark.parametrize("size", [(128, 72), (61, 19), (200, 33), (6, 5)])
@pytest.mark.parametrize("clamp", [False, True])
def test_emulated_rcas_kernel_within_fp16_tolerance(size, clamp):
    """rcas_h_packed_kernel: two pixels per lane, neighbours by warp shuffle, 60-pixel spans overlapping by 4, the unchecked
    interior path and the checked border path, out-of-image taps reading 0 or clamped."""
    w, h = size
    for gen in (F.uniform, F.structured):
        src = F.to_half(gen(w, h, 9))
        for sharp in (0.0, 0.25, 2.0):
            want = ol.rcas(src.astype(np.float32), ol.rcas_con(sharp), clamp)
            got = emu_rcas(src, sharp, clamp)
            assert np.abs(got.astype(np.float32) - want)[..., :3].max() <= 4e-3, (gen.__name__, sharp)
    y0, y1 = h // 3, 2 * h // 3 + 1
    part = emu_rcas(src, 0.25, clamp, y0=y0, y1=y1)
    full = emu_rcas(src, 0.25, clamp)
    assert np.array_equal(part[y0:y1].view(np.uint16), full[y0:y1].view(np.uint16))
    assert not part[:y0].view(np.uint16).any() and not part[y1:].view(np.uint16).any()


def _quantise(x, bits):
    s = np.float32((1 << bits) - 1)
    return (np.clip(x, 0.0, 1.0).astype(np.float32) * s + np.float32(0.5)).astype(np.uint32)


def _pack_unorm(q, bits):
    if bits == 8:
        return (q[..., 0] | (q[..., 1] << 8) | (q[..., 2] << 16) | (q[..., 3] << 24)).astype(np.uint32)
    return (q[..., 0] | (q[..., 1] << 10) | (q[..., 2] << 20) | (q[..., 3] << 30)).astype(np.uint32)


def _unpack_unorm(w, bits):
    if bits == 8:
        return np.stack([w & 255, (w >> 8) & 255, (w >> 16) & 255, w >> 24], axis=-1)
    return np.stack([w & 1023, (w >> 10) & 1023, (w >> 20) & 1023, w >> 30], axis=-1)


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("size", [(64, 36), (70, 23), (33, 17)])
def test_emulated_unorm_2x_easu_within_one_code(bits, size):
    """easu_u_quad2x_kernel (prepared, FSR1_UNORM_TILED=1): TMA box of 4-byte texels, decode to the half tile + fp32 luma,
    half-domain re-encode.  Against quantise(oracle(dequantise(input))): at most one code value off, and rarely."""
    iw, ih = size
    ow, oh = 2 * iw, 2 * ih
    rng = np.random.default_rng(3)
    top = (1 << bits) - 1
    for kind in ("noise", "smooth"):
        if kind == "noise":
            raw = rng.integers(0, top + 1, size=(ih, iw, 4), dtype=np.uint32)
        else:
            raw = _quantise(F.structured(iw, ih, 12), bits)
        raw[..., 3] = rng.integers(0, 4 if bits == 10 else 256, size=(ih, iw))
        fin = (raw.astype(np.float32) / np.float32(top)).astype(np.float32)
        want = _quantise(ol.easu(fin, ow, oh)[..., :3], bits)
        src = np.ascontiguousarray(_pack_unorm(raw, bits))
        out = np.zeros((oh, ow), np.uint32)
        con = (ctypes.c_uint32 * 16)(*ol.easu_con(iw, ih, ow, oh))
        rc = emu_lib().emu_easu_u_quad2x(bits, ctypes.c_void_p(src.ctypes.data), iw, ih, ctypes.c_longlong(src.strides[0]),
                                         ctypes.c_void_p(out.ctypes.data), ow, oh, ctypes.c_longlong(out.strides[0]), con, 0, oh, 3)
        assert rc == 0
        got = _unpack_unorm(out, bits)
        diff = np.abs(got[..., :3].astype(np.int64) - want.astype(np.int64))
        assert diff.max() <= (1 if bits == 8 else 3), (kind, int(diff.max()))     # 10-bit codes are finer than half's 11-bit mantissa
        assert (diff > 0).mean() < (0.10 if bits == 8 else 0.6), (kind, float((diff > 0).mean()))
        assert (got[..., 3] == (255 if bits == 8 else 3)).all()


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("clamp", [False, True])
def test_emulated_unorm_rcas_within_one_code(bits, clamp):
    """rcas_u_packed_kernel (prepared, FSR1_UNORM_TILED=1): decode two 4-byte pixels per lane, the half2 RCAS arithmetic of the
    production kernel, saturate, re-encode.  Against quantise(oracle(dequantise(input)))."""
    rng = np.random.default_rng(4)
    top = (1 << bits) - 1
    for (w, h) in ((128, 40), (61, 19), (6, 5)):
        for kind in ("noise", "smooth"):
            raw = rng.integers(0, top + 1, size=(h, w, 4), dtype=np.uint32) if kind == "noise" else _quantise(F.structured(w, h, 12), bits)
            raw[..., 3] = 3 if bits == 10 else 255
            fin = (raw.astype(np.float32) / np.float32(top)).astype(np.float32)
            src = np.ascontiguousarray(_pack_unorm(raw, bits))
            for sharp in (0.0, 0.25):
                want = _quantise(ol.rcas(fin, ol.rcas_con(sharp), clamp)[..., :3], bits)
                out = np.zeros((h, w), np.uint32)
                con = (ctypes.c_uint32 * 4)(*ol.rcas_con(sharp))
                rc = emu_lib().emu_rcas_u_packed(bits, ctypes.c_void_p(src.ctypes.data), ctypes.c_void_p(out.ctypes.data), w, h,
                                                 ctypes.c_longlong(src.strides[0]), ctypes.c_longlong(out.strides[0]), con,
                                                 1 if clamp else 0, 0, h)
                assert rc == 0
                got = _unpack_unorm(out, bits)
                diff = np.abs(got[..., :3].astype(np.int64) - want.astype(np.int64))
                assert diff.max() <= (1 if bits == 8 else 4), (w, h, kind, sharp, int(diff.max()))
                assert (got[..., 3] == (255 if bits == 8 else 3)).all()


def test_emulated_fp32_rcas_within_1e5(variant=1):
    """rcas_f32_packed_kernel (MUFU reciprocals): the fp32 fast path is held to
    1e-5 of the oracle (contraction reorders roundings; bit-exactness is FSR1_FLAG_EXACT's job)."""
    for (w, h) in ((128, 40), (61, 19), (6, 5)):
        for gen in (F.uniform, F.structured):
            src = np.ascontiguousarray(gen(w, h, 9))
            for clamp in (False, True):
                for sharp in (0.0, 0.25, 2.0):
                    con = (ctypes.c_uint32 * 4)(*ol.rcas_con(sharp))
                    out = np.zeros_like(src)
                    rc = emu_lib().emu_rcas_f32_packed(variant, ctypes.c_void_p(src.ctypes.data), ctypes.c_void_p(out.ctypes.data), w, h,
                                                       ctypes.c_longlong(src.strides[0]), ctypes.c_longlong(out.strides[0]), con,
                                                       1 if clamp else 0, 0, h)
                    assert rc == 0
                    want = ol.rcas(src, ol.rcas_con(sharp), clamp)
                    assert np.abs(out - want)[..., :3].max() <= 1e-5



def test_emulated_rcas_row_window_never_reads_past_the_stored_rows():
    """A row-slab window whose height is not a multiple of the 4 rows a lane walks (the default 8-GPU split: 270 rows per slab):
    the last partial chunk requests its rows up front and must not touch memory beyond the rows the window is required to
    hold (y1 included, y1+1.. not).  The window is placed so that it ENDS at a PROT_NONE guard page: a stray read faults."""
    import mmap
    libc = ctypes.CDLL(None, use_errno=True)
    libc.mprotect.argtypes = [ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int]
    w, h = 128, 40
    full = F.to_half(F.uniform(w, h, 21))
    pitch = w * 8
    page = mmap.PAGESIZE
    for (y0, y1) in ((0, 6), (8, 18), (3, 13)):
        need0, need1 = max(y0 - 1, 0), min(y1, h - 1)            # rows RCAS reads (fsr1_rcas's window contract)
        nbytes = (need1 - need0 + 1) * pitch
        total = ((nbytes + page - 1) // page + 1) * page
        buf = mmap.mmap(-1, total)
        base = ctypes.addressof(ctypes.c_char.from_buffer(buf))
        assert libc.mprotect(ctypes.c_void_p(base + total - page), page, 0) == 0        # PROT_NONE guard page
        start = base + total - page - nbytes                                            # window ends exactly at the guard page
        ctypes.memmove(start, np.ascontiguousarray(full[need0:need1 + 1]).ctypes.data, nbytes)
        out = np.zeros((h, w, 4), np.uint16)
        con = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
        rc = emu_lib().emu_rcas_h_packed_win(ctypes.c_void_p(start), need0, need1 - need0 + 1, ctypes.c_void_p(out.ctypes.data), w, h,
                                             ctypes.c_longlong(pitch), ctypes.c_longlong(out.strides[0]), con, 0, y0, y1)
        assert rc == 0
        want = emu_rcas(full, 0.25)
        assert np.array_equal(out[y0:y1], want[y0:y1].view(np.uint16))
        libc.mprotect(ctypes.c_void_p(base + total - page), page, 3)
        del start
        buf.close()


@pytest.mark.parametrize("opts", [1, 2, 3, 4, 5, 6, 7])
def test_emulated_rcas_options_on_the_packed_kernel(opts):
    """FSR_RCAS_DENOISE (bit 0), FSR_RCAS_PASSTHROUGH_ALPHA (bit 1) and the Sample.x output square (bit 2) are template bits of
    the production packed kernel (no fallback to the direct kernel, no extra pass): against the oracle built with the same
    options, RGBA16F and R8G8B8A8."""
    denoise, alpha, square = bool(opts & 1), bool(opts & 2), bool(opts & 4)
    w, h = 128, 40
    for gen in (F.uniform, F.structured):
        src = F.to_half(gen(w, h, 17))
        con = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
        for clamp in (False, True):
            want = ol.rcas(src.astype(np.float32), ol.rcas_con(0.25), clamp, denoise=denoise, alpha=alpha)
            if square:
                want[..., :3] = want[..., :3] * want[..., :3]
            s16 = np.ascontiguousarray(src.view(np.uint16))
            out = np.zeros((h, w, 4), np.uint16)
            rc = emu_lib().emu_rcas_h_packed_opt(ctypes.c_void_p(s16.ctypes.data), 0, h, ctypes.c_void_p(out.ctypes.data), w, h,
                                                 ctypes.c_longlong(s16.strides[0]), ctypes.c_longlong(out.strides[0]), con,
                                                 1 if clamp else 0, 0, h, opts)
            assert rc == 0
            got = out.view(np.float16).astype(np.float32)
            assert np.abs(got - want)[..., :3].max() <= 4e-3, (gen.__name__, clamp)
            if alpha:
                assert np.array_equal(out[..., 3], s16[..., 3])          # the centre pixel's alpha, bit for bit
            else:
                assert (out.view(np.float16)[..., 3] == np.float16(1.0)).all()
        # R8G8B8A8
        raw = _quantise(gen(w, h, 18), 8)
        raw[..., 3] = np.random.default_rng(3).integers(0, 256, size=(h, w))
        fin = (raw.astype(np.float32) / np.float32(255.0)).astype(np.float32)
        want = ol.rcas(fin, ol.rcas_con(0.25), False, denoise=denoise, alpha=alpha)
        if square:
            want[..., :3] = want[..., :3] * want[..., :3]
        wq = _quantise(want[..., :3], 8)
        src8 = np.ascontiguousarray(_pack_unorm(raw, 8))
        out8 = np.zeros_like(src8)
        rc = emu_lib().emu_rcas_u_packed_opt(8, ctypes.c_void_p(src8.ctypes.data), ctypes.c_void_p(out8.ctypes.data), w, h,
                                             ctypes.c_longlong(src8.strides[0]), ctypes.c_longlong(out8.strides[0]), con, 0, 0, h, opts)
        assert rc == 0
        got8 = _unpack_unorm(out8, 8)
        assert np.abs(got8[..., :3].astype(np.int64) - wq.astype(np.int64)).max() <= 1
        assert np.array_equal(got8[..., 3], raw[..., 3] if alpha else np.full((h, w), 255))


@pytest.mark.parametrize("size", [(64, 36), (70, 23), (33, 17), (99, 40), (5, 3)])
@pytest.mark.parametrize("ctas", [1, 3, 7])
def test_emulated_fused_kernel_is_bit_identical_to_the_two_kernel_path(size, ctas):
    """fused_h_quad2x_kernel (EASU -> shared-memory intermediate -> RCAS, column strips, rolling rows): the same bits as
    easu_h_quad2x_kernel followed by rcas_packed_kernel through an fp16 intermediate, for any number of CTAs (run boundaries
    fall anywhere), several strips (width > 62), image borders (out-of-image taps read 0), and row ranges (slabs)."""
    iw, ih = size
    ow, oh = 2 * iw, 2 * ih
    for gen in (F.uniform, F.structured):
        src = F.to_half(gen(iw, ih, 55))
        want = emu_rcas(emu_easu(PROD, src, ow, oh), 0.25)
        con = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
        s16 = np.ascontiguousarray(src.view(np.uint16))
        for (y0, y1) in ((0, oh), (oh // 3, 2 * oh // 3 + 1)):
            out = np.zeros((oh, ow, 4), np.uint16)
            rc = emu_lib().emu_fused_h(ctypes.c_void_p(s16.ctypes.data), iw, ih, ctypes.c_longlong(s16.strides[0]),
                                       ctypes.c_void_p(out.ctypes.data), ow, oh, ctypes.c_longlong(out.strides[0]), con, y0, y1, ctas)
            assert rc == 0
            assert np.array_equal(out[y0:y1], want.view(np.uint16)[y0:y1]), (gen.__name__, y0, y1)
            assert not out[:y0].any() and not out[y1:].any()


def emu_easu_f32_pairs(src, ow, oh, con, y0=0, y1=None, ctas=2):
    """easu_f32_pairs_kernel on a float32 image, or on a float16 image with fp32 arithmetic (FSR1_FLAG_PRECISE)."""
    ih, iw = src.shape[:2]
    y1 = oh if y1 is None else y1
    half_storage = src.dtype == np.float16
    s = np.ascontiguousarray(src.view(np.uint16) if half_storage else src)
    out = np.zeros((oh, ow, 4), np.uint16 if half_storage else np.float32)
    rc = emu_lib().emu_easu_f32_pairs(1 if half_storage else 0, ctypes.c_void_p(s.ctypes.data), iw, ih, ctypes.c_longlong(s.strides[0]),
                                      ctypes.c_void_p(out.ctypes.data), ow, oh, ctypes.c_longlong(out.strides[0]),
                                      (ctypes.c_uint32 * 16)(*con), y0, y1, ctas)
    assert rc == 0
    return out.view(np.float16) if half_storage else out


@pytest.mark.parametrize("shape", [(96, 54, 144, 81), (96, 54, 125, 70), (64, 64, 64, 64), (50, 20, 65, 26), (33, 17, 57, 31), (96, 54, 192, 81)])
@pytest.mark.parametrize("half_storage", [0, 1])
def test_emulated_any_scale_fp32_kernel(shape, half_storage, con=None):
    """easu_f32_pairs_kernel: RGBA32F images (or fp32 arithmetic on RGBA16F storage, FSR1_FLAG_PRECISE) at scales other than 2x —
    the structure of the fp16 any-scale kernel with pairwise fp32 tap weights; within 1e-5 of the oracle (fp32 storage) / one
    rounding to half (fp16 storage), row ranges included."""
    iw, ih, ow, oh = shape
    con = con or ol.easu_con(iw, ih, ow, oh)
    for gen in (F.uniform, F.structured):
        src = gen(iw, ih, 31)
        if half_storage:
            src = F.to_half(src)
        want = ol.easu(src.astype(np.float32), ow, oh, con)
        out = emu_easu_f32_pairs(src, ow, oh, con)
        got = out.astype(np.float32)
        assert np.abs(got - want)[..., :3].max() <= (6e-4 if half_storage else 1e-5)
        assert (got[..., 3] == 1.0).all()
        assert_within_cell_bounds(out, src, con, what=(shape, half_storage))
        y0, y1 = oh // 3, 2 * oh // 3 + 1
        part = emu_easu_f32_pairs(src, ow, oh, con, y0=y0, y1=y1, ctas=1)
        assert np.array_equal(part[y0:y1], out[y0:y1]) and not part[:y0].any() and not part[y1:].any()


# The geometry cases of tests/test_gpu_parity.py (GEOMETRY) at emulator size: viewports smaller than the resource, FsrEasuConOffset,
# non-uniform and extreme scales and "almost 2x" sizes.  Outputs span several 64x32 tiles, so one or two CTAs walk more than
# one tile (prefetch into the other buffer, mbarrier parity flip).  One axis downscaled selects the direct kernel, which the
# emulator does not build; the GPU suite covers it.
# id: (resource w, h, viewport w, h, offset or None, output w, h)
EMU_GEOMETRY = {
    "2x_viewport": (96, 40, 48, 20, None, 96, 40),
    "offset": (96, 40, 64, 26, (8, 4), 96, 39),
    "viewport_at_resource_edge": (96, 40, 48, 20, (48, 20), 96, 40),
    "anisotropic_x2_y1.5": (48, 26, 48, 26, None, 96, 39),
    "x1.5_y1": (64, 40, 64, 40, None, 96, 40),
    "x1_y1.5": (96, 26, 96, 26, None, 96, 39),
    "scale1": (96, 40, 96, 40, None, 96, 40),
    "3x": (32, 13, 32, 13, None, 96, 39),
    "4x": (24, 10, 24, 10, None, 96, 40),
    "almost_2x_41x47": (41, 47, 41, 47, None, 82, 94),
}


@pytest.mark.parametrize("case", list(EMU_GEOMETRY))
def test_emulated_geometry_against_oracle(case):
    """The tiled EASU kernels at this geometry against the oracle reading the whole resource with the same constants: the
    emulator tolerances, the de-ringing bound (no tolerance), one CTA == several CTAs and row ranges == the whole frame."""
    iw, ih, vw, vh, off, ow, oh = EMU_GEOMETRY[case]
    con = ol.easu_con(iw, ih, ow, oh, vw, vh, off=off)
    quad = con[:4] == [0x3F000000, 0x3F000000, 0xBE800000, 0xBE800000]
    y0, y1 = oh // 3, 2 * oh // 3 + 1
    for gen in (F.uniform, F.structured):
        src32 = gen(iw, ih, 77)
        src = F.to_half(src32)
        want = ol.easu(src.astype(np.float32), ow, oh, con)
        run = (lambda **kw: emu_easu(PROD, src, ow, oh, con=con, **kw)) if quad else (lambda **kw: emu_easu_pairs(src, ow, oh, con=con, **kw))
        got = run(ctas=2)
        assert np.abs(got.astype(np.float32) - want)[..., :3].max() <= 5e-3, (case, gen.__name__)
        assert_within_cell_bounds(got, src, con, what=(case, gen.__name__, "f16"))
        assert np.array_equal(run(ctas=1).view(np.uint16), got.view(np.uint16)), (case, "one CTA")
        part = run(y0=y0, y1=y1, ctas=1)
        assert np.array_equal(part[y0:y1].view(np.uint16), got[y0:y1].view(np.uint16)), (case, "rows")
        if quad:
            continue
        for s, tol in ((src32, 1e-5), (src, 6e-4)):                      # RGBA32F, and fp32 arithmetic on RGBA16F storage
            got = emu_easu_f32_pairs(s, ow, oh, con, ctas=2)
            assert np.abs(got.astype(np.float32) - ol.easu(s.astype(np.float32), ow, oh, con))[..., :3].max() <= tol, (case, s.dtype)
            assert_within_cell_bounds(got, s, con, what=(case, gen.__name__, str(s.dtype)))
            assert np.array_equal(emu_easu_f32_pairs(s, ow, oh, con, ctas=1), got), (case, s.dtype, "one CTA")
            part = emu_easu_f32_pairs(s, ow, oh, con, y0=y0, y1=y1, ctas=1)
            assert np.array_equal(part[y0:y1], got[y0:y1]), (case, s.dtype, "rows")
