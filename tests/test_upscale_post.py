"""fsr1_upscale_post: EASU -> RCAS with SRTM inverse, LFGA and TEPD applied in RCAS's store.  The contract is bit-equality with
fsr1_upscale followed by the separate passes through an RGBA16F intermediate.

Without a GPU: the device code of both epilogues (fused_h_quad2x_post_kernel, rcas_post_kernel) runs on the CPU emulator (tests/emu/emu_post.cpp) and
is compared with the oracle's chain on the emulated RCAS output; the ABI's validation is exercised on paths that return before any CUDA
call.  On the GPU: api.upscale_post against the sequence of existing calls, bit for bit."""
import ctypes
import itertools
import os
import subprocess

import numpy as np
import pytest

import fsr1_b200 as F
import oracle_lib as ol
from fsr1_b200 import _lib
from test_emu import EMU_DIR, emu_lib

SRTM, LFGA, T8, T10 = 1, 2, 4, 8
_post_lib = None


def post_lib():
    """tests/emu/emu_post.cpp: the epilogue kernels on CPU threads (a library of its own, tests/emu/post.mk)"""
    global _post_lib
    if _post_lib is None:
        subprocess.check_call(["make", "-s", "-C", EMU_DIR, "-f", "post.mk", "libfsr1_emu_post.so"])
        _post_lib = ctypes.CDLL(os.path.join(EMU_DIR, "libfsr1_emu_post.so"))
    return _post_lib


FMT = {np.float16: 1, np.float32: 2}


class EmuPost(ctypes.Structure):
    """struct EmuPost of tests/emu/emu_post.cpp"""
    _fields_ = [("ops", ctypes.c_int), ("amount", ctypes.c_float), ("frame", ctypes.c_uint32), ("grain", ctypes.c_void_p),
                ("gw", ctypes.c_int), ("gh", ctypes.c_int), ("gpitch", ctypes.c_longlong), ("gfmt", ctypes.c_int),
                ("dither", ctypes.c_void_p), ("dw", ctypes.c_int), ("dh", ctypes.c_int), ("dpitch", ctypes.c_longlong),
                ("dfmt", ctypes.c_int)]


def _emu_post(ops, grain, amount, dither, frame):
    g = d = (None, 0, 0, 0, 0)
    if grain is not None:
        g = (grain.ctypes.data, grain.shape[1], grain.shape[0], grain.strides[0], FMT[grain.dtype.type])
    if dither is not None:
        d = (dither.ctypes.data, dither.shape[1], dither.shape[0], dither.strides[0], FMT[dither.dtype.type])
    return EmuPost(ops, amount, frame, *g, *d)


def _out_buffer(h, w, out_format):
    return np.zeros((h, w, 4), np.uint16) if out_format == 1 else np.zeros((h, w), np.uint32)


def _to_unorm(x, scale):
    return (np.clip(np.nan_to_num(x, nan=0.0), 0.0, 1.0).astype(np.float32) * np.float32(scale) + np.float32(0.5)).astype(np.uint32)


def reference_chain(t16, ops, grain, amount, dither, frame, out_format):
    """The separate passes on the RCAS output t16 (float16 [H,W,4]): oracle fp32 steps, rounded to half between them (the RGBA16F
    intermediate), then the output store (half, or the UNORM code values of fsr1_tepd)."""
    c = np.ascontiguousarray(t16.astype(np.float32))
    if ops & SRTM:
        c = ol.srtm(c, inverse=True).astype(np.float16).astype(np.float32)
    if ops & LFGA:
        c = ol.lfga(c, np.ascontiguousarray(grain.astype(np.float32)), amount).astype(np.float16).astype(np.float32)
    if ops & (T8 | T10):
        d = np.ascontiguousarray(dither.astype(np.float32)) if dither is not None else None
        c = ol.tepd(c, 8 if ops & T8 else 10, frame=frame, dither=d)
    if out_format == 1:
        return c.astype(np.float16).view(np.uint16)
    if out_format == 3:
        q = [_to_unorm(c[..., i], 255.0) for i in range(4)]
        return q[0] | (q[1] << 8) | (q[2] << 16) | (q[3] << 24)
    q = [_to_unorm(c[..., i], 1023.0) for i in range(3)] + [_to_unorm(c[..., 3], 3.0)]
    return q[0] | (q[1] << 10) | (q[2] << 20) | (q[3] << 30)


def _tiles(seed):
    rng = np.random.default_rng(seed)
    grains = [(rng.random((5, 12, 4), np.float32) - 0.5).astype(np.float16),   # 12 x 5: widths that do not divide a strip
              (rng.random((7, 9, 4), np.float32) - 0.5).astype(np.float32)]     # 9 x 7, RGBA32F
    dither = np.ascontiguousarray(rng.random((3, 7, 4), np.float32) * 1.2 - 0.1)  # .w saturated: values outside [0,1] too
    return grains, dither


def _cases():
    """every subset of {SRTM_INVERSE, LFGA} x {no TEPD, TEPD8, TEPD10}; TEPD writes the UNORM code values (one case writes half)"""
    for srtm, lfga, tepd in itertools.product((0, SRTM), (0, LFGA), (0, T8, T10)):
        ops = srtm | lfga | tepd
        fmt = 3 if tepd == T8 else 4 if tepd == T10 else 1
        yield ops, fmt
    yield LFGA | T8, 1


CASES = list(_cases())


@pytest.mark.parametrize("ops,out_format", CASES)
def test_emulated_fused_epilogue_equals_the_pass_sequence(ops, out_format):
    """fused_h_quad2x_post_kernel on the CPU: odd output widths (partial pairs; 3 strips), a row slab, both grain tiles, a dither tile
    and the positional dither with frame != 0."""
    grains, dither_tile = _tiles(7)
    for k, (iw, ih, ow, oh) in enumerate([(40, 12, 79, 23), (70, 9, 139, 18)]):
        src = F.to_half(F.structured(iw, ih, 21 + k))
        s16 = np.ascontiguousarray(src.view(np.uint16))
        rcon = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
        grain = grains[k]
        dither = dither_tile if k == 0 else None
        for (y0, y1) in ((0, oh), (oh // 3, 2 * oh // 3 + 1)):
            plain = np.zeros((oh, ow, 4), np.uint16)
            assert emu_lib().emu_fused_h(ctypes.c_void_p(s16.ctypes.data), iw, ih, ctypes.c_longlong(s16.strides[0]),
                                         ctypes.c_void_p(plain.ctypes.data), ow, oh, ctypes.c_longlong(plain.strides[0]), rcon, y0, y1,
                                         3) == 0
            want = reference_chain(plain.view(np.float16), ops, grain, 0.375, dither, 5, out_format)
            out = _out_buffer(oh, ow, out_format)
            post = _emu_post(ops, grain, 0.375, dither, 5)
            assert post_lib().emu_fused_h_post(ctypes.c_void_p(s16.ctypes.data), iw, ih, ctypes.c_longlong(s16.strides[0]),
                                              ctypes.c_void_p(out.ctypes.data), ow, oh, ctypes.c_longlong(out.strides[0]), out_format,
                                              rcon, y0, y1, 3, ctypes.byref(post)) == 0
            assert np.array_equal(out[y0:y1], want[y0:y1]), (iw, ih, y0, y1)
            assert not out[:y0].any() and not out[y1:].any()


def test_emulated_fused_epilogue_with_no_ops_is_the_fused_kernel():
    iw, ih = 33, 17
    src = F.to_half(F.uniform(iw, ih, 3))
    want = np.zeros((2 * ih, 2 * iw, 4), np.uint16)
    s16 = np.ascontiguousarray(src.view(np.uint16))
    rcon = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.5))
    emu_lib().emu_fused_h(ctypes.c_void_p(s16.ctypes.data), iw, ih, ctypes.c_longlong(s16.strides[0]), ctypes.c_void_p(want.ctypes.data),
                          2 * iw, 2 * ih, ctypes.c_longlong(want.strides[0]), rcon, 0, 2 * ih, 2)
    out = np.zeros_like(want)
    post = _emu_post(0, None, 0.0, None, 0)
    post_lib().emu_fused_h_post(ctypes.c_void_p(s16.ctypes.data), iw, ih, ctypes.c_longlong(s16.strides[0]), ctypes.c_void_p(out.ctypes.data),
                               2 * iw, 2 * ih, ctypes.c_longlong(out.strides[0]), 1, rcon, 0, 2 * ih, 2, ctypes.byref(post))
    assert np.array_equal(out, want)


@pytest.mark.parametrize("ops,out_format", CASES)
@pytest.mark.parametrize("opts,clamp", [(0, 0), (0, 1), (1, 0), (2, 1), (4, 0), (7, 1)])
def test_emulated_rcas_epilogue_equals_the_pass_sequence(ops, out_format, opts, clamp):
    """rcas_post_kernel on the CPU with RCAS_CLAMP, DENOISE (opts bit 0), PASSTHROUGH_ALPHA (bit 1) and OUTPUT_SQUARE (bit 2): odd
    widths, interior and border spans, a row slab."""
    grains, dither_tile = _tiles(11)
    rng = np.random.default_rng(opts * 16 + ops)
    for k, (w, h) in enumerate([(61, 19), (131, 22)]):
        src = F.to_half(F.structured(w, h, 40 + k))
        src[..., 3] = rng.random((h, w)).astype(np.float16)   # alpha passes through with PASSTHROUGH_ALPHA
        s16 = np.ascontiguousarray(src.view(np.uint16))
        con = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
        grain = grains[k]
        dither = dither_tile if k == 1 else None
        y0, y1 = (0, h) if k == 0 else (5, h - 4)
        t = np.zeros((h, w, 4), np.uint16)
        assert emu_lib().emu_rcas_h_packed_opt(ctypes.c_void_p(s16.ctypes.data), 0, h, ctypes.c_void_p(t.ctypes.data), w, h,
                                               ctypes.c_longlong(s16.strides[0]), ctypes.c_longlong(t.strides[0]), con, clamp, y0, y1,
                                               opts) == 0
        want = reference_chain(t.view(np.float16), ops, grain, 0.5, dither, 3, out_format)
        out = _out_buffer(h, w, out_format)
        post = _emu_post(ops, grain, 0.5, dither, 3)
        assert post_lib().emu_rcas_h_packed_post(ctypes.c_void_p(s16.ctypes.data), ctypes.c_void_p(out.ctypes.data), w, h,
                                                ctypes.c_longlong(s16.strides[0]), ctypes.c_longlong(out.strides[0]), out_format, con,
                                                clamp, y0, y1, opts, ctypes.byref(post)) == 0
        assert np.array_equal(out[y0:y1], want[y0:y1]), (w, h)
        assert not out[:y0].any() and not out[y1:].any()


def test_upscale_post_validation_without_gpu():
    """The documented codes, all returned before any CUDA call."""
    L = _lib.lib()
    launches = L.fsr1_launch_count()   # the counter is process-wide: GPU tests may have run earlier in this process
    buf = (ctypes.c_uint8 * 65536)()
    addr = ctypes.addressof(buf)
    addr += (-addr) % 256
    econ = (ctypes.c_uint32 * 16)(*F.api.easu_con(8, 4, 8, 4, 16, 8))
    rcon = (ctypes.c_uint32 * 4)(*F.api.rcas_con(0.25))
    inp = _lib.Image(addr, 64, 8, 4, 0, 4, 1, 0)
    tmp = _lib.Image(addr + 4096, 128, 16, 8, 0, 8, 1, 0)
    out = _lib.Image(addr + 8192, 128, 16, 8, 0, 8, 1, 0)
    out8 = _lib.Image(addr + 8192, 64, 16, 8, 0, 8, 3, 0)
    out10 = _lib.Image(addr + 8192, 64, 16, 8, 0, 8, 4, 0)
    grain = _lib.Image(addr + 16384, 32, 4, 4, 0, 4, 1, 0)
    grain_win = _lib.Image(addr + 16384, 32, 4, 4, 1, 2, 1, 0)
    grain_u8 = _lib.Image(addr + 16384, 16, 4, 4, 0, 4, 3, 0)

    def call(i=inp, o=out, ops=_lib.POST_TEPD8, g=None, d=None, flags=0):
        post = _lib.Post(ops, 0.5, ctypes.pointer(g) if g is not None else None, ctypes.pointer(d) if d is not None else None, 0, 0)
        return L.fsr1_upscale_post(ctypes.byref(i), ctypes.byref(tmp), ctypes.byref(o), econ, rcon, ctypes.byref(post), 0, 0, flags, None)

    assert call(ops=1 << 4) == -1                                          # unknown ops bit
    assert call(ops=_lib.POST_TEPD8 | _lib.POST_TEPD10) == -1              # both TEPD bits
    assert call(ops=_lib.POST_LFGA) == -1                                  # LFGA without a grain tile
    assert call(ops=_lib.POST_LFGA, g=grain_win) == -1                     # an aux tile that is a window
    assert call(ops=_lib.POST_TEPD8, d=grain_win) == -1
    assert call(ops=_lib.POST_LFGA, g=grain_u8) == -2                      # grain is signed: float tiles only
    assert call(i=_lib.Image(addr, 128, 8, 4, 0, 4, 2, 0)) == -2          # RGBA32F input
    assert call(i=_lib.Image(addr, 32, 8, 4, 0, 4, 3, 0)) == -2           # UNORM input
    assert call(o=out10, ops=_lib.POST_TEPD8) == -2                        # TEPD8 writes RGBA8 codes, not RGB10A2
    assert call(o=out8, ops=_lib.POST_TEPD10) == -2
    assert call(o=out8, ops=_lib.POST_SRTM_INVERSE) == -2                  # UNORM out needs TEPD
    assert call(o=_lib.Image(addr + 8192, 256, 16, 8, 0, 8, 2, 0)) == -2   # RGBA32F out
    for flag in (F.api.FLAG_EXACT, F.api.FLAG_NO_RCAS, F.api.FLAG_RCAS_HX2, F.api.FLAG_FORCE_DIRECT, F.api.FLAG_H_REFERENCE):
        assert call(flags=flag) == -2, flag
    assert call(flags=1 << 20) == -1                                       # unknown flag
    assert call(o=_lib.Image(addr + 8192 + 8, 128, 16, 8, 0, 8, 1, 0)) == -2   # RGBA16F out not 16-byte aligned
    assert L.fsr1_context_upscale_post(None, None, 0, 0, 0, None, 0, ctypes.c_float(0.25), None, 0, None) == -1
    assert L.fsr1_launch_count() == launches                               # nothing was launched


# ---- on the GPU: against the sequence of existing calls ------------------------------------------------------------------------
def _gpu():
    import torch
    from fsr1_b200 import api
    return torch, api


def _sequence(api, torch, inp, econ, rcon, oh, ow, srtm_inverse, grain, amount, tepd_bits, dither, frame, out, y0=0, y1=0, flags=0):
    t = torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda")
    tmp = torch.zeros_like(t)
    api.upscale(inp, tmp, t, econ, rcon, y0, y1, flags)
    if srtm_inverse:
        api.srtm(t, t, inverse=True, y0=y0, y1=y1)
    if grain is not None:
        api.lfga(t, grain, t, amount, y0=y0, y1=y1)
    if tepd_bits:
        api.tepd(t, out, tepd_bits, frame=frame, dither=dither, y0=y0, y1=y1)
    else:
        out[y0:y1 if y1 else oh].copy_(t[y0:y1 if y1 else oh])


def _out_tensor(torch, oh, ow, bits, fill=0):
    if bits == 8:
        return torch.full((oh, ow, 4), fill, dtype=torch.uint8, device="cuda")
    if bits == 10:
        return torch.full((oh, ow), fill, dtype=torch.int32, device="cuda")
    return torch.full((oh, ow, 4), fill, dtype=torch.float16, device="cuda")


def _frame(torch, iw, ih, seed):
    return torch.from_numpy(F.to_half(F.structured(iw, ih, seed))).cuda()


def _grain(torch, seed, shape=(5, 12, 4), dtype=None):
    g = (np.random.default_rng(seed).random(shape, np.float32) - 0.5)
    return torch.from_numpy(g.astype(dtype or np.float16)).cuda()


def _check(torch, api, iw, ih, ow, oh, flags, srtm_inverse, grain, tepd_bits, dither, frame, y0=0, y1=0, tmp_none=False):
    inp = _frame(torch, iw, ih, iw + ih)
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    want = _out_tensor(torch, oh, ow, tepd_bits)
    _sequence(api, torch, inp, econ, rcon, oh, ow, srtm_inverse, grain, 0.3, tepd_bits, dither, frame, want, y0, y1, flags)
    got = _out_tensor(torch, oh, ow, tepd_bits)
    tmp = None if tmp_none else torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda")
    n0 = api.launch_count()
    api.upscale_post(inp, tmp, got, econ, rcon, srtm_inverse=srtm_inverse, grain=grain, amount=0.3, tepd_bits=tepd_bits, dither=dither,
                     frame=frame, y0=y0, y1=y1, flags=flags)
    torch.cuda.synchronize()
    launches, name = api.launch_count() - n0, api.last_kernel()
    assert torch.equal(got, want), (iw, ih, ow, oh, flags, srtm_inverse, grain is not None, tepd_bits, name)
    return launches, name


@pytest.mark.gpu
@pytest.mark.parametrize("srtm_inverse,lfga,tepd_bits", list(itertools.product((False, True), (False, True), (0, 8, 10))))
@pytest.mark.parametrize("scale", ["2x", "1.5x"])
def test_every_op_subset_equals_the_sequence(srtm_inverse, lfga, tepd_bits, scale):
    torch, api = _gpu()
    iw, ih, ow, oh = (160, 90, 320, 180) if scale == "2x" else (160, 90, 240, 135)
    grain = _grain(torch, 1) if lfga else None
    dither = _grain(torch, 2, (3, 7, 4), np.float32) + 0.5 if tepd_bits == 10 else None
    n, name = _check(torch, api, iw, ih, ow, oh, api.FLAG_FUSED, srtm_inverse, grain, tepd_bits, dither, 7)
    post = "post" if (srtm_inverse or lfga or tepd_bits) else "upscale"    # no ops: exactly fsr1_upscale
    if scale == "2x":
        assert n == 1 and name.startswith("fused_easu_rcas_h_quad2x") and (post in name) == (post == "post"), name
    else:
        assert n == 2 and name.startswith("rcas_h_packed") and (post in name) == (post == "post"), name


@pytest.mark.gpu
@pytest.mark.parametrize("size", [(1920, 1080, 3840, 2160), (2560, 1440, 3840, 2160), (1920, 1080, 2560, 1440)])
def test_display_chains_at_full_size(size):
    """The usual SDR ending (LFGA, TEPD 8-bit -> RGBA8) and HDR10-style ending (SRTM inverse, TEPD 10-bit -> RGB10A2)."""
    torch, api = _gpu()
    iw, ih, ow, oh = size
    _check(torch, api, iw, ih, ow, oh, api.FLAG_FUSED, False, _grain(torch, 3, (64, 64, 4)), 8, None, 11)
    _check(torch, api, iw, ih, ow, oh, api.FLAG_FUSED, True, None, 10, None, 12)


@pytest.mark.gpu
@pytest.mark.parametrize("flags", ["RCAS_CLAMP", "RCAS_DENOISE", "RCAS_PASSTHROUGH_ALPHA", "OUTPUT_SQUARE", "PRECISE"])
def test_rcas_options_on_the_two_kernel_path(flags):
    torch, api = _gpu()
    f = getattr(api, "FLAG_" + flags) | api.FLAG_FUSED
    n, name = _check(torch, api, 320, 180, 640, 360, f, True, _grain(torch, 4, (7, 9, 4), np.float32), 8, None, 2)
    assert n == 2 and name.startswith("rcas_h_packed_post"), name


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False])
def test_row_slab_leaves_other_rows_untouched(fused):
    torch, api = _gpu()
    iw, ih, ow, oh = (400, 200, 800, 400) if fused else (400, 200, 600, 300)
    y0, y1 = 101, 257
    inp = _frame(torch, iw, ih, 9)
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    grain = _grain(torch, 5)
    want = _out_tensor(torch, oh, ow, 8, fill=77)
    _sequence(api, torch, inp, econ, rcon, oh, ow, False, grain, 0.3, 8, None, 3, want, y0, y1, api.FLAG_FUSED)
    got = _out_tensor(torch, oh, ow, 8, fill=77)
    tmp = torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda")
    api.upscale_post(inp, tmp, got, econ, rcon, grain=grain, amount=0.3, tepd_bits=8, frame=3, y0=y0, y1=y1, flags=api.FLAG_FUSED)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert (got[:y0] == 77).all() and (got[y1:] == 77).all()


@pytest.mark.gpu
def test_fused_path_is_one_launch_without_tmp():
    torch, api = _gpu()
    n, name = _check(torch, api, 960, 540, 1920, 1080, api.FLAG_FUSED, True, _grain(torch, 6), 8, None, 1, tmp_none=True)
    assert n == 1 and name == "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba8>", name


@pytest.mark.gpu
def test_zero_ops_is_upscale():
    torch, api = _gpu()
    n, name = _check(torch, api, 160, 90, 320, 180, api.FLAG_FUSED, False, None, 0, None, 0)
    assert n == 1 and name == "fused_easu_rcas_h_quad2x<4w,7/sm,tma2,strips>", name


@pytest.mark.gpu
@pytest.mark.parametrize("render", [(0, 0), (701, 397)])
def test_context_variant_equals_the_sequence(render):
    torch, api = _gpu()
    iw, ih, ow, oh = 960, 540, 1920, 1080
    rw, rh = render[0] or iw, render[1] or ih
    inp = _frame(torch, iw, ih, 13)
    grain = _grain(torch, 7)
    econ, rcon = api.easu_con(rw, rh, rw, rh, ow, oh), api.rcas_con(0.5)
    want = _out_tensor(torch, oh, ow, 8)
    _sequence(api, torch, inp[:rh, :rw], econ, rcon, oh, ow, True, grain, 0.25, 8, None, 4, want, flags=api.FLAG_FUSED)
    ctx = api.HostContext(iw, ih, ow, oh)
    got = _out_tensor(torch, oh, ow, 8)
    ctx.upscale_post(inp, got, render[0], render[1], sharpness=0.5, srtm_inverse=True, grain=grain, amount=0.25, tepd_bits=8, frame=4)
    torch.cuda.synchronize()
    ctx.close()
    assert torch.equal(got, want)
