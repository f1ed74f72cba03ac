"""FSR1_FORMAT_R11G11B10_FLOAT input on the H100: every call on R11G11B10F codes is bit-identical to the same call on the RGBA16F image of
the decoded values (tests/test_r11g11b10.decode), and runs the tiled, fused or post kernel that the RGBA16F call runs, not a fallback.
Inputs are raw random 32-bit codes (every exponent, denormals, zeros, 65024, inf and NaN) or a linear HDR image for SRTM_INPUT."""
import ctypes
import fnmatch

import numpy as np
import pytest
import torch

import fsr1_b200 as F
from fsr1_b200 import _lib, api
from test_gpu_guards import Guarded, plain
from test_r11g11b10 import decode, hdr_codes, raw_codes

pytestmark = pytest.mark.gpu

R11 = api.FORMAT_R11G11B10_FLOAT
S = api.FLAG_SRTM_INPUT
BASELINE = [(1920, 1080, 3840, 2160), (2560, 1440, 3840, 2160), (2953, 1661, 3840, 2160)]
ODD = [(125, 67, 250, 134), (333, 97, 666, 194)]


def codes(kind, w, h, seed):
    """int32 [h, w] codes in rows padded to 16 bytes (the tiled kernels' layout)"""
    return plain((raw_codes if kind == "raw" else hdr_codes)(w, h, seed).view(np.int32))


def dec(c):
    """the RGBA16F image of the decoded values, float16 [H, W, 4], rows padded to 16 bytes"""
    return plain(decode(c.cpu().numpy().view(np.uint32)).view(np.float16))


def r11(t, height=None, row0=0):
    return api.image(t, height=height, row0=row0, format=R11)


def out16(oh, ow, fill=0.0):
    """float16 [oh, ow, 4] in rows padded to 16 bytes"""
    return torch.full((oh, ow + (ow & 1), 4), fill, dtype=torch.float16, device="cuda")[:, :ow]


def exact2x(iw, ih, ow, oh):
    """FsrEasuCon's constants are exactly 2x (41 -> 82 is not: 41 * fp32(1/82) != 0.5), so the 2x kernels run"""
    c = np.array(api.easu_con(iw, ih, iw, ih, ow, oh)[:4], np.uint32).view(np.float32)
    return tuple(c) == (0.5, 0.5, -0.25, -0.25)


def bits(t):
    return t.view(torch.int16) if t.dtype == torch.float16 else t


def same(a, b):
    return torch.equal(bits(a), bits(b))


def ran(pattern):
    k = api.last_kernel()
    assert fnmatch.fnmatchcase(k, pattern), k
    return k


# ---- fsr1_easu ---------------------------------------------------------------------------------------------------------------------
EASU_CASES = [  # (iw, ih, ow, oh, flags, kernel of the R11G11B10F call)
    (64, 36, 128, 72, 0, "easu_h_quad2x<4w,7/sm,tma2,r11g11b10f_in>"),
    (96, 54, 144, 81, 0, "easu_h_vpairs<*,r11g11b10f_in>"),                  # 1.5x
    (100, 60, 130, 78, 0, "easu_h_vpairs<*,r11g11b10f_in>"),                 # 1.3x
    (41, 23, 82, 46, 0, "easu_h_vpairs<*,r11g11b10f_in>"),                   # almost 2x (exact2x)
    (41, 23, 81, 45, 0, "easu_h_vpairs<*,r11g11b10f_in>"),
    (128, 72, 96, 54, 0, "easu_direct<r11g11b10f_in,f16out,fast>"),          # downscale
    (64, 36, 128, 72, api.FLAG_FORCE_DIRECT, "easu_direct<r11g11b10f_in,f16out,fast>"),
    (64, 36, 128, 72, S, "easu_h_quad2x<*,r11g11b10f_in,srtm_in>"),
    (96, 54, 144, 81, S, "easu_h_vpairs<*,r11g11b10f_in,srtm_in>"),
] + [(iw, ih, ow, oh, 0, "easu_h_vpairs<*,r11g11b10f_in>") for iw, ih, ow, oh in BASELINE[1:]] + [
    (1920, 1080, 3840, 2160, 0, "easu_h_quad2x<*,r11g11b10f_in>")] + [
    (iw, ih, ow, oh, 0, "easu_h_%s<*,r11g11b10f_in>" % ("quad2x" if exact2x(iw, ih, ow, oh) else "vpairs")) for iw, ih, ow, oh in ODD]


@pytest.mark.parametrize("iw,ih,ow,oh,flags,kernel", EASU_CASES)
def test_easu_equals_the_call_on_the_decoded_image(iw, ih, ow, oh, flags, kernel):
    c = codes("hdr" if flags & S else "raw", iw, ih, iw + ih)
    before = c.clone()
    con = api.easu_con(iw, ih, iw, ih, ow, oh)
    got, want = out16(oh, ow, 7.0), out16(oh, ow, 7.0)
    n0 = api.launch_count()
    api.easu(r11(c), got, con, flags=flags)
    assert api.launch_count() == n0 + 1
    k = ran(kernel)
    api.easu(dec(c), want, con, flags=flags)
    assert api.last_kernel() == k.replace(",r11g11b10f_in", "").replace("<r11g11b10f_in,f16out,", "<f16io,")
    assert same(got, want)
    assert torch.equal(c, before)


def test_easu_on_an_unaligned_pitch_takes_the_direct_kernel():
    iw, ih, ow, oh = 61, 33, 122, 66
    base = torch.from_numpy(raw_codes(iw + 1, ih, 5).view(np.int32)).cuda()
    c = base[:, :iw]                                         # pitch 248 bytes: not a multiple of 16
    got, want = out16(oh, ow), out16(oh, ow)
    con = api.easu_con(iw, ih, iw, ih, ow, oh)
    api.easu(r11(c), got, con)
    ran("easu_direct<r11g11b10f_in,f16out,fast>")
    api.easu(dec(c.contiguous()), want, con, flags=api.FLAG_FORCE_DIRECT)
    assert same(got, want)


def test_easu_row_slab_on_an_input_window():
    iw, ih, ow, oh = 320, 180, 640, 360
    c = codes("raw", iw, ih, 9)
    con = api.easu_con(iw, ih, iw, ih, ow, oh)
    y0, y1 = 101, 233
    r0, r1 = api.easu_input_rows(con, ih, y0, y1)
    got, want = out16(oh, ow, 3.0), out16(oh, ow, 3.0)
    api.easu(r11(c[r0:r1 + 1].clone(), height=ih, row0=r0), got, con, y0, y1)
    ran("easu_h_quad2x<*,r11g11b10f_in>")
    api.easu(dec(c), want, con, y0, y1)
    assert same(got, want)


# ---- fsr1_upscale ------------------------------------------------------------------------------------------------------------------
UPSCALE_FLAGS = [(api.FLAG_FUSED, "fused_easu_rcas_h_quad2x<4w,7/sm,tma2,strips,r11g11b10f_in>", 1),
                 (0, "rcas_h_packed*", 2), (api.FLAG_FUSED | api.FLAG_RCAS_CLAMP, "rcas_h_packed*", 2),
                 (api.FLAG_RCAS_DENOISE, "rcas_h_packed*", 2), (api.FLAG_RCAS_PASSTHROUGH_ALPHA, "rcas_h_packed*", 2),
                 (api.FLAG_OUTPUT_SQUARE, "rcas_h_packed*", 2), (api.FLAG_NO_RCAS, "easu_h_quad2x<*,r11g11b10f_in>", 1),
                 (api.FLAG_FUSED | S, "fused_easu_rcas_h_quad2x<4w,7/sm,tma2,strips,r11g11b10f_in,srtm_in>", 1)]


@pytest.mark.parametrize("size", BASELINE + ODD)
@pytest.mark.parametrize("flags,kernel,launches", UPSCALE_FLAGS)
def test_upscale_equals_the_call_on_the_decoded_image(size, flags, kernel, launches):
    iw, ih, ow, oh = size
    if not exact2x(iw, ih, ow, oh):
        kernel = kernel if kernel == "rcas_h_packed*" else ("rcas_h_packed*" if not flags & api.FLAG_NO_RCAS else "easu_h_vpairs<*")
        launches = 2 if not flags & api.FLAG_NO_RCAS else 1
    c = codes("hdr" if flags & S else "raw", iw, ih, iw * 7 + ih)
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    tmp, got = out16(oh, ow, 5.0), out16(oh, ow, 5.0)
    n0 = api.launch_count()
    api.upscale(r11(c), tmp, got, econ, rcon, flags=flags)
    assert api.launch_count() == n0 + launches
    ran(kernel)
    want = out16(oh, ow, 5.0)
    api.upscale(dec(c), out16(oh, ow, 5.0), want, econ, rcon, flags=flags)
    assert same(got, want)


# ---- fsr1_upscale_post -------------------------------------------------------------------------------------------------------------
def _post_out(oh, ow, bits_):
    if bits_ == 8:
        return torch.zeros((oh, ow, 4), dtype=torch.uint8, device="cuda")
    if bits_ == 10:
        return torch.zeros((oh, ow), dtype=torch.int32, device="cuda")
    return out16(oh, ow)


POST_OPS = [(s, g, t) for s in (False, True) for g in (False, True) for t in (0, 8, 10)]


@pytest.mark.parametrize("srtm_inverse,lfga,tepd_bits", POST_OPS)
@pytest.mark.parametrize("size,flags", [((960, 540, 1920, 1080), api.FLAG_FUSED), ((960, 540, 1920, 1080), api.FLAG_FUSED | S),
                                        ((333, 97, 666, 194), api.FLAG_FUSED), ((960, 540, 1440, 810), api.FLAG_FUSED),
                                        ((960, 540, 1920, 1080), api.FLAG_RCAS_DENOISE)])
def test_upscale_post_equals_the_call_on_the_decoded_image(srtm_inverse, lfga, tepd_bits, size, flags):
    iw, ih, ow, oh = size
    c = codes("hdr" if flags & S or srtm_inverse else "raw", iw, ih, ow + tepd_bits)
    grain = (torch.rand((5, 12, 4), device="cuda") - 0.5).half() if lfga else None
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    got, want = _post_out(oh, ow, tepd_bits), _post_out(oh, ow, tepd_bits)
    kw = dict(srtm_inverse=srtm_inverse, grain=grain, amount=0.375, tepd_bits=tepd_bits, frame=3, flags=flags)
    api.upscale_post(r11(c), out16(oh, ow), got, econ, rcon, **kw)
    k = api.last_kernel()
    fused = exact2x(iw, ih, ow, oh) and not flags & api.FLAG_RCAS_DENOISE
    ops = srtm_inverse or lfga or tepd_bits
    if fused:
        assert k.startswith("fused_easu_rcas_h_quad2x<") and "r11g11b10f_in" in k and (",post," in k) == bool(ops), k
    else:
        assert k.startswith("rcas_h_packed_post<" if ops else "rcas_h_packed<"), k
    api.upscale_post(dec(c), out16(oh, ow), want, econ, rcon, **kw)
    assert same(got, want)
    if fused:                                                                   # no intermediate needed
        got2 = _post_out(oh, ow, tepd_bits)
        api.upscale_post(r11(c), None, got2, econ, rcon, **kw)
        assert same(got2, want)


@pytest.mark.parametrize("size", BASELINE)
def test_hdr_round_trip_at_baseline_sizes(size):
    iw, ih, ow, oh = size
    c = codes("hdr", iw, ih, 77)
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    got, want = _post_out(oh, ow, 10), _post_out(oh, ow, 10)
    kw = dict(srtm_inverse=True, tepd_bits=10, frame=1, flags=api.FLAG_FUSED | S)
    api.upscale_post(r11(c), out16(oh, ow), got, econ, rcon, **kw)
    api.upscale_post(dec(c), out16(oh, ow), want, econ, rcon, **kw)
    assert same(got, want)


# ---- contexts ----------------------------------------------------------------------------------------------------------------------
def test_context_calls_equal_the_calls_on_the_decoded_image():
    iw, ih, ow, oh = 640, 360, 1280, 720
    c, h = codes("raw", iw, ih, 31), codes("hdr", iw, ih, 32)
    ctx, ref = api.HostContext(iw, ih, ow, oh, fmt=R11), api.HostContext(iw, ih, ow, oh)
    try:
        for flags, src in ((0, c), (S, h)):
            got, want = out16(oh, ow), out16(oh, ow)
            ctx.upscale(src, got, flags=flags)
            ran("fused_easu_rcas_h_quad2x<*,r11g11b10f_in*")
            ref.upscale(dec(src), want, flags=flags)
            assert same(got, want)
            got, want = out16(oh, ow), out16(oh, ow)
            ctx.upscale_render(src, 480, 270, got, flags=flags)
            ref.upscale_render(dec(src), 480, 270, want, flags=flags)
            assert same(got, want)
            for bits_ in (0, 8, 10):
                got, want = _post_out(oh, ow, bits_), _post_out(oh, ow, bits_)
                ctx.upscale_post(src, got, srtm_inverse=True, tepd_bits=bits_, frame=2, flags=flags)
                ref.upscale_post(dec(src), want, srtm_inverse=True, tepd_bits=bits_, frame=2, flags=flags)
                assert same(got, want)
        hin = c.cpu().pin_memory()
        hgot, hwant = torch.zeros((oh, ow, 4), dtype=torch.float16).pin_memory(), torch.zeros((oh, ow, 4), dtype=torch.float16).pin_memory()
        ctx.upscale_host(hin, hgot)
        ref.upscale_host(dec(c).cpu().pin_memory(), hwant)
        torch.cuda.synchronize()
        assert torch.equal(hgot.view(torch.int16), hwant.view(torch.int16))
    finally:
        ctx.close()
        ref.close()


# ---- shards ------------------------------------------------------------------------------------------------------------------------
def _whole(frame, rw, rh, ow, oh, flags, sharpness=0.25):
    """the whole frame on one GPU: fused upscale of the decoded render region"""
    d = dec(frame[:rh, :rw].contiguous())
    out = out16(oh, ow)
    api.upscale(d, out16(oh, ow), out, api.easu_con(rw, rh, rw, rh, ow, oh), api.rcas_con(sharpness), flags=flags | api.FLAG_FUSED)
    return out


def test_single_rank_shard_and_its_geometry():
    for iw, ih, ow, oh in [(1920, 1080, 3840, 2160), (1920, 1080, 2880, 1620)]:
        up = F.ShardedUpscaler(iw, ih, ow, oh, 1, 0, slots=2, halo="p2p", in_format=R11)
        try:
            assert up.input(0).dtype == torch.int32 and up.output(0).dtype == torch.float16
            s = torch.cuda.current_stream()
            frames = [codes("raw", iw, ih, 50 + k) for k in range(2)]
            for k in range(2):
                up.input(k).copy_(frames[k])
                up.submit(k, s)
                ran("fused_easu_rcas_h_quad2x<*,r11g11b10f_in>" if ow == 2 * iw else "rcas_h_packed*")
            for k in range(2):
                up.wait(k, s)
            torch.cuda.synchronize()
            up.status()
            for k in range(2):
                assert same(up.output(k), _whole(frames[k], iw, ih, ow, oh, 0))
        finally:
            up.close()


@pytest.mark.parametrize("world", [2, 8])
def test_shard_geometry_is_sized_at_4_bytes_per_pixel(world):
    iw, ih, ow, oh = 640, 360, 1280, 720
    for r in range(world):
        a = F.ShardedUpscaler(iw, ih, ow, oh, world, r, slots=2, halo="p2p", attach=False, in_format=R11)
        b = F.ShardedUpscaler(iw, ih, ow, oh, world, r, slots=2, halo="p2p", attach=False)
        try:
            assert a.info.halo_recv_bytes == a.plan.halo_bytes(r, iw, 4) == b.info.halo_recv_bytes // 2
            lo, hi = a.plan.window_rows(r)
            assert a.window.shape == (hi - lo, iw) and a.window.stride(0) * 4 == -(-iw * 4 // 128) * 128
            rows = max(a.plan.window_rows(q)[1] - a.plan.window_rows(q)[0] for q in range(world))   # every rank's arena: the tallest window
            assert a.info.arena_bytes == 4096 + 2 * (-(-rows * (-(-iw * 4 // 128) * 128) // 256) * 256)
            assert a.info.arena_bytes < b.info.arena_bytes
        finally:
            a.close()
            b.close()


@pytest.mark.parametrize("dynamic", [False, True])
@pytest.mark.parametrize("srtm", [False, True])
def test_eight_ranks_on_one_device(dynamic, srtm):
    iw, ih, ow, oh, world, nslots, nframes = 960, 540, 1920, 1080, 8, 2, 4
    flags = S if srtm else 0
    ups = [F.ShardedUpscaler(iw, ih, ow, oh, world, r, slots=nslots, halo="p2p", attach=False, flags=flags, dynamic=dynamic, in_format=R11)
           for r in range(world)]
    sizes = [(iw, ih), (800, 450), (iw, ih), (720, 400)] if dynamic else [(iw, ih)] * nframes
    try:
        for r, u in enumerate(ups):
            u.attach_local(ups[r - 1] if r > 0 else None, ups[r + 1] if r + 1 < world else None)
        frames = [codes("hdr" if srtm else "raw", iw, ih, 70 + i) for i in range(nframes)]
        s = torch.cuda.current_stream()
        got = []
        for i, fr in enumerate(frames):
            k = i % nslots
            if i >= nslots:
                for u in ups:
                    u.wait(k, s)
                got.append(torch.cat([u.output(k) for u in ups]).clone())
            rw, rh = sizes[i]
            for r, u in enumerate(ups):
                owned = u.frame(k, rw, rh) if dynamic else u.input(k)
                o0 = owned.shape[0]
                a0 = (r * rh) // world
                owned.copy_(fr[a0:a0 + o0, :rw])
            for u in ups:
                n0 = api.launch_count()
                u.submit(k, s)
                assert api.launch_count() == n0 + (1 if (rw, rh) == (iw, ih) else 2)
                if (rw, rh) == (iw, ih):
                    ran("fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,r11g11b10f_in%s>" % (",srtm_in" if srtm else ""))
        for i in range(nframes - nslots, nframes):
            for u in ups:
                u.wait(i % nslots, s)
            got.append(torch.cat([u.output(i % nslots) for u in ups]).clone())
        torch.cuda.synchronize()
        for u in ups:
            u.status()
        for i in range(nframes):
            rw, rh = sizes[i]
            assert same(got[i], _whole(frames[i], rw, rh, ow, oh, flags)), "frame %d" % i
    finally:
        for u in ups:
            u.close()


def test_shard_with_display_steps():
    iw, ih, ow, oh, world = 640, 360, 1280, 720, 4
    ups = [F.ShardedUpscaler(iw, ih, ow, oh, world, r, halo="p2p", attach=False, flags=S, srtm_inverse=True, tepd_bits=10,
                             in_format=R11) for r in range(world)]
    try:
        for r, u in enumerate(ups):
            u.attach_local(ups[r - 1] if r > 0 else None, ups[r + 1] if r + 1 < world else None)
        fr = codes("hdr", iw, ih, 99)
        s = torch.cuda.current_stream()
        for r, u in enumerate(ups):
            o0, o1 = u.plan.owned_in_rows(r)
            u.input(0).copy_(fr[o0:o1])
        for u in ups:
            u.submit(0, s)
            ran("fused_easu_rcas_h_quad2x<*,post,rgb10a2,r11g11b10f_in,srtm_in>")
        for u in ups:
            u.wait(0, s)
        torch.cuda.synchronize()
        for u in ups:
            u.status()
        got = torch.cat([u.output(0) for u in ups])
        want = _post_out(oh, ow, 10)
        api.upscale_post(dec(fr), None, want, api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25), srtm_inverse=True,
                         tepd_bits=10, flags=api.FLAG_FUSED | S)
        assert torch.equal(got, want)
    finally:
        for u in ups:
            u.close()


# ---- guards: every kernel family reads and writes only its own pixels ---------------------------------------------------------------
GUARD_CASES = [(64, 36, 128, 72, 0), (96, 54, 144, 81, 0), (64, 36, 128, 72, api.FLAG_FORCE_DIRECT), (128, 72, 96, 54, 0),
               (64, 36, 128, 72, api.FLAG_FUSED), (125, 33, 250, 66, api.FLAG_FUSED | S), (64, 36, 128, 72, -1)]


@pytest.mark.parametrize("poison", ["nan", "big", "atlas"])
@pytest.mark.parametrize("iw,ih,ow,oh,flags", GUARD_CASES)
def test_kernels_stay_inside_their_images(iw, ih, ow, oh, flags, poison):
    """The input inside a poisoned int32 allocation, the outputs inside poisoned half ones.  flags -1: fsr1_upscale_post with TEPD10."""
    src = raw_codes(iw, ih, iw + ih).view(np.int32)
    gin = Guarded("u10", ih, iw, poison, seed=31)
    gin.set(src)
    gtmp, gout = Guarded("f16", oh, ow, poison, seed=32), Guarded("f16", oh, ow, poison, seed=33)
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    inp = r11(gin.img)
    c = torch.from_numpy(src).cuda()
    if flags == -1:
        gout = Guarded("u10", oh, ow, poison, seed=34)
        api.upscale_post(inp, gtmp.image(), gout.image(), econ, rcon, srtm_inverse=True, tepd_bits=10, flags=api.FLAG_FUSED)
        want = _post_out(oh, ow, 10)
        api.upscale_post(dec(c), None, want, econ, rcon, srtm_inverse=True, tepd_bits=10, flags=api.FLAG_FUSED)
        gtmp.assert_untouched("tmp of a fused post frame")
    elif flags & api.FLAG_FUSED:
        api.upscale(inp, gtmp.image(), gout.image(), econ, rcon, flags=flags)
        want = out16(oh, ow)
        api.upscale(dec(c), out16(oh, ow), want, econ, rcon, flags=flags)
        gtmp.assert_untouched("tmp of a fused frame")
    else:
        api.easu(inp, gout.image(), econ, flags=flags)
        want = out16(oh, ow)
        api.easu(dec(c), want, econ, flags=flags)
    torch.cuda.synchronize()
    what = (iw, ih, ow, oh, flags, poison, api.last_kernel())
    gin.assert_untouched("input %s" % (what,))                                 # not even the image itself is written
    gout.assert_untouched("output %s" % (what,), 0, oh)
    assert same(gout.img, want), what
