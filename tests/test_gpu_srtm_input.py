"""FSR1_FLAG_SRTM_INPUT on the GPU: every call that takes the flag against fsr1_srtm(in, I, 0) followed by the same call without it,
bit for bit (torch.equal), with the kernel that ran, the launch count, and the caller's input unchanged byte for byte."""
import numpy as np
import pytest
import torch

import fsr1_b200 as F
from test_gpu_guards import Guarded, plain
from test_srtm_input import hdr_frame, sdr_frame

pytestmark = pytest.mark.gpu
api = F.api
S = api.FLAG_SRTM_INPUT
FRAMES = {"hdr": hdr_frame, "sdr": sdr_frame}
QUAD = "easu_h_quad2x<4w,7/sm,tma2,srtm_in>"
VPAIRS = "easu_h_vpairs<64x32,persistent,tma2,srtm_in>"
FUSED7 = "fused_easu_rcas_h_quad2x<4w,7/sm,tma2,strips,srtm_in>"


def _frame(kind, iw, ih, seed):
    """rows padded to 16 bytes (plain): odd widths such as 2953 still meet the tiled kernels' alignment"""
    return plain(FRAMES[kind](iw, ih, seed))


def _srtm(inp, height=None, row0=0):
    """I = fsr1_srtm(inp, I, 0) over inp's rows (a window: rows [row0, row0 + rows) of an image `height` tall)."""
    i = plain(np.zeros(tuple(inp.shape), np.float16))
    rows = inp.shape[0]
    api.srtm(api.image(inp, height=height, row0=row0), api.image(i, height=height, row0=row0), y0=row0, y1=row0 + rows)
    return i


class Call:
    """Runs fn(), then checks the launch count, the last kernel's name and that `inputs` kept every byte."""

    def __init__(self, *inputs):
        self.inputs = inputs
        self.before = [t.clone() for t in inputs]

    def run(self, fn, launches, name):
        n0 = api.launch_count()
        fn()
        torch.cuda.synchronize()
        got_n, got_name = api.launch_count() - n0, api.last_kernel()
        assert got_n == launches, (got_n, got_name)
        assert (got_name.startswith(name[:-1]) if name.endswith("*") else got_name == name), got_name
        for t, b in zip(self.inputs, self.before):
            assert torch.equal(t.view(torch.int16), b.view(torch.int16)), "the input was written"


def _out(oh, ow, fill=0.0):
    return torch.full((oh, ow, 4), fill, dtype=torch.float16, device="cuda")


# ---- fsr1_easu ---------------------------------------------------------------------------------------------------------------
EASU_SIZES = {"1080p-4k": (1920, 1080, 3840, 2160, QUAD), "1440p-4k": (2560, 1440, 3840, 2160, VPAIRS),
              "1.3x": (2953, 1661, 3840, 2160, VPAIRS), "aniso-1.5x2": (1280, 1080, 1920, 2160, VPAIRS)}


@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("size", list(EASU_SIZES))
def test_easu_equals_srtm_then_easu(size, frame):
    iw, ih, ow, oh, name = EASU_SIZES[size]
    inp = _frame(frame, iw, ih, iw + ih)
    con = api.easu_con(iw, ih, iw, ih, ow, oh)
    want = _out(oh, ow)
    api.easu(_srtm(inp), want, con)
    got = _out(oh, ow)
    Call(inp).run(lambda: api.easu(inp, got, con, flags=S), 1, name)
    assert torch.equal(got, want)


@pytest.mark.parametrize("size", ["1080p-4k", "1440p-4k"])
def test_easu_row_slab_on_an_input_window(size):
    iw, ih, ow, oh, name = EASU_SIZES[size]
    y0, y1 = 301, 777
    full = _frame("hdr", iw, ih, 5)
    con = api.easu_con(iw, ih, iw, ih, ow, oh)
    r0, r1 = api.easu_input_rows(con, ih, y0, y1)
    win = plain(full[r0:r1 + 1].cpu().numpy())
    want = _out(oh, ow, 3.0)
    api.easu(api.image(_srtm(win, ih, r0), height=ih, row0=r0), want, con, y0=y0, y1=y1)
    got = _out(oh, ow, 3.0)
    Call(win).run(lambda: api.easu(api.image(win, height=ih, row0=r0), got, con, y0=y0, y1=y1, flags=S), 1, name)
    assert torch.equal(got, want)
    assert (got[:y0] == 3.0).all() and (got[y1:] == 3.0).all()


# ---- fsr1_upscale ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("frame", list(FRAMES))
@pytest.mark.parametrize("size", [(1920, 1080, 3840, 2160), (3840, 2160, 7680, 4320)], ids=["1080p-4k", "2160p-8k"])
def test_fused_upscale_equals_srtm_then_upscale(size, frame):
    iw, ih, ow, oh = size
    inp = _frame(frame, iw, ih, 17)
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    tmp = _out(oh, ow)
    want = _out(oh, ow)
    api.upscale(_srtm(inp), tmp, want, econ, rcon, flags=api.FLAG_FUSED)
    got = _out(oh, ow)
    Call(inp).run(lambda: api.upscale(inp, tmp, got, econ, rcon, flags=api.FLAG_FUSED | S), 1, FUSED7)
    assert torch.equal(got, want)


TWO_KERNEL = {"clamp": (api.FLAG_RCAS_CLAMP, 2, "rcas_h_packed*"), "denoise": (api.FLAG_RCAS_DENOISE, 2, "rcas_h_packed*"),
              "passthrough_alpha": (api.FLAG_RCAS_PASSTHROUGH_ALPHA, 2, "rcas_h_packed*"),
              "output_square": (api.FLAG_OUTPUT_SQUARE, 2, "rcas_h_packed*"), "no_rcas": (api.FLAG_NO_RCAS, 1, QUAD),
              "plain_1.5x": (0, 2, "rcas_h_packed*")}


@pytest.mark.parametrize("case", list(TWO_KERNEL))
def test_two_kernel_upscale_equals_srtm_then_upscale(case):
    flags, launches, name = TWO_KERNEL[case]
    iw, ih, ow, oh = (640, 360, 960, 540) if case == "plain_1.5x" else (640, 360, 1280, 720)
    inp = _frame("hdr", iw, ih, 23)
    inp[..., 3] = torch.rand((ih, iw), device="cuda").half()               # alpha passes through with PASSTHROUGH_ALPHA
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    tmp = _out(oh, ow)
    want = _out(oh, ow)
    api.upscale(_srtm(inp), tmp, want, econ, rcon, flags=flags | api.FLAG_FUSED)
    got = _out(oh, ow)
    Call(inp).run(lambda: api.upscale(inp, tmp, got, econ, rcon, flags=flags | api.FLAG_FUSED | S), launches, name)
    assert torch.equal(got, want)


# ---- fsr1_upscale_post: the HDR round trip -----------------------------------------------------------------------------------
POST = {"rgba16f": (0, None), "tepd10": (10, None), "lfga_tepd8": (8, "grain")}


def _post_out(oh, ow, bits):
    if bits == 8:
        return torch.zeros((oh, ow, 4), dtype=torch.uint8, device="cuda")
    if bits == 10:
        return torch.zeros((oh, ow), dtype=torch.int32, device="cuda")
    return _out(oh, ow)


@pytest.mark.parametrize("case", list(POST))
@pytest.mark.parametrize("scale", ["2x", "1.5x", "2x-no-tmp"])
def test_upscale_post_round_trip_equals_srtm_then_upscale_post(case, scale):
    bits, g = POST[case]
    iw, ih = 960, 540
    ow, oh = (1440, 810) if scale == "1.5x" else (1920, 1080)
    inp = _frame("hdr", iw, ih, 29)
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    grain = torch.from_numpy((np.random.default_rng(3).random((7, 9, 4), np.float32) - 0.5).astype(np.float16)).cuda() if g else None
    tmp = None if scale == "2x-no-tmp" else _out(oh, ow)
    kw = dict(srtm_inverse=True, grain=grain, amount=0.3, tepd_bits=bits, frame=4)
    want = _post_out(oh, ow, bits)
    api.upscale_post(_srtm(inp), tmp, want, econ, rcon, flags=api.FLAG_FUSED, **kw)
    got = _post_out(oh, ow, bits)
    fmt = {0: "rgba16f", 8: "rgba8", 10: "rgb10a2"}[bits]
    fused = scale != "1.5x"
    name = "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,%s,srtm_in>" % fmt if fused else "rcas_h_packed_post*"
    Call(inp).run(lambda: api.upscale_post(inp, tmp, got, econ, rcon, flags=api.FLAG_FUSED | S, **kw), 1 if fused else 2, name)
    assert torch.equal(got, want)


# ---- fsr1_context_* ----------------------------------------------------------------------------------------------------------
def test_context_calls_equal_srtm_then_the_same_call():
    iw, ih, ow, oh = 960, 540, 1920, 1080
    inp = _frame("hdr", iw, ih, 31)
    ref = _srtm(inp)
    ctx = api.HostContext(iw, ih, ow, oh)
    try:
        c = Call(inp)
        want, got = _out(oh, ow), _out(oh, ow)
        ctx.upscale(ref, want, 0.5)
        c.run(lambda: ctx.upscale(inp, got, 0.5, flags=S), 1, FUSED7)
        assert torch.equal(got, want)
        # a smaller render size: not 2x, so EASU (the vpairs kernel with the prologue) + RCAS through the context's intermediate
        rw, rh = 701, 397
        sub_ref = _srtm(inp[:rh, :rw].contiguous())
        inp_pad = inp.clone()
        inp_pad[:rh, :rw] = sub_ref
        want, got = _out(oh, ow), _out(oh, ow)
        ctx.upscale_render(inp_pad, rw, rh, want, 0.5)
        c.run(lambda: ctx.upscale_render(inp, rw, rh, got, 0.5, flags=S), 2, "rcas_h_packed*")
        assert torch.equal(got, want)
        want, got = _post_out(oh, ow, 10), _post_out(oh, ow, 10)
        ctx.upscale_post(ref, want, sharpness=0.5, srtm_inverse=True, tepd_bits=10, frame=2)
        c.run(lambda: ctx.upscale_post(inp, got, sharpness=0.5, srtm_inverse=True, tepd_bits=10, frame=2, flags=S), 1,
              "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgb10a2,srtm_in>")
        assert torch.equal(got, want)
        hin, href = inp.cpu().pin_memory(), ref.cpu().pin_memory()
        hwant, hgot = torch.empty((oh, ow, 4), dtype=torch.float16).pin_memory(), torch.empty((oh, ow, 4), dtype=torch.float16).pin_memory()
        ctx.upscale_host(href, hwant, 0.5)
        hc = Call(hin)
        hc.run(lambda: ctx.upscale_host(hin, hgot, 0.5, flags=S), 1, FUSED7)
        assert torch.equal(hgot, hwant)
    finally:
        ctx.close()


# ---- fsr1_shard_* ------------------------------------------------------------------------------------------------------------
def _chain(frame, ow, oh):
    """The single-GPU chain: fsr1_srtm into a scratch image, then EASU + RCAS through an intermediate."""
    ih, iw = frame.shape[:2]
    i = _srtm(frame)
    tmp, out = _out(oh, ow), _out(oh, ow)
    api.easu(i, tmp, api.easu_con(iw, ih, iw, ih, ow, oh))
    api.rcas(tmp, out, api.rcas_con(0.25))
    return out


@pytest.mark.parametrize("shape,name", [((1920, 1080, 3840, 2160), FUSED7), ((1920, 1080, 2880, 1620), "rcas_h_packed*")],
                         ids=["1080p-4k-fused", "1.5x-two-kernels"])
def test_single_rank_shard_equals_the_chain(shape, name):
    iw, ih, ow, oh = shape
    slots = 3
    up = F.ShardedUpscaler(iw, ih, ow, oh, 1, 0, slots=slots, halo="p2p", flags=S)
    frames = [_frame("hdr", iw, ih, 40 + k) for k in range(slots)]
    s = torch.cuda.current_stream()
    try:
        for k in range(slots):
            up.input(k).copy_(frames[k])
            c = Call(up.input(k))
            c.run(lambda: up.submit(k, s), 1 if name == FUSED7 else 2, name)
        for k in range(slots):
            up.wait(k, s)
        torch.cuda.synchronize()
        up.status()
        for k in range(slots):
            assert torch.equal(up.input(k), frames[k]), "slot %d input" % k
            assert torch.equal(up.output(k), _chain(frames[k], ow, oh)), "slot %d" % k
    finally:
        up.close()


@pytest.mark.parametrize("world", [2, 8])
def test_ranks_on_one_device_run_the_fused_prologue_with_the_halo_inside(world):
    """The halo carries raw input rows; each rank transforms its window as it loads it.  6 CTAs per SM (the push kernel fits)."""
    iw, ih, ow, oh = 640, 360, 1280, 720
    nslots, nframes = 2, 4
    ups = [F.ShardedUpscaler(iw, ih, ow, oh, world, r, slots=nslots, halo="p2p", attach=False, flags=S) for r in range(world)]
    try:
        for r, u in enumerate(ups):
            u.attach_local(ups[r - 1] if r > 0 else None, ups[r + 1] if r + 1 < world else None)
        frames = [_frame("hdr", iw, ih, 60 + i) for i in range(nframes)]
        s = torch.cuda.current_stream()
        got = []
        for i, fr in enumerate(frames):
            k = i % nslots
            if i >= nslots:
                for u in ups:
                    u.wait(k, s)
                got.append(torch.cat([u.output(k) for u in ups]).clone())
            for r, u in enumerate(ups):
                o0, o1 = u.plan.owned_in_rows(r)
                u.input(k).copy_(fr[o0:o1])
            for u in ups:
                n0 = api.launch_count()
                u.submit(k, s)
                assert api.launch_count() == n0 + 1
                assert api.last_kernel() == "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,srtm_in>", api.last_kernel()
        for i in range(nframes - nslots, nframes):
            for u in ups:
                u.wait(i % nslots, s)
            got.append(torch.cat([u.output(i % nslots) for u in ups]).clone())
        torch.cuda.synchronize()
        for u in ups:
            u.status()
        for i in range(nframes):
            assert torch.equal(got[i], _chain(frames[i], ow, oh)), "frame %d" % i
    finally:
        for u in ups:
            u.close()


# ---- guards: the prologue variants inside poisoned allocations ---------------------------------------------------------------
GUARD_CASES = {"quad2x": (2.0, "easu"), "vpairs_1.5x": (1.5, "easu"), "fused": (2.0, "upscale"), "fused_post": (2.0, "post"),
               "rcas_post_1.5x": (1.5, "post")}
GUARD_SHAPES = [(1, 2), (61, 15), (125, 17), (129, 33)]


def _geometry(ow, oh, scale):
    from test_gpu_guards import easu_geometry
    return easu_geometry(ow, oh, scale)


def run_guarded(case, ow, oh, poison, y0=0, y1=None):
    scale, call = GUARD_CASES[case]
    y1 = oh if y1 is None else y1
    iw, ih, econ = _geometry(ow, oh, scale)
    rcon = api.rcas_con(0.25)
    src = hdr_frame(iw, ih, ow * 5 + oh)
    e0, e1 = (y0, y1) if call == "easu" else (max(y0 - 1, 0), min(y1 + 1, oh))
    r0, r1 = api.easu_input_rows(econ, ih, e0, e1)
    gin = Guarded("f16", r1 - r0 + 1, iw, poison, seed=21)
    gin.set(src[r0:r1 + 1])
    gtmp = Guarded("f16", oh, ow, poison, seed=22)
    gout = Guarded("f16", oh, ow, poison, seed=23)
    # the flag-free call on I = fsr1_srtm(src) allocated alone
    ref_in = _srtm(plain(src))
    want = plain(np.zeros((oh, ow, 4), np.float16))
    post_kw = dict(srtm_inverse=True, tepd_bits=0, frame=1)
    if call == "easu":
        api.easu(ref_in, want, econ, y0=y0, y1=y1)
        api.easu(gin.image(height=ih, row0=r0), gout.image(), econ, y0=y0, y1=y1, flags=S)
    elif call == "upscale":
        api.upscale(ref_in, plain(np.zeros((oh, ow, 4), np.float16)), want, econ, rcon, y0, y1, api.FLAG_FUSED)
        api.upscale(gin.image(height=ih, row0=r0), gtmp.image(), gout.image(), econ, rcon, y0, y1, api.FLAG_FUSED | S)
    else:
        api.upscale_post(ref_in, plain(np.zeros((oh, ow, 4), np.float16)), want, econ, rcon, y0=y0, y1=y1, flags=api.FLAG_FUSED, **post_kw)
        api.upscale_post(gin.image(height=ih, row0=r0), gtmp.image(), gout.image(), econ, rcon, y0=y0, y1=y1, flags=api.FLAG_FUSED | S,
                         **post_kw)
    torch.cuda.synchronize()
    what = (case, ow, oh, poison, y0, y1, api.last_kernel())
    assert "srtm_in" in api.last_kernel() or case == "rcas_post_1.5x", what
    assert np.array_equal(gout.numpy()[y0:y1].view(np.uint16), want.cpu().numpy()[y0:y1].view(np.uint16)), what
    gin.assert_untouched(what + ("input",))
    if case == "rcas_post_1.5x":
        gtmp.assert_untouched(what + ("tmp",), e0, e1)
    else:
        gtmp.assert_untouched(what + ("tmp",))
    gout.assert_untouched(what + ("output",), y0, y1)


@pytest.mark.parametrize("poison", ["nan", "big", "atlas"])
@pytest.mark.parametrize("case", list(GUARD_CASES))
def test_prologue_variants_stay_inside_their_images(case, poison):
    for ow, oh in GUARD_SHAPES:
        run_guarded(case, ow, oh, poison)
    run_guarded(case, 125, 33, poison, 3, 20)
    run_guarded(case, 1920, 1080, poison, 301, 777)
