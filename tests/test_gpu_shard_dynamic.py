"""Dynamic resolution in the sharded frame stream on the GPU (FSR1_SHARD_DYNAMIC, fsr1_shard_frame): every frame of the stream has
its own render size and sharpness, slots are reused with a different size on consecutive uses, and each frame equals the one-frame
fsr1_context_upscale_render of the same render region bit for bit, on one rank and on 2 and 8 ranks in one process."""
import ctypes

import numpy as np
import pytest
import torch

import fsr1_b200 as F
from fsr1_b200 import _lib
from fsr1_b200.sharded import _tensor_of
from test_gpu_guards import POISON_BITS
from test_shard_dynamic import accepted_heights, capacity, frame_plan, neighbours_only
from test_srtm_input import hdr_frame

pytestmark = pytest.mark.gpu
api = F.api

# render sizes of a 1920x1080 resource upscaled to 3840x2160: exactly 2x, 1.5x, 2x-and-a-bit, an odd size, and almost 2x
CYCLE_4K = [(1920, 1080), (1600, 900), (1280, 720), (1477, 831), (1919, 1079)]
# the same shapes for a 640x360 resource upscaled to 1280x720
CYCLE_720 = [(640, 360), (500, 300), (333, 217), (639, 359), (480, 270)]
SHARPNESS = [0.25, 0.0, 1.0, 0.5, 2.0, 0.125, 1.5]


def _resources(iw, ih, n, seed, hdr=False):
    """n distinct resources on the device (rows padded to 16 bytes): one frame rolled by a different number of columns each."""
    base = hdr_frame(iw, ih, seed) if hdr else F.to_half(F.uniform(iw, ih, seed))
    base = torch.from_numpy(np.ascontiguousarray(base)).cuda()
    return [torch.roll(base, 7 * t, dims=1).contiguous() for t in range(n)]


class Reference:
    """fsr1_context_upscale_render of the same render region: the one-frame path the stream is held to."""

    def __init__(self, iw, ih, ow, oh):
        self.ctx = api.HostContext(iw, ih, ow, oh)
        self.ow, self.oh = ow, oh

    def __call__(self, res, rw, rh, sharp, flags=0):
        out = torch.empty((self.oh, self.ow, 4), dtype=torch.float16, device="cuda")
        self.ctx.upscale_render(res, rw, rh, out, sharp, flags)
        return out

    def close(self):
        self.ctx.close()


def _ranks(iw, ih, ow, oh, world, slots, **kw):
    ups = [F.ShardedUpscaler(iw, ih, ow, oh, world, r, slots=slots, halo="p2p", attach=False, **kw) for r in range(world)]
    for r, u in enumerate(ups):
        u.attach_local(ups[r - 1] if r > 0 else None, ups[r + 1] if r + 1 < world else None)
    return ups


def _slot_memory(u, k):
    """The whole of slot k's window capacity as a half tensor (the rows of every frame size, and those beyond)."""
    pitch = u.inputs[k].stride(0) * 2
    rows = (u.info.arena_bytes - 4096) // u.slots // pitch
    img = _lib.Image(u.windows[k].data_ptr(), pitch, pitch // 8, rows, 0, rows, _lib.FORMAT_RGBA16F, 0)
    return _tensor_of(img, u.device)


def _poison16(poison):
    """the poison's half bit pattern as an int16 fill value"""
    b = POISON_BITS[poison]["f16"]
    return b - (1 << 16) if b >= 1 << 15 else b


def _is_2x(rw, rh, ow, oh):
    return 2 * rw == ow and 2 * rh == oh


def run_stream(ups, frames, nslots, describe=True, poison=None, flags=0):
    """Feeds frames (resource, rw, rh, sharpness) through the ranks, frame i in slot i % nslots, and returns each frame's gathered
    output.  Checks the rows every rank was given and the kernels every submit launched.  poison: fill each rank's whole slot
    with that bit pattern before the frame is written."""
    world, s = len(ups), torch.cuda.current_stream()
    ow, oh = ups[0].out_w, ups[0].out_h
    got, pending = [None] * len(frames), {}
    for i, (res, rw, rh, sharp) in enumerate(frames):
        k = i % nslots
        if k in pending:                                  # collect the slot's previous frame before reusing it
            for u in ups:
                u.wait(k, s)
            got[pending.pop(k)] = torch.cat([u.output(k) for u in ups]).clone()
        if poison:
            for u in ups:
                _slot_memory(u, k).view(torch.int16).fill_(_poison16(poison))
        plan = frame_plan(rw, rh, ow, oh, world)
        for r, u in enumerate(ups):
            owned = u.frame(k, rw, rh, sharp) if describe else u.input(k)
            o0, o1 = plan.owned_in_rows(r)
            w0, w1 = plan.window_rows(r)
            assert tuple(owned.shape) == (o1 - o0, rw, 4) and tuple(u.windows[k].shape) == (w1 - w0, rw, 4)
            assert owned.data_ptr() == u.windows[k].data_ptr() + (o0 - w0) * owned.stride(0) * 2
            owned.copy_(res[o0:o1, :rw])
        for u in ups:
            n0 = api.launch_count()
            u.submit(k, s)
            n, name = api.launch_count() - n0, api.last_kernel()
            if _is_2x(rw, rh, ow, oh):
                assert n == 1 and name.startswith("fused_easu_rcas_h_quad2x<4w,%d/sm" % (7 if world == 1 else 6)), (i, n, name)
                assert ("srtm_in" in name) == bool(flags & api.FLAG_SRTM_INPUT), name
            else:
                assert n == 2 and name.startswith("rcas_h_packed"), (i, rw, rh, n, name)
        pending[k] = i
    for k, i in pending.items():
        for u in ups:
            u.wait(k, s)
        got[i] = torch.cat([u.output(k) for u in ups]).clone()
    torch.cuda.synchronize()
    for u in ups:
        u.status()
    return got


def _bits(t):
    return t.contiguous().view(torch.int16)


def _check(got, frames, ref, flags=0):
    for i, (res, rw, rh, sharp) in enumerate(frames):
        want = ref(res, rw, rh, sharp, flags)
        assert torch.equal(_bits(got[i]), _bits(want)), "frame %d (%dx%d, sharpness %g)" % (i, rw, rh, sharp)


def test_one_rank_eight_slots_every_render_size():
    iw, ih, ow, oh = 1920, 1080, 3840, 2160
    nslots, nframes = 8, 24                               # slot k's uses i, i + 8, i + 16 have three different render sizes
    res = _resources(iw, ih, 6, 31)
    frames = [(res[i % 6], *CYCLE_4K[i % 5], SHARPNESS[i % 7]) for i in range(nframes)]
    ups, ref = _ranks(iw, ih, ow, oh, 1, nslots, dynamic=True), Reference(iw, ih, ow, oh)
    try:
        got = run_stream(ups, frames, nslots)
        _check(got, frames, ref)
    finally:
        ref.close()
        for u in ups:
            u.close()


@pytest.mark.parametrize("world", [2, 8])
def test_ranks_on_one_device_every_render_size(world):
    iw, ih, ow, oh = 640, 360, 1280, 720
    nslots, nframes = 2, 11
    res = _resources(iw, ih, 4, 77)
    frames = [(res[i % 4], *CYCLE_720[i % 5], SHARPNESS[i % 7]) for i in range(nframes)]
    ups, ref = _ranks(iw, ih, ow, oh, world, nslots, dynamic=True), Reference(iw, ih, ow, oh)
    try:
        pitch = ups[0].inputs[0].stride(0) * 2
        cap = capacity(iw, ih, ow, oh, world)
        for u in ups:                                     # every slot sized for the tallest window of any accepted height
            assert u.info.arena_bytes == 4096 + nslots * (-(-cap * pitch // 256) * 256)
        got = run_stream(ups, frames, nslots)
        _check(got, frames, ref)
    finally:
        ref.close()
        for u in ups:
            u.close()


def test_eight_ranks_thinnest_accepted_frames_after_tall_ones_in_one_slot():
    """One slot, so every use changes height: the thinnest heights a dynamic shard accepts at 8 ranks (26-30 rows, a few per rank)
    after taller frames, each still the one-frame result; poison shows any row that went stale."""
    iw, ih, ow, oh, world = 640, 360, 1280, 720, 8
    sizes = [(180, 100), (40, 26), (333, 217), (64, 27), (640, 360), (50, 28), (120, 100), (44, 29), (639, 359), (48, 30)]
    assert min(accepted_heights(iw, ih, ow, oh, world)) == 26
    res = _resources(iw, ih, 3, 19)
    frames = [(res[i % 3], *sizes[i], SHARPNESS[i % 7]) for i in range(len(sizes))]
    ups, ref = _ranks(iw, ih, ow, oh, world, 1, dynamic=True), Reference(iw, ih, ow, oh)
    try:
        got = run_stream(ups, frames, 1, poison="nan")
        _check(got, frames, ref)
    finally:
        ref.close()
        for u in ups:
            u.close()


@pytest.mark.parametrize("poison", ["nan", "big"])
@pytest.mark.parametrize("world", [1, 2])
def test_poison_outside_the_frame_changes_nothing(world, poison):
    """The resource outside the render region and every byte of each slot's window capacity hold NaN (or 65504) before each frame:
    a stale halo row of a taller previous frame, or a tap outside the render region, would show."""
    iw, ih, ow, oh = 640, 360, 1280, 720
    nslots, nframes = 2, 10
    clean = _resources(iw, ih, 3, 91)
    frames = [(clean[i % 3], *CYCLE_720[i % 5], SHARPNESS[i % 7]) for i in range(nframes)]
    ups, ref = _ranks(iw, ih, ow, oh, world, nslots, dynamic=True), Reference(iw, ih, ow, oh)
    try:
        got = run_stream(ups, frames, nslots, poison=poison)
        _check(got, frames, ref)
        # the one-frame path agrees on a resource poisoned outside the region
        for res, rw, rh, sharp in frames[:5]:
            p = torch.empty_like(res).view(torch.int16).fill_(_poison16(poison)).view(torch.float16)
            p[:rh, :rw] = res[:rh, :rw]
            assert torch.equal(_bits(ref(p, rw, rh, sharp)), _bits(ref(res, rw, rh, sharp)))
    finally:
        ref.close()
        for u in ups:
            u.close()


@pytest.mark.parametrize("world", [1, 2])
def test_srtm_input_on_a_dynamic_shard(world):
    iw, ih, ow, oh = 640, 360, 1280, 720
    S = api.FLAG_SRTM_INPUT
    nslots, nframes = 2, 7
    res = _resources(iw, ih, 3, 43, hdr=True)
    frames = [(res[i % 3], *CYCLE_720[i % 5], SHARPNESS[i % 7]) for i in range(nframes)]
    ups, ref = _ranks(iw, ih, ow, oh, world, nslots, dynamic=True, flags=S), Reference(iw, ih, ow, oh)
    try:
        got = run_stream(ups, frames, nslots, flags=S)
        _check(got, frames, ref, flags=S)
    finally:
        ref.close()
        for u in ups:
            u.close()


def test_refusals_launch_nothing_and_keep_the_description():
    L = _lib.lib()
    iw, ih, ow, oh, world = 640, 360, 1280, 720, 8
    f = ctypes.c_float(0.25)
    static = F.ShardedUpscaler(iw, ih, ow, oh, 1, 0, slots=2, halo="p2p")
    ups = _ranks(iw, ih, ow, oh, world, 2, dynamic=True)
    try:
        n0 = api.launch_count()
        assert L.fsr1_shard_frame(static._shard, 0, 320, 180, f) == -1          # created without FSR1_SHARD_DYNAMIC
        with pytest.raises(ValueError):
            static.frame(0, 320, 180)
        h = ups[3]._shard
        before = ups[3].input(1)
        assert L.fsr1_shard_frame(h, 2, 320, 180, f) == -1                      # bad slot
        assert L.fsr1_shard_frame(h, 1, 0, 180, f) == -1                        # zero render size
        assert L.fsr1_shard_frame(h, 1, 320, 0, f) == -1
        assert L.fsr1_shard_frame(h, 1, iw + 1, 180, f) == -1                   # larger than the resource
        assert L.fsr1_shard_frame(h, 1, 320, ih + 1, f) == -1
        assert L.fsr1_shard_frame(h, 1, 320, world - 1, f) == -1                # world > render height
        accepted = set(accepted_heights(iw, ih, ow, oh, world))
        thin = [rh for rh in range(world, ih + 1) if rh not in accepted]
        assert thin and not neighbours_only(frame_plan(320, min(thin), ow, oh, world))
        assert neighbours_only(frame_plan(320, 21, ow, oh, world)) and 21 in thin
        for rh in (min(thin), 21, max(thin)):     # halo from beyond the neighbours; rows a push of another height reads
            assert L.fsr1_shard_frame(h, 1, 320, rh, f) == -2, rh
        with pytest.raises(_lib.Fsr1Error):
            ups[3].frame(1, 320, max(thin))
        assert api.launch_count() == n0
        a = _lib.Image()
        assert L.fsr1_shard_input(h, 1, ctypes.byref(a)) == 0                   # the slot kept its description
        assert (a.data, a.width, a.height, a.rows) == (before.data_ptr(), iw, ih, before.shape[0])
        assert L.fsr1_shard_frame(h, 1, 320, max(thin) + 1, f) == 0            # the first accepted height
        assert api.launch_count() == n0
    finally:
        static.close()
        for u in ups:
            u.close()


@pytest.mark.parametrize("shape,world", [((1920, 1080, 3840, 2160), 1), ((640, 360, 1280, 720), 2), ((2560, 1440, 3840, 2160), 1)],
                         ids=["1080p-4k", "360p-720p-2ranks", "1440p-4k"])
def test_an_undescribed_dynamic_shard_launches_what_a_static_shard_launches(shape, world):
    iw, ih, ow, oh = shape
    nslots, nframes = 2, 4
    res = _resources(iw, ih, nframes, 55)
    outs, launches = {}, {}
    for dynamic in (False, True):
        ups = _ranks(iw, ih, ow, oh, world, nslots, dynamic=dynamic)
        try:
            seen = []
            s = torch.cuda.current_stream()
            got = []
            for i in range(nframes):
                k = i % nslots
                if i >= nslots:
                    for u in ups:
                        u.wait(k, s)
                    got.append(torch.cat([u.output(k) for u in ups]).clone())
                for r, u in enumerate(ups):
                    o0, o1 = u.plan.owned_in_rows(r)
                    u.input(k).copy_(res[i][o0:o1])
                for u in ups:
                    n0 = api.launch_count()
                    u.submit(k, s)
                    seen.append((api.launch_count() - n0, api.last_kernel()))
            for i in range(nframes - nslots, nframes):
                for u in ups:
                    u.wait(i % nslots, s)
                got.append(torch.cat([u.output(i % nslots) for u in ups]).clone())
            torch.cuda.synchronize()
            for u in ups:
                u.status()
            outs[dynamic], launches[dynamic] = got, seen
        finally:
            for u in ups:
                u.close()
    assert launches[True] == launches[False]
    for a, b in zip(outs[True], outs[False]):
        assert torch.equal(_bits(a), _bits(b))
