"""Display output from the sharded frame stream on the GPU (fsr1_shard_create_post, fsr1_shard_post): every rank's slab equals, bit for
bit, the same rows of fsr1_context_upscale_post on the whole frame, for the fused 2x post kernel and for EASU + the RCAS post kernel, on
1, 2, 3 and 8 ranks in one process on one device (attach_local), on a dynamic shard, at 1080p -> 4K, and between two processes."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import fsr1_b200 as F
from fsr1_b200 import _lib
from test_srtm_input import hdr_frame

pytestmark = pytest.mark.gpu
api = F.api

S = api.FLAG_SRTM_INPUT
# op sets: constructor keywords of ShardedUpscaler (tiles by name), kernel flags, HDR input
OPS = {
    "srtm_inverse": (dict(srtm_inverse=True), 0, False),
    "lfga_tepd8": (dict(grain="grain", amount=0.375, tepd_bits=8), 0, False),       # positional dither
    "tepd10_tile": (dict(tepd_bits=10, dither="dither"), 0, False),
    "srtm_in_inverse_tepd10": (dict(srtm_inverse=True, tepd_bits=10), S, True),
}
FMT_TAG = {0: "rgba16f", 8: "rgba8", 10: "rgb10a2"}
SCALES = {"2x": (640, 360, 1280, 720), "1.5x": (640, 360, 960, 540)}


def _tiles():
    rng = np.random.default_rng(5)
    grain = torch.from_numpy((rng.random((5, 12, 4), np.float32) - 0.5).astype(np.float16)).cuda()       # 12 x 5 RGBA16F
    grain2 = torch.from_numpy((rng.random((7, 9, 4), np.float32) - 0.5).astype(np.float32)).cuda()       # 9 x 7 RGBA32F
    dither = torch.from_numpy(rng.random((3, 7, 4), np.float32) * 1.2 - 0.1).cuda()                      # .w saturated
    dither2 = torch.from_numpy(rng.random((4, 5, 4), np.float32).astype(np.float16)).cuda()
    return {"grain": grain, "grain2": grain2, "dither": dither, "dither2": dither2}


def _post_kw(name, tiles):
    kw, flags, hdr = OPS[name]
    return {k: tiles[v] if isinstance(v, str) else v for k, v in kw.items()}, flags, hdr


def _resources(iw, ih, n, seed, hdr=False):
    base = hdr_frame(iw, ih, seed) if hdr else F.to_half(F.uniform(iw, ih, seed))
    base = torch.from_numpy(np.ascontiguousarray(base)).cuda()
    return [torch.roll(base, 7 * t, dims=1).contiguous() for t in range(n)]


def _display(oh, ow, tepd_bits):
    if tepd_bits == 8:
        return torch.empty((oh, ow, 4), dtype=torch.uint8, device="cuda")
    if tepd_bits == 10:
        return torch.empty((oh, ow), dtype=torch.int32, device="cuda")
    return torch.empty((oh, ow, 4), dtype=torch.float16, device="cuda")


class Reference:
    """fsr1_context_upscale_post on the whole frame: the one-frame path every slab is held to."""

    def __init__(self, iw, ih, ow, oh):
        self.ctx = api.HostContext(iw, ih, ow, oh)
        self.ow, self.oh = ow, oh

    def __call__(self, res, rw, rh, sharp, kw, flags, frame=0):
        out = _display(self.oh, self.ow, kw.get("tepd_bits", 0))
        self.ctx.upscale_post(res, out, rw, rh, sharp, frame=frame, flags=flags, **kw)
        return out

    def close(self):
        self.ctx.close()


def _ranks(iw, ih, ow, oh, world, slots, **kw):
    ups = [F.ShardedUpscaler(iw, ih, ow, oh, world, r, slots=slots, halo="p2p", attach=False, **kw) for r in range(world)]
    for r, u in enumerate(ups):
        u.attach_local(ups[r - 1] if r > 0 else None, ups[r + 1] if r + 1 < world else None)
    return ups


def _bits(t):
    return t.contiguous().view(torch.uint8)


def _poison(t):
    """every pixel of an output slab set to a pattern no frame here produces in all of them (half NaN / 0xA5 bytes)"""
    if t.dtype == torch.float16:
        t.view(torch.int16).fill_(0x7E01)
    elif t.dtype == torch.uint8:
        t.fill_(0xA5)
    else:
        t.fill_(-0x5A5A5A5B)


def run_stream(ups, frames, nslots, kw, flags, poison=False):
    """frames: (resource, rw, rh, sharpness, post) with post = keywords of ShardedUpscaler.post (None: no description), frame i in
    slot i % nslots.  Checks the kernels every submit launched; returns each frame's gathered output."""
    s = torch.cuda.current_stream()
    ow, oh, world = ups[0].out_w, ups[0].out_h, len(ups)
    bits = kw.get("tepd_bits", 0)
    got, pending = [None] * len(frames), {}
    for i, (res, rw, rh, sharp, post) in enumerate(frames):
        k = i % nslots
        if k in pending:
            for u in ups:
                u.wait(k, s)
            got[pending.pop(k)] = torch.cat([u.output(k) for u in ups]).clone()
        if poison:
            for u in ups:
                _poison(u.output(k))
        plan = F.SlabPlan(rh, oh, world, api.easu_con(rw, rh, rw, rh, ow, oh))
        for r, u in enumerate(ups):
            if post is not None:
                u.post(k, **post)
            owned = u.frame(k, rw, rh, sharp) if u.dynamic else u.input(k)
            o0, o1 = plan.owned_in_rows(r)
            owned.copy_(res[o0:o1, :rw])
        for u in ups:
            n0 = api.launch_count()
            u.submit(k, s)
            n, name = api.launch_count() - n0, api.last_kernel()
            if 2 * rw == ow and 2 * rh == oh:
                assert n == 1 and name.startswith("fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,%s" % FMT_TAG[bits]), (i, n, name)
                assert ("srtm_in" in name) == bool(flags & S), name
            else:
                assert n == 2 and name == "rcas_h_packed_post<2px,4rows,shfl60,%s>" % FMT_TAG[bits], (i, rw, rh, n, name)
        pending[k] = i
    for k, i in pending.items():
        for u in ups:
            u.wait(k, s)
        got[i] = torch.cat([u.output(k) for u in ups]).clone()
    torch.cuda.synchronize()
    for u in ups:
        u.status()
    return got


def _check(got, frames, ref, kw, flags):
    for i, (res, rw, rh, sharp, post) in enumerate(frames):
        use = dict(kw)
        frame = 0
        if post:
            post = dict(post)
            frame = post.pop("frame", 0)
            use.update({k: v for k, v in post.items() if v is not None})
        want = ref(res, rw, rh, sharp, use, flags, frame)
        assert torch.equal(_bits(got[i]), _bits(want)), "frame %d (%dx%d)" % (i, rw, rh)


@pytest.mark.parametrize("ops", list(OPS))
@pytest.mark.parametrize("scale", list(SCALES))
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_slabs_equal_the_context_call(world, scale, ops):
    iw, ih, ow, oh = SCALES[scale]
    tiles = _tiles()
    kw, flags, hdr = _post_kw(ops, tiles)
    nslots, nframes = 2, 4
    res = _resources(iw, ih, 3, 61 + world, hdr)
    frames = [(res[i % 3], iw, ih, 0.25, {"frame": 3 * i + 1}) for i in range(nframes)]
    ups, ref = _ranks(iw, ih, ow, oh, world, nslots, flags=flags, **kw), Reference(iw, ih, ow, oh)
    try:
        bits = kw.get("tepd_bits", 0)
        for r, u in enumerate(ups):                               # slabs in the display format: 4 B/px with TEPD
            out = u.output(0)
            y0, y1 = u.plan.out_rows(r)
            assert out.dtype == {0: torch.float16, 8: torch.uint8, 10: torch.int32}[bits] and out.shape[:2] == (y1 - y0, ow)
            assert out.stride(0) * out.element_size() == -(-ow * (4 if bits else 8) // 128) * 128
        got = run_stream(ups, frames, nslots, kw, flags)
        _check(got, frames, ref, kw, flags)
    finally:
        ref.close()
        for u in ups:
            u.close()


@pytest.mark.parametrize("scale", list(SCALES))
def test_the_hand_shake_rides_inside_the_post_kernels(scale):
    """trace stamps [0] (wait began), [1] (halo present) and [2] (last CTA done, credit sent) come from the kernel that reads the window:
    the fused post kernel at 2x, the tiled EASU kernel before the RCAS post kernel otherwise; halo_wait_kernel sets none of them."""
    iw, ih, ow, oh = SCALES[scale]
    tiles = _tiles()
    kw, flags, _ = _post_kw("lfga_tepd8", tiles)
    world, nslots, nframes = 3, 2, 6
    res = _resources(iw, ih, 2, 17)
    frames = [(res[i % 2], iw, ih, 0.25, None) for i in range(nframes)]
    ups = _ranks(iw, ih, ow, oh, world, nslots, trace=True, flags=flags, **kw)
    try:
        run_stream(ups, frames, nslots, kw, flags)
        for u in ups:
            tr = u.trace().astype(np.int64)
            assert tr.shape == (nframes, 8)
            assert (tr[:, :3] > 0).all(), tr
            assert (tr[:, 1] >= tr[:, 0]).all() and (tr[:, 2] >= tr[:, 1]).all(), tr
    finally:
        for u in ups:
            u.close()


@pytest.mark.parametrize("scale", list(SCALES))
def test_each_use_of_a_slot_has_its_own_description(scale):
    """fsr1_shard_post per use: the TEPD frame, the LFGA amount and the grain tile change from one use of a slot to the next; each frame
    equals the context call with that description, and a different `frame` changes the output."""
    iw, ih, ow, oh = SCALES[scale]
    tiles = _tiles()
    kw, flags, _ = _post_kw("lfga_tepd8", tiles)
    world, nslots = 2, 2
    res = _resources(iw, ih, 1, 23)[0]
    posts = [{"frame": 0}, {"frame": 1}, {"frame": 1, "amount": 0.125}, {"frame": 7, "grain": tiles["grain2"]},
             {"frame": 2, "amount": 0.5, "grain": tiles["grain"]}, None, {"frame": 0}]
    frames = [(res, iw, ih, 0.25, p) for p in posts]
    ups, ref = _ranks(iw, ih, ow, oh, world, nslots, **kw), Reference(iw, ih, ow, oh)
    try:
        got = run_stream(ups, frames, nslots, kw, flags)
        # frame 5 has no description: slot 1 keeps that of frame 3
        frames[5] = (res, iw, ih, 0.25, posts[3])
        _check(got, frames, ref, kw, flags)
        assert not torch.equal(got[0], got[1])                  # the positional dither moves with `frame`
        assert torch.equal(got[0], got[6])
    finally:
        ref.close()
        for u in ups:
            u.close()


def test_post_refusals_launch_nothing_and_keep_the_description():
    L = _lib.lib()
    iw, ih, ow, oh = SCALES["2x"]
    tiles = _tiles()
    kw, flags, _ = _post_kw("lfga_tepd8", tiles)
    plain = F.ShardedUpscaler(iw, ih, ow, oh, 1, 0, slots=2, halo="p2p")
    u = F.ShardedUpscaler(iw, ih, ow, oh, 1, 0, slots=2, halo="p2p", **kw)
    tepd10 = F.ShardedUpscaler(iw, ih, ow, oh, 1, 0, slots=1, halo="p2p", tepd_bits=10)
    try:
        grain = api.image(tiles["grain"])
        win = api.image(tiles["grain"][1:3], height=5, row0=1)
        good = _lib.Post(_lib.POST_LFGA | _lib.POST_TEPD8, 0.25, ctypes.pointer(grain), None, 9, 0)
        n0 = api.launch_count()
        assert L.fsr1_shard_post(plain._shard, 0, ctypes.byref(good)) == -1            # created without post
        with pytest.raises(ValueError):
            plain.post(0, frame=1)
        assert L.fsr1_shard_post(tepd10._shard, 0, ctypes.byref(good)) == -1           # other ops
        for ops in (_lib.POST_TEPD8, _lib.POST_LFGA | _lib.POST_TEPD10, _lib.POST_LFGA | _lib.POST_TEPD8 | _lib.POST_SRTM_INVERSE):
            bad = _lib.Post(ops, 0.25, ctypes.pointer(grain), None, 9, 0)
            assert L.fsr1_shard_post(u._shard, 0, ctypes.byref(bad)) == -1, ops
        assert L.fsr1_shard_post(u._shard, 2, ctypes.byref(good)) == -1                # bad slot
        assert L.fsr1_shard_post(u._shard, 0, None) == -1
        nogr = _lib.Post(_lib.POST_LFGA | _lib.POST_TEPD8, 0.25, None, None, 9, 0)
        assert L.fsr1_shard_post(u._shard, 0, ctypes.byref(nogr)) == -1                # LFGA without a grain tile
        wpost = _lib.Post(_lib.POST_LFGA | _lib.POST_TEPD8, 0.25, ctypes.pointer(win), None, 9, 0)
        assert L.fsr1_shard_post(u._shard, 0, ctypes.byref(wpost)) == -1               # a tile that is a window
        u8 = api.image(torch.zeros((2, 2, 4), dtype=torch.uint8, device="cuda"))
        upost = _lib.Post(_lib.POST_LFGA | _lib.POST_TEPD8, 0.25, ctypes.pointer(u8), None, 9, 0)
        assert L.fsr1_shard_post(u._shard, 0, ctypes.byref(upost)) == -2               # grain must be a float tile
        assert api.launch_count() == n0
        # the slot kept its create-time description: frame 0, the constructor's amount and grain
        res = _resources(iw, ih, 1, 3)[0]
        got = run_stream([u], [(res, iw, ih, 0.25, None)], 1, kw, flags)
        ref = Reference(iw, ih, ow, oh)
        try:
            _check(got, [(res, iw, ih, 0.25, None)], ref, kw, flags)
        finally:
            ref.close()
    finally:
        for x in (plain, u, tepd10):
            x.close()


@pytest.mark.parametrize("ops", ["lfga_tepd8", "srtm_in_inverse_tepd10"])
def test_dynamic_shard_with_post_eight_ranks(ops):
    """Render sizes cycle through 2x, other scales and the thinnest accepted heights after tall ones; every slab pixel is poisoned before
    its frame and must come out written and equal to the context call."""
    iw, ih, ow, oh, world = 640, 360, 1280, 720, 8
    tiles = _tiles()
    kw, flags, hdr = _post_kw(ops, tiles)
    sizes = [(640, 360), (500, 300), (40, 26), (333, 217), (640, 360), (64, 27), (480, 270), (50, 28), (639, 359), (48, 30)]
    res = _resources(iw, ih, 3, 47, hdr)
    frames = [(res[i % 3], *sizes[i], [0.25, 0.0, 1.0, 0.5][i % 4], {"frame": i}) for i in range(len(sizes))]
    ups, ref = _ranks(iw, ih, ow, oh, world, 2, dynamic=True, flags=flags, **kw), Reference(iw, ih, ow, oh)
    try:
        got = run_stream(ups, frames, 2, kw, flags, poison=True)
        _check(got, frames, ref, kw, flags)
    finally:
        ref.close()
        for u in ups:
            u.close()


def test_1080p_to_4k_eight_ranks_on_one_device():
    """2x fused-post frames of 1920x1080 -> 3840x2160 through 8 slots on 8 ranks sharing one GPU: the one-warp halo push must fit beside
    the six post CTAs per SM of every rank.  The stream runs its normal schedule and ends with fsr1_shard_status OK."""
    iw, ih, ow, oh, world, nslots, nframes = 1920, 1080, 3840, 2160, 8, 8, 40
    tiles = _tiles()
    kw, flags, _ = _post_kw("lfga_tepd8", tiles)
    res = _resources(iw, ih, 2, 71)
    frames = [(res[i % 2], iw, ih, 0.25, {"frame": i}) for i in range(nframes)]
    ups, ref = _ranks(iw, ih, ow, oh, world, nslots, **kw), Reference(iw, ih, ow, oh)
    try:
        got = run_stream(ups, frames, nslots, kw, flags)            # ends with status() on every rank
        _check(got[-2:], frames[-2:], ref, kw, flags)
    finally:
        ref.close()
        for u in ups:
            u.close()


def _ipc_worker(rank, world, port, shape, tmpdir):
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch.distributed as dist
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)      # only carries the 64-byte IPC handles
    iw, ih, ow, oh = shape
    nslots, nframes = 2, 4
    up = F.ShardedUpscaler(iw, ih, ow, oh, world, rank, slots=nslots, halo="p2p", device=dev, tepd_bits=8)
    o0, o1 = up.plan.owned_in_rows(rank)
    s = torch.cuda.current_stream()
    outs = []
    for i in range(nframes):
        k = i % nslots
        if i >= nslots:
            up.wait(k, s)
            outs.append(up.output(k).clone())
        up.post(k, frame=5 * i)
        up.input(k).copy_(torch.from_numpy(F.to_half(F.uniform(iw, ih, 800 + i))[o0:o1].copy()).to(dev))
        up.submit(k, s)
    for i in range(nframes - nslots, nframes):
        up.wait(i % nslots, s)
        outs.append(up.output(i % nslots).clone())
    torch.cuda.synchronize()
    up.status()
    np.save(os.path.join(tmpdir, "slab%d.npy" % rank), torch.stack(outs).cpu().numpy())
    dist.barrier()
    up.close()
    dist.destroy_process_group()


def test_two_processes_over_cuda_ipc_tepd8(tmp_path):
    shape = (320, 180, 640, 360)
    world = 2
    port = 36500 + (os.getpid() % 2000)
    mp.spawn(_ipc_worker, args=(world, port, shape, str(tmp_path)), nprocs=world, join=True)
    iw, ih, ow, oh = shape
    got = np.concatenate([np.load(os.path.join(str(tmp_path), "slab%d.npy" % r)) for r in range(world)], axis=1)
    ref = Reference(iw, ih, ow, oh)
    try:
        for i in range(got.shape[0]):
            res = torch.from_numpy(F.to_half(F.uniform(iw, ih, 800 + i))).cuda()
            want = ref(res, iw, ih, 0.25, {"tepd_bits": 8}, 0, 5 * i)
            assert np.array_equal(got[i], want.cpu().numpy()), "frame %d" % i
    finally:
        ref.close()
