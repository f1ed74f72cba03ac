"""The fused EASU->RCAS kernel as the default of the schedules that own their intermediate (fsr1_shard_*): 2x RGBA16F frames
without RCAS options run as one fused kernel per frame, every other frame still as EASU + RCAS, and either way the output is
the two-kernel result bit for bit.  The emulator part runs the fused kernel's device code (interior and border steps) on the CPU."""
import ctypes

import numpy as np
import pytest
import torch

import fsr1_b200 as F
import oracle_lib as ol
from test_emu import PROD, emu_easu, emu_lib, emu_rcas

api = F.api


def _frames(iw, ih, n, seed, dtype=torch.float16):
    """n distinct frames on the device: one LCG frame rolled by a different number of columns each."""
    f = F.uniform(iw, ih, seed)
    if dtype == torch.uint8:
        base = torch.from_numpy(np.floor(f * 255.0 + 0.5).astype(np.uint8)).cuda()
    else:
        base = torch.from_numpy(f).cuda().to(dtype)
    return [torch.roll(base, 7 * t, dims=1).contiguous() for t in range(n)]


def _two_kernels(frame, ow, oh, flags=0):
    """api.easu then api.rcas through an intermediate: the reference the library's schedules are held to."""
    ih, iw = frame.shape[:2]
    tmp = torch.empty((oh, ow, 4), dtype=frame.dtype, device=frame.device)
    out = torch.empty_like(tmp)
    api.easu(frame, tmp, api.easu_con(iw, ih, iw, ih, ow, oh), flags=flags)
    api.rcas(tmp, out, api.rcas_con(0.25), flags=flags)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(1920, 1080, 3840, 2160), (3840, 2160, 7680, 4320)], ids=["1080p-4k", "2160p-8k"])
def test_shard_runs_each_2x_fp16_frame_as_one_fused_kernel(shape):
    iw, ih, ow, oh = shape
    slots = 8
    up = F.ShardedUpscaler(iw, ih, ow, oh, 1, 0, slots=slots, halo="p2p")
    frames = _frames(iw, ih, slots, 31)
    s = torch.cuda.current_stream()
    for k in range(slots):
        up.input(k).copy_(frames[k])
    for k in range(slots):
        n0 = api.launch_count()
        up.submit(k, s)
        assert api.launch_count() == n0 + 1
        assert api.last_kernel().startswith("fused_easu_rcas_h"), api.last_kernel()
    for k in range(slots):
        up.wait(k, s)
    torch.cuda.synchronize()
    up.status()
    for k in range(slots):
        assert torch.equal(up.output(k), _two_kernels(frames[k], ow, oh)), "slot %d" % k
    up.close()


TWO_KERNEL_CASES = [
    ((2560, 1440, 3840, 2160), torch.float16, 0, "rcas_h_packed"),             # 1.5x: no fused kernel at this scale
    ((480, 270, 960, 540), torch.float32, 0, "rcas_f32_packed"),
    ((480, 270, 960, 540), torch.uint8, 0, "rcas_u8_packed"),
    ((480, 270, 960, 540), torch.float16, api.FLAG_RCAS_DENOISE, "rcas_h_packed"),
    ((480, 270, 960, 540), torch.float16, api.FLAG_RCAS_CLAMP, "rcas_h_packed"),
    ((480, 270, 960, 540), torch.float16, api.FLAG_RCAS_PASSTHROUGH_ALPHA, "rcas_h_packed"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("shape,dtype,flags,rcas_kernel", TWO_KERNEL_CASES,
                         ids=["1440p-4k-f16", "f32", "u8", "denoise", "clamp", "passthrough-alpha"])
def test_shard_frames_the_fused_kernel_does_not_cover_stay_on_two_kernels(shape, dtype, flags, rcas_kernel):
    iw, ih, ow, oh = shape
    slots = 2
    up = F.ShardedUpscaler(iw, ih, ow, oh, 1, 0, dtype=dtype, flags=flags, slots=slots, halo="p2p")
    frames = _frames(iw, ih, slots, 47, dtype)
    s = torch.cuda.current_stream()
    for k in range(slots):
        up.input(k).copy_(frames[k])
        n0 = api.launch_count()
        up.submit(k, s)
        assert api.launch_count() == n0 + 2
        assert api.last_kernel().startswith(rcas_kernel), api.last_kernel()
    for k in range(slots):
        up.wait(k, s)
    torch.cuda.synchronize()
    up.status()
    for k in range(slots):
        assert torch.equal(up.output(k), _two_kernels(frames[k], ow, oh, flags)), "slot %d" % k
    up.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 8])
def test_ranks_on_one_device_run_the_fused_kernel_with_the_halo_inside(world):
    """Several ranks in one process on one device: the fused kernel carries the halo hand-shake (6 CTAs per SM so the push
    kernel fits beside it), slots are reused, and the frame equals the single-GPU two-kernel frame bit for bit."""
    iw, ih, ow, oh = 640, 360, 1280, 720
    nslots, nframes = 2, 5
    ups = [F.ShardedUpscaler(iw, ih, ow, oh, world, r, slots=nslots, halo="p2p", attach=False) for r in range(world)]
    for r, u in enumerate(ups):
        u.attach_local(ups[r - 1] if r > 0 else None, ups[r + 1] if r + 1 < world else None)
    frames = _frames(iw, ih, nframes, 77)
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
            assert api.last_kernel().startswith("fused_easu_rcas_h_quad2x<4w,6/sm"), api.last_kernel()
    for i in range(nframes - nslots, nframes):
        for u in ups:
            u.wait(i % nslots, s)
        got.append(torch.cat([u.output(i % nslots) for u in ups]).clone())
    torch.cuda.synchronize()
    for u in ups:
        u.status()
    for i in range(nframes):
        assert torch.equal(got[i], _two_kernels(frames[i], ow, oh)), "frame %d" % i
    for u in ups:
        u.close()


@pytest.mark.parametrize("size", [(200, 120), (257, 67), (130, 200)])
@pytest.mark.parametrize("ctas", [1, 5, 13])
def test_emulated_fused_kernel_interior_steps_match_the_two_kernel_path(size, ctas):
    """Sizes with interior strips (the predicate-free step), runs spanning many steps, and a row slab: the fused kernel's
    device code on the CPU emulator gives the bits of EASU followed by RCAS."""
    iw, ih = size
    ow, oh = 2 * iw, 2 * ih
    src = F.to_half(F.uniform(iw, ih, 61))
    want = emu_rcas(emu_easu(PROD, src, ow, oh), 0.25).view(np.uint16)
    con = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
    s16 = np.ascontiguousarray(src.view(np.uint16))
    for (y0, y1) in ((0, oh), (oh // 4 + 1, 3 * oh // 4)):
        out = np.zeros((oh, ow, 4), np.uint16)
        rc = emu_lib().emu_fused_h(ctypes.c_void_p(s16.ctypes.data), iw, ih, ctypes.c_longlong(s16.strides[0]),
                                   ctypes.c_void_p(out.ctypes.data), ow, oh, ctypes.c_longlong(out.strides[0]), con, y0, y1, ctas)
        assert rc == 0
        assert np.array_equal(out[y0:y1], want[y0:y1]), (y0, y1)
        assert not out[:y0].any() and not out[y1:].any()
