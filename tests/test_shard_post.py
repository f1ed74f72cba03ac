"""Display output from the sharded frame stream (fsr1_shard_create_post, fsr1_shard_post), the parts that need no GPU: every refusal
of fsr1_upscale_post's rule set returns before any CUDA call (no device, nothing launched), and the binding's refusals."""
import ctypes

import pytest

import fsr1_b200 as F
from fsr1_b200 import _lib

T8, T10, LFGA, SRTM = _lib.POST_TEPD8, _lib.POST_TEPD10, _lib.POST_LFGA, _lib.POST_SRTM_INVERSE
F16, F32, U8, U10 = _lib.FORMAT_RGBA16F, _lib.FORMAT_RGBA32F, _lib.FORMAT_RGBA8_UNORM, _lib.FORMAT_RGB10A2_UNORM


@pytest.fixture(scope="module")
def tiles():
    """host-side descriptors only: nothing dereferences them before the rules pass"""
    buf = (ctypes.c_uint8 * 8192)()
    addr = ctypes.addressof(buf)
    addr += (-addr) % 256
    return {"buf": buf, "grain": _lib.Image(addr, 32, 4, 4, 0, 4, F16, 0), "grain_win": _lib.Image(addr, 32, 4, 4, 1, 2, F16, 0),
            "grain_u8": _lib.Image(addr, 16, 4, 4, 0, 4, U8, 0)}


def _create(fmt=F16, out_fmt=U8, ops=T8, grain=None, dither=None, flags=0, world=2, rank=0, post=True):
    L = _lib.lib()
    h = ctypes.c_void_p()
    p = _lib.Post(ops, 0.5, ctypes.pointer(grain) if grain is not None else None, ctypes.pointer(dither) if dither is not None else None,
                  3, 0)
    rc = L.fsr1_shard_create_post(ctypes.byref(h), 64, 36, 128, 72, fmt, out_fmt, ctypes.byref(p) if post else None, world, rank, 2,
                                  ctypes.c_float(0.25), flags)
    assert not h.value
    return rc


def test_create_post_refusals_return_before_any_cuda_call(tiles):
    L = _lib.lib()
    n0 = L.fsr1_launch_count()
    g = tiles["grain"]
    assert _create(ops=1 << 4) == -1                                         # unknown ops bit
    assert _create(ops=T8 | T10) == -1                                       # both TEPD bits
    assert _create(ops=LFGA | T8) == -1                                      # LFGA without a grain tile
    assert _create(ops=LFGA | T8, grain=tiles["grain_win"]) == -1           # a tile that is a window
    assert _create(ops=T8, dither=tiles["grain_win"]) == -1
    assert _create(ops=LFGA | T8, grain=tiles["grain_u8"]) == -2            # grain is signed: float tiles only
    assert _create(ops=T8, flags=1 << 25) == -1                              # unknown kernel flag
    assert _create(fmt=F32, out_fmt=F32, ops=SRTM) == -2                    # input RGBA16F only
    assert _create(fmt=U8, out_fmt=U8, ops=T8) == -2
    assert _create(out_fmt=U10, ops=T8) == -2                                # TEPD8 writes RGBA8 codes
    assert _create(out_fmt=U8, ops=T10) == -2
    assert _create(out_fmt=U8, ops=SRTM) == -2                               # UNORM slabs need TEPD
    assert _create(out_fmt=F32, ops=SRTM) == -2
    assert _create(out_fmt=9, ops=SRTM) == -1                                # unknown format
    for flag in (_lib.FLAG_EXACT, _lib.FLAG_FORCE_DIRECT, _lib.FLAG_H_REFERENCE, _lib.FLAG_RCAS_HX2, _lib.FLAG_NO_RCAS):
        assert _create(flags=flag) == -2, flag
        assert _create(flags=flag | _lib.SHARD_DYNAMIC | _lib.SHARD_ONE_STREAM) == -2, flag
    assert _create(post=False, out_fmt=U8) == -2                             # no post: the slabs are in the input's format
    assert _create(ops=0, out_fmt=U8) == -2                                  # ops == 0 is no post
    assert _create(world=0) == -1 and _create(rank=2) == -1                 # the arguments fsr1_shard_create checks
    assert L.fsr1_launch_count() == n0


def test_shard_post_refuses_a_null_shard_without_a_gpu(tiles):
    L = _lib.lib()
    p = _lib.Post(T8, 0.0, None, None, 1, 0)
    assert L.fsr1_shard_post(None, 0, ctypes.byref(p)) == -1


def test_post_needs_the_p2p_data_plane():
    with pytest.raises(ValueError):
        F.ShardedUpscaler(64, 64, 128, 128, 2, 0, halo="nccl", tepd_bits=8, device="cpu")
    with pytest.raises(ValueError):
        F.ShardedUpscaler(64, 64, 128, 128, 2, 0, halo="nccl", srtm_inverse=True, device="cpu")
