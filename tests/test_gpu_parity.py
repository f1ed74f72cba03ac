"""Parity of the CUDA kernels (through the C ABI) against the CPU oracle.

Tolerances (BASELINE.json north_star / SURVEY.md §8(d)):
  fp32 images, FSR1_FLAG_EXACT : bit-exact to the oracle (reference source built with -ffp-contract=off)
  fp32 images, default          : max-abs <= 1e-5
  fp16 images                   : max-abs <= 1e-2 against the fp32 oracle reading the SAME half-quantised input
"""
import os

import numpy as np
import pytest
import torch

import fsr1_b200 as F
import oracle_lib as ol
from easu_checks import assert_within_cell_bounds, expected_easu_kernel

pytestmark = pytest.mark.gpu
api = F.api
TOL32, TOL16 = 1e-5, 1e-2
G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fsr1_golden.npz"))
GSIZES = {"x2.0": (64, 36), "x1.5": (48, 27), "x1.3": (41, 23), "x1.0": (32, 18), "x2.0x1.5": (64, 27)}


def _padded(w, itemsize):
    """Row length in pixels of a 16-byte multiple (and even, as the fp16 / fp32 images always were)."""
    per = max(2, 16 // (4 * itemsize))
    return -(-w // per) * per


def dev(a):
    """Upload [H,W,4]; rows are padded to a 16-byte multiple (like any real texture allocation) so that the
    production kernels apply to odd widths too; the returned tensor is the [H,W,4] view."""
    h, w = a.shape[:2]
    t = torch.zeros((h, _padded(w, a.itemsize), 4), dtype=torch.from_numpy(a[:0]).dtype, device="cuda")
    t[:, :w] = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t[:, :w]


def empty_like_image(h, w, dtype):
    return torch.zeros((h, _padded(w, torch.empty(0, dtype=dtype).element_size()), 4), dtype=dtype, device="cuda")[:, :w]


def fmt_of(a):
    return {np.dtype(np.float16): api.FORMAT_RGBA16F, np.dtype(np.float32): api.FORMAT_RGBA32F,
            np.dtype(np.uint8): api.FORMAT_RGBA8_UNORM}[np.dtype(a.dtype)]


def assert_kernel(con, src, flags=0):
    """The kernel family of the last launch is the one the launchers' selection rule gives for these constants."""
    want = expected_easu_kernel(con, fmt_of(src), flags)
    assert api.last_kernel().startswith(want), (api.last_kernel(), want)


def gpu_easu(src, ow, oh, flags=0, con=None, y0=0, y1=0):
    ih, iw = src.shape[:2]
    con = con or api.easu_con(iw, ih, iw, ih, ow, oh)
    out = empty_like_image(oh, ow, torch.from_numpy(src[:0]).dtype)
    api.easu(dev(src), out, con, y0=y0, y1=y1, flags=flags)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def gpu_rcas(src, sharp, flags=0, y0=0, y1=0):
    out = empty_like_image(src.shape[0], src.shape[1], torch.float16 if src.dtype == np.float16 else torch.float32)
    api.rcas(dev(src), out, api.rcas_con(sharp), y0=y0, y1=y1, flags=flags)
    torch.cuda.synchronize()
    return out.cpu().numpy()


# (41, 47, 82, 94): twice the size, but fp32 41 * rcp(82) = 0.49999997, so not the 2x kernels
SHAPES = [(96, 54, 192, 108), (96, 54, 144, 81), (96, 54, 125, 70), (33, 17, 57, 31), (7, 5, 14, 10), (64, 64, 64, 64),
          (3, 3, 9, 9), (1, 1, 4, 4), (50, 20, 65, 26), (130, 70, 259, 141), (200, 40, 401, 79), (41, 47, 82, 94)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("gen", ["uniform", "structured"])
def test_fp32_exact_is_bit_identical(shape, gen):
    iw, ih, ow, oh = shape
    src = getattr(F, gen)(iw, ih, 31)
    want = ol.easu(src, ow, oh)
    got = gpu_easu(src, ow, oh, api.FLAG_EXACT)
    assert api.last_kernel().startswith("easu_direct<f32,exact")
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    for clamp in (0, api.FLAG_RCAS_CLAMP):
        for sharp in (0.0, 0.25, 1.0):
            r = gpu_rcas(want, sharp, api.FLAG_EXACT | clamp)
            assert np.array_equal(r.view(np.uint32), ol.rcas(want, ol.rcas_con(sharp), bool(clamp)).view(np.uint32))


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("gen", ["uniform", "structured"])
def test_fp32_default_within_1e5(shape, gen):
    iw, ih, ow, oh = shape
    src = getattr(F, gen)(iw, ih, 32)
    want = ol.easu(src, ow, oh)
    got = gpu_easu(src, ow, oh)
    # a TMA-tiled kernel at every upscale: the quad kernel at exactly 2x, the vertical-pair kernel otherwise (never easu_direct)
    assert_kernel(api.easu_con(iw, ih, iw, ih, ow, oh), src)
    assert np.abs(got - want).max() <= TOL32
    alt = gpu_easu(src, ow, oh, api.FLAG_FORCE_DIRECT)
    assert api.last_kernel().startswith("easu_direct<f32,fast") and np.abs(alt - want).max() <= TOL32
    for clamp in (0, api.FLAG_RCAS_CLAMP):
        r = gpu_rcas(want, 0.25, clamp)
        assert api.last_kernel().startswith("rcas_f32_packed"), api.last_kernel()
        assert np.abs(r - ol.rcas(want, ol.rcas_con(0.25), bool(clamp))).max() <= TOL32


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("gen", ["uniform", "structured"])
def test_fp16_kernels_within_1e2_of_fp32_oracle(shape, gen):
    iw, ih, ow, oh = shape
    src = F.to_half(getattr(F, gen)(iw, ih, 33))
    want = ol.easu(src.astype(np.float32), ow, oh)       # fp32 algorithm on the quantised input
    got = gpu_easu(src, ow, oh)
    assert_kernel(api.easu_con(iw, ih, iw, ih, ow, oh), src)
    assert got.dtype == np.float16 and np.all(got[..., 3] == 1.0)
    assert np.abs(got.astype(np.float32) - want).max() <= TOL16
    # the fp32-math / fp16-storage fallback kernel is held to the same bound
    alt = gpu_easu(src, ow, oh, api.FLAG_FORCE_DIRECT)
    assert np.abs(alt.astype(np.float32) - want).max() <= TOL16
    for clamp in (0, api.FLAG_RCAS_CLAMP):
        for sharp in (0.0, 0.25, 2.0):
            mid = got                                        # RCAS stage on its own: same half input both sides
            r = gpu_rcas(mid, sharp, clamp)
            assert api.last_kernel().startswith("rcas_h_packed")
            wr = ol.rcas(mid.astype(np.float32), ol.rcas_con(sharp), bool(clamp))
            assert np.abs(r.astype(np.float32) - wr).max() <= TOL16
            assert np.all(r[..., 3] == 1.0)


@pytest.mark.parametrize("kind", ["uniform", "structured"])
@pytest.mark.parametrize("tag", list(GSIZES))
def test_against_committed_golden_vectors(kind, tag):
    """Golden vectors were produced by executing the reference's own source (tests/golden/make_golden.py)."""
    ow, oh = GSIZES[tag]
    src = G[kind + "_in_f32"]
    got = gpu_easu(src, ow, oh, api.FLAG_EXACT)
    assert np.array_equal(got.view(np.uint32), G["%s_%s_easu_f32" % (kind, tag)].view(np.uint32))
    src_h = G[kind + "_in_f16"].view(np.float16)
    got_h = gpu_easu(src_h, ow, oh).astype(np.float32)
    assert np.abs(got_h - G["%s_%s_easu_f32_of_f16" % (kind, tag)]).max() <= TOL16
    key = "%s_%s_rcas_s0.25_c0_f32" % (kind, tag)
    r = gpu_rcas(G["%s_%s_easu_f32" % (kind, tag)], 0.25, api.FLAG_EXACT)
    assert np.array_equal(r.view(np.uint32), G[key].view(np.uint32))


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("gen", ["uniform", "structured"])
def test_h_reference_mode_is_bit_identical_to_the_packed_half_source(shape, gen):
    """FSR1_FLAG_H_REFERENCE = the literal FsrEasuH / FsrRcasH arithmetic.  The H-path oracle is bit-equal to the
    reference's own H source compiled for the host (tests/test_oracle.py), so this pins the kernels to it."""
    iw, ih, ow, oh = shape
    src = F.to_half(getattr(F, gen)(iw, ih, 34))
    want = ol.easu(src, ow, oh)                      # half input -> the H-path model
    got = gpu_easu(src, ow, oh, api.FLAG_H_REFERENCE)
    assert api.last_kernel().startswith("easu_href")
    assert np.array_equal(got.view(np.uint16), want.view(np.uint16))
    for clamp in (0, api.FLAG_RCAS_CLAMP):
        for sharp in (0.0, 0.25, 1.0):
            r = gpu_rcas(want, sharp, api.FLAG_H_REFERENCE | clamp)
            assert np.array_equal(r.view(np.uint16), ol.rcas(want, ol.rcas_con(sharp), bool(clamp)).view(np.uint16))


def test_h_reference_mode_against_golden_vectors():
    for kind in ("uniform", "structured"):
        for tag, (ow, oh) in GSIZES.items():
            src_h = G[kind + "_in_f16"].view(np.float16)
            got = gpu_easu(src_h, ow, oh, api.FLAG_H_REFERENCE)
            assert np.array_equal(got.view(np.uint16), G["%s_%s_easu_h16" % (kind, tag)])
            key = "%s_%s_rcas_s0.25_c0_h16" % (kind, tag)
            r = gpu_rcas(G["%s_%s_easu_h16" % (kind, tag)].view(np.float16), 0.25, api.FLAG_H_REFERENCE)
            assert np.array_equal(r.view(np.uint16), G[key])


@pytest.mark.parametrize("denoise,alpha", [(True, False), (False, True), (True, True)])
def test_rcas_denoise_and_alpha_passthrough_options(denoise, alpha):
    """The reference's compile-time RCAS options (FSR_RCAS_DENOISE, FSR_RCAS_PASSTHROUGH_ALPHA) as run-time flags."""
    fl = (api.FLAG_RCAS_DENOISE if denoise else 0) | (api.FLAG_RCAS_PASSTHROUGH_ALPHA if alpha else 0)
    for gen in ("uniform", "structured"):
        img = getattr(F, gen)(77, 45, 36)
        for clamp in (0, api.FLAG_RCAS_CLAMP):
            rc = ol.rcas_con(0.25)
            want = ol.rcas(img, rc, bool(clamp), denoise=denoise, alpha=alpha)
            got = gpu_rcas(img, 0.25, fl | clamp | api.FLAG_EXACT)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32))            # fp32 exact: bit-identical
            assert np.abs(gpu_rcas(img, 0.25, fl | clamp) - want).max() <= TOL32          # fp32 fast
            imh = F.to_half(img)
            goth = gpu_rcas(imh, 0.25, fl | clamp).astype(np.float32)                     # fp16 storage, fp32 math
            assert np.abs(goth - ol.rcas(imh.astype(np.float32), rc, bool(clamp), denoise=denoise, alpha=alpha)).max() <= TOL16
            href = gpu_rcas(imh, 0.25, fl | clamp | api.FLAG_H_REFERENCE)                 # literal FsrRcasH + options
            assert np.array_equal(href.view(np.uint16), ol.rcas(imh, rc, bool(clamp), denoise=denoise, alpha=alpha).view(np.uint16))
            if alpha:
                assert np.array_equal(got[..., 3], img[..., 3]) and np.array_equal(href[..., 3], imh[..., 3])


def _q(x, n):
    """D3D float -> unorm: clamp, scale by 2^n-1, add 0.5, truncate (NaN -> 0)."""
    s = np.float32((1 << n) - 1)
    return (np.nan_to_num(np.clip(x, 0.0, 1.0), nan=0.0).astype(np.float32) * s + np.float32(0.5)).astype(np.uint32)


@pytest.mark.parametrize("shape", [(96, 54, 192, 108), (50, 20, 65, 26), (33, 17, 57, 31)])
def test_unorm_formats_exact(shape):
    """R8G8B8A8_UNORM / R10G10B10A2_UNORM images (what the sample renders into): fp32 F-path arithmetic between the D3D
    unorm<->float conversions; with FSR1_FLAG_EXACT the stored integers equal quantise(oracle(dequantise(input)))."""
    iw, ih, ow, oh = shape
    rng = np.random.default_rng(5)
    for bits in (8, 10):
        s = np.float32((1 << bits) - 1)
        raw = rng.integers(0, 1 << bits, size=(ih, iw, 4), dtype=np.uint32)
        if bits == 10:
            raw[..., 3] = rng.integers(0, 4, size=(ih, iw))
        fin = (raw.astype(np.float32) / s).astype(np.float32)                     # c / (2^n - 1), correctly rounded
        fin[..., 3] = raw[..., 3].astype(np.float32) / np.float32(255.0 if bits == 8 else 3.0)
        e_want = ol.easu(fin, ow, oh)
        def pack(q):
            if bits == 8:
                return torch.from_numpy(q.astype(np.uint8)).cuda()
            w = (q[..., 0] | (q[..., 1] << 10) | (q[..., 2] << 20) | (q[..., 3] << 30)).astype(np.uint32)
            return torch.from_numpy(w.view(np.int32)).cuda()
        def unpack(t):
            a = t.cpu().numpy()
            if bits == 8:
                return a.astype(np.uint32)
            w = a.view(np.uint32)
            return np.stack([w & 1023, (w >> 10) & 1023, (w >> 20) & 1023, w >> 30], axis=-1)
        din = pack(raw)
        dout = torch.zeros((oh, ow, 4), dtype=torch.uint8, device="cuda") if bits == 8 else torch.zeros((oh, ow), dtype=torch.int32, device="cuda")
        api.easu(din, dout, api.easu_con(iw, ih, iw, ih, ow, oh), flags=api.FLAG_EXACT)
        torch.cuda.synchronize()
        assert api.last_kernel() == "easu_direct<unorm%d,exact>" % bits
        got = unpack(dout)
        want = np.concatenate([_q(e_want[..., :3], bits), np.full((oh, ow, 1), (1 << bits) - 1 if bits == 8 else 3, np.uint32)], axis=-1)
        assert np.array_equal(got, want)
        # RCAS on the quantised EASU output
        mid = (want.astype(np.float32) / s).astype(np.float32)
        mid[..., 3] = 1.0
        r_want = ol.rcas(mid, ol.rcas_con(0.25))
        rout = torch.zeros_like(dout)
        api.rcas(dout, rout, api.rcas_con(0.25), flags=api.FLAG_EXACT)
        torch.cuda.synchronize()
        rw = np.concatenate([_q(r_want[..., :3], bits), np.full((oh, ow, 1), (1 << bits) - 1 if bits == 8 else 3, np.uint32)], axis=-1)
        assert np.array_equal(unpack(rout), rw)
        # default (contracted) arithmetic may move a value across a rounding boundary: at most one code value
        api.easu(din, dout, api.easu_con(iw, ih, iw, ih, ow, oh))
        torch.cuda.synchronize()
        assert np.abs(unpack(dout).astype(np.int64) - want.astype(np.int64)).max() <= 1


def test_precise_flag_fp32_math_on_fp16_storage():
    """FSR1_FLAG_PRECISE at 2x: fp32 arithmetic on RGBA16F images; only the final rounding to half is left."""
    for gen in ("uniform", "structured"):
        iw, ih, ow, oh = 200, 120, 400, 240
        src = F.to_half(getattr(F, gen)(iw, ih, 35))
        want = ol.easu(src.astype(np.float32), ow, oh)
        got = gpu_easu(src, ow, oh, api.FLAG_PRECISE)
        assert_kernel(api.easu_con(iw, ih, iw, ih, ow, oh), src, api.FLAG_PRECISE)
        assert np.abs(got.astype(np.float32) - want).max() <= 6e-4      # half ulp at 1.0 is 4.9e-4
        assert np.all(got[..., 3] == 1.0)
        mid = gpu_rcas(got, 0.25)
        e2e_check(mid, ol.rcas(want, ol.rcas_con(0.25)), ("precise", gen), tight=True)
        for (ow2, oh2) in ((300, 180), (261, 157)):                       # 1.5x and ~1.3x: the any-scale fp32-math kernel
            want2 = ol.easu(src.astype(np.float32), ow2, oh2)
            got2 = gpu_easu(src, ow2, oh2, api.FLAG_PRECISE)
            assert_kernel(api.easu_con(iw, ih, iw, ih, ow2, oh2), src, api.FLAG_PRECISE)
            assert np.abs(got2.astype(np.float32) - want2).max() <= 6e-4


def e2e_check(got, want, what, tight=False):
    """End to end (EASU -> fp16 intermediate -> RCAS) against the fp32 oracle end to end: max-abs <= 1e-2.
    RCAS amplifies differences in its input 4-7x, so this is the demanding check; measured at 4K: 6.4e-3 max,
    4e-4 mean (DESIGN.md "numerics").  tight = the FSR1_FLAG_PRECISE path, held to 4e-3."""
    d = np.abs(got.astype(np.float32) - want)[..., :3]
    assert d.max() <= (4e-3 if tight else TOL16), (what, d.max())
    assert d.mean() <= 1e-3, (what, d.mean())


def test_end_to_end_fp16_pipeline():
    for gen in ("uniform", "structured"):
        for (iw, ih, ow, oh) in [(192, 108, 384, 216), (192, 108, 288, 162), (192, 108, 250, 141)]:
            src = F.to_half(getattr(F, gen)(iw, ih, 7))
            want = ol.rcas(ol.easu(src.astype(np.float32), ow, oh), ol.rcas_con(0.25))
            flt = F.FSR_Filter()
            flt.OnCreate()
            flt.OnCreateWindowSizeDependentResources(iw, ih, ow, oh)
            out = empty_like_image(oh, ow, torch.float16)
            flt.Upscale(dev(src), out, ow, oh, F.State(renderWidth=iw, renderHeight=ih, rcasAttenuation=0.25))
            torch.cuda.synchronize()
            e2e_check(out.cpu().numpy(), want, (gen, iw, ih, ow, oh))
            flt.OnDestroy()


def test_flat_frames_and_nan_paths():
    for v in (0.0, 1.0, 0.5):
        for dt in (np.float16, np.float32):
            src = np.full((23, 37, 4), v, dt)
            e = gpu_easu(src, 74, 46)
            assert np.all(e[..., :3] == dt(v))
            for clamp in (0, api.FLAG_RCAS_CLAMP):
                r = gpu_rcas(e, 0.0, clamp)
                assert np.isfinite(r.astype(np.float32)).all()
                w = ol.rcas(e.astype(np.float32), ol.rcas_con(0.0), bool(clamp))
                assert np.abs(r.astype(np.float32) - w).max() <= (TOL16 if dt == np.float16 else TOL32)


def test_padded_pitch_odd_sizes_and_unaligned_fallback():
    iw, ih, ow, oh = 45, 29, 77, 51
    src = F.to_half(F.uniform(iw, ih, 11))
    want = ol.easu(src.astype(np.float32), ow, oh)
    con = api.easu_con(iw, ih, iw, ih, ow, oh)
    # padded row pitch (multiple of 16 B): production kernels
    big_in = torch.zeros((ih, iw + 3, 4), dtype=torch.float16, device="cuda")
    big_in[:, :iw] = dev(src)
    big_out = torch.zeros((oh, ow + 5, 4), dtype=torch.float16, device="cuda")
    api.easu(big_in[:, :iw], big_out[:, :ow], con)
    assert api.last_kernel().startswith("easu_h_")
    assert np.abs(big_out[:, :ow].cpu().numpy().astype(np.float32) - want).max() <= TOL16
    assert torch.all(big_out[:, ow:] == 0)                      # nothing written outside the image
    # pitch that is only 8-byte aligned: TMA / 128-bit stores impossible -> direct kernels, same answer
    odd_in = torch.zeros((ih, iw + 2, 4), dtype=torch.float16, device="cuda")[:, 1:iw + 1]
    odd_in.copy_(dev(src))
    odd_out = torch.zeros((oh, ow + 2, 4), dtype=torch.float16, device="cuda")[:, 1:ow + 1]
    api.easu(odd_in, odd_out, con)
    assert api.last_kernel().startswith("easu_direct<f16io")
    assert np.abs(odd_out.cpu().numpy().astype(np.float32) - want).max() <= TOL16
    r_out = torch.zeros_like(odd_out)
    api.rcas(odd_out, r_out, api.rcas_con(0.25))
    assert api.last_kernel().startswith("rcas_direct<f16io")
    wr = ol.rcas(odd_out.cpu().numpy().astype(np.float32), ol.rcas_con(0.25))
    assert np.abs(r_out.cpu().numpy().astype(np.float32) - wr).max() <= TOL16


def test_dynamic_resolution_viewport_and_offset():
    """viewport != resource size and FsrEasuConOffset (ffx_fsr1.h:161-169, 205-225)."""
    iw, ih, ow, oh = 80, 60, 96, 72
    src = F.uniform(iw, ih, 12)
    for con in (api.easu_con(60, 40, iw, ih, ow, oh), api.easu_con_offset(48, 36, iw, ih, ow, oh, 16.0, 8.0)):
        want = ol.easu(src, ow, oh, con)
        got = gpu_easu(src, ow, oh, api.FLAG_EXACT, con=con)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        goth = gpu_easu(F.to_half(src), ow, oh, con=con).astype(np.float32)
        assert np.abs(goth - ol.easu(F.to_half(src).astype(np.float32), ow, oh, con)).max() <= TOL16


@pytest.mark.parametrize("shape", [(64, 60, 128, 120), (64, 60, 96, 90), (70, 50, 91, 65)])
@pytest.mark.parametrize("dt", [np.float16, np.float32])
def test_slabs_compose(dt, shape):
    """Row windows (the multi-GPU slabs) give exactly the bytes of the whole-frame run — for the 2x kernels, the
    generic kernel (1.5x, 1.3x) and the direct kernels alike."""
    iw, ih, ow, oh = shape
    check_slabs_compose(F.uniform(iw, ih, 13).astype(dt), ow, oh, api.easu_con(iw, ih, iw, ih, ow, oh))


def check_slabs_compose(src, ow, oh, econ):
    """Three row slabs, each with the input window SlabPlan gives it, reproduce the bytes of the whole-frame upscale."""
    ih = src.shape[0]
    tdt = torch.from_numpy(src[:0]).dtype
    rcon = api.rcas_con(0.25)
    full_in = dev(src)
    tmp = empty_like_image(oh, ow, tdt)
    whole = empty_like_image(oh, ow, tdt)
    api.upscale(full_in, tmp, whole, econ, rcon)
    parts = []
    for world in (3,):
        plan = F.SlabPlan(ih, oh, world, econ)
        for r in range(world):
            n0, n1 = plan.needed_in_rows(r)
            e0, e1 = plan.easu_rows(r)
            y0, y1 = plan.out_rows(r)
            win = full_in[n0:n1]
            t = empty_like_image(e1 - e0, ow, tdt)
            o = empty_like_image(y1 - y0, ow, tdt)
            api.upscale(api.image(win, height=ih, row0=n0), api.image(t, height=oh, row0=e0),
                        api.image(o, height=oh, row0=y0), econ, rcon, y0=y0, y1=y1)
            parts.append(o)
    torch.cuda.synchronize()
    assert torch.equal(torch.cat(parts), whole)


def test_sharded_upscaler_single_rank_equals_plain_upscale():
    """world = 1: the sharded path issues no communication and must give exactly the plain result (the N > 1 exchange
    is covered on CPU over gloo, tests/test_sharding.py, and by bench.py --gpus N)."""
    iw, ih, ow, oh = 160, 90, 320, 180
    src = torch.from_numpy(F.to_half(F.structured(iw, ih, 15))).cuda()
    up = F.ShardedUpscaler(iw, ih, ow, oh, 1, 0)
    up.owned.copy_(src)
    got = up.upscale().clone()
    got2 = up.upscale().clone()          # second call re-launches the prepared descriptors
    tmp = torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda")
    want = torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda")
    api.upscale(src, tmp, want, api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25))
    torch.cuda.synchronize()
    assert torch.equal(got, want) and torch.equal(got2, want)


def test_plain_c_host_program(tmp_path):
    """examples/fsr1_demo.c run on the GPU; its checksum against the oracle on the same gradient frame."""
    import subprocess
    from test_abi import _build_c_demo
    out = subprocess.check_output([str(_build_c_demo(tmp_path))]).decode()
    assert "easu" in out or "rcas" in out
    rw, rh, dw, dh = 640, 360, 1280, 720
    y, x = np.mgrid[0:rh, 0:rw]
    frame = np.stack([x / np.float32(rw), y / np.float32(rh), (((x // 16 + y // 16) & 1) == 1).astype(np.float32),
                      np.ones((rh, rw), np.float32)], axis=-1).astype(np.float32)
    want = ol.rcas(ol.easu(frame, dw, dh), ol.rcas_con(0.25))[..., :3].astype(np.float64).sum()
    got = float(out.split("checksum")[1].split(",")[0])
    assert abs(got - want) <= 1e-6 * want + 0.5


def test_frame_pipeline_equals_sequential():
    """api.FramePipeline (RCAS of frame i overlapped with EASU of frame i+1 on two streams) changes scheduling, not
    results: every frame equals the one-stream upscale, also when slots are reused many times."""
    iw, ih, ow, oh = 256, 144, 512, 288
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    nslots, nframes = 3, 11
    frames = [torch.from_numpy(F.to_half(F.uniform(iw, ih, 100 + t))).cuda() for t in range(nframes)]
    want = []
    for fr in frames:
        t = torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda")
        o = torch.zeros_like(t)
        api.upscale(fr, t, o, econ, rcon)
        want.append(o)
    ins = [torch.zeros_like(frames[0]) for _ in range(nslots)]
    tmps = [torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda") for _ in range(nslots)]
    outs = [torch.zeros_like(tmps[0]) for _ in range(nslots)]
    pipe = api.FramePipeline(list(zip(ins, tmps, outs)), econ, rcon)
    got = []
    for i, fr in enumerate(frames):
        s = i % nslots
        if i >= nslots:                               # collect the slot's previous result before reusing it
            pipe.end()
            got.append(outs[s].clone())
        ins[s].copy_(fr)
        pipe.begin()
        pipe.submit(s)
    pipe.end()
    torch.cuda.synchronize()
    for i in range(nframes - nslots, nframes):
        got.append(outs[i % nslots].clone())
    assert len(got) == nframes and all(torch.equal(a, b) for a, b in zip(got, want))


def test_host_frame_entry_point():
    iw, ih, ow, oh = 120, 68, 240, 136
    src = F.to_half(F.structured(iw, ih, 14))
    ctx = api.HostContext(iw, ih, ow, oh, api.FORMAT_RGBA16F)
    hin = torch.from_numpy(src).pin_memory()
    hout = torch.zeros((oh, ow, 4), dtype=torch.float16).pin_memory()
    ctx.upscale_host(hin, hout, 0.25)
    torch.cuda.synchronize()
    e2e_check(hout.numpy(), ol.rcas(ol.easu(src.astype(np.float32), ow, oh), ol.rcas_con(0.25)), "host frames")
    ctx.close()


def test_full_size_1080p_to_4k_against_oracle():
    """BASELINE.json config 2 at full size: every pixel against the oracle (the C oracle does 4K in ~1 s)."""
    iw, ih, ow, oh = 1920, 1080, 3840, 2160
    src = F.to_half(F.structured(iw, ih, 2024))
    din = dev(src)
    tmp = torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda")
    out = torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda")
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    api.upscale(din, tmp, out, econ, rcon)
    torch.cuda.synchronize()
    e_want = ol.easu(src.astype(np.float32), ow, oh)
    e_got = tmp.cpu().numpy()
    assert np.abs(e_got.astype(np.float32) - e_want).max() <= TOL16
    r_want = ol.rcas(e_got.astype(np.float32), ol.rcas_con(0.25))
    assert np.abs(out.cpu().numpy().astype(np.float32) - r_want).max() <= TOL16
    e2e_check(out.cpu().numpy(), ol.rcas(e_want, ol.rcas_con(0.25)), "1080p->4K structured")
    # size-independent property: the de-ringing clamp — every EASU output lies within the min/max of its 2x2 cell
    assert_within_cell_bounds(e_got, src, econ, what="1080p->4K")


# ---- BASELINE.json configs at their own size (every pixel against the oracle) ----------------------------------------
def _full_size_fp16(iw, ih, ow, oh, gen, seed, kernel_prefix):
    src = F.to_half(getattr(F, gen)(iw, ih, seed))
    din = dev(src)
    tmp = torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda")
    out = torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda")
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    api.easu(din, tmp, econ)
    assert api.last_kernel().startswith(kernel_prefix), api.last_kernel()     # the production kernel, not a fallback
    api.rcas(tmp, out, rcon)
    assert api.last_kernel().startswith("rcas_h_packed"), api.last_kernel()
    torch.cuda.synchronize()
    e_want = ol.easu(src.astype(np.float32), ow, oh)
    e_got = tmp.cpu().numpy()
    assert np.abs(e_got.astype(np.float32) - e_want).max() <= TOL16
    assert np.all(e_got[..., 3] == np.float16(1.0))
    r_want = ol.rcas(e_got.astype(np.float32), ol.rcas_con(0.25))
    assert np.abs(out.cpu().numpy().astype(np.float32) - r_want).max() <= TOL16
    e2e_check(out.cpu().numpy(), ol.rcas(e_want, ol.rcas_con(0.25)), (iw, ih, ow, oh, gen))


@pytest.mark.parametrize("gen", ["uniform", "structured"])
def test_full_size_1080p_to_4k_noise_and_structured(gen):
    """BASELINE configs[1] (the headline), LCG noise and the structured frame."""
    _full_size_fp16(1920, 1080, 3840, 2160, gen, 12345, "easu_h_quad2x")


@pytest.mark.parametrize("gen", ["uniform", "structured"])
@pytest.mark.parametrize("size", [(2560, 1440), (2953, 1661)])
def test_full_size_configs2_1440p_and_ultra_quality_to_4k(size, gen):
    """BASELINE configs[2]: 2560x1440 -> 4K (1.5x) and the true Ultra Quality 2953x1661 -> 4K (1.3x, odd width: padded
    pitch); the any-scale kernel with its per-launch TMA box."""
    _full_size_fp16(size[0], size[1], 3840, 2160, gen, 12345, "easu_h_vpairs")


@pytest.mark.parametrize("gen", ["uniform", "structured"])
def test_full_size_configs3_fp32_1080p_to_4k(gen):
    """BASELINE configs[3]: RGBA32F at 1080p -> 4K, fast path within 1e-5; and the fp16 path against it (tolerance sweep)."""
    iw, ih, ow, oh = 1920, 1080, 3840, 2160
    src = getattr(F, gen)(iw, ih, 12345)
    din = dev(src)
    tmp = torch.zeros((oh, ow, 4), dtype=torch.float32, device="cuda")
    out = torch.zeros((oh, ow, 4), dtype=torch.float32, device="cuda")
    for sharp in (0.0, 0.25, 1.0, 2.0):
        api.upscale(din, tmp, out, api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(sharp))
        torch.cuda.synchronize()
        if sharp == 0.0:
            e_want = ol.easu(src, ow, oh)
            assert np.abs(tmp.cpu().numpy() - e_want).max() <= TOL32
        r_want = ol.rcas(tmp.cpu().numpy(), ol.rcas_con(sharp))
        assert np.abs(out.cpu().numpy() - r_want).max() <= TOL32, sharp
        assert np.abs(out.cpu().numpy() - ol.rcas(e_want, ol.rcas_con(sharp)))[..., :3].max() <= 5e-5, sharp   # end to end (RCAS amplifies)


def test_full_size_configs4_2160p_to_8k_in_8_slabs():
    """BASELINE configs[4]: 3840x2160 -> 7680x4320 RGBA16F cut into 8 row slabs of 540 rows (2 halo rows each side,
    61 440 B per message) through the sharded data plane (8 ranks on this one device, halo by direct stores), bit-identical
    to the single-GPU frame, and that against the oracle on bands that straddle every slab boundary."""
    iw, ih, ow, oh, world = 3840, 2160, 7680, 4320, 8
    src = F.to_half(F.structured(iw, ih, 4242))
    frame = torch.from_numpy(src).cuda()
    ups = [F.ShardedUpscaler(iw, ih, ow, oh, world, r, slots=1, halo="p2p", attach=False) for r in range(world)]
    for r, u in enumerate(ups):
        u.attach_local(ups[r - 1] if r > 0 else None, ups[r + 1] if r + 1 < world else None)
        assert u.plan.halo_bytes(r, iw, 8) == (2 if 0 < r < world - 1 else 1) * 61440
    s = torch.cuda.current_stream()
    for r, u in enumerate(ups):
        o0, o1 = u.plan.owned_in_rows(r)
        u.input(0).copy_(frame[o0:o1])
    for u in ups:
        u.submit(0, s)
    for u in ups:
        u.wait(0, s)
    sharded = torch.cat([u.output(0) for u in ups])
    tmp = torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda")
    whole = torch.zeros_like(tmp)
    api.upscale(frame, tmp, whole, api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25))
    torch.cuda.synchronize()
    for u in ups:
        u.status()
    assert torch.equal(sharded, whole)
    got = whole.cpu().numpy().astype(np.float32)
    f32 = src.astype(np.float32)
    for r in range(1, world):
        yb = r * oh // world
        y0, y1 = yb - 24, yb + 24
        e = ol.easu(f32, ow, oh, y0=y0 - 1, y1=y1 + 1)
        want = ol.rcas(e, ol.rcas_con(0.25), y0=y0, y1=y1)
        assert np.abs(got[y0:y1] - want[y0:y1])[..., :3].max() <= TOL16, r
    for u in ups:
        u.close()


@pytest.mark.parametrize("opts", [1, 2, 3, 4, 5, 6, 7])
def test_rcas_options_run_on_the_packed_kernels(opts):
    """FSR_RCAS_DENOISE / FSR_RCAS_PASSTHROUGH_ALPHA / the Sample.x square are template bits of the production kernels
    (RGBA16F, RGBA32F, R8G8B8A8): same kernel family as the plain configuration, no extra pass, results against the oracle
    built with the same options (ffx_fsr1.h:688-702,731-739,761-763; FSR_Pass.hlsl:93-94)."""
    denoise, alpha, square = bool(opts & 1), bool(opts & 2), bool(opts & 4)
    fl = (api.FLAG_RCAS_DENOISE if denoise else 0) | (api.FLAG_RCAS_PASSTHROUGH_ALPHA if alpha else 0) | (api.FLAG_OUTPUT_SQUARE if square else 0)
    w, h = 259, 141
    for gen in ("uniform", "structured"):
        img = getattr(F, gen)(w, h, 36)
        for clamp in (0, api.FLAG_RCAS_CLAMP):
            rc = ol.rcas_con(0.25)
            def want_of(x):
                r = ol.rcas(x, rc, bool(clamp), denoise=denoise, alpha=alpha)
                if square:
                    r[..., :3] = r[..., :3] * r[..., :3]
                return r
            n0 = api.launch_count()
            got = gpu_rcas(img, 0.25, fl | clamp)
            assert api.last_kernel().startswith("rcas_f32_packed") and api.launch_count() == n0 + 1
            assert np.abs(got - want_of(img))[..., :3].max() <= (TOL32 if not square else 2e-5)
            assert np.array_equal(got[..., 3], img[..., 3] if alpha else np.ones((h, w), np.float32))
            imh = F.to_half(img)
            n0 = api.launch_count()
            goth = gpu_rcas(imh, 0.25, fl | clamp)
            assert api.last_kernel().startswith("rcas_h_packed") and api.launch_count() == n0 + 1
            assert np.abs(goth.astype(np.float32) - want_of(imh.astype(np.float32)))[..., :3].max() <= TOL16
            assert np.array_equal(goth[..., 3].view(np.uint16), imh[..., 3].view(np.uint16) if alpha else np.full((h, w), 0x3c00, np.uint16))
    # R8G8B8A8
    raw = (np.random.default_rng(7).integers(0, 256, size=(h, w, 4))).astype(np.uint8)
    fin = raw.astype(np.float32) / np.float32(255.0)
    want = ol.rcas(fin, ol.rcas_con(0.25), False, denoise=denoise, alpha=alpha)
    if square:
        want[..., :3] = want[..., :3] * want[..., :3]
    wq = _q(want[..., :3], 8)
    out = torch.zeros((h, w + (-w) % 2, 4), dtype=torch.uint8, device="cuda")[:, :w]
    src = torch.zeros((h, w + (-w) % 2, 4), dtype=torch.uint8, device="cuda")[:, :w]
    src.copy_(torch.from_numpy(raw))
    api.rcas(src, out, api.rcas_con(0.25), flags=fl)
    torch.cuda.synchronize()
    assert api.last_kernel().startswith("rcas_u8_packed"), api.last_kernel()
    got8 = out.cpu().numpy()
    assert np.abs(got8[..., :3].astype(np.int64) - wq.astype(np.int64)).max() <= 1
    assert np.array_equal(got8[..., 3], raw[..., 3] if alpha else np.full((h, w), 255, np.uint8))


def test_unorm8_production_kernels_within_one_code():
    """R8G8B8A8_UNORM (what the sample renders into, FSR_Filter.cpp:72-73) at 2x takes the TMA-tiled EASU and the packed RCAS:
    each within one code value of quantise(oracle(dequantise(input))), per kernel, at 1080p -> 4K."""
    iw, ih, ow, oh = 1920, 1080, 3840, 2160
    raw = np.floor(F.uniform(iw, ih, 12345) * 255.0 + 0.5).astype(np.uint8)
    raw[::64, ::64] = 0
    raw[32::64, 32::64] = 255
    fin = raw.astype(np.float32) / np.float32(255.0)
    din = torch.from_numpy(raw).cuda()
    tmp = torch.zeros((oh, ow, 4), dtype=torch.uint8, device="cuda")
    out = torch.zeros_like(tmp)
    api.easu(din, tmp, api.easu_con(iw, ih, iw, ih, ow, oh))
    assert api.last_kernel().startswith("easu_u8_quad2x"), api.last_kernel()
    api.rcas(tmp, out, api.rcas_con(0.25))
    assert api.last_kernel().startswith("rcas_u8_packed"), api.last_kernel()
    torch.cuda.synchronize()
    e_got = tmp.cpu().numpy()
    e_want = _q(ol.easu(fin, ow, oh)[..., :3], 8)
    d = np.abs(e_got[..., :3].astype(np.int64) - e_want.astype(np.int64))
    assert d.max() <= 1 and (d > 0).mean() < 0.10, (int(d.max()), float((d > 0).mean()))
    assert (e_got[..., 3] == 255).all()
    mid = e_got.astype(np.float32) / np.float32(255.0)
    r_want = _q(ol.rcas(mid, ol.rcas_con(0.25))[..., :3], 8)
    d = np.abs(out.cpu().numpy()[..., :3].astype(np.int64) - r_want.astype(np.int64))
    assert d.max() <= 1, int(d.max())


# ---- the fused EASU -> RCAS kernel (FSR1_FLAG_FUSED) -------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(96, 54, 192, 108), (33, 17, 66, 34), (130, 70, 260, 140), (5, 3, 10, 6), (1, 1, 2, 2), (200, 40, 400, 80)])
@pytest.mark.parametrize("gen", ["uniform", "structured"])
def test_fused_kernel_is_bit_identical_to_the_two_kernel_path(shape, gen):
    """FSR1_FLAG_FUSED at 2x RGBA16F: the intermediate stays in shared memory (rounded to fp16 exactly as the intermediate image
    would be), so every output bit equals fsr1_easu + fsr1_rcas; `tmp` is not touched; row ranges (slabs) compose."""
    iw, ih, ow, oh = shape
    src = F.to_half(getattr(F, gen)(iw, ih, 91))
    din = dev(src)
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    tmp, want = empty_like_image(oh, ow, torch.float16), empty_like_image(oh, ow, torch.float16)
    api.upscale(din, tmp, want, econ, rcon)
    sentinel = torch.full((oh, (ow + 1) & ~1, 4), 7.0, dtype=torch.float16, device="cuda")[:, :ow]
    got = empty_like_image(oh, ow, torch.float16)
    api.upscale(din, sentinel, got, econ, rcon, flags=api.FLAG_FUSED)
    assert api.last_kernel().startswith("fused_easu_rcas_h"), api.last_kernel()
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert (sentinel == 7.0).all()                                   # no intermediate image
    if oh >= 30:
        parts = empty_like_image(oh, ow, torch.float16)
        for (y0, y1) in ((0, oh // 3), (oh // 3, oh // 3 + 5), (oh // 3 + 5, oh)):
            api.upscale(din, sentinel, parts, econ, rcon, y0=y0, y1=y1, flags=api.FLAG_FUSED)
        torch.cuda.synchronize()
        assert torch.equal(parts, want)
    # other scales and options fall back to the two kernels (same results by construction)
    api.upscale(din, tmp, got, econ, rcon, flags=api.FLAG_FUSED | api.FLAG_RCAS_CLAMP)
    assert api.last_kernel().startswith("rcas_h_packed")


@pytest.mark.parametrize("gen", ["uniform", "structured"])
def test_fused_kernel_full_size_1080p_to_4k(gen):
    iw, ih, ow, oh = 1920, 1080, 3840, 2160
    src = F.to_half(getattr(F, gen)(iw, ih, 12345))
    din = dev(src)
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    tmp = torch.zeros((oh, ow, 4), dtype=torch.float16, device="cuda")
    want, got = torch.zeros_like(tmp), torch.zeros_like(tmp)
    api.upscale(din, tmp, want, econ, rcon)
    api.upscale(din, tmp, got, econ, rcon, flags=api.FLAG_FUSED)
    assert api.last_kernel().startswith("fused_easu_rcas_h"), api.last_kernel()
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    e2e_check(got.cpu().numpy(), ol.rcas(ol.easu(src.astype(np.float32), ow, oh), ol.rcas_con(0.25)), ("fused", gen))


# ---- geometry: viewports, offsets, non-uniform and extreme scales, multi-wave launches ------------------------------------
# Each output is about 1080p or larger, so every persistent kernel walks more tiles than it has CTAs (prefetch into the other
# buffer, mbarrier parity flip, tile walk after the first tile).  The kernel family is predicted from the constant block.
# id: (resource w, h, viewport w, h, offset or None, output w, h)
GEOMETRY = {
    "2x_viewport": (1920, 1080, 960, 540, None, 1920, 1080),
    "offset_1280x720_at_16_8": (1920, 1080, 1280, 720, (16, 8), 2560, 1440),
    "viewport_at_resource_edge": (1920, 1080, 960, 540, (960, 540), 1920, 1080),
    "anisotropic_x2_y1.5": (1920, 1080, 1920, 1080, None, 3840, 1620),
    "anisotropic_x1.34_y1.33": (2560, 1080, 2560, 1080, None, 3440, 1440),
    "x1.5_y1": (1280, 1080, 1280, 1080, None, 1920, 1080),
    "x1_y1.5": (1920, 720, 1920, 720, None, 1920, 1080),
    "scale1": (1920, 1080, 1920, 1080, None, 1920, 1080),
    "3x": (640, 360, 640, 360, None, 1920, 1080),
    "4x": (480, 270, 480, 270, None, 1920, 1080),
    "y_downscaled": (1920, 1080, 1920, 1080, None, 2880, 900),
    "almost_2x_949x564": (949, 564, 949, 564, None, 1898, 1128),
    "almost_2x_41x47": (41, 47, 41, 47, None, 82, 94),
}


def geometry_con(iw, ih, vw, vh, off, ow, oh):
    if off is None:
        return api.easu_con(vw, vh, iw, ih, ow, oh)
    return api.easu_con_offset(vw, vh, iw, ih, ow, oh, float(off[0]), float(off[1]))


def report(case, what, got, want):
    """Max / mean abs error of one kernel against its oracle, printed with the kernel that ran (pytest -s shows it)."""
    d = np.abs(got[..., :3].astype(np.float64) - want[..., :3].astype(np.float64))
    print("EASU %-28s %-16s %-52s max %.3g mean %.3g" % (case, what, api.last_kernel(), d.max(), d.mean()))
    return d


@pytest.mark.parametrize("case", list(GEOMETRY))
def test_geometry_against_oracle(case):
    """Every format's EASU kernel at this geometry against the oracle reading the whole resource with the same constants: the
    suite's contract per format, the de-ringing bound, the kernel family the constants select, and row slabs that compose."""
    iw, ih, vw, vh, off, ow, oh = GEOMETRY[case]
    con = geometry_con(iw, ih, vw, vh, off, ow, oh)
    src = F.uniform(iw, ih, 4000 + iw + ih)
    src_h = F.to_half(src)
    f_h = src_h.astype(np.float32)
    raw = np.floor(src * 255.0 + 0.5).astype(np.uint8)
    fin = raw.astype(np.float32) / np.float32(255.0)

    want = ol.easu(src, ow, oh, con)
    got = gpu_easu(src, ow, oh, con=con)                                     # RGBA32F, default
    assert_kernel(con, src)
    assert report(case, "f32", got, want).max() <= TOL32
    assert_within_cell_bounds(got, src, con, what=(case, "f32"))
    got = gpu_easu(src, ow, oh, api.FLAG_EXACT, con=con)                    # RGBA32F, EXACT: bit for bit
    assert_kernel(con, src, api.FLAG_EXACT)
    report(case, "f32 exact", got, want)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert_within_cell_bounds(got, src, con, what=(case, "f32 exact"))

    want = ol.easu(f_h, ow, oh, con)                                         # fp32 algorithm on the half input
    got = gpu_easu(src_h, ow, oh, con=con)                                   # RGBA16F, default
    assert_kernel(con, src_h)
    assert report(case, "f16", got, want).max() <= TOL16
    assert_within_cell_bounds(got, src_h, con, what=(case, "f16"))
    got = gpu_easu(src_h, ow, oh, api.FLAG_PRECISE, con=con)                # RGBA16F, PRECISE
    assert_kernel(con, src_h, api.FLAG_PRECISE)
    assert report(case, "f16 precise", got, want).max() <= 6e-4
    assert_within_cell_bounds(got, src_h, con, what=(case, "f16 precise"))
    got = gpu_easu(src_h, ow, oh, api.FLAG_H_REFERENCE, con=con)            # RGBA16F, the literal FsrEasuH: bit for bit
    assert_kernel(con, src_h, api.FLAG_H_REFERENCE)
    want_h = ol.easu(src_h, ow, oh, con)
    report(case, "f16 href", got, want_h)
    assert np.array_equal(got.view(np.uint16), want_h.view(np.uint16))
    assert_within_cell_bounds(got, src_h, con, what=(case, "f16 href"))

    want8 = _q(ol.easu(fin, ow, oh, con)[..., :3], 8)                        # R8G8B8A8: code values
    got = gpu_easu(raw, ow, oh, con=con)
    assert_kernel(con, raw)
    assert report(case, "u8 (codes)", got, want8).max() <= 1
    assert_within_cell_bounds(got, raw, con, what=(case, "u8"))

    econ_is_2x = expected_easu_kernel(con, api.FORMAT_RGBA16F) == "easu_h_quad2x"
    if econ_is_2x:                                                           # fused == two kernels, bit for bit
        din, rcon = dev(src_h), api.rcas_con(0.25)
        tmp, two = empty_like_image(oh, ow, torch.float16), empty_like_image(oh, ow, torch.float16)
        api.upscale(din, tmp, two, con, rcon)
        fused = empty_like_image(oh, ow, torch.float16)
        api.upscale(din, tmp, fused, con, rcon, flags=api.FLAG_FUSED)
        assert api.last_kernel().startswith("fused_easu_rcas_h"), api.last_kernel()
        torch.cuda.synchronize()
        assert torch.equal(fused, two)
    for s in (src_h, src, raw):
        check_slabs_compose(s, ow, oh, con)


@pytest.mark.parametrize("gen", ["uniform", "structured"])
def test_full_size_fp32_and_precise_1440p_to_4k(gen):
    """The fp32 any-scale kernels (the slow fallback at the Quality preset) at full size: 1020 tiles against at most 2 x 132 CTAs."""
    iw, ih, ow, oh = 2560, 1440, 3840, 2160
    src = getattr(F, gen)(iw, ih, 12345)
    econ, rcon = api.easu_con(iw, ih, iw, ih, ow, oh), api.rcas_con(0.25)
    tmp = torch.zeros((oh, ow, 4), dtype=torch.float32, device="cuda")
    out = torch.zeros_like(tmp)
    api.upscale(dev(src), tmp, out, econ, rcon)
    torch.cuda.synchronize()
    e_want = ol.easu(src, ow, oh)
    e_got = tmp.cpu().numpy()
    api.easu(dev(src), tmp, econ)
    assert_kernel(econ, src)
    assert report("1440p->4K " + gen, "f32", e_got, e_want).max() <= TOL32
    assert_within_cell_bounds(e_got, src, econ, what="f32 1440p->4K")
    got = out.cpu().numpy()
    assert np.abs(got - ol.rcas(e_got, rcon)).max() <= TOL32                  # RCAS on the kernel's own intermediate
    assert np.abs(got - ol.rcas(e_want, rcon))[..., :3].max() <= 5e-5         # end to end
    src_h = F.to_half(src)
    got_h = gpu_easu(src_h, ow, oh, api.FLAG_PRECISE)
    assert_kernel(econ, src_h, api.FLAG_PRECISE)
    assert report("1440p->4K " + gen, "f16 precise", got_h, ol.easu(src_h.astype(np.float32), ow, oh)).max() <= 6e-4
    assert_within_cell_bounds(got_h, src_h, econ, what="precise 1440p->4K")


# ---- dynamic resolution: one context, the render size changing from frame to frame --------------------------------------
SEQUENCE = [(960, 540), (1280, 720), (1129, 635), (1476, 830), (1920, 1080), (640, 360), (949, 540), (960, 540)]


@pytest.mark.parametrize("fmt,flags", [("f16", 0), ("f32", 0), ("u8", 0), ("f16", api.FLAG_FUSED), ("f16", api.FLAG_PRECISE)],
                         ids=["f16", "f32", "u8", "f16-fused", "f16-precise"])
def test_dynamic_resolution_frame_sequence(fmt, flags):
    """fsr1_context_upscale_render (the path of the C++ FSR_Filter) and the Python FSR_Filter on a 1920x1080 buffer whose top-left
    render region changes size every frame, so the kernels move between the quad, vertical-pair and direct families.  Every texel
    outside the render region holds a sentinel; a tap that reads it breaks the de-ringing bound.  Each frame equals fsr1_upscale
    on the cropped view, bit for bit, and is held to the format's contract against the oracle."""
    W, H = 1920, 1080
    dt = {"f16": np.float16, "f32": np.float32, "u8": np.uint8}[fmt]
    tdt = torch.from_numpy(np.zeros(0, dt)).dtype
    fmt_id = {"f16": api.FORMAT_RGBA16F, "f32": api.FORMAT_RGBA32F, "u8": api.FORMAT_RGBA8_UNORM}[fmt]
    sentinel = 255 if fmt == "u8" else 4.0
    rcon = api.rcas_con(0.25)
    ctx = api.HostContext(W, H, W, H, fmt_id)
    flt = F.FSR_Filter()
    flt.OnCreate(dtype=tdt)
    flt.flags = flags
    flt.OnCreateWindowSizeDependentResources(W, H, W, H)
    buf = torch.full((H, W, 4), sentinel, dtype=tdt, device="cuda")
    for i, (rw, rh) in enumerate(SEQUENCE):
        f32 = F.uniform(rw, rh, 500 + i)
        content = np.floor(f32 * 255.0 + 0.5).astype(np.uint8) if fmt == "u8" else f32.astype(dt)
        buf.fill_(sentinel)
        buf[:rh, :rw] = torch.from_numpy(content).cuda()
        crop = buf[:rh, :rw]
        con = api.easu_con(rw, rh, rw, rh, W, H)
        out_ctx = torch.zeros((H, W, 4), dtype=tdt, device="cuda")
        ctx.upscale_render(buf, rw, rh, out_ctx, 0.25, flags)
        tmp, want = torch.zeros_like(out_ctx), torch.zeros_like(out_ctx)
        api.upscale(crop, tmp, want, con, rcon, flags=flags)
        if flags & api.FLAG_FUSED:
            two_x = expected_easu_kernel(con, fmt_id) == "easu_h_quad2x"
            assert api.last_kernel().startswith("fused_easu_rcas_h" if two_x else "rcas_h_packed"), (rw, rh, api.last_kernel())
        out_flt = torch.zeros_like(out_ctx)
        flt.Upscale(buf, out_flt, W, H, F.State(renderWidth=rw, renderHeight=rh, rcasAttenuation=0.25))
        e_flags = flags & ~api.FLAG_FUSED
        api.easu(crop, tmp, con, flags=e_flags)
        assert_kernel(con, content, e_flags)
        kernel = api.last_kernel()
        torch.cuda.synchronize()
        assert torch.equal(out_ctx, want), (rw, rh)
        assert torch.equal(out_flt, out_ctx), (rw, rh)
        e_got, got = tmp.cpu().numpy(), out_ctx.cpu().numpy()
        what = "%dx%d %s flags=%d" % (rw, rh, fmt, flags)
        assert_within_cell_bounds(e_got, content, con, what=what)
        if fmt == "u8":
            fin = content.astype(np.float32) / np.float32(255.0)
            d = np.abs(e_got[..., :3].astype(np.int64) - _q(ol.easu(fin, W, H)[..., :3], 8).astype(np.int64))
            mid = e_got.astype(np.float32) / np.float32(255.0)
            r = np.abs(got[..., :3].astype(np.int64) - _q(ol.rcas(mid, rcon)[..., :3], 8).astype(np.int64))
            print("frame %-24s %-52s EASU max %d codes mean %.3g; RCAS max %d codes" % (what, kernel, d.max(), d.mean(), r.max()))
            assert d.max() <= 1 and r.max() <= 1, (what, int(d.max()), int(r.max()))
            continue
        e_want = ol.easu(content.astype(np.float32), W, H)
        d = np.abs(e_got.astype(np.float32) - e_want)[..., :3]
        print("frame %-24s %-52s EASU max %.3g mean %.3g" % (what, kernel, d.max(), d.mean()))
        assert d.max() <= (TOL32 if fmt == "f32" else 6e-4 if flags & api.FLAG_PRECISE else TOL16), (what, d.max())
        if fmt == "f32":
            assert np.abs(got - ol.rcas(e_got, rcon)).max() <= TOL32, what
            assert np.abs(got - ol.rcas(e_want, rcon))[..., :3].max() <= 5e-5, what
        else:
            assert np.abs(got.astype(np.float32) - ol.rcas(e_got.astype(np.float32), rcon))[..., :3].max() <= TOL16, what
            if not flags & api.FLAG_PRECISE and W > 2.1 * rw:
                # Not held end to end above 2x.  At 3x (640x360) the half-arithmetic EASU is within its own bounds (2.7e-3 of the
                # oracle, inside every cell's texel range), but on that smooth 3x content RCAS amplifies EASU errors of at most
                # 9e-4 around one pixel about 20x, to 1.9e-2, past the 1e-2 measured at 2x.  The CPU emulator, which runs the same
                # device code, gives the same numbers.
                continue
            e2e_check(got, ol.rcas(e_want, rcon), what, tight=bool(flags & api.FLAG_PRECISE))
    # a render size larger than the context's input is refused before anything is launched, even where the caller's buffer
    # is large enough to read from
    big = torch.zeros((H + 8, W + 16, 4), dtype=tdt, device="cuda")
    n0 = api.launch_count()
    for (rw, rh) in ((W + 16, H), (W, H + 8), (W + 16, H + 8)):
        with pytest.raises(api.Fsr1Error):
            ctx.upscale_render(big, rw, rh, out_ctx, 0.25, flags)
        with pytest.raises(api.Fsr1Error):
            flt.Upscale(buf, out_flt, W, H, F.State(renderWidth=rw, renderHeight=rh))
    assert api.launch_count() == n0
    ctx.close()
    flt.OnDestroy()
