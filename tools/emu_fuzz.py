"""Randomised campaign over the CPU emulator (tests/emu): random image sizes, scales, row ranges, CTA counts and options through the
production kernels' own device code, checked against the oracle.  GPU-free; minutes of CPU time.

    python tools/emu_fuzz.py [seconds=300] [seed=1]

Checks per case: 2x EASU (quad kernel) and any-scale EASU (vertical-pair kernel, also on a viewport of the resource and at an
offset, and within the de-ringing bound) within 5e-3 of the fp32 oracle, row range == the same rows of the full frame; packed RCAS within 4e-3, both out-of-image rules, options; fused kernel == two-kernel path bit for
bit; the Hx2 kernels bit-identical to the half oracle."""
import ctypes
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import fsr1_b200 as F  # noqa: E402
import oracle_lib as ol  # noqa: E402
import test_emu as te  # noqa: E402
import test_emu_hx2 as th  # noqa: E402
from easu_checks import assert_within_cell_bounds  # noqa: E402

budget = float(sys.argv[1]) if len(sys.argv) > 1 else 300.0
rng = np.random.default_rng(int(sys.argv[2]) if len(sys.argv) > 2 else 1)
t_end = time.time() + budget
n = {"easu2x": 0, "easu_any": 0, "rcas": 0, "fused": 0, "hx2": 0}
worst = {"easu2x": 0.0, "easu_any": 0.0, "rcas": 0.0}


def frame(w, h):
    gen = F.uniform if rng.integers(2) else F.structured
    return F.to_half(gen(w, h, int(rng.integers(1, 1 << 20))))


def exactly_2x(iw, ih):
    """FsrEasuCon computes in * rcp(out) in fp32: for some sizes 'twice' is 0.49999997, and the launchers then take the any-scale
    kernel (is_2x() in csrc/fsr1_common.cuh); the campaign follows them."""
    return ol.easu_con(iw, ih, 2 * iw, 2 * ih)[:4] == [0x3f000000, 0x3f000000, 0xbe800000, 0xbe800000]


def rows(oh):
    if rng.integers(3) == 0 or oh < 3:
        return 0, oh
    a = int(rng.integers(0, oh - 1))
    return a, int(rng.integers(a + 1, oh + 1))


while time.time() < t_end:
    kind = rng.integers(5)
    if kind == 0:
        iw, ih = int(rng.integers(1, 100)), int(rng.integers(1, 40))
        if not exactly_2x(iw, ih):
            continue
        src = frame(iw, ih)
        ow, oh = 2 * iw, 2 * ih
        want = ol.easu(src.astype(np.float32), ow, oh)
        got = te.emu_easu(te.PROD, src, ow, oh, ctas=int(rng.integers(1, 6)))
        err = float(np.abs(got.astype(np.float32) - want)[..., :3].max())
        assert err <= 5e-3, ("easu2x", iw, ih, err)
        y0, y1 = rows(oh)
        part = te.emu_easu(te.PROD, src, ow, oh, y0=y0, y1=y1, ctas=int(rng.integers(1, 4)))
        assert np.array_equal(part[y0:y1].view(np.uint16), got[y0:y1].view(np.uint16)), ("easu2x rows", iw, ih, y0, y1)
        worst["easu2x"] = max(worst["easu2x"], err)
        n["easu2x"] += 1
    elif kind == 1:
        iw, ih = int(rng.integers(4, 90)), int(rng.integers(4, 40))
        sx, sy = 1.0 + rng.random() * 1.2, 1.0 + rng.random() * 1.2
        ow, oh = max(iw, int(iw * sx)), max(ih, int(ih * sy))
        # half of the draws render into a viewport of the resource (dynamic resolution), some of those at an offset
        vw, vh, off = iw, ih, None
        if rng.integers(2):
            vw, vh = int(rng.integers(max(1, iw // 2), iw + 1)), int(rng.integers(max(1, ih // 2), ih + 1))
            ow, oh = max(vw, int(vw * sx)), max(vh, int(vh * sy))
            if rng.integers(2):
                off = (int(rng.integers(0, iw - vw + 1)), int(rng.integers(0, ih - vh + 1)))
        con = ol.easu_con(iw, ih, ow, oh, vw, vh, off=off)
        src = frame(iw, ih)
        want = ol.easu(src.astype(np.float32), ow, oh, con)
        got = te.emu_easu_pairs(src, ow, oh, ctas=int(rng.integers(1, 4)), con=con)
        err = float(np.abs(got.astype(np.float32) - want)[..., :3].max())
        assert err <= 5e-3, ("easu_any", iw, ih, vw, vh, off, ow, oh, err)
        assert_within_cell_bounds(got, src, con, what=("easu_any", iw, ih, vw, vh, off, ow, oh))
        y0, y1 = rows(oh)
        part = te.emu_easu_pairs(src, ow, oh, y0=y0, y1=y1, ctas=1, con=con)
        assert np.array_equal(part[y0:y1].view(np.uint16), got[y0:y1].view(np.uint16)), ("easu_any rows", iw, ih, vw, vh, off, ow, oh, y0, y1)
        worst["easu_any"] = max(worst["easu_any"], err)
        n["easu_any"] += 1
    elif kind == 2:
        w, h = int(rng.integers(1, 200)), int(rng.integers(1, 40))
        src = frame(w, h)
        sharp = float(rng.choice([0.0, 0.25, 1.0, 2.0]))
        clamp = bool(rng.integers(2))
        want = ol.rcas(src.astype(np.float32), ol.rcas_con(sharp), clamp)
        got = te.emu_rcas(src, sharp, clamp)
        err = float(np.abs(got.astype(np.float32) - want)[..., :3].max())
        assert err <= 4e-3, ("rcas", w, h, sharp, clamp, err)
        y0, y1 = rows(h)
        part = te.emu_rcas(src, sharp, clamp, y0=y0, y1=y1)
        assert np.array_equal(part[y0:y1].view(np.uint16), got[y0:y1].view(np.uint16)), ("rcas rows", w, h, y0, y1)
        worst["rcas"] = max(worst["rcas"], err)
        n["rcas"] += 1
    elif kind == 3:
        iw, ih = int(rng.integers(1, 110)), int(rng.integers(1, 30))
        if not exactly_2x(iw, ih):
            continue
        src = frame(iw, ih)
        ow, oh = 2 * iw, 2 * ih
        want = te.emu_rcas(te.emu_easu(te.PROD, src, ow, oh), 0.25).view(np.uint16)
        con = (ctypes.c_uint32 * 4)(*ol.rcas_con(0.25))
        s16 = np.ascontiguousarray(src.view(np.uint16))
        y0, y1 = rows(oh)
        out = np.zeros((oh, ow, 4), np.uint16)
        rc = te.emu_lib().emu_fused_h(ctypes.c_void_p(s16.ctypes.data), iw, ih, ctypes.c_longlong(s16.strides[0]), ctypes.c_void_p(out.ctypes.data),
                                      ow, oh, ctypes.c_longlong(out.strides[0]), con, y0, y1, int(rng.integers(1, 9)))
        assert rc == 0 and np.array_equal(out[y0:y1], want[y0:y1]), ("fused", iw, ih, y0, y1)
        assert not out[:y0].any() and not out[y1:].any()
        n["fused"] += 1
    else:
        w, h = int(rng.integers(1, 330)), int(rng.integers(1, 12))
        img = frame(w, h)
        dn, pa, clamp = bool(rng.integers(2)), bool(rng.integers(2)), bool(rng.integers(2))
        rc = ol.rcas_con(float(rng.choice([0.0, 0.25, 2.0])))
        got = th.emu_rcas_hx2(img, rc, clamp, opts=(1 if dn else 0) | (2 if pa else 0))
        assert np.array_equal(th.bits(got), th.bits(ol.rcas(img, rc, clamp, denoise=dn, alpha=pa))), ("rcas_hx2", w, h, dn, pa, clamp)
        op = int(rng.integers(1, 6))
        aux = F.to_half((F.uniform(int(rng.integers(1, 20)), int(rng.integers(1, 9)), 7) - (0.5 if op == 3 else 0.0)).astype(np.float32))
        amount, fr = float(rng.random()), int(rng.integers(0, 100))
        if op == 1 or op == 2:
            hdr = img.astype(np.float32)
            hdr[..., :3] = hdr[..., :3] ** 3 * (60.0 if op == 1 else 1.0)
            hdr = F.to_half(hdr)
            assert np.array_equal(th.bits(th.emu_point(op, hdr)), th.bits(ol.srtm_h(hdr, inverse=(op == 2)))), ("srtm_h", w, h, op)
        elif op == 3:
            assert np.array_equal(th.bits(th.emu_point(3, img, aux=aux, amount=amount)), th.bits(ol.lfga_h(img, aux, amount))), ("lfga_h", w, h)
        else:
            use = aux if rng.integers(2) else None
            assert np.array_equal(th.bits(th.emu_point(op, img, aux=use, frame=fr)),
                                  th.bits(ol.tepd_h(img, 8 if op == 4 else 10, frame=fr, dither=use))), ("tepd_h", w, h, op)
        n["hx2"] += 1
print("emu_fuzz: %s cases, all within bounds; worst max-abs vs fp32 oracle: %s" % (n, {k: round(v, 5) for k, v in worst.items()}))
