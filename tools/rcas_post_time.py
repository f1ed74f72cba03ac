"""Times fsr1_rcas_post (a frame rendered at display size, sharpened straight to display output in one kernel) against the routes it
replaces, in one process with the legs alternated.

    python tools/rcas_post_time.py [--frames 100] [--reps 5] [--ring 4]

Legs at 3840x2160:
  sdr:   fsr1_rcas + fsr1_lfga + fsr1_tepd(8) -> RGBA8                vs  fsr1_rcas_post(LFGA | TEPD8)
  hdr:   fsr1_srtm + fsr1_rcas + fsr1_srtm(inverse) + fsr1_tepd(10)   vs  fsr1_rcas_post(SRTM_INPUT; SRTM_INVERSE | TEPD10) -> RGB10A2
  r11:   that fsr1_rcas_post call on R11G11B10F codes                 vs  on the RGBA16F image of their values
  ctx:   fsr1_context_upscale_post at render size = display size (EASU at 1x + RCAS with the epilogue), the one call available before,
         with the hdr leg's steps; timed for its cost only (it runs EASU, so its bits differ)
Each leg walks a ring of frame sets larger than the 50 MB L2 and is timed with CUDA events over --frames frames after a warm-up; the
compared legs' outputs are checked bit-identical before any timing.  Prints the card, its power limit and SM clock (before and after),
then one line per leg: median us per frame over --reps alternations and the spread (max - min) / median.  Needs a GPU."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from srtm_input_time import gpu_info, hdr, report, timed  # noqa: E402


def r11_of(x16):
    """R11G11B10F codes (int32 [H, W]) of an RGBA16F image of non-negative finite values, each half truncated to the format's mantissa"""
    import torch
    b = x16.view(torch.int16).to(torch.int32) & 0x7FFF
    return (b[..., 0] >> 4) | ((b[..., 1] >> 4) << 11) | ((b[..., 2] >> 5) << 22)


def decode(codes):
    import torch
    c = codes.to(torch.int64) & 0xFFFFFFFF
    r, g, b = (c & 0x7FF) << 4, ((c >> 11) & 0x7FF) << 4, ((c >> 22) & 0x3FF) << 5
    return torch.stack([r, g, b, torch.full_like(r, 0x3C00)], dim=-1).to(torch.int16).view(torch.float16)


def check_equal(outs, what):
    import torch
    torch.cuda.synchronize()
    a, b = list(outs.values())
    for i in range(len(a)):
        assert torch.equal(a[i].view(torch.uint8), b[i].view(torch.uint8)), (what, i)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ring", type=int, default=4)
    a = ap.parse_args()
    import torch
    import fsr1_b200 as F
    from fsr1_b200 import api
    assert torch.cuda.is_available(), "rcas_post_time.py needs a GPU"
    print("gpu: %s" % gpu_info())
    w, h = 3840, 2160
    rcon = api.rcas_con(0.25)
    S = api.FLAG_SRTM_INPUT
    grain = torch.from_numpy((np.random.default_rng(1).random((64, 64, 4), np.float32) - 0.5).astype(np.float16)).cuda()
    sdr = [torch.from_numpy(F.to_half(F.uniform(w, h, 100 + i))).cuda() for i in range(a.ring)]
    hdr16 = [torch.from_numpy(hdr(w, h, 200 + i)).cuda() for i in range(a.ring)]
    r11 = [r11_of(x) for x in hdr16]
    dec = [decode(c) for c in r11]
    t1 = [torch.empty((h, w, 4), dtype=torch.float16, device="cuda") for _ in range(a.ring)]
    t2 = [torch.empty_like(x) for x in t1]
    u8 = {k: [torch.empty((h, w, 4), dtype=torch.uint8, device="cuda") for _ in range(a.ring)] for k in ("passes", "rcas_post")}
    u10 = {k: [torch.empty((h, w), dtype=torch.int32, device="cuda") for _ in range(a.ring)] for k in ("passes", "rcas_post", "ctx")}
    print("compulsory bytes per pixel: sdr passes 44, rcas_post 12; hdr passes 60, rcas_post 12; r11 rcas_post 8")

    def sdr_passes(i):
        api.rcas(sdr[i], t1[i], rcon)
        api.lfga(t1[i], grain, t1[i], 0.3)
        api.tepd(t1[i], u8["passes"][i], 8, frame=i)

    def sdr_post(i):
        api.rcas_post(sdr[i], u8["rcas_post"][i], rcon, grain=grain, amount=0.3, tepd_bits=8, frame=i)

    def hdr_passes(i):
        api.srtm(hdr16[i], t1[i])
        api.rcas(t1[i], t2[i], rcon)
        api.srtm(t2[i], t2[i], inverse=True)
        api.tepd(t2[i], u10["passes"][i], 10, frame=i)

    def hdr_post(i):
        api.rcas_post(hdr16[i], u10["rcas_post"][i], rcon, srtm_inverse=True, tepd_bits=10, frame=i, flags=S)

    r11_out = {k: [torch.empty((h, w), dtype=torch.int32, device="cuda") for _ in range(a.ring)] for k in ("r11", "rgba16f")}

    def r11_post(i):
        api.rcas_post(api.image(r11[i], format=api.FORMAT_R11G11B10_FLOAT), r11_out["r11"][i], rcon, srtm_inverse=True, tepd_bits=10,
                      frame=i, flags=S)

    def h16_post(i):
        api.rcas_post(dec[i], r11_out["rgba16f"][i], rcon, srtm_inverse=True, tepd_bits=10, frame=i, flags=S)

    ctx = api.HostContext(w, h, w, h)

    def ctx_post(i):
        ctx.upscale_post(hdr16[i], u10["ctx"][i], sharpness=0.25, srtm_inverse=True, tepd_bits=10, frame=i, flags=S)

    for i in range(a.ring):
        for fn in (sdr_passes, sdr_post, hdr_passes, hdr_post, r11_post, h16_post, ctx_post):
            fn(i)
    check_equal(u8, "sdr")
    check_equal({k: u10[k] for k in ("passes", "rcas_post")}, "hdr")
    check_equal(r11_out, "r11")
    report("3840x2160 sdr (LFGA, TEPD8)", timed({"passes": sdr_passes, "rcas_post": sdr_post}, a))
    report("3840x2160 hdr (SRTM, SRTM_INV, TEPD10)", timed({"passes": hdr_passes, "rcas_post": hdr_post}, a))
    report("3840x2160 hdr rcas_post input", timed({"r11": r11_post, "rgba16f": h16_post}, a))
    report("3840x2160 hdr, context at 1x", timed({"ctx_1x": ctx_post, "rcas_post": hdr_post}, a))
    ctx.close()
    print("gpu: %s" % gpu_info())


if __name__ == "__main__":
    main()
