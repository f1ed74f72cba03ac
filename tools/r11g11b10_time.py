"""Times R11G11B10_FLOAT input against RGBA16F input holding the same values, in one process with the legs alternated.

    python tools/r11g11b10_time.py [--frames 200] [--reps 5] [--ring 8]

Legs, each pair on the same values (r11: raw R11G11B10F codes, 4 B/px; rgba16f: the decoded RGBA16F image, 8 B/px):
  1080p -> 4K  fsr1_upscale(FUSED)                                (the fused EASU->RCAS kernel)
  1440p -> 4K  fsr1_upscale(FUSED)                                (1.5x: EASU + RCAS through the intermediate)
  1080p -> 4K  fsr1_upscale_post(FUSED | SRTM_INPUT, SRTM_INVERSE | TEPD10)   (the HDR round trip, linear HDR input)
Each leg walks a ring of frame sets larger than the 50 MB L2 and is timed with CUDA events over --frames frames after a warm-up; the two
legs' outputs are checked bit-identical before any timing.  Prints the card, its power limit and SM clock (before and after), then one
line per leg: median us per frame over --reps alternations and the spread (max - min) / median.  Needs a GPU; there is no CPU fallback."""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from srtm_input_time import gpu_info, report, timed  # noqa: E402


def codes(iw, ih, seed, hdr):
    """R11G11B10F codes: raw random words, or (hdr) linear HDR values (the LCG frame times 2^e, e in [-8, 16)) truncated to the format"""
    rng = np.random.default_rng(seed)
    if not hdr:
        return rng.integers(0, 1 << 32, size=(ih, iw), dtype=np.uint64).astype(np.uint32)
    import fsr1_b200 as F
    f = F.uniform(iw, ih, seed).astype(np.float32) * np.exp2(rng.integers(-8, 16, size=(ih, iw, 4)).astype(np.float32))
    x = np.clip(f, 0.0, 65024.0).astype(np.float16).view(np.uint16).astype(np.uint32)
    return (x[..., 0] >> 4) | ((x[..., 1] >> 4) << 11) | ((x[..., 2] >> 5) << 22)


def decode(c):
    """the RGBA16F image of the codes' values (exact: shifts only), as float16 [H, W, 4]"""
    r, g, b = (c & 0x7FF) << 4, ((c >> 11) & 0x7FF) << 4, ((c >> 22) & 0x3FF) << 5
    return np.stack([r, g, b, np.full_like(r, 0x3C00)], axis=-1).astype(np.uint16).view(np.float16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ring", type=int, default=8)
    a = ap.parse_args()
    import torch
    from fsr1_b200 import api
    assert torch.cuda.is_available(), "r11g11b10_time.py needs a GPU"
    print("gpu: %s" % gpu_info())
    rcon = api.rcas_con(0.25)
    R11 = api.FORMAT_R11G11B10_FLOAT
    for iw, ih, ow, oh, post in ((1920, 1080, 3840, 2160, False), (2560, 1440, 3840, 2160, False), (1920, 1080, 3840, 2160, True)):
        econ = api.easu_con(iw, ih, iw, ih, ow, oh)
        c = [codes(iw, ih, 100 + i, post) for i in range(a.ring)]
        srcs = {"r11": [torch.from_numpy(x.view(np.int32)).cuda() for x in c], "rgba16f": [torch.from_numpy(decode(x)).cuda() for x in c]}
        ins = {"r11": [api.image(t, format=R11) for t in srcs["r11"]], "rgba16f": [api.image(t) for t in srcs["rgba16f"]]}
        tmps = [torch.empty((oh, ow, 4), dtype=torch.float16, device="cuda") for _ in range(a.ring)]
        if post:
            outs = {k: [torch.empty((oh, ow), dtype=torch.int32, device="cuda") for _ in range(a.ring)] for k in ins}
        else:
            outs = {k: [torch.empty((oh, ow, 4), dtype=torch.float16, device="cuda") for _ in range(a.ring)] for k in ins}

        def leg(k):
            if post:
                return lambda i: api.upscale_post(ins[k][i], tmps[i], outs[k][i], econ, rcon, srtm_inverse=True, tepd_bits=10, frame=i,
                                                  flags=api.FLAG_FUSED | api.FLAG_SRTM_INPUT)
            return lambda i: api.upscale(ins[k][i], tmps[i], outs[k][i], econ, rcon, flags=api.FLAG_FUSED)

        legs = {k: leg(k) for k in ins}
        names = {}
        for i in range(a.ring):
            for k, fn in legs.items():
                fn(i)
                names[k] = api.last_kernel()
        torch.cuda.synchronize()
        for i in range(a.ring):
            assert torch.equal(outs["r11"][i].view(torch.int16 if not post else torch.int32),
                               outs["rgba16f"][i].view(torch.int16 if not post else torch.int32)), (iw, ih, i)
        print("  kernels: %s" % names)
        report("%dx%d->%dx%d %s" % (iw, ih, ow, oh, "hdr round trip" if post else "upscale"), timed(legs, a))
        del ins, srcs, tmps, outs
        torch.cuda.empty_cache()
    print("gpu: %s" % gpu_info())


if __name__ == "__main__":
    main()
