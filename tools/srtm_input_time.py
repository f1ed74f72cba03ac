"""Times FSR1_FLAG_SRTM_INPUT against the separate fsr1_srtm pass it replaces, in one process with the legs alternated.

    python tools/srtm_input_time.py [--frames 200] [--reps 5] [--ring 8]

Legs, each on linear HDR RGBA16F frames:
  1080p -> 4K and 2160p -> 8K (2x: the fused EASU->RCAS kernel), 1440p -> 4K (1.5x: EASU + RCAS):
    pass:  fsr1_srtm(in, I) + fsr1_upscale(I, FUSED)            prologue:  fsr1_upscale(in, FUSED | SRTM_INPUT)
  1080p -> 4K, the HDR round trip to RGB10A2:
    pass:  fsr1_srtm + fsr1_upscale_post(SRTM_INVERSE | TEPD10)  prologue:  fsr1_upscale_post(FUSED | SRTM_INPUT, SRTM_INVERSE | TEPD10)
  and the fsr1_srtm pass alone at 1080p and 2160p.
Each leg walks a ring of frame sets larger than the 50 MB L2 and is timed with CUDA events over --frames frames after a warm-up; the two
legs' outputs are checked bit-identical before any timing.  Prints the card, its power limit and SM clock (before and after), then one
line per leg: median us per frame over --reps alternations and the spread (max - min) / median.  Needs a GPU; there is no CPU fallback."""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "nvidia-smi unavailable"


def hdr(iw, ih, seed):
    """linear HDR half values: the LCG frame times 2^e, e in [-8, 16)"""
    import fsr1_b200 as F
    f = F.uniform(iw, ih, seed).astype(np.float32)
    e = np.random.default_rng(seed).integers(-8, 16, size=f.shape).astype(np.float32)
    return np.clip(f * np.exp2(e), 0.0, 65504.0).astype(np.float16)


def timed(legs, a):
    import torch
    times = {k: [] for k in legs}
    for _ in range(a.reps):
        for name, fn in legs.items():
            for f in range(a.warmup):
                fn(f % a.ring)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for f in range(a.frames):
                fn(f % a.ring)
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1) * 1000.0 / a.frames)
    return times


def report(label, times):
    for name, t in times.items():
        t = np.array(t)
        print("%-34s %-9s %8.1f us/frame (spread %.1f%%)" % (label, name, np.median(t), 100.0 * (t.max() - t.min()) / np.median(t)))
    sys.stdout.flush()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ring", type=int, default=8)
    a = ap.parse_args()
    import torch
    from fsr1_b200 import api
    assert torch.cuda.is_available(), "srtm_input_time.py needs a GPU"
    print("gpu: %s" % gpu_info())
    rcon = api.rcas_con(0.25)
    S = api.FLAG_SRTM_INPUT
    for iw, ih, ow, oh in ((1920, 1080, 3840, 2160), (3840, 2160, 7680, 4320), (2560, 1440, 3840, 2160)):
        econ = api.easu_con(iw, ih, iw, ih, ow, oh)
        ins = [torch.from_numpy(hdr(iw, ih, 100 + i)).cuda() for i in range(a.ring)]
        mids = [torch.empty_like(x) for x in ins]
        tmps = [torch.empty((oh, ow, 4), dtype=torch.float16, device="cuda") for _ in range(a.ring)]
        outs = {k: [torch.empty((oh, ow, 4), dtype=torch.float16, device="cuda") for _ in range(a.ring)] for k in ("pass", "prologue")}

        def pass_leg(i):
            api.srtm(ins[i], mids[i])
            api.upscale(mids[i], tmps[i], outs["pass"][i], econ, rcon, flags=api.FLAG_FUSED)

        def prologue_leg(i):
            api.upscale(ins[i], tmps[i], outs["prologue"][i], econ, rcon, flags=api.FLAG_FUSED | S)

        legs = {"pass": pass_leg, "prologue": prologue_leg}
        for i in range(a.ring):
            pass_leg(i)
            prologue_leg(i)
        torch.cuda.synchronize()
        for i in range(a.ring):
            assert torch.equal(outs["pass"][i], outs["prologue"][i]), (iw, ih, i)
        report("%dx%d->%dx%d upscale" % (iw, ih, ow, oh), timed(legs, a))
        if ow == 2 * iw and iw <= 1920:
            r10 = {k: [torch.empty((oh, ow), dtype=torch.int32, device="cuda") for _ in range(a.ring)] for k in legs}

            def pass_post(i):
                api.srtm(ins[i], mids[i])
                api.upscale_post(mids[i], tmps[i], r10["pass"][i], econ, rcon, srtm_inverse=True, tepd_bits=10, frame=i,
                                 flags=api.FLAG_FUSED)

            def prologue_post(i):
                api.upscale_post(ins[i], tmps[i], r10["prologue"][i], econ, rcon, srtm_inverse=True, tepd_bits=10, frame=i,
                                 flags=api.FLAG_FUSED | S)

            post_legs = {"pass": pass_post, "prologue": prologue_post}
            for i in range(a.ring):
                pass_post(i)
                prologue_post(i)
            torch.cuda.synchronize()
            for i in range(a.ring):
                assert torch.equal(r10["pass"][i], r10["prologue"][i]), ("post", iw, ih, i)
            report("%dx%d->%dx%d hdr round trip" % (iw, ih, ow, oh), timed(post_legs, a))
        if ow == 2 * iw:
            report("%dx%d fsr1_srtm alone (%.1f MB)" % (iw, ih, 2 * 8 * iw * ih / 1e6), timed({"srtm": lambda i: api.srtm(ins[i], mids[i])}, a))
        del ins, mids, tmps, outs
        torch.cuda.empty_cache()
    print("gpu: %s" % gpu_info())


if __name__ == "__main__":
    main()
