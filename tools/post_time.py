"""Times fsr1_upscale_post against the sequence of calls it replaces, in one process with the legs alternated.

    python tools/post_time.py [--frames 200] [--reps 5] [--ring 8]

Two display chains at two scales:
  sdr:  upscale, LFGA, TEPD 8-bit -> RGBA8_UNORM          (sequence: fsr1_upscale(FUSED) + fsr1_lfga + fsr1_tepd)
  hdr:  upscale, TEPD 10-bit -> RGB10A2_UNORM             (sequence: fsr1_upscale(FUSED) + fsr1_tepd)
  1080p -> 4K (2x: the fused EASU->RCAS kernel) and 1440p -> 4K (1.5x: EASU + RCAS).
Each leg walks a ring of frame sets larger than the 50 MB L2, is timed with CUDA events over --frames frames after a warm-up, and
the two legs' outputs are checked bit-identical before any timing.  Prints one line per (scale, chain, leg): median us per frame over
--reps alternations, and the compulsory HBM bytes per output pixel.  Needs a GPU; there is no CPU fallback."""
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


def compulsory_bytes(iw, ih, ow, oh, chain, fused_leg):
    """HBM bytes per output pixel the algorithm must move: input once, every intermediate image written and read once, output once."""
    inp = 8.0 * iw * ih / (ow * oh)
    two_x = 2 * iw == ow and 2 * ih == oh
    up = 0.0 if two_x else 16.0                        # EASU -> RCAS intermediate (8 B written, 8 B read) off the fused path
    out = 4.0
    if fused_leg:
        return inp + up + out
    steps = (16.0 if chain == "sdr" else 0.0) + 8.0    # LFGA reads + writes RGBA16F; TEPD reads RGBA16F
    return inp + up + 8.0 + steps + out                # + the RGBA16F upscale output


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ring", type=int, default=8)
    a = ap.parse_args()
    import torch
    import fsr1_b200 as F
    from fsr1_b200 import api
    assert torch.cuda.is_available(), "post_time.py needs a GPU"
    print("gpu: %s" % gpu_info())
    grain = torch.from_numpy((np.random.default_rng(1).random((64, 64, 4), np.float32) - 0.5).astype(np.float16)).cuda()
    rcon = api.rcas_con(0.25)
    for iw, ih, ow, oh in ((1920, 1080, 3840, 2160), (2560, 1440, 3840, 2160)):
        econ = api.easu_con(iw, ih, iw, ih, ow, oh)
        ins = [torch.from_numpy(F.to_half(F.uniform(iw, ih, 100 + i))).cuda() for i in range(a.ring)]
        tmps = [torch.empty((oh, ow, 4), dtype=torch.float16, device="cuda") for _ in range(a.ring)]
        mids = [torch.empty((oh, ow, 4), dtype=torch.float16, device="cuda") for _ in range(a.ring)]
        for chain in ("sdr", "hdr"):
            bits = 8 if chain == "sdr" else 10
            g = grain if chain == "sdr" else None

            def outs():
                if bits == 8:
                    return [torch.empty((oh, ow, 4), dtype=torch.uint8, device="cuda") for _ in range(a.ring)]
                return [torch.empty((oh, ow), dtype=torch.int32, device="cuda") for _ in range(a.ring)]
            seq_out, post_out = outs(), outs()

            def seq(i):
                api.upscale(ins[i], tmps[i], mids[i], econ, rcon, flags=api.FLAG_FUSED)
                if g is not None:
                    api.lfga(mids[i], g, mids[i], 0.25)
                api.tepd(mids[i], seq_out[i], bits, frame=i)

            def post(i):
                api.upscale_post(ins[i], tmps[i], post_out[i], econ, rcon, grain=g, amount=0.25, tepd_bits=bits, frame=i,
                                 flags=api.FLAG_FUSED)

            for i in range(a.ring):
                seq(i)
                post(i)
            torch.cuda.synchronize()
            for i in range(a.ring):
                assert torch.equal(seq_out[i], post_out[i]), (iw, ih, chain, i)
            legs = {"sequence": seq, "fused": post}
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
            for name in legs:
                t = np.array(times[name])
                print("%dx%d->%dx%d %s %-8s %8.1f us/frame (spread %.1f%%)  compulsory %.1f B/px" % (
                    iw, ih, ow, oh, chain, name, np.median(t), 100.0 * (t.max() - t.min()) / np.median(t),
                    compulsory_bytes(iw, ih, ow, oh, chain, name == "fused")))
            sys.stdout.flush()
    print("gpu: %s" % gpu_info())


if __name__ == "__main__":
    main()
