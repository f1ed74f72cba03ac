"""Times the dynamic-resolution frame stream (FSR1_SHARD_DYNAMIC, fsr1_shard_frame) on one GPU, one rank, 1920x1080 -> 3840x2160.

    python tools/shard_dynamic_time.py [--frames 200] [--rounds 5] [--slots 8] [--json OUT]

(a) a static shard against a dynamic shard that is given fsr1_shard_frame(1920, 1080) before every submit, legs alternated, --rounds
    rounds of --frames frames each.  Both run the same kernel (the fused one), so a difference is host cost: reported as GPU time per
    frame (CUDA events) and host time per frame of the submission loop (fsr1_shard_frame + fsr1_shard_submit, through ctypes).
(b) GPU time per frame of the dynamic shard fed each render size of a cycle (2x, 1.5x, 1.5x-and-a-bit, an odd size, almost 2x) for
    --frames frames, median over --rounds.
(c) 8 ranks in one process on one device (attach_local), static against dynamic at the resource size, legs alternated: the whole
    frame (all ranks) per frame.  Both run the same kernels and protocol, so a difference is host cost.
Slots are cycled without rewriting their input (the shard orders a slot's reuse after its previous frame).  Prints the card, its power
limit and SM clock before and after.  Needs a GPU; there is no CPU fallback."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(1920, 1080), (1600, 900), (1280, 720), (1477, 831), (1919, 1079)]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--slots", type=int, default=8)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    import fsr1_b200 as F
    from fsr1_b200 import _lib
    assert torch.cuda.is_available(), "shard_dynamic_time.py needs a GPU"
    L = _lib.lib()
    iw, ih, ow, oh = 1920, 1080, 3840, 2160
    result = {"gpu_before": gpu_info(), "shape": [iw, ih, ow, oh], "frames": a.frames, "rounds": a.rounds, "slots": a.slots}
    print("gpu: %s" % result["gpu_before"])
    src = torch.from_numpy(F.to_half(F.uniform(iw, ih, 5))).cuda()
    static = F.ShardedUpscaler(iw, ih, ow, oh, 1, 0, slots=a.slots, halo="p2p")
    dyn = F.ShardedUpscaler(iw, ih, ow, oh, 1, 0, slots=a.slots, halo="p2p", dynamic=True)
    stream = torch.cuda.current_stream()
    sp = ctypes.c_void_p(stream.cuda_stream)
    sharp = ctypes.c_float(0.25)
    for k in range(a.slots):
        static.input(k).copy_(src)
        dyn.input(k).copy_(src)

    def leg(up, size, n):
        """n frames; returns (us/frame from the first submit to the last frame's end on the GPU (CUDA events on the caller's
        stream, joined to the shard's streams with fsr1_shard_wait), host us/frame of the submission loop)"""
        h, rw, rh = up._shard, size[0], size[1]
        describe = up.dynamic
        for f in range(a.warmup):
            if describe:
                _lib.check(L.fsr1_shard_frame(h, f % a.slots, rw, rh, sharp))
            _lib.check(L.fsr1_shard_submit(h, f % a.slots, sp))
        for k in range(a.slots):                          # the frames run on the shard's own streams: join them
            _lib.check(L.fsr1_shard_wait(h, k, sp))
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        bad = 0
        t0 = time.perf_counter()
        for f in range(n):
            if describe:
                bad |= L.fsr1_shard_frame(h, f % a.slots, rw, rh, sharp)
            bad |= L.fsr1_shard_submit(h, f % a.slots, sp)
        t1 = time.perf_counter()
        for k in range(a.slots):
            bad |= L.fsr1_shard_wait(h, k, sp)
        e1.record()
        e1.synchronize()
        assert bad == 0, bad
        return e0.elapsed_time(e1) * 1000.0 / n, (t1 - t0) * 1e6 / n

    # (a) static against dynamic at the resource size, legs alternated
    gpu = {"static": [], "dynamic": []}
    host = {"static": [], "dynamic": []}
    for _ in range(a.rounds):
        for name, up in (("static", static), ("dynamic", dyn)):
            g, hh = leg(up, (iw, ih), a.frames)
            gpu[name].append(g)
            host[name].append(hh)
    static.status()
    dyn.status()
    result["a"] = {}
    for name in ("static", "dynamic"):
        g, hh = np.array(gpu[name]), np.array(host[name])
        result["a"][name] = {"gpu_us_per_frame": float(np.median(g)), "gpu_spread": float((g.max() - g.min()) / np.median(g)),
                             "host_us_per_frame": float(np.median(hh)), "all_gpu": g.tolist(), "all_host": hh.tolist()}
        print("(a) %-8s %8.1f us/frame GPU (spread %.1f%%)  %6.2f us/frame host" % (
            name, np.median(g), 100.0 * (g.max() - g.min()) / np.median(g), np.median(hh)))
    # (b) each render size of the cycle on the dynamic shard
    result["b"] = {}
    for size in SIZES:
        g = np.array([leg(dyn, size, a.frames)[0] for _ in range(a.rounds)])
        result["b"]["%dx%d" % size] = {"gpu_us_per_frame": float(np.median(g)), "gpu_spread": float((g.max() - g.min()) / np.median(g))}
        print("(b) %4dx%-4d %8.1f us/frame GPU (spread %.1f%%)" % (size[0], size[1], np.median(g), 100.0 * (g.max() - g.min()) / np.median(g)))
    torch.cuda.synchronize()
    dyn.status()
    static.close()
    dyn.close()
    # (c) 8 ranks in one process on this device, static against dynamic at the resource size
    result["c"] = {}
    world = 8
    legs = {}
    for name, dynamic in (("static", False), ("dynamic", True)):
        ups = [F.ShardedUpscaler(iw, ih, ow, oh, world, r, slots=a.slots, halo="p2p", attach=False, dynamic=dynamic) for r in range(world)]
        for r, u in enumerate(ups):
            u.attach_local(ups[r - 1] if r > 0 else None, ups[r + 1] if r + 1 < world else None)
            o0, o1 = u.plan.owned_in_rows(r)
            for k in range(a.slots):
                u.input(k).copy_(src[o0:o1])
        legs[name] = ups

    def ranks_leg(ups, n):
        for f in range(a.warmup + n):
            if f == a.warmup:
                for u in ups:
                    for k in range(a.slots):
                        _lib.check(L.fsr1_shard_wait(u._shard, k, sp))
                torch.cuda.synchronize()
                e0.record()
            for u in ups:
                if u.dynamic:
                    _lib.check(L.fsr1_shard_frame(u._shard, f % a.slots, iw, ih, sharp))
                _lib.check(L.fsr1_shard_submit(u._shard, f % a.slots, sp))
        for u in ups:
            for k in range(a.slots):
                _lib.check(L.fsr1_shard_wait(u._shard, k, sp))
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) * 1000.0 / n

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = {"static": [], "dynamic": []}
    for _ in range(a.rounds):
        for name in ("static", "dynamic"):
            times[name].append(ranks_leg(legs[name], a.frames))
    for name, ups in legs.items():
        for u in ups:
            u.status()
        g = np.array(times[name])
        result["c"][name] = {"us_per_frame": float(np.median(g)), "spread": float((g.max() - g.min()) / np.median(g)), "all": g.tolist()}
        print("(c) 8 ranks %-8s %8.1f us/frame (all ranks, spread %.1f%%)" % (name, np.median(g), 100.0 * (g.max() - g.min()) / np.median(g)))
        for u in ups:
            u.close()
    result["gpu_after"] = gpu_info()
    print("gpu: %s" % result["gpu_after"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
