"""Times display output from the sharded frame stream (fsr1_shard_create_post) against the plain RGBA16F shard followed by the separate
display passes over each slab, in one process with the legs alternated.

    python tools/shard_post_time.py [--frames 200] [--warmup 20] [--rounds 5] [--slots 8] [--json OUT]

Workloads: 1920x1080 -> 3840x2160 (2x: the fused kernels) and 2560x1440 -> 3840x2160 (1.5x: EASU + RCAS), each at 1 rank and at 8 ranks
in one process on one device (attach_local).  Display chains:
  sdr  {LFGA, TEPD8} -> RGBA8_UNORM, positional dither with the frame number
  hdr  FSR1_FLAG_SRTM_INPUT + {SRTM_INVERSE, TEPD10} -> RGB10A2_UNORM
Legs:
  A  the post shard: fsr1_shard_post(slot, frame) + fsr1_shard_submit per rank and frame; the slabs are the display image.
  B  the RGBA16F shard (same flags), then per rank, on one consumer stream after fsr1_shard_wait(slot, consumer): fsr1_srtm(inverse) /
     fsr1_lfga in place on the slab and fsr1_tepd into a UNORM slab of the caller's.  The submitting stream waits only for the passes
     of a slot's previous use before reusing it.  At 8 ranks on one device leg B has ended with FSR1_ERR_TIMEOUT in every run so
     far, with its passes on either stream: DESIGN.md §6 "Display output".  The tool checks fsr1_shard_status after every round
     and stops at the first timeout, naming the leg and rank; the JSON keeps the configurations measured before it.
Both legs' display slabs are checked bit-identical over a whole ring of slots before any timing.  Per leg: median GPU us per frame (all
ranks; CUDA events on the caller's stream, joined to the shards' streams with fsr1_shard_wait) over --rounds alternations, the spread
((max - min) / median), host us per frame of the submission loop, and the slab bytes per slot computed from the slab shapes (leg B: the
RGBA16F slab and the caller's UNORM slab).  Inputs are written once per slot; the slots are cycled without rewriting them.  Prints the
card, its power limit and SM clock (one nvidia-smi query) before and after.  Needs a GPU; there is no CPU fallback."""
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
# 8 ranks on one device use 24 streams, and a rank's flag-waiting kernel must never share a hardware work queue with the push it waits
# for: more queues than the default 8 (the driver reads this when the context is created; tests/conftest.py does the same)
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

WORKLOADS = [(1920, 1080, 3840, 2160), (2560, 1440, 3840, 2160)]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or "nvidia-smi unavailable"


def hdr(f, seed):
    """linear HDR half values: the frame times 2^e, e in [-8, 16) per texel and channel, clipped to the half range"""
    e = np.random.default_rng(seed).integers(-8, 16, size=f.shape)
    return np.clip(f.astype(np.float64) * np.exp2(e), 0.0, 65504.0).astype(np.float16)


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
    from fsr1_b200 import _lib, api
    from fsr1_b200.sharded import _DevBuf
    assert torch.cuda.is_available(), "shard_post_time.py needs a GPU"
    L = _lib.lib()
    result = {"gpu_before": gpu_info(), "frames": a.frames, "rounds": a.rounds, "slots": a.slots, "runs": []}
    print("gpu: %s" % result["gpu_before"])
    stream = torch.cuda.current_stream()
    sp = ctypes.c_void_p(stream.cuda_stream)
    grain = torch.from_numpy((np.random.default_rng(1).random((64, 64, 4), np.float32) - 0.5).astype(np.float16)).cuda()
    nslots = a.slots

    def dump():  # after every configuration, so a run that stops early keeps what it measured
        if a.json:
            os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
            with open(a.json, "w") as fh:
                json.dump(result, fh, indent=1)

    # every 1-rank configuration first, then the 8-rank ones
    for world, (iw, ih, ow, oh), chain in [(w, s, c) for w in (1, 8) for s in WORKLOADS for c in ("sdr", "hdr")]:
        bits, flags = (8, 0) if chain == "sdr" else (10, api.FLAG_SRTM_INPUT)
        post_kw = dict(grain=grain, amount=0.25, tepd_bits=8) if chain == "sdr" else dict(srtm_inverse=True, tepd_bits=10)
        srcs = []
        for k in range(nslots):
            f = F.uniform(iw, ih, 300 + k)
            srcs.append(torch.from_numpy(np.ascontiguousarray(F.to_half(f) if chain == "sdr" else hdr(f, k))).cuda())
        legs = {}
        for leg in ("A", "B"):
            kw = post_kw if leg == "A" else {}
            ups = [F.ShardedUpscaler(iw, ih, ow, oh, world, r, slots=nslots, halo="p2p", attach=False, flags=flags, **kw)
                   for r in range(world)]
            for r, u in enumerate(ups):
                u.attach_local(ups[r - 1] if r > 0 else None, ups[r + 1] if r + 1 < world else None)
                o0, o1 = u.plan.owned_in_rows(r)
                for k in range(nslots):
                    u.input(k).copy_(srcs[k][o0:o1])
            legs[leg] = ups
        # leg A: one fsr1_post per rank, its frame set before every submit
        posts_a = []
        for u in legs["A"]:
            g = api.image(grain) if chain == "sdr" else None
            ops = (_lib.POST_LFGA | _lib.POST_TEPD8) if chain == "sdr" else (_lib.POST_SRTM_INVERSE | _lib.POST_TEPD10)
            posts_a.append((_lib.Post(ops, 0.25, ctypes.pointer(g) if g is not None else None, None, 0, 0), g))
        # leg B: the passes over each slab, marshalled once: (slab image, display image, rows) per rank and slot.  They run on a
        # consumer stream ordered after fsr1_shard_wait, so the submitting stream never waits for a frame
        consumer = torch.cuda.Stream()
        csp = ctypes.c_void_p(consumer.cuda_stream)
        passes_done = [torch.cuda.Event() for _ in range(nslots)]
        for ev in passes_done:
            ev.record(consumer)
        disp_b, b_args = [], []
        g_img = api.image(grain)
        for r, u in enumerate(legs["B"]):
            y0, y1 = u.plan.out_rows(r)
            per = []
            for k in range(nslots):
                d = torch.empty((y1 - y0, ow, 4), dtype=torch.uint8, device="cuda") if bits == 8 else \
                    torch.empty((y1 - y0, ow), dtype=torch.int32, device="cuda")
                disp_b.append(d)
                per.append((api.image(u.output(k), height=oh, row0=y0), api.image(d, height=oh, row0=y0), y0, y1))
            b_args.append(per)

        def submit_a(f):
            k = f % nslots
            bad = 0
            for u, (p, _) in zip(legs["A"], posts_a):
                p.frame = f
                bad |= L.fsr1_shard_post(u._shard, k, ctypes.byref(p))
                bad |= L.fsr1_shard_submit(u._shard, k, sp)
            return bad

        def submit_b(f):
            k = f % nslots
            bad = 0
            stream.wait_event(passes_done[k])               # the passes of the slot's previous use have read its slab
            for u in legs["B"]:
                bad |= L.fsr1_shard_submit(u._shard, k, sp)
            for u, per in zip(legs["B"], b_args):
                slab, disp, y0, y1 = per[k]
                bad |= L.fsr1_shard_wait(u._shard, k, csp)
                if chain == "sdr":
                    bad |= L.fsr1_lfga(ctypes.byref(slab), ctypes.byref(g_img), ctypes.byref(slab), ctypes.c_float(0.25), y0, y1, csp)
                else:
                    bad |= L.fsr1_srtm(ctypes.byref(slab), ctypes.byref(slab), 1, y0, y1, csp)
                bad |= L.fsr1_tepd(ctypes.byref(slab), None, ctypes.byref(disp), bits, f, y0, y1, csp)
            passes_done[k].record(consumer)
            return bad

        def check(phase):
            """fsr1_shard_status of every rank of both legs; on a timeout, which shard and the non-zero words of its flags page"""
            torch.cuda.synchronize()
            for name, ups in legs.items():
                for u in ups:
                    rc = L.fsr1_shard_status(u._shard)
                    if rc:
                        page = torch.as_tensor(_DevBuf(L.fsr1_shard_arena(u._shard), (1024,), (4,), "<i4"), device="cuda")
                        nz = {i: int(v) for i, v in enumerate(page.cpu().tolist()) if v}
                        raise RuntimeError("%s: leg %s rank %d status %d (detail %d); non-zero flag words %s" % (
                            phase, name, u.rank, rc, L.fsr1_last_cuda_error(), nz))

        def join(name):
            bad = 0
            for u in legs[name]:
                for k in range(nslots):
                    bad |= L.fsr1_shard_wait(u._shard, k, sp)
            if name == "B":
                stream.wait_stream(consumer)
            return bad

        # bit-identity over a whole ring before timing
        check("after create")
        for f in range(nslots):
            assert submit_a(f) == 0 and submit_b(f) == 0
        assert join("A") == 0 and join("B") == 0
        check("after the first ring")
        for k in range(nslots):
            a_img = torch.cat([u.output(k) for u in legs["A"]])
            b_img = torch.cat([disp_b[r * nslots + k] for r in range(world)])
            assert torch.equal(a_img, b_img), (iw, ih, chain, world, k)
        fns = {"A": submit_a, "B": submit_b}
        gpu, host = {"A": [], "B": []}, {"A": [], "B": []}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(a.rounds):
            for name in ("A", "B"):
                fn = fns[name]
                bad = 0
                for f in range(a.warmup):
                    bad |= fn(f)
                bad |= join(name)
                torch.cuda.synchronize()
                e0.record()
                t0 = time.perf_counter()
                for f in range(a.frames):
                    bad |= fn(f)
                t1 = time.perf_counter()
                bad |= join(name)
                e1.record()
                e1.synchronize()
                assert bad == 0, bad
                gpu[name].append(e0.elapsed_time(e1) * 1000.0 / a.frames)
                host[name].append((t1 - t0) * 1e6 / a.frames)
                check("after a timed round of leg %s" % name)
        # slab bytes per slot, all ranks, from the slab shapes (pitch x rows)
        slab_a = sum(u.output(0).stride(0) * u.output(0).element_size() * u.output(0).shape[0] for u in legs["A"])
        slab_b = sum(u.output(0).stride(0) * 2 * u.output(0).shape[0] for u in legs["B"]) + \
            sum(disp_b[r * nslots].stride(0) * disp_b[r * nslots].element_size() * disp_b[r * nslots].shape[0] for r in range(world))
        run = {"shape": [iw, ih, ow, oh], "chain": chain, "world": world, "slab_bytes_per_slot": {"A": slab_a, "B": slab_b}}
        for name in ("A", "B"):
            g, h = np.array(gpu[name]), np.array(host[name])
            run[name] = {"gpu_us_per_frame": float(np.median(g)), "spread": float((g.max() - g.min()) / np.median(g)),
                         "host_us_per_frame": float(np.median(h)), "all_gpu": g.tolist()}
            print("%dx%d->%dx%d %s world %d leg %s %8.1f us/frame GPU (spread %4.1f%%)  host %7.1f us/frame  slabs %6.1f MB/slot" % (
                iw, ih, ow, oh, chain, world, name, np.median(g), 100.0 * (g.max() - g.min()) / np.median(g), np.median(h),
                run["slab_bytes_per_slot"][name] / 1e6))
        sys.stdout.flush()
        result["runs"].append(run)
        dump()
        for ups in legs.values():
            for u in ups:
                u.close()
    result["gpu_after"] = gpu_info()
    print("gpu: %s" % result["gpu_after"])
    dump()


if __name__ == "__main__":
    main()
