"""Times the two-kernel schedule against the fused EASU->RCAS kernel for 2x RGBA16F frames, in one process.

    python tools/fused_schedule.py [--rounds 5] [--frames 200] [--json OUT]

Legs, per workload (1080p->4K and 2160p->8K fp16, ring of 8 frame sets > L2, inputs resident in HBM):
  two_kernel  fsr1_easu + fsr1_rcas per frame, whole frames on two streams in turn (the schedule fsr1_shard_submit used
              before the fused kernel became its default for these frames)
  fused       fsr1_upscale with FSR1_FLAG_FUSED, frames on two streams in turn
  easu, rcas, fused_alone   each kernel on its own, one stream
Pipelined legs alternate A/B in every round; each leg reports the median and the min..max over the rounds.  CUDA events on
the launching stream.  The GPU's name, enforced power limit and SM clock (sampled right after each round) go with the numbers.
Reads device state only; changes none.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import fsr1_b200 as F  # noqa: E402

api = F.api
WORKLOADS = {"1080p-4k-fp16": (1920, 1080, 3840, 2160), "2160p-8k-fp16": (3840, 2160, 7680, 4320)}
RING = 8
BPP = 8


def device_info():
    """(name, power limit W, SM clock MHz) of cuda:0 — queries only."""
    name = torch.cuda.get_device_name(0)
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(0)
        return name, pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0, pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)
    except Exception:  # noqa: BLE001
        try:
            out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader,nounits"],
                                          text=True).strip().split(",")
            return name, float(out[0]), float(out[1])
        except Exception:  # noqa: BLE001
            return name, None, None


class Workload:
    def __init__(self, iw, ih, ow, oh):
        self.iw, self.ih, self.ow, self.oh = iw, ih, ow, oh
        dev = torch.device("cuda", 0)
        self.ins = [torch.from_numpy(F.to_half(F.uniform(iw, ih, 12345 + t))).to(dev) for t in range(RING)]
        self.tmps = [torch.empty((oh, ow, 4), dtype=torch.float16, device=dev) for _ in range(RING)]
        self.outs = [torch.empty((oh, ow, 4), dtype=torch.float16, device=dev) for _ in range(RING)]
        self.outs_f = [torch.empty((oh, ow, 4), dtype=torch.float16, device=dev) for _ in range(RING)]
        self.ei = [api.image(t) for t in self.ins]
        self.ti = [api.image(t) for t in self.tmps]
        self.oi = [api.image(t) for t in self.outs]
        self.fi = [api.image(t) for t in self.outs_f]
        self.econ = (ctypes.c_uint32 * 16)(*api.easu_con(iw, ih, iw, ih, ow, oh))
        self.rcon = (ctypes.c_uint32 * 4)(*api.rcas_con(0.25))
        self.L = F._lib.lib()
        self.main = torch.cuda.current_stream()
        self.streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        self.sp = [ctypes.c_void_p(s.cuda_stream) for s in self.streams]
        self.mp = ctypes.c_void_p(self.main.cuda_stream)
        self.done = [torch.cuda.Event() for _ in range(RING)]

    # one frame of each schedule; slot k always lands on the same stream (RING is even), as in fsr1_shard_submit
    def easu(self, i, s):
        k = i % RING
        rc = self.L.fsr1_easu(ctypes.byref(self.ei[k]), ctypes.byref(self.ti[k]), self.econ, 0, self.oh, 0, s)
        assert rc == 0, rc

    def rcas(self, i, s):
        k = i % RING
        rc = self.L.fsr1_rcas(ctypes.byref(self.ti[k]), ctypes.byref(self.oi[k]), self.rcon, 0, self.oh, 0, s)
        assert rc == 0, rc

    def fused(self, i, s):
        k = i % RING
        rc = self.L.fsr1_upscale(ctypes.byref(self.ei[k]), ctypes.byref(self.ti[k]), ctypes.byref(self.fi[k]), self.econ, self.rcon,
                                 0, self.oh, api.FLAG_FUSED, s)
        assert rc == 0, rc

    def two_kernel(self, i, s):
        self.easu(i, s)
        self.rcas(i, s)

    def timed(self, frame, n, pipelined):
        """ms per frame over n frames."""
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(self.main)
        if pipelined:
            for st in self.streams:
                st.wait_stream(self.main)
            for i in range(n):
                frame(i, self.sp[i & 1])
            for st in self.streams:
                self.main.wait_stream(st)
        else:
            for i in range(n):
                frame(i, self.mp)
        b.record(self.main)
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n


def stats(v):
    v = sorted(v)
    return {"median": float(np.median(v)), "min": v[0], "max": v[-1], "spread_pct": 100.0 * (v[-1] - v[0]) / float(np.median(v))}


def run(name, dims, rounds, n, warm):
    iw, ih, ow, oh = dims
    w = Workload(*dims)
    pin, pout = iw * ih, ow * oh
    alg = {"two_kernel": BPP * (pin + pout) + BPP * 2 * pout, "fused": BPP * (pin + pout), "easu": BPP * (pin + pout),
           "rcas": BPP * 2 * pout, "fused_alone": BPP * (pin + pout)}
    legs = [("two_kernel", w.two_kernel, True), ("fused", w.fused, True), ("easu", w.easu, False), ("rcas", w.rcas, False),
            ("fused_alone", w.fused, False)]
    kernels = {}
    for leg, fn, pip in legs:
        w.timed(fn, warm, pip)
        kernels[leg] = api.last_kernel()
    # the fused output equals the two-kernel output bit for bit on every slot
    for i in range(RING):
        w.two_kernel(i, w.mp)
        w.fused(i, w.mp)
    torch.cuda.synchronize()
    identical = all(torch.equal(w.outs[k], w.outs_f[k]) for k in range(RING))
    t = {leg: [] for leg, _, _ in legs}
    clocks = []
    for r in range(rounds):
        order = legs if r % 2 == 0 else [legs[1], legs[0]] + legs[2:]
        for leg, fn, pip in order:
            t[leg].append(w.timed(fn, n, pip) * 1e3)
        clocks.append(device_info()[2])
    res = {"workload": name, "fused_equals_two_kernel": identical, "sm_mhz_after_rounds": clocks, "legs": {}}
    for leg, _, _ in legs:
        s = stats(t[leg])
        s.update({"kernel": kernels[leg], "us": t[leg], "mpix_s": pout / s["median"], "alg_GBps": alg[leg] / (s["median"] * 1e-6) / 1e9})
        res["legs"][leg] = s
    res["fused_speedup"] = res["legs"]["two_kernel"]["median"] / res["legs"]["fused"]["median"]
    del w
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=200, help="frames per timed leg")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--workload", action="append", choices=list(WORKLOADS), help="default: all")
    ap.add_argument("--json", default=None, help="also write the results here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fused_schedule.py times kernels: it needs a CUDA device")
    torch.cuda.set_device(0)
    gpu, limit, sm = device_info()
    out = {"gpu": gpu, "power_limit_w": limit, "sm_mhz_at_start": sm, "rounds": args.rounds, "frames_per_leg": args.frames, "results": []}
    print("%s, power limit %s W, SM clock %s MHz at start; %d rounds x %d frames per leg, A/B alternated" % (
        gpu, limit, sm, args.rounds, args.frames))
    for name in args.workload or list(WORKLOADS):
        r = run(name, WORKLOADS[name], args.rounds, args.frames, args.warmup)
        out["results"].append(r)
        print("%s: fused output == two-kernel output on every slot: %s; SM MHz after each round %s" % (
            name, r["fused_equals_two_kernel"], r["sm_mhz_after_rounds"]))
        for leg, s in r["legs"].items():
            print("  %-12s %8.1f us/frame  (min %.1f max %.1f, spread %.1f%%)  %7.0f Mpix/s  %6.0f GB/s algorithmic  %s" % (
                leg, s["median"], s["min"], s["max"], s["spread_pct"], s["mpix_s"], s["alg_GBps"], s["kernel"]))
        print("  fused / two_kernel speed-up (medians): %.3fx" % r["fused_speedup"])
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
