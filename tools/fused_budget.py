"""Instruction budget of the fused 2x RGBA16F kernel (fused_h_quad2x_kernel, csrc/fsr1_fused.cu) and its issue floor.

    python tools/fused_budget.py [--size 3840x2160] [--y0 Y] [--y1 Y] [--per-sm 7] [--sms 132] [--sm-mhz 1980] [--time] [--json OUT]

Static part (no GPU needed): compiles csrc/fsr1_fused.cu to a cubin, reads its SASS with `nvdisasm -g -gi` and files every
instruction of the kernel under one region by the source lines of its inline chain:
  phase1   luma per texel (the texel_luma loop of fused_body)
  phase2   terms per texel (the texel_terms loop)
  quad     EASU of one cell row by a warp (fused_step's quad loop, quad_compute)
  rcas     fused_step after the quad barrier: the mid-row loads, rcas_pair, the stores
  control  the rest of the step loop (iterator, TMA, barriers, the mid-row carry)
  clamp    the clamp-to-edge fix-up of a box that reaches outside the input
  setup    fused_body outside the step loop
and, for quad and rcas, the interior copy (fused_step<true>) or the edge copy (fused_step<false>).
Trip counts come from a Python copy of FusedIter and fused_setup's grid (shares, runs, steps, interior or edge); the static
counts are multiplied by them per warp:
  quad      count of the copy per cell row the warp computes
  rcas      count of the copy once per step
  phase1/2  count per loop iteration (region count over the shared stores it holds, one per iteration) times the warp's
            iterations
  control   count once per step
  clamp     count once per step whose box reaches outside the input
  setup     count once per CTA
This is an estimate of issued warp instructions: branches not taken inside a region are counted, loop overhead is not
separated.  The floor is (warp instructions) / (4 schedulers x SMs x clock), one instruction per clock per scheduler.

--time (needs a GPU) also times fused frames pipelined on two streams, as tools/fused_schedule.py does, and prints the
fraction of the floor reached, with the GPU's name, power limit and SM clock.
"""
import argparse
import collections
import json
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "fidelityfx-fsr_b200", "csrc")
SRC = os.path.join(CSRC, "fsr1_fused.cu")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVDISASM = os.path.join(os.path.dirname(NVCC), "nvdisasm")
KERNEL = "_ZN4fsr121fused_h_quad2x_kernelILi4ELi7EEEvNS_11FusedParamsE14CUtensorMap_st"

# the geometry of fsr1_fused.cu / fsr1_easu_quad.cuh at NW = 4
NW, NT = 4, 128
CY = 2 * NW
FBW, FSW, STRIP = 38, 36, 31


def source_lines():
    """Line numbers (1-based) of fsr1_fused.cu that delimit the regions, found by their text."""
    src = open(SRC).read().splitlines()

    def find(pat, start=0):
        for i in range(start, len(src)):
            if re.search(pat, src[i]):
                return i + 1
        raise RuntimeError("fused_budget: %r not found in %s" % (pat, SRC))

    step = find(r"^__device__ __forceinline__ void fused_step\(")
    quad0 = find(r"for \(int q = 0; q < 2; q\+\+\)", step)
    rcas0 = find(r"__syncthreads\(\);", quad0)
    body = find(r"^__device__ __forceinline__ void fused_body\(", rcas0)
    return {
        "quad": (quad0, rcas0 - 1),
        "rcas": (rcas0 + 1, body - 1),
        "phase1": (find(r"texel_luma\(tile\[i\]\)", body),) * 2,
        "phase2": (find(r"idx < kFSW \* \(n \+ 1\)", body), find(r"sm\.S\[idx\] = texel_terms", body)),
        "clamp": (find(r"clamp_fixup\(", body), find(r"clamp_fixup\(", body) + 2),
        "loop": (find(r"for \(int it = 0; has; it\+\+\)", body), find(r"halo_sync_end", body) - 1),
        "interior": find(r"fused_step<true,", body),
        "edge": find(r"fused_step<false,", body),
    }


def sass(cubin_dir):
    cubin = os.path.join(cubin_dir, "fused.cubin")
    subprocess.run([NVCC, "-cubin", "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-o", cubin, SRC],
                   check=True)
    return subprocess.run([NVDISASM, "-g", "-gi", "-c", cubin], check=True, capture_output=True, text=True).stdout


def static_counts(text, lines):
    """{(region, copy): instructions} and {region: shared stores} of KERNEL; copy is 'interior', 'edge' or '-'."""
    fused = os.path.basename(SRC)
    counts, stores = collections.Counter(), collections.Counter()
    cur, chain, fresh = None, [], True
    for ln in text.splitlines():
        m = re.match(r"\s*\.text\.(\S+):", ln)
        if m:
            cur = m.group(1)
            chain = []
            continue
        if cur != KERNEL:
            continue
        if ln.lstrip().startswith("//##"):  # a location block: it holds for every instruction up to the next block
            if fresh:
                chain, fresh = [], False
            chain += [(os.path.basename(f), int(n)) for f, n in re.findall(r'File "([^"]+)", line (\d+)', ln)]
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+([^;]+);", ln)
        if not m:
            continue
        ins = m.group(1).strip()
        fl = [n for f, n in chain if f == fused]
        region = "control"
        for r in ("quad", "rcas", "phase1", "phase2", "clamp", "loop"):
            a, b = lines[r]
            if any(a <= n <= b for n in fl):
                region = r
                break
        region = {"loop": "control", "control": "setup"}.get(region, region)
        copy = "interior" if lines["interior"] in fl else "edge" if lines["edge"] in fl else "-"
        counts[(region, copy)] += 1
        op = ins.split()[1] if ins.startswith("@") else ins.split()[0]
        if op.startswith("STS"):
            stores[region] += 1
        fresh = True
    if not counts:
        raise RuntimeError("fused_budget: kernel %s not found in the SASS" % KERNEL)
    return counts, stores


# ---- Python copies of fused_setup's grid and FusedIter --------------------------------------------------------------
def grid_of(ow, oh, y0, y1, per_sm, sms):
    n_strips = ((ow + 1) // 2 + STRIP - 1) // STRIP
    units = n_strips * ((y1 - y0 + 1) // 2)
    g = per_sm * sms
    g = min(g, (units + 7) // 8)
    return max(g, 1), n_strips


def steps_of(ow, oh, y0, y1, n_strips, cta, ctas):
    """The FusedStep list (tx, m0, n, ya, yb) of CTA `cta`, as FusedIter::next yields it."""
    if y1 <= y0:
        return []
    mfirst, mlast = (y0 - 2) >> 1, (y1 - 1) >> 1
    S, C = n_strips, mlast - mfirst + 1
    if ctas < S:
        runs = [(s, mfirst, mlast) for s in range(S * cta // ctas, S * (cta + 1) // ctas)]
    else:
        s = ((cta + 1) * S - 1) // ctas
        g0 = ctas * s // S
        g, i = ctas * (s + 1) // S - g0, cta - g0
        T = (C + g - 1 + CY - 1) // CY
        if T < g:
            T = (C - 1 + CY - 2) // (CY - 1)
        a, k = T * i // g, T * (i + 1) // g - T * i // g
        ma = mfirst + CY * a - min(i, a)
        runs = [] if k == 0 or 2 * ma + 2 >= y1 else [(s, ma, min(ma + CY * k - 1, mlast))]
    out = []
    for s, ma, mb in runs:
        m = ma
        while m <= mb:
            n = min(mb - m + 1, CY)
            out.append((s, m, n, max(2 * ma + 2, y0), min(2 * mb + 2, y1)))
            m += n
    return out


def interior(ow, oh, s):
    tx, m0, n, ya, yb = s
    k0 = STRIP * tx - 1
    return k0 >= 0 and 2 * (k0 + 31) + 2 < ow and m0 >= 0 and 2 * (m0 + CY) < oh and n == CY and 2 * m0 + 2 >= ya and 2 * (m0 + CY) <= yb


def box_clamped(s, iw, ih):
    """the step's TMA box reaches outside the input: fused_body rewrites its zero fill to clamp-to-edge"""
    gx, gy = (STRIP * s[0] - 2) & ~1, s[1] - 1
    return gx < 0 or gy < 0 or gx + FBW > iw or gy + CY + 3 > ih


def warp_iters(total, warp):
    """loop iterations of warp `warp` in `for (i = tid; i < total; i += NT)` (a warp issues while any lane is in)."""
    return len(range(warp * 32, total, NT))


def budget(counts, stores, ow, oh, y0, y1, per_sm, sms):
    ctas, n_strips = grid_of(ow, oh, y0, y1, per_sm, sms)
    per = lambda r, c: counts.get((r, c), 0)  # noqa: E731
    region = lambda r: sum(v for (rr, _), v in counts.items() if rr == r)  # noqa: E731
    iw, ih = ow // 2, oh // 2
    phase_it = {r: sum(v for (rr, _), v in counts.items() if rr == r) / max(stores[r], 1) for r in ("phase1", "phase2")}
    tot = collections.Counter()
    geo = collections.Counter()
    for c in range(ctas):
        st = steps_of(ow, oh, y0, y1, n_strips, c, ctas)
        geo["steps"] += len(st)
        geo["max_steps_per_cta"] = max(geo["max_steps_per_cta"], len(st))
        runs = set((s[0], s[3]) for s in st)
        geo["runs"] += len(runs)
        geo["ctas_over_two_strips"] += len(set(s[0] for s in st)) > 1
        tot["setup"] += NW * region("setup")
        for s in st:
            n = s[2]
            cp = "interior" if interior(ow, oh, s) else "edge"
            geo[cp + "_steps"] += 1
            geo["partial_steps"] += n < CY
            for w in range(NW):
                rows = sum(1 for q in range(2) if w + q * NW < n)
                tot["quad"] += rows * per("quad", cp)
                tot["rcas"] += per("rcas", cp)
                tot["phase1"] += warp_iters(FBW * (n + 3), w) * phase_it["phase1"]
                tot["phase2"] += warp_iters(FSW * (n + 1), w) * phase_it["phase2"]
                tot["control"] += region("control")
                tot["clamp"] += region("clamp") if box_clamped(s, iw, ih) else 0
    geo["ctas"] = ctas
    geo["strips"] = n_strips
    return tot, geo


def device_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.sm", "--format=csv,noheader,nounits"],
                                      text=True).strip().split(",")
        return name, float(out[0]), float(out[1])
    except Exception:  # noqa: BLE001
        return name, None, None


def time_fused(ow, oh, frames, rounds):
    """µs per frame of fused frames pipelined on two streams (median, min, max over rounds)."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import fused_schedule as fs
    import numpy as np
    w = fs.Workload(ow // 2, oh // 2, ow, oh)
    w.timed(w.fused, 20, True)
    kernel = fs.api.last_kernel()
    t = sorted(w.timed(w.fused, frames, True) * 1e3 for _ in range(rounds))
    return float(np.median(t)), t[0], t[-1], kernel


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", default="3840x2160", help="output size (the input is half of it)")
    ap.add_argument("--y0", type=int, default=0)
    ap.add_argument("--y1", type=int, default=-1, help="default: the output height")
    ap.add_argument("--per-sm", type=int, default=7, help="CTAs per SM of the launch (7; 6 with a halo hand-shake)")
    ap.add_argument("--sms", type=int, default=132, help="SMs (132 on an H100 SXM)")
    ap.add_argument("--sm-mhz", type=float, default=1980.0, help="SM clock for the floor")
    ap.add_argument("--time", action="store_true", help="also time the kernel on cuda:0 and print the fraction of the floor")
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    ow, oh = (int(v) for v in args.size.split("x"))
    y1 = oh if args.y1 < 0 else args.y1
    lines = source_lines()
    with tempfile.TemporaryDirectory() as d:
        counts, stores = static_counts(sass(d), lines)
    tot, geo = budget(counts, stores, ow, oh, args.y0, y1, args.per_sm, args.sms)
    pix = ow * (y1 - args.y0)
    allw = sum(tot.values())
    floor_us = allw / (4 * args.sms * args.sm_mhz * 1e6) * 1e6
    print("static SASS of fused_h_quad2x_kernel<4,7> by region (copy):")
    for (r, c), v in sorted(counts.items()):
        print("  %-8s %-9s %6d" % (r, c, v))
    print("geometry at %dx%d rows [%d, %d): %s" % (ow, oh, args.y0, y1, dict(geo)))
    print("warp instructions per output pixel:")
    for r in ("phase1", "phase2", "quad", "rcas", "control", "clamp", "setup"):
        print("  %-8s %6.3f   (%.1f M per frame)" % (r, tot[r] / pix, tot[r] / 1e6))
    print("  %-8s %6.3f   (%.1f M per frame)" % ("total", allw / pix, allw / 1e6))
    print("issue floor at %d SMs x 4 schedulers x %.0f MHz: %.1f us per frame" % (args.sms, args.sm_mhz, floor_us))
    res = {"size": [ow, oh], "rows": [args.y0, y1], "static": {"%s/%s" % k: v for k, v in counts.items()}, "geometry": dict(geo),
           "per_pixel": {r: tot[r] / pix for r in tot}, "per_pixel_total": allw / pix, "floor_us": floor_us, "sm_mhz": args.sm_mhz}
    if args.time:
        import torch
        if not torch.cuda.is_available():
            sys.exit("fused_budget.py --time needs a CUDA device")
        gpu, limit, mhz = device_info()
        med, lo, hi, kernel = time_fused(ow, oh, args.frames, args.rounds)
        _, _, mhz_after = device_info()
        floor_at = allw / (4 * args.sms * (mhz_after or args.sm_mhz) * 1e6) * 1e6
        print("%s, power limit %s W, SM clock %s MHz before / %s MHz after: %s %.1f us per frame pipelined (min %.1f max %.1f); "
              "floor at that clock %.1f us = %.2f of issue" % (gpu, limit, mhz, mhz_after, kernel, med, lo, hi, floor_at, floor_at / med))
        res.update({"gpu": gpu, "power_limit_w": limit, "sm_mhz_measured": [mhz, mhz_after], "us": [med, lo, hi], "kernel": kernel,
                    "floor_fraction": floor_at / med})
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
