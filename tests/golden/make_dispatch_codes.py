"""Generates tests/golden/dispatch_codes.json: the return code of every entry point of the dispatch layer for a deterministic list
of calls, on a machine WITHOUT a CUDA device.

There every call either returns a refusal (FSR1_ERR_INVALID_ARGUMENT, _UNSUPPORTED, _WINDOW) before any CUDA call, or reaches a
launch and returns FSR1_ERR_CUDA; fsr1_shard_create_post returns FSR1_ERR_NO_DEVICE at that point.  The tiled launchers decline
every frame there (no tensor-map encoder can be resolved without a driver), so FSR1_FLAG_SRTM_INPUT calls are refused with
FSR1_ERR_UNSUPPORTED.  The mapping is deterministic and depends on the dispatch code only: which check runs first, and which
rules exist.  tests/test_dispatch_codes.py rebuilds the same cases and compares.

    python tests/golden/make_dispatch_codes.py [--lib PATH] [--out PATH]

--lib loads another build of the library (for instance one of the parent commit) instead of the one in the tree.
"""
import argparse
import ctypes
import itertools
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
GOLDEN = os.path.join(HERE, "dispatch_codes.json")
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from fsr1_b200 import _lib  # noqa: E402

I = _lib
F16, F32, U8, U10, R11, BAD = 1, 2, 3, 4, 5, 9
BPP = {F16: 8, F32: 16, U8: 4, U10: 4, R11: 4, BAD: 8}

# the axes of a call; the first value of each is the one the base frames use unless the base says otherwise
FLAGS = [0, I.FLAG_RCAS_CLAMP, I.FLAG_EXACT, I.FLAG_FORCE_DIRECT, I.FLAG_NO_RCAS, I.FLAG_H_REFERENCE, I.FLAG_PRECISE,
         I.FLAG_RCAS_DENOISE, I.FLAG_RCAS_PASSTHROUGH_ALPHA, I.FLAG_OUTPUT_SQUARE, I.FLAG_FUSED, I.FLAG_RCAS_HX2,
         I.FLAG_SRTM_INPUT, 1 << 20,
         I.FLAG_FUSED | I.FLAG_SRTM_INPUT, I.FLAG_SRTM_INPUT | I.FLAG_PRECISE, I.FLAG_FUSED | I.FLAG_RCAS_CLAMP,
         I.FLAG_OUTPUT_SQUARE | I.FLAG_FUSED, I.FLAG_FUSED | I.FLAG_PRECISE, I.FLAG_FUSED | I.FLAG_NO_RCAS,
         I.FLAG_SRTM_INPUT | I.FLAG_NO_RCAS, I.FLAG_SRTM_INPUT | I.FLAG_FORCE_DIRECT, I.FLAG_FUSED | I.FLAG_EXACT,
         I.FLAG_FUSED | I.FLAG_H_REFERENCE, I.FLAG_FUSED | I.FLAG_RCAS_HX2, I.FLAG_FUSED | I.FLAG_RCAS_DENOISE,
         I.FLAG_FUSED | I.FLAG_RCAS_PASSTHROUGH_ALPHA, I.FLAG_SRTM_INPUT | I.FLAG_OUTPUT_SQUARE,
         I.FLAG_PRECISE | I.FLAG_OUTPUT_SQUARE, I.FLAG_FUSED | I.FLAG_SRTM_INPUT | I.FLAG_NO_RCAS,
         I.FLAG_FUSED | I.FLAG_SRTM_INPUT | I.FLAG_OUTPUT_SQUARE, I.FLAG_EXACT | I.FLAG_SRTM_INPUT,
         I.FLAG_H_REFERENCE | I.FLAG_SRTM_INPUT, I.FLAG_RCAS_HX2 | I.FLAG_SRTM_INPUT, I.FLAG_NO_RCAS | I.FLAG_OUTPUT_SQUARE,
         I.FLAG_FUSED | I.SHARD_DYNAMIC, I.SHARD_ONE_STREAM | I.SHARD_TRACE]
POST_OPS = [0, I.POST_SRTM_INVERSE, I.POST_LFGA, I.POST_TEPD8, I.POST_TEPD10, I.POST_TEPD8 | I.POST_TEPD10,
            I.POST_LFGA | I.POST_TEPD8, I.POST_SRTM_INVERSE | I.POST_LFGA | I.POST_TEPD10, I.POST_SRTM_INVERSE | I.POST_TEPD8,
            1 << 4]
FORMATS = [F16, F32, U8, U10, R11, BAD]
ALIGNS = ["a256", "a8", "a4", "data8", "pitch8", "small_pitch"]
WINDOWS = ["whole", "top", "bottom", "mid", "past", "no_rows"]
AXES = {
    "con": ["match", "2x", "up", "1to1", "down", "aniso"],
    "in_fmt": FORMATS, "tmp_fmt": FORMATS, "out_fmt": FORMATS,
    "flags": FLAGS,
    "in_align": ALIGNS, "tmp_align": ALIGNS, "out_align": ALIGNS,
    "in_win": WINDOWS, "tmp_win": WINDOWS, "out_win": WINDOWS,
    "in_size": ["ok", "zero", "huge"],
    "rows": ["whole", "explicit", "slab", "bottom", "empty", "past", "inverted"],
    "null": ["none", "in", "tmp", "out", "econ", "rcon", "post", "grain", "dither"],
    "alias": ["none", "tmp_out", "in_tmp"],
    "post_ops": POST_OPS,
    "grain": [F16, F32, U8, R11, "partial"],
    "dither": [U8, F16, U10, R11, "partial"],
    "bits": [8, 10, 9],
    "shard": [(1, 0, 1), (4, 1, 2), (4, 4, 1), (0, 0, 1), (1, 0, 0), (1, 0, 200), (64, 0, 1)],
}
SCALES = {"2x": (16, 8, 32, 16), "1.5x": (16, 8, 24, 12), "down": (32, 16, 16, 8)}
BASE_FORMATS = [(F16, F16), (R11, F16), (F32, F32), (U8, U8)]
N_SAMPLED = 1500  # from the whole product: mostly refusals
N_NEAR = 3000     # near the base frames: more accepted calls, and refusals that meet several at once
REGION = 1 << 16  # bytes per image region: in, tmp, out, grain, dither


def bases():
    for scale, (fi, fo) in itertools.product(SCALES, BASE_FORMATS):
        c = {k: v[0] for k, v in AXES.items()}
        c.update(scale=scale, in_fmt=fi, tmp_fmt=fo, out_fmt=fo)
        yield c


def cases():
    """The case list: every single-axis variation of each base frame, then a seeded sample of the product of the axes, then
    seeded variations of the base frames in several axes at once (each axis changes with probability 1/4)."""
    out = []
    for b in bases():
        out.append(dict(b))
        for k, vals in AXES.items():
            for v in vals:
                if v != b[k]:
                    c = dict(b)
                    c[k] = v
                    out.append(c)
    rng = random.Random(20261017)
    for _ in range(N_SAMPLED):
        c = {k: rng.choice(v) for k, v in AXES.items()}
        c["scale"] = rng.choice(sorted(SCALES))
        out.append(c)
    base_list = list(bases())
    for _ in range(N_NEAR):
        c = dict(rng.choice(base_list))
        for k, vals in AXES.items():
            if rng.random() < 0.25:
                c[k] = rng.choice(vals)
        out.append(c)
    return out


class Arena:
    def __init__(self):
        self.buf = (ctypes.c_uint8 * (5 * REGION + 256))()
        a = ctypes.addressof(self.buf)
        self.base = a + (-a) % 256

    def image(self, region, w, h, fmt, align, win):
        bpp = BPP[fmt]
        row = w * bpp
        data, pitch = 0, (row + 255) // 256 * 256
        if align in ("a8", "a4"):
            data, pitch = (8, (row + 15) // 16 * 16 + 8) if align == "a8" else (4, (row + 15) // 16 * 16 + 4)
        elif align == "data8":
            data = 8
        elif align == "pitch8":
            pitch = (row + 15) // 16 * 16 + 8
        elif align == "small_pitch":
            pitch = max(row - bpp, 0)
        row0, rows = {"whole": (0, h), "top": (0, h // 2), "bottom": (h // 2, h - h // 2), "mid": (h // 4, h // 2),
                      "past": (h // 2, h), "no_rows": (0, 0)}[win]
        return I.Image(self.base + region * REGION + data, pitch, w, h, row0, rows, fmt, 0)


def con_words(L, kind, in_w, in_h, out_w, out_h):
    ow, oh = {"match": (out_w, out_h), "2x": (2 * in_w, 2 * in_h), "up": (3 * in_w // 2, 3 * in_h // 2), "1to1": (in_w, in_h),
              "down": (in_w // 2, in_h // 2), "aniso": (2 * in_w, 3 * in_h // 2)}[kind]
    econ = (ctypes.c_uint32 * 16)()
    f = ctypes.c_float
    L.fsr1_easu_con(econ, f(in_w), f(in_h), f(in_w), f(in_h), f(ow), f(oh))
    return econ


ENTRY_POINTS = ["fsr1_easu", "fsr1_rcas", "fsr1_upscale", "fsr1_upscale_post", "fsr1_srtm", "fsr1_lfga", "fsr1_tepd",
                "fsr1_srtm_h", "fsr1_lfga_h", "fsr1_tepd_h", "fsr1_shard_create_post"]


def run(L, arena, c):
    """The return code of every entry point for case `c`, in ENTRY_POINTS order."""
    in_w, in_h, out_w, out_h = SCALES[c["scale"]]
    if c["in_size"] == "zero":
        in_w = 0
    elif c["in_size"] == "huge":
        in_w = 40000
    in_region, tmp_region = 0, 1
    if c["alias"] == "tmp_out":
        tmp_region = 2
    elif c["alias"] == "in_tmp":
        in_region = 1
    im_in = arena.image(in_region, in_w, in_h, c["in_fmt"], c["in_align"], c["in_win"])
    im_tmp = arena.image(tmp_region, out_w, out_h, c["tmp_fmt"], c["tmp_align"], c["tmp_win"])
    im_out = arena.image(2, out_w, out_h, c["out_fmt"], c["out_align"], c["out_win"])
    tiles = {}
    for name, region in (("grain", 3), ("dither", 4)):
        v = c[name]
        tiles[name] = arena.image(region, 5, 4, F16 if v == "partial" else v, "a256", "mid" if v == "partial" else "whole")
    econ = con_words(L, c["con"], in_w or 1, in_h, out_w, out_h)
    rcon = (ctypes.c_uint32 * 4)()
    L.fsr1_rcas_con(rcon, ctypes.c_float(0.25))
    y0, y1 = {"whole": (0, 0), "explicit": (0, out_h), "slab": (out_h // 4, out_h // 2), "bottom": (out_h // 2, out_h),
              "empty": (3, 3), "past": (0, out_h + 1), "inverted": (5, 2)}[c["rows"]]
    null = c["null"]
    ref = ctypes.pointer
    p_in = None if null == "in" else ref(im_in)
    p_tmp = None if null == "tmp" else ref(im_tmp)
    p_out = None if null == "out" else ref(im_out)
    p_econ = None if null == "econ" else econ
    p_rcon = None if null == "rcon" else rcon
    p_grain = None if null == "grain" else ref(tiles["grain"])
    p_dither = None if null == "dither" else ref(tiles["dither"])
    post = I.Post(c["post_ops"], 0.5, p_grain, p_dither, 7, 0)
    p_post = None if null == "post" else ref(post)
    flags, bits, inverse = c["flags"], c["bits"], 1 if c["bits"] == 10 else 0
    world, rank, slots = c["shard"]
    h = ctypes.c_void_p()
    codes = [
        L.fsr1_easu(p_in, p_tmp, p_econ, y0, y1, flags, None),
        L.fsr1_rcas(p_tmp, p_out, p_rcon, y0, y1, flags, None),
        L.fsr1_upscale(p_in, p_tmp, p_out, p_econ, p_rcon, y0, y1, flags, None),
        L.fsr1_upscale_post(p_in, p_tmp, p_out, p_econ, p_rcon, p_post, y0, y1, flags, None),
        L.fsr1_srtm(p_tmp, p_out, inverse, y0, y1, None),
        L.fsr1_lfga(p_tmp, p_grain, p_out, ctypes.c_float(0.5), y0, y1, None),
        L.fsr1_tepd(p_tmp, p_dither, p_out, bits, 7, y0, y1, None),
        L.fsr1_srtm_h(p_tmp, p_out, inverse, y0, y1, None),
        L.fsr1_lfga_h(p_tmp, p_grain, p_out, ctypes.c_float(0.5), y0, y1, None),
        L.fsr1_tepd_h(p_tmp, p_dither, p_out, bits, 7, y0, y1, None),
        L.fsr1_shard_create_post(ref(h), in_w, in_h, out_w, out_h, c["in_fmt"], c["out_fmt"], p_post, world, rank, slots,
                                 ctypes.c_float(0.25), flags),
    ]
    assert not h.value, "a shard was created: this must run without a CUDA device"
    return codes


def codes_of(L):
    """{entry point: one character per case, the negated return code}"""
    arena = Arena()
    per_entry = [[] for _ in ENTRY_POINTS]
    for c in cases():
        for i, rc in enumerate(run(L, arena, c)):
            assert -9 <= rc <= 0, rc
            per_entry[i].append(str(-rc))
    return {name: "".join(s) for name, s in zip(ENTRY_POINTS, per_entry)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="the library to load instead of the tree's")
    ap.add_argument("--out", default=GOLDEN)
    args = ap.parse_args()
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    L = _lib.lib()
    n0 = L.fsr1_launch_count()
    codes = codes_of(L)
    assert L.fsr1_launch_count() == n0
    with open(args.out, "w") as f:
        json.dump({"cases": len(cases()), "codes": codes}, f, indent=1)
        f.write("\n")
    for name, s in codes.items():
        print(name, {ch: s.count(ch) for ch in sorted(set(s))})


if __name__ == "__main__":
    main()
