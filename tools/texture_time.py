"""Times reading the render target through a texture object (FSR1_FLAG_IN_TEXTURE) against the other ways to feed EASU from a CUDA array,
in one process with the legs alternated.

    python tools/texture_time.py [--frames 200] [--reps 5] [--ring 8]

Legs, on the same pixels, all writing the same output:
  linear   the call on a linear input buffer
  copies   cuMemcpy2DAsync of the input array into a linear buffer, then the linear call (the route of a render target that only has
           sampled usage, before FSR1_FLAG_IN_TEXTURE)
  surface  the call with FSR1_FLAG_IN_SURFACE on a surface object (an array mapped with surface load/store; RGBA16F only)
  texture  the call with FSR1_FLAG_IN_TEXTURE on a texture object of an array mapped WITHOUT surface load/store
Workloads, each on RGBA16F input and on R11G11B10F input (no surface leg): 1080p -> 4K fsr1_upscale(FUSED) (the fused kernel), 1440p -> 4K
fsr1_upscale (1.5x: EASU + RCAS), and the HDR round trip fsr1_upscale_post(FUSED | SRTM_INPUT, SRTM_INVERSE | TEPD10) at 1080p -> 4K into
an RGB10A2 array (FSR1_FLAG_OUT_SURFACE in every leg but linear; on R11G11B10F input into a linear RGB10A2 buffer in every leg, because
no kernel reads linear R11G11B10F input and stores through a surface).  Each leg walks a ring of frame sets larger than the 50 MB L2 and is timed
with CUDA events over --frames frames after a warm-up; every leg's output is checked bit-identical to the linear call's before any
timing.  Prints the card, its power limit and SM clock (before and after), the kernels each leg ran, then one line per leg: median us
per frame over --reps alternations and the spread (max - min) / median.  CUDA arrays are made with the driver API through ctypes
(libcuda.so.1, torch's primary context).  Needs a GPU."""
import argparse
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from srtm_input_time import gpu_info, hdr, report, timed  # noqa: E402
from surface_time import _Copy2D, _Desc3D, _ResDesc, _ok  # noqa: E402


class _TexDesc(ctypes.Structure):  # CUDA_TEXTURE_DESC
    _fields_ = [("addressMode", ctypes.c_int * 3), ("filterMode", ctypes.c_int), ("flags", ctypes.c_uint), ("maxAnisotropy", ctypes.c_uint),
                ("mipmapFilterMode", ctypes.c_int), ("mipmapLevelBias", ctypes.c_float), ("minMipmapLevelClamp", ctypes.c_float),
                ("maxMipmapLevelClamp", ctypes.c_float), ("borderColor", ctypes.c_float * 4), ("reserved", ctypes.c_int * 12)]


class Array:
    """a 2D CUDA array of unsigned-integer texels (16,16,16,16 or 32), with surface load/store and a surface object when `surface`, else a
    texture object (point filtering, element reads, unnormalized coordinates); prepared copies to / from a linear tensor"""

    def __init__(self, cu, w, h, elem, surface):
        self.cu, self.w, self.h, self.elem, self.surface = cu, w, h, elem, surface
        fmt, ch = (0x02, 4) if elem == 8 else (0x03, 1)
        self.arr, obj = ctypes.c_void_p(), ctypes.c_uint64()
        _ok(cu.cuArray3DCreate_v2(ctypes.byref(self.arr), ctypes.byref(_Desc3D(w, h, 0, fmt, ch, 0x02 if surface else 0))))
        if surface:
            _ok(cu.cuSurfObjectCreate(ctypes.byref(obj), ctypes.byref(_ResDesc(0, self.arr))))
        else:
            d = _TexDesc()
            d.addressMode[0] = d.addressMode[1] = d.addressMode[2] = 1   # clamp
            d.filterMode, d.flags = 0, 0x01                              # point, CU_TRSF_READ_AS_INTEGER
            _ok(cu.cuTexObjectCreate(ctypes.byref(obj), ctypes.byref(_ResDesc(0, self.arr)), ctypes.byref(d), None))
        self.handle = obj.value

    def copy_desc(self, t, to_array):
        c = _Copy2D()
        pitch = t.stride(0) * t.element_size()
        if to_array:
            c.srcMemoryType, c.srcDevice, c.srcPitch, c.dstMemoryType, c.dstArray = 2, t.data_ptr(), pitch, 3, self.arr
        else:
            c.srcMemoryType, c.srcArray, c.dstMemoryType, c.dstDevice, c.dstPitch = 3, self.arr, 2, t.data_ptr(), pitch
        c.WidthInBytes, c.Height = self.w * self.elem, self.h
        return c

    def close(self):
        if self.surface:
            self.cu.cuSurfObjectDestroy(ctypes.c_uint64(self.handle))
        else:
            self.cu.cuTexObjectDestroy(ctypes.c_uint64(self.handle))
        self.cu.cuArrayDestroy(self.arr)


def r11_codes(x16):
    """R11G11B10F codes of an RGBA16F numpy image (each half truncated to the format's mantissa), int32 [h, w]"""
    import numpy as np
    x = x16.view(np.uint16).astype(np.uint32) & 0x7FFF
    return ((x[..., 0] >> 4) | ((x[..., 1] >> 4) << 11) | ((x[..., 2] >> 5) << 22)).astype(np.uint32).view(np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ring", type=int, default=8)
    a = ap.parse_args()
    import torch
    from fsr1_b200 import api
    assert torch.cuda.is_available(), "texture_time.py needs a GPU"
    torch.zeros(1, device="cuda")
    cu = ctypes.CDLL("libcuda.so.1")
    print("gpu: %s" % gpu_info())
    rcon = api.rcas_con(0.25)
    for r11 in (False, True):
        fmt, elem = (api.FORMAT_R11G11B10_FLOAT, 4) if r11 else (api.FORMAT_RGBA16F, 8)
        for iw, ih, ow, oh, post in ((1920, 1080, 3840, 2160, False), (2560, 1440, 3840, 2160, False), (1920, 1080, 3840, 2160, True)):
            econ = api.easu_con(iw, ih, iw, ih, ow, oh)
            stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            ins = [torch.from_numpy(r11_codes(hdr(iw, ih, 100 + i)) if r11 else hdr(iw, ih, 100 + i)).cuda() for i in range(a.ring)]
            stage_in = [torch.empty_like(x) for x in ins]
            tmps = [torch.empty((oh, ow, 4), dtype=torch.float16, device="cuda") for _ in range(a.ring)]
            lin_in = [api.image(x, format=api.FORMAT_R11G11B10_FLOAT if r11 else None) for x in ins]
            stage_img = [api.image(x, format=api.FORMAT_R11G11B10_FLOAT if r11 else None) for x in stage_in]
            in_arr = {k: [Array(cu, iw, ih, elem, k == "surface") for _ in range(a.ring)] for k in (("texture",) if r11 else ("surface", "texture"))}
            torch.cuda.synchronize()
            for arrs in in_arr.values():
                for i in range(a.ring):
                    _ok(cu.cuMemcpy2D_v2(ctypes.byref(arrs[i].copy_desc(ins[i], True))))
            copy_in = [in_arr["texture"][i].copy_desc(stage_in[i], False) for i in range(a.ring)]
            images = {"texture": [api.texture_image(x.handle, iw, ih, fmt) for x in in_arr["texture"]]}
            if not r11:
                images["surface"] = [api.surface_image(x.handle, iw, ih, fmt) for x in in_arr["surface"]]
            flags = api.FLAG_FUSED | (api.FLAG_SRTM_INPUT if post else 0)
            arr_out = post and not r11
            if arr_out:   # the display image: an RGB10A2 array per leg (the linear leg: a linear buffer)
                outs = {k: [Array(cu, ow, oh, 4, True) for _ in range(a.ring)] for k in ("copies", "surface", "texture")}
                out_img = {k: [api.surface_image(x.handle, ow, oh, api.FORMAT_RGB10A2_UNORM) for x in v] for k, v in outs.items()}
                lin_out = [torch.empty((oh, ow), dtype=torch.int32, device="cuda") for _ in range(a.ring)]
                oflag = api.FLAG_OUT_SURFACE
            else:
                def out_tensor():
                    return torch.empty((oh, ow), dtype=torch.int32, device="cuda") if post else torch.empty((oh, ow, 4), dtype=torch.float16,
                                                                                                           device="cuda")
                out_img = {k: [out_tensor() for _ in range(a.ring)] for k in ("copies", "surface", "texture")}
                lin_out, oflag = [out_tensor() for _ in range(a.ring)], 0

            def call(i, inp, out, f):
                if post:
                    api.upscale_post(inp, tmps[i], out, econ, rcon, srtm_inverse=True, tepd_bits=10, frame=i, flags=f)
                else:
                    api.upscale(inp, tmps[i], out, econ, rcon, flags=f)

            def copies(i):
                _ok(cu.cuMemcpy2DAsync_v2(ctypes.byref(copy_in[i]), stream))
                call(i, stage_img[i], out_img["copies"][i], flags | oflag)

            legs = {"linear": lambda i: call(i, lin_in[i], lin_out[i], flags), "copies": copies}
            if not r11:
                legs["surface"] = lambda i: call(i, images["surface"][i], out_img["surface"][i], flags | oflag | api.FLAG_IN_SURFACE)
            legs["texture"] = lambda i: call(i, images["texture"][i], out_img["texture"][i], flags | oflag | api.FLAG_IN_TEXTURE)
            names = {}
            for i in range(a.ring):
                for k, fn in legs.items():
                    fn(i)
                    names[k] = api.last_kernel()
            torch.cuda.synchronize()
            view = torch.int32 if post else torch.int16
            for k in legs:
                if k == "linear":
                    continue
                for i in range(a.ring):
                    if arr_out:
                        got = torch.empty_like(lin_out[i])
                        _ok(cu.cuMemcpy2D_v2(ctypes.byref(outs[k][i].copy_desc(got, False))))
                    else:
                        got = out_img[k][i]
                    assert torch.equal(got.view(view), lin_out[i].view(view)), (k, iw, ih, i)
            print("  kernels: %s" % names)
            label = "%s %dx%d->%dx%d %s" % ("r11" if r11 else "rgba16f", iw, ih, ow, oh, "hdr rt rgb10a2" if post else "upscale")
            report(label, timed(legs, a))
            torch.cuda.synchronize()
            for x in sum(in_arr.values(), []) + (sum(outs.values(), []) if arr_out else []):
                x.close()
            del ins, stage_in, tmps, lin_out, out_img
            torch.cuda.empty_cache()
    print("gpu: %s" % gpu_info())


if __name__ == "__main__":
    main()
