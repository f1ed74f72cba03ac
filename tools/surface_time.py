"""Times upscaling from and into CUDA arrays: the surface call against today's interop route and against linear buffers, in one process
with the legs alternated.

    python tools/surface_time.py [--frames 200] [--reps 5] [--ring 8]

Legs, on the same pixels:
  linear   the call on linear buffers (what the copies of the interop route feed)
  copies   cudaMemcpy2DFromArrayAsync of the input into a linear buffer, the linear call, cudaMemcpy2DToArrayAsync of the output
           (the driver's cuMemcpy2DAsync on the same stream)
  surface  the call with FSR1_FLAG_IN_SURFACE | FSR1_FLAG_OUT_SURFACE on surface objects of the same arrays
  in_only, out_only   the call with one of the two flags (the other image linear): where the surface call's time goes
Workloads: 1080p -> 4K fsr1_upscale(FUSED) (the fused kernel), 1440p -> 4K fsr1_upscale(FUSED) (1.5x: EASU + RCAS), and the HDR round
trip fsr1_upscale_post(FUSED | SRTM_INPUT, SRTM_INVERSE | TEPD10) at 1080p -> 4K into an RGB10A2 array.  Each leg walks a ring of frame
sets larger than the 50 MB L2 and is timed with CUDA events over --frames frames after a warm-up; the arrays written by the copies and
surface legs (and the in_only leg's linear output) are checked bit-identical to the linear call's output before any timing.  Prints the
card, its power limit and SM clock (before and after), the kernels each leg ran, then one line per leg: median us per frame over --reps
alternations and the spread (max - min) / median.  CUDA arrays are made with the driver API through ctypes (libcuda.so.1, torch's
primary context).  Needs a GPU."""
import argparse
import ctypes
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from srtm_input_time import gpu_info, hdr, report, timed  # noqa: E402


class _Desc3D(ctypes.Structure):
    _fields_ = [("Width", ctypes.c_size_t), ("Height", ctypes.c_size_t), ("Depth", ctypes.c_size_t), ("Format", ctypes.c_int),
                ("NumChannels", ctypes.c_uint), ("Flags", ctypes.c_uint)]


class _ResDesc(ctypes.Structure):  # CUDA_RESOURCE_DESC with the array member of its union
    _fields_ = [("resType", ctypes.c_int), ("hArray", ctypes.c_void_p), ("reserved", ctypes.c_int * 30), ("flags", ctypes.c_uint)]


class _Copy2D(ctypes.Structure):  # CUDA_MEMCPY2D
    _fields_ = [("srcXInBytes", ctypes.c_size_t), ("srcY", ctypes.c_size_t), ("srcMemoryType", ctypes.c_int), ("srcHost", ctypes.c_void_p),
                ("srcDevice", ctypes.c_uint64), ("srcArray", ctypes.c_void_p), ("srcPitch", ctypes.c_size_t),
                ("dstXInBytes", ctypes.c_size_t), ("dstY", ctypes.c_size_t), ("dstMemoryType", ctypes.c_int), ("dstHost", ctypes.c_void_p),
                ("dstDevice", ctypes.c_uint64), ("dstArray", ctypes.c_void_p), ("dstPitch", ctypes.c_size_t),
                ("WidthInBytes", ctypes.c_size_t), ("Height", ctypes.c_size_t)]


def _ok(rc):
    assert rc == 0, "CUDA driver error %d" % rc


class CudaArray:
    """a 2D CUDA array with surface load/store, a surface object on it, and prepared copies to / from a linear tensor"""
    KINDS = {"rgba16f": (0x10, 4, 8), "u32": (0x03, 1, 4)}   # CUarray_format, channels, bytes per element

    def __init__(self, cu, w, h, kind):
        fmt, ch, self.elem = self.KINDS[kind]
        self.cu, self.w, self.h = cu, w, h
        self.arr, s = ctypes.c_void_p(), ctypes.c_uint64()
        _ok(cu.cuArray3DCreate_v2(ctypes.byref(self.arr), ctypes.byref(_Desc3D(w, h, 0, fmt, ch, 0x02))))
        _ok(cu.cuSurfObjectCreate(ctypes.byref(s), ctypes.byref(_ResDesc(0, self.arr))))
        self.handle = s.value

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
        self.cu.cuSurfObjectDestroy(ctypes.c_uint64(self.handle))
        self.cu.cuArrayDestroy(self.arr)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ring", type=int, default=8)
    a = ap.parse_args()
    import torch
    from fsr1_b200 import api
    assert torch.cuda.is_available(), "surface_time.py needs a GPU"
    torch.zeros(1, device="cuda")
    cu = ctypes.CDLL("libcuda.so.1")
    print("gpu: %s" % gpu_info())
    rcon = api.rcas_con(0.25)
    IN, OUT = api.FLAG_IN_SURFACE, api.FLAG_OUT_SURFACE
    for iw, ih, ow, oh, post in ((1920, 1080, 3840, 2160, False), (2560, 1440, 3840, 2160, False), (1920, 1080, 3840, 2160, True)):
        econ = api.easu_con(iw, ih, iw, ih, ow, oh)
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        ins = [torch.from_numpy(hdr(iw, ih, 100 + i)).cuda() for i in range(a.ring)]
        stage_in = [torch.empty_like(x) for x in ins]
        tmps = [torch.empty((oh, ow, 4), dtype=torch.float16, device="cuda") for _ in range(a.ring)]

        def out_tensor():
            return torch.empty((oh, ow), dtype=torch.int32, device="cuda") if post else torch.empty((oh, ow, 4), dtype=torch.float16, device="cuda")
        lin_out, stage_out, in_only_out = ([out_tensor() for _ in range(a.ring)] for _ in range(3))
        kind, ofmt = ("u32", api.FORMAT_RGB10A2_UNORM) if post else ("rgba16f", api.FORMAT_RGBA16F)
        in_arr = [CudaArray(cu, iw, ih, "rgba16f") for _ in range(a.ring)]
        out_arr = {k: [CudaArray(cu, ow, oh, kind) for _ in range(a.ring)] for k in ("copies", "surface")}
        torch.cuda.synchronize()
        for i in range(a.ring):
            _ok(cu.cuMemcpy2D_v2(ctypes.byref(in_arr[i].copy_desc(ins[i], True))))
        copy_in = [in_arr[i].copy_desc(stage_in[i], False) for i in range(a.ring)]
        copy_out = [out_arr["copies"][i].copy_desc(stage_out[i], True) for i in range(a.ring)]
        s_in = [api.surface_image(x.handle, iw, ih, api.FORMAT_RGBA16F) for x in in_arr]
        s_out = [api.surface_image(x.handle, ow, oh, ofmt) for x in out_arr["surface"]]
        flags = api.FLAG_FUSED | (api.FLAG_SRTM_INPUT if post else 0)

        def call(i, inp, out, f):
            if post:
                api.upscale_post(inp, tmps[i], out, econ, rcon, srtm_inverse=True, tepd_bits=10, frame=i, flags=f)
            else:
                api.upscale(inp, tmps[i], out, econ, rcon, flags=f)

        def copies(i):
            _ok(cu.cuMemcpy2DAsync_v2(ctypes.byref(copy_in[i]), stream))
            call(i, stage_in[i], stage_out[i], flags)
            _ok(cu.cuMemcpy2DAsync_v2(ctypes.byref(copy_out[i]), stream))

        legs = {"linear": lambda i: call(i, ins[i], lin_out[i], flags), "copies": copies,
                "surface": lambda i: call(i, s_in[i], s_out[i], flags | IN | OUT),
                "in_only": lambda i: call(i, s_in[i], in_only_out[i], flags | IN),
                "out_only": lambda i: call(i, ins[i], s_out[i], flags | OUT)}
        names = {}
        for i in range(a.ring):
            for k, fn in legs.items():
                fn(i)
                names[k] = api.last_kernel()
        torch.cuda.synchronize()
        view = torch.int32 if post else torch.int16
        for i in range(a.ring):
            assert torch.equal(in_only_out[i].view(view), lin_out[i].view(view)), ("in_only", iw, ih, i)
        for k in ("copies", "surface"):
            for i in range(a.ring):
                got = torch.empty_like(lin_out[i])
                _ok(cu.cuMemcpy2D_v2(ctypes.byref(out_arr[k][i].copy_desc(got, False))))
                assert torch.equal(got.view(view), lin_out[i].view(view)), (k, iw, ih, i)
        print("  kernels: %s" % names)
        label = "%dx%d->%dx%d %s" % (iw, ih, ow, oh, "hdr round trip rgb10a2" if post else "upscale")
        report(label, timed(legs, a))
        torch.cuda.synchronize()
        for x in in_arr + out_arr["copies"] + out_arr["surface"]:
            x.close()
        del ins, stage_in, tmps, lin_out, stage_out, in_only_out
        torch.cuda.empty_cache()
    print("gpu: %s" % gpu_info())


if __name__ == "__main__":
    main()
