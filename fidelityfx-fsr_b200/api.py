"""Thin Python layer over the C ABI: torch tensors are used ONLY as device memory + stream handles.

Images are torch CUDA tensors of shape [rows, width, 4], dtype float16 (RGBA16F) or float32 (RGBA32F),
contiguous in the last two dimensions (the row stride may be padded).
"""
import ctypes

import torch

from . import _lib
from ._lib import FORMAT_R11G11B10_FLOAT, FORMAT_RGB10A2_UNORM, FORMAT_RGBA8_UNORM  # noqa: F401
from ._lib import FLAG_FUSED, FLAG_OUTPUT_SQUARE, FLAG_RCAS_HX2, FLAG_SRTM_INPUT  # noqa: F401
from ._lib import FLAG_IN_SURFACE, FLAG_OUT_SURFACE, FLAG_IN_TEXTURE  # noqa: F401
from ._lib import POST_LFGA, POST_SRTM_INVERSE, POST_TEPD10, POST_TEPD8  # noqa: F401
from ._lib import (FLAG_EXACT, FLAG_FORCE_DIRECT, FLAG_H_REFERENCE, FLAG_NO_RCAS, FLAG_PRECISE, FLAG_RCAS_DENOISE, FLAG_RCAS_PASSTHROUGH_ALPHA, FLAG_RCAS_CLAMP, FORMAT_RGBA16F,  # noqa: F401
                   FORMAT_RGBA32F, Fsr1Error, Image)


def _u32(n):
    return (ctypes.c_uint32 * n)()


def easu_con(in_viewport_w, in_viewport_h, in_size_w, in_size_h, out_w, out_h):
    """FsrEasuCon (reference ffx-fsr/ffx_fsr1.h:156-202): returns the 16 constant words con0..con3."""
    con = _u32(16)
    f = ctypes.c_float
    _lib.lib().fsr1_easu_con(con, f(in_viewport_w), f(in_viewport_h), f(in_size_w), f(in_size_h), f(out_w), f(out_h))
    return list(con)


def easu_con_offset(in_viewport_w, in_viewport_h, in_size_w, in_size_h, out_w, out_h, off_x, off_y):
    """FsrEasuConOffset (reference ffx-fsr/ffx_fsr1.h:205-225)."""
    con = _u32(16)
    f = ctypes.c_float
    _lib.lib().fsr1_easu_con_offset(con, f(in_viewport_w), f(in_viewport_h), f(in_size_w), f(in_size_h), f(out_w),
                                    f(out_h), f(off_x), f(off_y))
    return list(con)


def rcas_con(sharpness_stops):
    """FsrRcasCon (reference ffx-fsr/ffx_fsr1.h:662-672): returns the 4 constant words."""
    con = _u32(4)
    _lib.lib().fsr1_rcas_con(con, ctypes.c_float(sharpness_stops))
    return list(con)


def easu_input_rows(con, in_height, y0, y1):
    a, b = ctypes.c_uint32(), ctypes.c_uint32()
    _lib.check(_lib.lib().fsr1_easu_input_rows((ctypes.c_uint32 * 16)(*con), in_height, y0, y1, ctypes.byref(a),
                                               ctypes.byref(b)))
    return a.value, b.value


def image(t, height=None, row0=0, format=None):
    """Describe tensor `t` ([rows, W, 4]) as logical rows [row0, row0+rows) of an image `height` rows tall.
    An int32 [rows, W] tensor is RGB10A2_UNORM, or R11G11B10_FLOAT (an input format only) with format=FORMAT_R11G11B10_FLOAT."""
    if not t.is_cuda:
        raise Fsr1Error("fsr1 kernels run on CUDA tensors only (no CPU path)")
    if format not in (None, FORMAT_R11G11B10_FLOAT):
        raise Fsr1Error("format: None (from the tensor) or FORMAT_R11G11B10_FLOAT")
    if format == FORMAT_R11G11B10_FLOAT and not (t.dim() == 2 and t.dtype == torch.int32 and t.stride(1) == 1):
        raise Fsr1Error("R11G11B10_FLOAT images are [rows, width] int32 tensors (one 32-bit code per pixel)")
    if t.dim() == 2 and t.dtype == torch.int32 and t.stride(1) == 1:      # one 32-bit code per pixel
        fmt = FORMAT_R11G11B10_FLOAT if format == FORMAT_R11G11B10_FLOAT else FORMAT_RGB10A2_UNORM
    else:
        if t.dim() != 3 or t.shape[2] != 4 or t.stride(2) != 1 or t.stride(1) != 4:
            raise Fsr1Error("image tensors must be [rows, width, 4] with contiguous pixels (or [rows, width] int32 for RGB10A2)")
        fmt = {torch.float16: FORMAT_RGBA16F, torch.float32: FORMAT_RGBA32F, torch.uint8: FORMAT_RGBA8_UNORM}.get(t.dtype)
        if fmt is None:
            raise Fsr1Error("unsupported dtype %s" % t.dtype)
    rows, w = int(t.shape[0]), int(t.shape[1])
    return Image(t.data_ptr(), t.stride(0) * t.element_size(), w, int(height if height is not None else rows), row0,
                 rows, fmt, 0)


def surface_image(handle, width, height, format):
    """A surface image (FLAG_IN_SURFACE / FLAG_OUT_SURFACE): the CUDA surface object `handle` (an int) on a 2D CUDA array, of which
    the top-left width x height is the image.  Pitch 0, the whole image (never a window)."""
    if not isinstance(handle, int) or handle <= 0:
        raise Fsr1Error("a surface image is a nonzero cudaSurfaceObject_t handle (int)")
    return Image(handle, 0, int(width), int(height), 0, int(height), int(format), 0)


def texture_image(handle, width, height, format):
    """A texture image (FLAG_IN_TEXTURE): the CUDA texture object `handle` (an int) on a 2D CUDA array with unsigned-integer channels
    (16,16,16,16 for FORMAT_RGBA16F, 32 for FORMAT_R11G11B10_FLOAT), point filtering, unnormalized coordinates, element read mode; the
    top-left width x height of the array is the image.  Pitch 0, the whole image (never a window)."""
    if not isinstance(handle, int) or handle <= 0:
        raise Fsr1Error("a texture image is a nonzero cudaTextureObject_t handle (int)")
    return Image(handle, 0, int(width), int(height), 0, int(height), int(format), 0)


def _stream(stream):
    if stream is None:
        stream = torch.cuda.current_stream()
    return ctypes.c_void_p(stream.cuda_stream)


def _as_img(x):
    return x if isinstance(x, Image) else image(x)


def easu(inp, out, con, y0=0, y1=0, flags=0, stream=None):
    """EASU over output rows [y0,y1) — the shader dispatch FsrEasuF/H (ffx_fsr1.h:315-437,505-593)."""
    a, b = _as_img(inp), _as_img(out)
    _lib.check(_lib.lib().fsr1_easu(ctypes.byref(a), ctypes.byref(b), (ctypes.c_uint32 * 16)(*con), y0, y1, flags,
                                    _stream(stream)))


def rcas(inp, out, con, y0=0, y1=0, flags=0, stream=None):
    """RCAS over rows [y0,y1) — FsrRcasF/H (ffx_fsr1.h:684-769,782-866)."""
    a, b = _as_img(inp), _as_img(out)
    _lib.check(_lib.lib().fsr1_rcas(ctypes.byref(a), ctypes.byref(b), (ctypes.c_uint32 * 4)(*con), y0, y1, flags,
                                    _stream(stream)))


def upscale(inp, tmp, out, econ, rcon, y0=0, y1=0, flags=0, stream=None):
    """EASU -> RCAS, the body of FSR_Filter::Upscale (sample/src/DX12/FSR_Filter.cpp:101-141)."""
    a, t, b = _as_img(inp), _as_img(tmp), _as_img(out)
    _lib.check(_lib.lib().fsr1_upscale(ctypes.byref(a), ctypes.byref(t), ctypes.byref(b), (ctypes.c_uint32 * 16)(*econ),
                                       (ctypes.c_uint32 * 4)(*rcon), y0, y1, flags, _stream(stream)))


def _post(srtm_inverse, grain, amount, tepd_bits, dither, frame):
    """struct fsr1_post for the given steps, and the image descriptors it points at (kept alive by the caller)."""
    if tepd_bits not in (0, 8, 10):
        raise Fsr1Error("tepd_bits must be 0, 8 or 10")
    ops = (_lib.POST_SRTM_INVERSE if srtm_inverse else 0) | (_lib.POST_LFGA if grain is not None else 0)
    ops |= {0: 0, 8: _lib.POST_TEPD8, 10: _lib.POST_TEPD10}[tepd_bits]
    g = _as_img(grain) if grain is not None else None
    d = _as_img(dither) if dither is not None and tepd_bits else None
    post = _lib.Post(ops, amount, ctypes.pointer(g) if g is not None else None, ctypes.pointer(d) if d is not None else None, frame, 0)
    return post, (g, d)


def upscale_post(inp, tmp, out, econ, rcon, srtm_inverse=False, grain=None, amount=0.0, tepd_bits=0, dither=None, frame=0, y0=0, y1=0,
                 flags=0, stream=None):
    """upscale() followed by SRTM inverse, LFGA (when `grain` is given) and TEPD (tepd_bits 8 / 10), applied inside RCAS's store:
    the bits of upscale + srtm(inverse) + lfga + tepd through an RGBA16F intermediate, written once.  `out` is float16 [H,W,4], or with
    TEPD uint8 [H,W,4] (8 bits) / int32 [H,W] (10 bits), as tepd() accepts.  `tmp` may be None when the frame takes the fused kernel
    (FLAG_FUSED, exactly 2x, no RCAS option)."""
    a, b = _as_img(inp), _as_img(out)
    t = _as_img(tmp) if tmp is not None else None
    post, keep = _post(srtm_inverse, grain, amount, tepd_bits, dither, frame)
    _lib.check(_lib.lib().fsr1_upscale_post(ctypes.byref(a), ctypes.byref(t) if t is not None else None, ctypes.byref(b),
                                            (ctypes.c_uint32 * 16)(*econ), (ctypes.c_uint32 * 4)(*rcon), ctypes.byref(post), y0, y1,
                                            flags, _stream(stream)))
    del keep


def rcas_post(inp, out, rcon, srtm_inverse=False, grain=None, amount=0.0, tepd_bits=0, dither=None, frame=0, y0=0, y1=0, flags=0,
              stream=None):
    """fsr1_rcas_post: a frame rendered at display size, sharpened straight to the display output in one kernel.  The bits of
    rcas() on the RGBA16F image of `inp` (through srtm() first with FLAG_SRTM_INPUT), then srtm(inverse), lfga and tepd as in
    upscale_post().  `inp` is float16 [H,W,4], or int32 [H,W] R11G11B10F codes described by image(t, format=FORMAT_R11G11B10_FLOAT);
    `out` as upscale_post(), or a surface_image() with FLAG_OUT_SURFACE."""
    a, b = _as_img(inp), _as_img(out)
    post, keep = _post(srtm_inverse, grain, amount, tepd_bits, dither, frame)
    _lib.check(_lib.lib().fsr1_rcas_post(ctypes.byref(a), ctypes.byref(b), (ctypes.c_uint32 * 4)(*rcon), ctypes.byref(post), y0, y1, flags,
                                         _stream(stream)))
    del keep


def srtm(inp, out, inverse=False, y0=0, y1=0, stream=None):
    """FsrSrtmF / FsrSrtmInvF (ffx_fsr1.h:1044,1046) over rows [y0,y1); `out` may be `inp` (in place)."""
    a, b = _as_img(inp), _as_img(out)
    _lib.check(_lib.lib().fsr1_srtm(ctypes.byref(a), ctypes.byref(b), 1 if inverse else 0, y0, y1, _stream(stream)))


def lfga(inp, grain, out, amount, y0=0, y1=0, stream=None):
    """FsrLfgaF (ffx_fsr1.h:1014): film grain from the tiled RGB `grain` image ({-0.5..0.5})."""
    a, g, b = _as_img(inp), _as_img(grain), _as_img(out)
    _lib.check(_lib.lib().fsr1_lfga(ctypes.byref(a), ctypes.byref(g), ctypes.byref(b), ctypes.c_float(amount), y0, y1,
                                    _stream(stream)))


def tepd(inp, out, bits, frame=0, dither=None, y0=0, y1=0, stream=None):
    """FsrTepdC8F / FsrTepdC10F (ffx_fsr1.h:1100-1126); dither None -> FsrTepdDitF(pixel, frame), else the .w channel of
    the tiled `dither` image.  `out` may be a UNORM image (uint8 [H,W,4] for 8 bits, int32 [H,W] for 10)."""
    a, b = _as_img(inp), _as_img(out)
    d = _as_img(dither) if dither is not None else None
    _lib.check(_lib.lib().fsr1_tepd(ctypes.byref(a), ctypes.byref(d) if d is not None else None, ctypes.byref(b), bits,
                                    frame, y0, y1, _stream(stream)))


def srtm_h(inp, out, inverse=False, y0=0, y1=0, stream=None):
    """FsrSrtmH / FsrSrtmHx2 and the inverses (ffx_fsr1.h:1049-1055): half arithmetic, packed calling convention; RGBA16F."""
    a, b = _as_img(inp), _as_img(out)
    _lib.check(_lib.lib().fsr1_srtm_h(ctypes.byref(a), ctypes.byref(b), 1 if inverse else 0, y0, y1, _stream(stream)))


def lfga_h(inp, grain, out, amount, y0=0, y1=0, stream=None):
    """FsrLfgaH / FsrLfgaHx2 (ffx_fsr1.h:1019-1024); `grain` is an RGBA16F tile."""
    a, g, b = _as_img(inp), _as_img(grain), _as_img(out)
    _lib.check(_lib.lib().fsr1_lfga_h(ctypes.byref(a), ctypes.byref(g), ctypes.byref(b), ctypes.c_float(amount), y0, y1,
                                      _stream(stream)))


def tepd_h(inp, out, bits, frame=0, dither=None, y0=0, y1=0, stream=None):
    """FsrTepdC8H / C10H and the Hx2 forms (ffx_fsr1.h:1137-1199); dither None -> FsrTepdDitH / DitHx2(pixel, frame), else the .w
    channel of the tiled RGBA16F `dither` image."""
    a, b = _as_img(inp), _as_img(out)
    d = _as_img(dither) if dither is not None else None
    _lib.check(_lib.lib().fsr1_tepd_h(ctypes.byref(a), ctypes.byref(d) if d is not None else None, ctypes.byref(b), bits,
                                      frame, y0, y1, _stream(stream)))


class PreparedUpscale:
    """fsr1_upscale with every argument marshalled once: the per-frame host cost is one foreign call.
    (Streams of frames through fixed buffers — the sharded path, the bench — re-launch the same descriptors.)"""

    def __init__(self, inp, tmp, out, econ, rcon, y0=0, y1=0, flags=0):
        self._a, self._t, self._b = _as_img(inp), _as_img(tmp), _as_img(out)
        self._econ, self._rcon = (ctypes.c_uint32 * 16)(*econ), (ctypes.c_uint32 * 4)(*rcon)
        self._args = (ctypes.byref(self._a), ctypes.byref(self._t), ctypes.byref(self._b), self._econ, self._rcon, y0, y1, flags)
        self._fn = _lib.lib().fsr1_upscale

    def launch(self, stream=None):
        rc = self._fn(*self._args, _stream(stream))
        if rc:
            _lib.check(rc)


class FramePipeline:
    """A stream of frames over fixed buffer sets, software-pipelined on two CUDA streams with the plain entry points: RCAS of frame
    i runs on stream B while EASU of frame i+1 runs on stream A.  (The C ABI's fsr1_shard_* runs whole frames on two streams in turn
    instead — three driver calls fewer per frame — and is what bench.py uses at every GPU count.)  EASU is FMA-pipe-bound and RCAS ALU/XU/issue-bound, and both
    have ragged tails (persistent CTAs / last wave), so letting them share the SMs raises throughput over running the
    two kernels of every frame back to back (bench.py: value vs unpipelined_value).  Per-slot events keep a
    slot's intermediate from being overwritten before its RCAS has read it.

    sets: list of (inp, tmp, out) images/tensors; econ/rcon: the constant blocks shared by all frames."""

    def __init__(self, sets, econ, rcon, flags=0, device=None, priorities=None, easu_rows=(0, 0), rcas_rows=(0, 0)):
        """priorities: optional (easu, rcas) CUDA stream priorities (lower = more urgent); None = default streams.
        easu_rows / rcas_rows: output row ranges [y0,y1) of the two passes when the images are row-slab windows
        (EASU covers the slab plus the one-row apron RCAS reads); (0, 0) = the whole image."""
        self._erows, self._rrows = tuple(int(v) for v in easu_rows), tuple(int(v) for v in rcas_rows)
        self._L = _lib.lib()
        self._econ, self._rcon = (ctypes.c_uint32 * 16)(*econ), (ctypes.c_uint32 * 4)(*rcon)
        self._imgs = [(_as_img(a), _as_img(t), _as_img(b)) for a, t, b in sets]
        self._rcas_flags = flags & ~FLAG_SRTM_INPUT         # the input tonemap belongs to EASU's loads only
        self._easu_flags = flags & ~FLAG_OUTPUT_SQUARE      # the Sample.x hook belongs to the LAST pass only
        if priorities is None:
            self.stream_easu, self.stream_rcas = torch.cuda.Stream(device=device), torch.cuda.Stream(device=device)
        else:
            self.stream_easu = torch.cuda.Stream(device=device, priority=priorities[0])
            self.stream_rcas = torch.cuda.Stream(device=device, priority=priorities[1])
        self._easu_done = [torch.cuda.Event() for _ in sets]
        self._rcas_done = [None for _ in sets]

    def begin(self, stream=None):
        """Order both pipeline streams after `stream` (default: the current stream)."""
        stream = stream or torch.cuda.current_stream()
        self.stream_easu.wait_stream(stream)
        self.stream_rcas.wait_stream(stream)

    def submit(self, slot):
        a, t, b = self._imgs[slot]
        sa, sb = self.stream_easu, self.stream_rcas
        if self._rcas_done[slot] is not None:
            sa.wait_event(self._rcas_done[slot])       # the slot's intermediate is free again
        rc = self._L.fsr1_easu(ctypes.byref(a), ctypes.byref(t), self._econ, self._erows[0], self._erows[1], self._easu_flags,
                               ctypes.c_void_p(sa.cuda_stream))
        if rc:
            _lib.check(rc)
        self._easu_done[slot].record(sa)
        sb.wait_event(self._easu_done[slot])
        rc = self._L.fsr1_rcas(ctypes.byref(t), ctypes.byref(b), self._rcon, self._rrows[0], self._rrows[1], self._rcas_flags,
                               ctypes.c_void_p(sb.cuda_stream))
        if rc:
            _lib.check(rc)
        if self._rcas_done[slot] is None:
            self._rcas_done[slot] = torch.cuda.Event()
        self._rcas_done[slot].record(sb)

    def end(self, stream=None):
        """Order `stream` after everything submitted so far."""
        stream = stream or torch.cuda.current_stream()
        stream.wait_stream(self.stream_easu)
        stream.wait_stream(self.stream_rcas)


def last_kernel():
    return _lib.lib().fsr1_last_kernel_name().decode()


def launch_count():
    return int(_lib.lib().fsr1_launch_count())


def _dev(x, flags, flag):
    """(address, pitch) of a device image argument of the context calls: a tensor, or with a bit of `flag` in `flags` a surface or
    texture object handle (int) with pitch 0."""
    if flags & flag:
        if not isinstance(x, int):
            raise Fsr1Error("with FLAG_IN_SURFACE / FLAG_IN_TEXTURE / FLAG_OUT_SURFACE the matching image is a surface or texture object "
                            "handle (int)")
        return ctypes.c_void_p(x), 0
    return ctypes.c_void_p(x.data_ptr()), x.stride(0) * x.element_size()


class HostContext:
    """fsr1_context_*: owns the intermediate and device staging; frames live in (pinned) host memory.
    fmt: the input's format; the output is in it too, but float16 [H, W, 4] (RGBA16F) for FORMAT_R11G11B10_FLOAT input (int32 [H, W]).
    The device-frame calls take a surface object handle (int) in place of `in_dev` / `out_dev` with FLAG_IN_SURFACE / FLAG_OUT_SURFACE,
    and a texture object handle in place of `in_dev` with FLAG_IN_TEXTURE."""

    def __init__(self, in_w, in_h, out_w, out_h, fmt=FORMAT_RGBA16F):
        self._h = ctypes.c_void_p()
        self.shape = (in_w, in_h, out_w, out_h)
        _lib.check(_lib.lib().fsr1_context_create(ctypes.byref(self._h), in_w, in_h, out_w, out_h, fmt))

    def upscale_host(self, in_host, out_host, sharpness=0.25, flags=0, stream=None):
        _lib.check(_lib.lib().fsr1_context_upscale_host(
            self._h, ctypes.c_void_p(in_host.data_ptr()), in_host.stride(0) * in_host.element_size(),
            ctypes.c_void_p(out_host.data_ptr()), out_host.stride(0) * out_host.element_size(),
            ctypes.c_float(sharpness), flags, _stream(stream)))

    def upscale(self, in_dev, out_dev, sharpness=0.25, flags=0, stream=None):
        (a, ap), (b, bp) = _dev(in_dev, flags, FLAG_IN_SURFACE | FLAG_IN_TEXTURE), _dev(out_dev, flags, FLAG_OUT_SURFACE)
        _lib.check(_lib.lib().fsr1_context_upscale(self._h, a, ap, b, bp, ctypes.c_float(sharpness), flags, _stream(stream)))

    def upscale_render(self, in_dev, render_w, render_h, out_dev, sharpness=0.25, flags=0, stream=None):
        """One frame rendered at render_w x render_h (dynamic resolution): the top-left render region of `in_dev`, upscaled to the
        context's output size with constants rebuilt from this frame's render size."""
        (a, ap), (b, bp) = _dev(in_dev, flags, FLAG_IN_SURFACE | FLAG_IN_TEXTURE), _dev(out_dev, flags, FLAG_OUT_SURFACE)
        _lib.check(_lib.lib().fsr1_context_upscale_render(self._h, a, ap, render_w, render_h, b, bp, ctypes.c_float(sharpness), flags,
                                                          _stream(stream)))

    def upscale_post(self, in_dev, out_dev, render_w=0, render_h=0, sharpness=0.25, srtm_inverse=False, grain=None, amount=0.0,
                     tepd_bits=0, dither=None, frame=0, flags=0, stream=None):
        """fsr1_context_upscale_post: upscale_render followed by the display steps of api.upscale_post; `out_dev` is uint8 [H,W,4]
        with tepd_bits 8, int32 [H,W] with 10, float16 [H,W,4] otherwise.  render size 0 = the context's input size."""
        post, keep = _post(srtm_inverse, grain, amount, tepd_bits, dither, frame)
        (a, ap), (b, bp) = _dev(in_dev, flags, FLAG_IN_SURFACE | FLAG_IN_TEXTURE), _dev(out_dev, flags, FLAG_OUT_SURFACE)
        _lib.check(_lib.lib().fsr1_context_upscale_post(self._h, a, ap, render_w, render_h, b, bp, ctypes.c_float(sharpness),
                                                        ctypes.byref(post), flags, _stream(stream)))
        del keep

    def close(self):
        if self._h:
            _lib.lib().fsr1_context_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
