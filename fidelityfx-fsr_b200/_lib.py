"""ctypes binding of the C ABI in include/fsr1_b200.h.  There is NO fallback: if the CUDA library is
missing or cannot be loaded every entry point raises, loudly."""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libfsr1_b200.so")

FSR1_OK = 0
FORMAT_RGBA16F, FORMAT_RGBA32F, FORMAT_RGBA8_UNORM, FORMAT_RGB10A2_UNORM = 1, 2, 3, 4
FORMAT_R11G11B10_FLOAT = 5  # input only: 4 B/px, int32 [H, W] tensors with api.image(t, format=FORMAT_R11G11B10_FLOAT)
FLAG_RCAS_CLAMP, FLAG_EXACT, FLAG_FORCE_DIRECT, FLAG_NO_RCAS, FLAG_H_REFERENCE, FLAG_PRECISE = 1, 2, 4, 8, 16, 32
FLAG_RCAS_DENOISE, FLAG_RCAS_PASSTHROUGH_ALPHA, FLAG_OUTPUT_SQUARE, FLAG_FUSED, FLAG_RCAS_HX2 = 64, 128, 256, 512, 1024
FLAG_SRTM_INPUT = 2048
FLAG_IN_SURFACE, FLAG_OUT_SURFACE = 1 << 12, 1 << 13  # `in` / `out` is a CUDA surface object (api.surface_image)
FLAG_IN_TEXTURE = 1 << 14  # `in` is a CUDA texture object (api.texture_image)
POST_SRTM_INVERSE, POST_LFGA, POST_TEPD8, POST_TEPD10 = 1, 2, 4, 8
SHARD_ONE_STREAM, SHARD_SKIP_HALO, SHARD_TRACE, SHARD_HANDLE_BYTES = 1 << 16, 1 << 17, 1 << 18, 64
SHARD_DYNAMIC = 1 << 19

# every symbol include/fsr1_b200.h declares
SYMBOLS = ["fsr1_easu", "fsr1_rcas", "fsr1_easu_input_rows", "fsr1_upscale", "fsr1_upscale_post", "fsr1_context_create",
           "fsr1_context_destroy", "fsr1_context_upscale", "fsr1_context_upscale_render", "fsr1_context_upscale_post", "fsr1_context_upscale_host", "fsr1_easu_con",
           "fsr1_easu_con_offset", "fsr1_rcas_con", "fsr1_abi_version", "fsr1_error_string",
           "fsr1_last_cuda_error", "fsr1_launch_count", "fsr1_last_kernel_name", "fsr1_srtm", "fsr1_lfga", "fsr1_tepd",
           "fsr1_srtm_h", "fsr1_lfga_h", "fsr1_tepd_h",
           "fsr1_shard_create", "fsr1_shard_destroy", "fsr1_shard_geometry", "fsr1_shard_export", "fsr1_shard_attach",
           "fsr1_shard_attach_local", "fsr1_shard_input", "fsr1_shard_window", "fsr1_shard_output", "fsr1_shard_arena",
           "fsr1_shard_frame", "fsr1_shard_submit", "fsr1_shard_wait", "fsr1_shard_status", "fsr1_shard_trace",
           "fsr1_shard_create_post", "fsr1_shard_post", "fsr1_rcas_post"]


class Image(ctypes.Structure):
    """struct fsr1_image"""
    _fields_ = [("data", ctypes.c_void_p), ("pitch_bytes", ctypes.c_uint64), ("width", ctypes.c_uint32),
                ("height", ctypes.c_uint32), ("row0", ctypes.c_uint32), ("rows", ctypes.c_uint32),
                ("format", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class Post(ctypes.Structure):
    """struct fsr1_post"""
    _fields_ = [("ops", ctypes.c_uint32), ("lfga_amount", ctypes.c_float), ("grain", ctypes.POINTER(Image)),
                ("dither", ctypes.POINTER(Image)), ("frame", ctypes.c_uint32), ("reserved", ctypes.c_uint32)]


class ShardInfo(ctypes.Structure):
    """struct fsr1_shard_info"""
    _fields_ = [(n, ctypes.c_uint32) for n in (
        "out_row0", "out_row1", "easu_row0", "easu_row1", "owned_row0", "owned_row1", "needed_row0", "needed_row1",
        "window_row0", "window_row1", "send_up_row0", "send_up_row1", "send_down_row0", "send_down_row1")] + [
        ("halo_recv_bytes", ctypes.c_uint64), ("arena_bytes", ctypes.c_uint64)]


class Fsr1Error(RuntimeError):
    pass


_lib = None


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise Fsr1Error("%s is missing: run `python fidelityfx-fsr_b200/build.py` (needs nvcc). "
                        "There is no CPU fallback." % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    u32p, imgp, vp = ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(Image), ctypes.c_void_p
    u32, u64, f32 = ctypes.c_uint32, ctypes.c_uint64, ctypes.c_float
    L.fsr1_easu.argtypes = [imgp, imgp, u32p, u32, u32, u32, vp]
    L.fsr1_rcas.argtypes = [imgp, imgp, u32p, u32, u32, u32, vp]
    L.fsr1_easu_input_rows.argtypes = [u32p, u32, u32, u32, u32p, u32p]
    L.fsr1_upscale.argtypes = [imgp, imgp, imgp, u32p, u32p, u32, u32, u32, vp]
    postp = ctypes.POINTER(Post)
    L.fsr1_upscale_post.argtypes = [imgp, imgp, imgp, u32p, u32p, postp, u32, u32, u32, vp]
    L.fsr1_context_upscale_post.argtypes = [vp, vp, u64, u32, u32, vp, u64, f32, postp, u32, vp]
    L.fsr1_rcas_post.argtypes = [imgp, imgp, u32p, postp, u32, u32, u32, vp]
    L.fsr1_context_create.argtypes = [ctypes.POINTER(vp), u32, u32, u32, u32, u32]
    L.fsr1_context_destroy.argtypes = [vp]
    L.fsr1_context_destroy.restype = None
    L.fsr1_context_upscale.argtypes = [vp, vp, u64, vp, u64, f32, u32, vp]
    L.fsr1_context_upscale_host.argtypes = [vp, vp, u64, vp, u64, f32, u32, vp]
    L.fsr1_context_upscale_render.argtypes = [vp, vp, u64, u32, u32, vp, u64, f32, u32, vp]
    L.fsr1_easu_con.argtypes = [u32p] + [f32] * 6
    L.fsr1_easu_con.restype = None
    L.fsr1_easu_con_offset.argtypes = [u32p] + [f32] * 8
    L.fsr1_easu_con_offset.restype = None
    L.fsr1_rcas_con.argtypes = [u32p, f32]
    L.fsr1_rcas_con.restype = None
    L.fsr1_srtm.argtypes = [imgp, imgp, ctypes.c_int, u32, u32, vp]
    L.fsr1_lfga.argtypes = [imgp, imgp, imgp, f32, u32, u32, vp]
    L.fsr1_tepd.argtypes = [imgp, imgp, imgp, ctypes.c_int, u32, u32, u32, vp]
    L.fsr1_srtm_h.argtypes = [imgp, imgp, ctypes.c_int, u32, u32, vp]
    L.fsr1_lfga_h.argtypes = [imgp, imgp, imgp, f32, u32, u32, vp]
    L.fsr1_tepd_h.argtypes = [imgp, imgp, imgp, ctypes.c_int, u32, u32, u32, vp]
    L.fsr1_shard_create.argtypes = [ctypes.POINTER(vp), u32, u32, u32, u32, u32, u32, u32, u32, f32, u32]
    L.fsr1_shard_create_post.argtypes = [ctypes.POINTER(vp), u32, u32, u32, u32, u32, u32, postp, u32, u32, u32, f32, u32]
    L.fsr1_shard_post.argtypes = [vp, u32, postp]
    L.fsr1_shard_destroy.argtypes = [vp]
    L.fsr1_shard_destroy.restype = None
    L.fsr1_shard_geometry.argtypes = [vp, ctypes.POINTER(ShardInfo)]
    L.fsr1_shard_export.argtypes = [vp, vp]
    L.fsr1_shard_attach.argtypes = [vp, ctypes.c_char_p, u32]
    L.fsr1_shard_attach_local.argtypes = [vp, vp, vp]
    for fn in (L.fsr1_shard_input, L.fsr1_shard_window, L.fsr1_shard_output):
        fn.argtypes = [vp, u32, imgp]
    L.fsr1_shard_arena.argtypes = [vp]
    L.fsr1_shard_arena.restype = vp
    L.fsr1_shard_frame.argtypes = [vp, u32, u32, u32, f32]
    L.fsr1_shard_submit.argtypes = [vp, u32, vp]
    L.fsr1_shard_wait.argtypes = [vp, u32, vp]
    L.fsr1_shard_status.argtypes = [vp]
    L.fsr1_shard_trace.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64), u32, u32p]
    L.fsr1_error_string.restype = ctypes.c_char_p
    L.fsr1_error_string.argtypes = [ctypes.c_int]
    L.fsr1_last_kernel_name.restype = ctypes.c_char_p
    L.fsr1_launch_count.restype = ctypes.c_uint64
    _lib = L
    return L


def check(rc):
    if rc != FSR1_OK:
        L = lib()
        raise Fsr1Error("fsr1: %s (code %d, cuda error %d)" % (L.fsr1_error_string(rc).decode(), rc,
                                                              L.fsr1_last_cuda_error()))
