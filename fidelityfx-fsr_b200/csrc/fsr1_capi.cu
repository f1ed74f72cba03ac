// fsr1_capi.cu — the C ABI declared in include/fsr1_b200.h: argument validation, kernel selection,
// the resource-owning context, and the constant-setup entry points.
#include <atomic>
#include <math.h>
#include <new>
#include <string.h>

#include <nvtx3/nvToolsExt.h>  // header-only NVTX 3: ranges "EASU" / "RCAS" / "FSR1" around the launches, as the sample's
                               // user markers do (sample/src/DX12/FSR_Filter.cpp:118,128); no-ops unless a profiler is attached

#include "../../include/fsr1_b200.h"
#include "../../include/fsr1_host.h"
#include "fsr1_common.cuh"
#include "fsr1_post.cuh"

using namespace fsr1;

namespace {

struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

thread_local int t_last_cuda = 0;
thread_local const char* t_last_kernel = "";
std::atomic<unsigned long long> g_launches{0};

}  // namespace
namespace fsr1 {
void set_last_detail(int v) { t_last_cuda = v; }  // fsr1_shard_status: which wait timed out, reported through fsr1_last_cuda_error()
}
namespace {

int cuda_fail(cudaError_t e) {
  t_last_cuda = (int)e;
  return FSR1_ERR_CUDA;
}

// a kernel launched: fsr1_last_kernel_name and fsr1_launch_count
void launched(const char* name) {
  t_last_kernel = name;
  g_launches.fetch_add(1);
}

// R11G11B10_FLOAT input runs on the RGBA16F production kernels (and the fast direct kernel); the parity and fp32 paths do not take it
constexpr uint32_t kR11Refused = FSR1_FLAG_EXACT | FSR1_FLAG_H_REFERENCE | FSR1_FLAG_PRECISE | FSR1_FLAG_RCAS_HX2;

// the flags that keep a frame off the fused EASU->RCAS kernels (plain and post): the other arithmetic paths, and the RCAS options and
// output step the fused kernels do not have
constexpr uint32_t kNotFused = FSR1_FLAG_EXACT | FSR1_FLAG_FORCE_DIRECT | FSR1_FLAG_H_REFERENCE | FSR1_FLAG_PRECISE | FSR1_FLAG_RCAS_CLAMP |
                               FSR1_FLAG_RCAS_DENOISE | FSR1_FLAG_RCAS_PASSTHROUGH_ALPHA | FSR1_FLAG_OUTPUT_SQUARE | FSR1_FLAG_RCAS_HX2;

int check_image(const fsr1_image* im) {
  if (!im || !im->data || im->width == 0 || im->height == 0 || im->rows == 0) return FSR1_ERR_INVALID_ARGUMENT;
  const int bpp = bytes_per_pixel(im->format);
  if (!bpp) return FSR1_ERR_INVALID_ARGUMENT;
  if (im->width > 32768u || im->height > 32768u) return FSR1_ERR_INVALID_ARGUMENT;
  if (im->pitch_bytes < (uint64_t)im->width * bpp || (im->pitch_bytes % bpp) != 0) return FSR1_ERR_INVALID_ARGUMENT;
  if ((uintptr_t)im->data % bpp != 0) return FSR1_ERR_INVALID_ARGUMENT;
  if ((uint64_t)im->row0 + im->rows > im->height) return FSR1_ERR_INVALID_ARGUMENT;
  return FSR1_OK;
}

ImgView view_of(const fsr1_image* im) {
  ImgView v;
  v.base = static_cast<unsigned char*>(im->data);
  v.pitch = (long long)im->pitch_bytes;
  v.w = (int)im->width;
  v.h = (int)im->height;
  v.row0 = (int)im->row0;
  v.rows = (int)im->rows;
  return v;
}

// identical float arithmetic to easu_pos() on the device and to the oracle
int host_cell(uint32_t o, float scale, float offset) {
  volatile float m = (float)o * scale;
  volatile float s = m + offset;
  return (int)floorf(s);
}

// every flag include/fsr1_b200.h defines
constexpr uint32_t kAllFlags = FSR1_FLAG_RCAS_CLAMP | FSR1_FLAG_EXACT | FSR1_FLAG_FORCE_DIRECT | FSR1_FLAG_NO_RCAS |
                               FSR1_FLAG_H_REFERENCE | FSR1_FLAG_PRECISE | FSR1_FLAG_RCAS_DENOISE |
                               FSR1_FLAG_RCAS_PASSTHROUGH_ALPHA | FSR1_FLAG_OUTPUT_SQUARE | FSR1_FLAG_FUSED | FSR1_FLAG_RCAS_HX2 |
                               FSR1_FLAG_SRTM_INPUT | FSR1_FLAG_IN_SURFACE | FSR1_FLAG_OUT_SURFACE | FSR1_FLAG_IN_TEXTURE;

// ---- array images (FSR1_FLAG_IN_SURFACE / FSR1_FLAG_IN_TEXTURE / FSR1_FLAG_OUT_SURFACE, include/fsr1_b200.h) -----------------------
constexpr uint32_t kArrayIn = FSR1_FLAG_IN_SURFACE | FSR1_FLAG_IN_TEXTURE;  // `in` is a CUDA array: at most one of them
constexpr uint32_t kArrayFlags = kArrayIn | FSR1_FLAG_OUT_SURFACE;
// the array stages exist in the RGBA16F production kernels only (tiled EASU, packed RCAS, fused, post) and their R11G11B10F variants
constexpr uint32_t kSurfRefused = FSR1_FLAG_EXACT | FSR1_FLAG_FORCE_DIRECT | FSR1_FLAG_H_REFERENCE | FSR1_FLAG_PRECISE | FSR1_FLAG_RCAS_HX2;

// flags the call cannot take whatever it is: an unknown bit, or both kinds of array input
bool bad_flags(uint32_t flags) { return (flags & ~kAllFlags) || (flags & kArrayIn) == kArrayIn; }

// The layout of an array image (a surface or texture image): a handle, pitch 0, the whole image (never a window).  No CUDA call.
int check_array(const fsr1_image* im) {
  if (!im || !im->data || im->width == 0 || im->height == 0 || im->width > 32768u || im->height > 32768u) return FSR1_ERR_INVALID_ARGUMENT;
  if (!bytes_per_pixel(im->format) || im->pitch_bytes != 0 || im->row0 != 0 || im->rows != im->height) return FSR1_ERR_INVALID_ARGUMENT;
  return FSR1_OK;
}
// an image the call reads or writes: an array image when a flag that describes it is set, a linear one otherwise
int check_io(const fsr1_image* im, bool array) { return array ? check_array(im) : check_image(im); }
// where EASU's load stage reads `in` from under `flags`
InSrc in_src(uint32_t flags) {
  return (flags & FSR1_FLAG_IN_TEXTURE) ? kInTex : (flags & FSR1_FLAG_IN_SURFACE) ? kInSurf : kInTma;
}

// The CUDA array behind a surface image: a 2D array (not layered, not 3D) whose element is the format's size and whose extent holds
// width x height.  An unknown handle: FSR1_ERR_INVALID_ARGUMENT (the failed query's error is cleared: nothing has launched).
int surface_fits(const fsr1_image* im) {
  cudaResourceDesc rd;
  cudaChannelFormatDesc cd;
  cudaExtent ext;
  unsigned int aflags = 0;
  if (cudaGetSurfaceObjectResourceDesc(&rd, (cudaSurfaceObject_t)(uintptr_t)im->data) != cudaSuccess) {
    cudaGetLastError();
    return FSR1_ERR_INVALID_ARGUMENT;
  }
  if (rd.resType != cudaResourceTypeArray) return FSR1_ERR_UNSUPPORTED;
  if (cudaArrayGetInfo(&cd, &ext, &aflags, rd.res.array.array) != cudaSuccess) {
    cudaGetLastError();
    return FSR1_ERR_INVALID_ARGUMENT;
  }
  if (ext.depth != 0 || (aflags & cudaArrayLayered)) return FSR1_ERR_UNSUPPORTED;
  if ((cd.x + cd.y + cd.z + cd.w) != 8 * bytes_per_pixel(im->format)) return FSR1_ERR_UNSUPPORTED;
  if (ext.width < im->width || ext.height < im->height) return FSR1_ERR_INVALID_ARGUMENT;
  return FSR1_OK;
}

// The texture object behind a texture image: a level-0 2D array resource (not layered, not 3D) whose channels are unsigned integers of
// the format's layout (16,16,16,16 for RGBA16F, 32 for R11G11B10F), read in element mode at unnormalized coordinates with point
// filtering and no sRGB decode, so that every fetch returns the texel's raw bits; its extent holds width x height.  An unknown handle or
// a short extent: FSR1_ERR_INVALID_ARGUMENT (a failed query's error is cleared: nothing has launched); anything else that differs:
// FSR1_ERR_UNSUPPORTED.  The address mode is free: every fetch is inside the logical image.
int texture_fits(const fsr1_image* im) {
  const cudaTextureObject_t t = (cudaTextureObject_t)(uintptr_t)im->data;
  cudaResourceDesc rd;
  cudaTextureDesc td;
  cudaChannelFormatDesc cd;
  cudaExtent ext;
  unsigned int aflags = 0;
  if (cudaGetTextureObjectResourceDesc(&rd, t) != cudaSuccess || cudaGetTextureObjectTextureDesc(&td, t) != cudaSuccess) {
    cudaGetLastError();
    return FSR1_ERR_INVALID_ARGUMENT;
  }
  if (rd.resType != cudaResourceTypeArray) return FSR1_ERR_UNSUPPORTED;  // pitch2D, linear and mipmapped resources
  if (td.readMode != cudaReadModeElementType || td.normalizedCoords || td.filterMode != cudaFilterModePoint || td.sRGB)
    return FSR1_ERR_UNSUPPORTED;
  if (cudaArrayGetInfo(&cd, &ext, &aflags, rd.res.array.array) != cudaSuccess) {
    cudaGetLastError();
    return FSR1_ERR_INVALID_ARGUMENT;
  }
  if (ext.depth != 0 || (aflags & cudaArrayLayered)) return FSR1_ERR_UNSUPPORTED;
  const bool bits = im->format == FSR1_FORMAT_RGBA16F ? cd.x == 16 && cd.y == 16 && cd.z == 16 && cd.w == 16
                  : im->format == FSR1_FORMAT_R11G11B10_FLOAT && cd.x == 32 && cd.y == 0 && cd.z == 0 && cd.w == 0;
  if (cd.f != cudaChannelFormatKindUnsigned || !bits) return FSR1_ERR_UNSUPPORTED;  // a float kind would convert, losing the bits
  if (ext.width < im->width || ext.height < im->height) return FSR1_ERR_INVALID_ARGUMENT;
  return FSR1_OK;
}
// the CUDA array behind an array input
int in_array_fits(const fsr1_image* in, uint32_t flags) { return (flags & FSR1_FLAG_IN_TEXTURE) ? texture_fits(in) : surface_fits(in); }

// Every refusal of the array flags of a call that may take both sides (fsr1_upscale, fsr1_upscale_post), before anything launches, so
// that the two-kernel path never runs EASU and then refuses RCAS's store: the flag and format rules first, then the arrays.  unorm_out:
// the output may also be RGBA8 / RGB10A2 (fsr1_upscale_post's TEPD; its format rules are post_params').  The layouts were checked already.
int array_rules(const fsr1_image* in, const fsr1_image* out, const uint32_t* easu_con, uint32_t flags, bool unorm_out) {
  if (flags & kSurfRefused) return FSR1_ERR_UNSUPPORTED;
  // the array twins are those of the RGBA16F kernels, and with a texture input those of their R11G11B10F variants
  const bool tex_r11 = (flags & FSR1_FLAG_IN_TEXTURE) && in->format == FSR1_FORMAT_R11G11B10_FLOAT;
  if (in->format != FSR1_FORMAT_RGBA16F && !tex_r11) return FSR1_ERR_UNSUPPORTED;
  if (flags & kArrayIn) {
    if (!is_upscale(word_as_float(easu_con[0]), word_as_float(easu_con[1]))) return FSR1_ERR_UNSUPPORTED;  // no direct kernel reads one
  }
  if (flags & FSR1_FLAG_OUT_SURFACE) {
    if (flags & FSR1_FLAG_NO_RCAS) return FSR1_ERR_UNSUPPORTED;  // EASU stores to linear images only
    const bool ok = out->format == FSR1_FORMAT_RGBA16F ||
                    (unorm_out && (out->format == FSR1_FORMAT_RGBA8_UNORM || out->format == FSR1_FORMAT_RGB10A2_UNORM));
    if (!ok) return FSR1_ERR_UNSUPPORTED;
  }
  int rc;
  if ((flags & kArrayIn) && (rc = in_array_fits(in, flags)) != FSR1_OK) return rc;
  if ((flags & FSR1_FLAG_OUT_SURFACE) && (rc = surface_fits(out)) != FSR1_OK) return rc;
  return FSR1_OK;
}

bool window_holds(const fsr1_image* im, int first, int last) {  // logical rows [first,last]
  return first >= (int)im->row0 && last < (int)(im->row0 + im->rows);
}

// RCAS reads neighbours of every pixel it writes: an output whose storage overlaps the input's is a race
bool overlaps(const fsr1_image* a, const fsr1_image* b) {
  const uintptr_t a0 = (uintptr_t)a->data, a1 = a0 + (uintptr_t)a->pitch_bytes * a->rows;
  const uintptr_t b0 = (uintptr_t)b->data, b1 = b0 + (uintptr_t)b->pitch_bytes * b->rows;
  return a0 < b1 && b0 < a1;
}

EasuParams easu_params(const fsr1_image* in, const fsr1_image* out, const uint32_t con[16], uint32_t y0, uint32_t y1) {
  EasuParams p;
  p.in = view_of(in);
  p.out = view_of(out);
  p.c0x = word_as_float(con[0]); p.c0y = word_as_float(con[1]); p.c0z = word_as_float(con[2]); p.c0w = word_as_float(con[3]);
  p.y0 = (int)y0; p.y1 = (int)y1;
  return p;
}

// options: the RCAS flags of every kernel (bit 2, the Sample.x hook, is added where a kernel folds it into its store)
RcasParams rcas_params(const fsr1_image* in, const fsr1_image* out, const uint32_t con[4], uint32_t y0, uint32_t y1, uint32_t flags) {
  RcasParams p;
  p.in = view_of(in);
  p.out = view_of(out);
  p.sharp = word_as_float(con[0]);
  p.sharp_h2 = con[1];
  p.y0 = (int)y0; p.y1 = (int)y1;
  p.clamp = (flags & FSR1_FLAG_RCAS_CLAMP) ? 1 : 0;
  p.options = ((flags & FSR1_FLAG_RCAS_DENOISE) ? 1 : 0) | ((flags & FSR1_FLAG_RCAS_PASSTHROUGH_ALPHA) ? 2 : 0);
  return p;
}

// FSR1_FLAG_SRTM_INPUT: only the TMA-tiled RGBA16F EASU kernels (and the fused kernels built on them) apply FsrSrtmF as they load,
// so everything those kernels decline is refused here, before any CUDA call, instead of falling back to a kernel that would ignore
// the flag.  `out`: the image EASU writes (the intermediate, or the output of a fused frame); null when not checked here.
int srtm_input_check(const fsr1_image* in, const fsr1_image* out, const uint32_t con[16], uint32_t flags) {
  if (in->format != FSR1_FORMAT_RGBA16F && in->format != FSR1_FORMAT_R11G11B10_FLOAT) return FSR1_ERR_UNSUPPORTED;
  if (flags & (FSR1_FLAG_EXACT | FSR1_FLAG_FORCE_DIRECT | FSR1_FLAG_H_REFERENCE | FSR1_FLAG_PRECISE)) return FSR1_ERR_UNSUPPORTED;
  if (!(flags & kArrayIn) && (((uintptr_t)in->data & 15) || (in->pitch_bytes & 15))) return FSR1_ERR_UNSUPPORTED;  // TMA
  if (out && (((uintptr_t)out->data & 15) || (out->pitch_bytes & 15))) return FSR1_ERR_UNSUPPORTED;  // 16-byte pixel-pair stores
  if (!is_upscale(word_as_float(con[0]), word_as_float(con[1]))) return FSR1_ERR_UNSUPPORTED;
  return FSR1_OK;
}

// The images of an RCAS pass over rows [y0, y1) (y1 == 0 becomes the last row): the same logical size, a row range inside the image,
// windows that hold the rows written and the rows read, linear storage that does not overlap; then the array behind a surface output
// (the only CUDA call).  fsr1_rcas and fsr1_rcas_post.
int rcas_images(const fsr1_image* in, const fsr1_image* out, uint32_t y0, uint32_t& y1, bool surf_out) {
  if (in->width != out->width || in->height != out->height) return FSR1_ERR_INVALID_ARGUMENT;
  if (y1 == 0) y1 = out->height;
  if (y0 >= y1 || y1 > out->height) return FSR1_ERR_INVALID_ARGUMENT;
  if (!window_holds(out, (int)y0, (int)y1 - 1)) return FSR1_ERR_WINDOW;
  const Rows need = easu_rows(y0, y1, out->height);
  if (!window_holds(in, (int)need.a, (int)need.b - 1)) return FSR1_ERR_WINDOW;
  if (!surf_out && overlaps(in, out)) return FSR1_ERR_INVALID_ARGUMENT;
  if (surf_out) return surface_fits(out);
  return FSR1_OK;
}

// the Sample.x hook: `c *= c` in place on the rows the last pass wrote (a separate streaming pass)
int square_rows(const fsr1_image* img, uint32_t y0, uint32_t y1, cudaStream_t s) {
  const ImgView v = view_of(img);
  const char* name = "";
  cudaError_t e = launch_pointwise(6, v, (int)img->format, v, (int)img->format, nullptr, 0, 0.0f, 0u, (int)y0, (int)y1, s, &name);
  if (e != cudaSuccess) return cuda_fail(e);
  launched(name);
  return FSR1_OK;
}

// The pointwise companions: any format but R11G11B10_FLOAT (launch_pointwise), or with `half` the H / Hx2 forms, RGBA16F everywhere
// (launch_pointwise_hx2).
int pointwise(int op, bool half, const fsr1_image* in, const fsr1_image* aux, const fsr1_image* out, float amount, uint32_t frame,
              uint32_t y0, uint32_t y1, void* stream) {
  int rc;
  if ((rc = check_image(in)) != FSR1_OK || (rc = check_image(out)) != FSR1_OK) return rc;
  if (aux && (rc = check_image(aux)) != FSR1_OK) return rc;
  if (aux && (aux->row0 != 0 || aux->rows != aux->height)) return FSR1_ERR_INVALID_ARGUMENT;  // tiles are whole images
  if (in->width != out->width || in->height != out->height) return FSR1_ERR_INVALID_ARGUMENT;
  const bool formats_ok = half ? in->format == FSR1_FORMAT_RGBA16F && out->format == FSR1_FORMAT_RGBA16F &&
                                     (!aux || aux->format == FSR1_FORMAT_RGBA16F)
                              : in->format != FSR1_FORMAT_R11G11B10_FLOAT && out->format != FSR1_FORMAT_R11G11B10_FLOAT &&
                                     (!aux || aux->format != FSR1_FORMAT_R11G11B10_FLOAT);  // an EASU input format only
  if (!formats_ok) return FSR1_ERR_UNSUPPORTED;
  if (y1 == 0) y1 = out->height;
  if (y0 >= y1 || y1 > out->height) return FSR1_ERR_INVALID_ARGUMENT;
  if (!window_holds(out, (int)y0, (int)y1 - 1) || !window_holds(in, (int)y0, (int)y1 - 1)) return FSR1_ERR_WINDOW;
  const ImgView vi = view_of(in), vo = view_of(out);
  ImgView va;
  if (aux) va = view_of(aux);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const char* name = "";
  const cudaError_t e =
      half ? launch_pointwise_hx2(op, vi, vo, aux ? &va : nullptr, amount, frame, (int)y0, (int)y1, s, &name)
           : launch_pointwise(op, vi, (int)in->format, vo, (int)out->format, aux ? &va : nullptr, aux ? (int)aux->format : 0, amount,
                              frame, (int)y0, (int)y1, s, &name);
  if (e == cudaErrorNotSupported && !half) return FSR1_ERR_UNSUPPORTED;  // launch_pointwise declines the format combination
  if (e != cudaSuccess) return cuda_fail(e);
  launched(name);
  return FSR1_OK;
}

// The fused EASU -> RCAS kernel for output rows [y0, y1) of `out`, with the display epilogue `q` when not null: cudaErrorNotSupported
// when it does not cover the frame.  A sharded frame's neighbour hand-shake (`sync`) rides inside the kernel.
cudaError_t launch_fused(const fsr1_image* in, const fsr1_image* out, const uint32_t easu_con[16], const uint32_t rcas_con[4],
                         const PostParams* q, uint32_t y0, uint32_t y1, uint32_t flags, void* stream, const HaloSync* sync,
                         bool* sync_taken) {
  EasuParams p = easu_params(in, out, easu_con, y0, y1);
  if (sync) p.sync = *sync;
  const bool srtm_in = (flags & FSR1_FLAG_SRTM_INPUT) != 0, r11 = in->format == FSR1_FORMAT_R11G11B10_FLOAT;
  const InSrc src = in_src(flags);
  const bool surf_out = (flags & FSR1_FLAG_OUT_SURFACE) != 0;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const char* name = "";
  const cudaError_t e = q ? launch_fused_h_post(p, rcas_con[1], *q, (int)out->format, s, &name, srtm_in, r11, src, surf_out)
                          : launch_fused_h(p, rcas_con[1], 0, s, &name, srtm_in, r11, src, surf_out);
  if (e != cudaSuccess) return e;
  launched(name);
  if (sync) *sync_taken = true;
  return cudaSuccess;
}

// ---- upscale straight to the display output: the rules of the post description ----------------------------------------------
constexpr uint32_t kAllPost = FSR1_POST_SRTM_INVERSE | FSR1_POST_LFGA | FSR1_POST_TEPD8 | FSR1_POST_TEPD10;

// an aux tile of the epilogue: a whole image (not a window), described as 1 x 1 when the ops do not read it
int post_tile(const fsr1_image* im, bool used, ImgView& v, int& fmt) {
  v = ImgView{nullptr, 0, 1, 1, 0, 1};
  fmt = 0;
  if (!used || !im) return FSR1_OK;
  const int rc = check_image(im);
  if (rc != FSR1_OK) return rc;
  if (im->row0 != 0 || im->rows != im->height) return FSR1_ERR_INVALID_ARGUMENT;
  v = view_of(im);
  fmt = (int)im->format;
  return FSR1_OK;
}

// the epilogue's parameters from a post description with ops != 0, under the rules that depend on the description, the formats and
// the flags only (fsr1::post_rules)
int post_params(const fsr1_post* post, uint32_t in_format, uint32_t out_format, uint32_t flags, PostParams& q) {
  const uint32_t ops = post->ops;
  if (ops & ~kAllPost) return FSR1_ERR_INVALID_ARGUMENT;
  if ((ops & FSR1_POST_TEPD8) && (ops & FSR1_POST_TEPD10)) return FSR1_ERR_INVALID_ARGUMENT;
  if ((ops & FSR1_POST_LFGA) && !post->grain) return FSR1_ERR_INVALID_ARGUMENT;
  if (bad_flags(flags)) return FSR1_ERR_INVALID_ARGUMENT;
  int rc;
  const bool tepd = (ops & (FSR1_POST_TEPD8 | FSR1_POST_TEPD10)) != 0;
  if ((rc = post_tile(post->grain, (ops & FSR1_POST_LFGA) != 0, q.grain, q.grain_fmt)) != FSR1_OK) return rc;
  if ((rc = post_tile(post->dither, tepd, q.dither, q.dither_fmt)) != FSR1_OK) return rc;
  if (q.grain_fmt && q.grain_fmt != FSR1_FORMAT_RGBA16F && q.grain_fmt != FSR1_FORMAT_RGBA32F) return FSR1_ERR_UNSUPPORTED;  // signed values
  if (q.dither_fmt == FSR1_FORMAT_R11G11B10_FLOAT) return FSR1_ERR_UNSUPPORTED;  // an EASU input format only
  q.ops = (int)ops;
  q.amount = post->lfga_amount;
  q.frame = post->frame;
  // formats: RGBA16F or R11G11B10_FLOAT in; RGBA16F out, or with TEPD the matching UNORM code values (the rule of fsr1_tepd)
  if (in_format != FSR1_FORMAT_RGBA16F && in_format != FSR1_FORMAT_R11G11B10_FLOAT) return FSR1_ERR_UNSUPPORTED;
  if (in_format == FSR1_FORMAT_R11G11B10_FLOAT && (flags & kR11Refused)) return FSR1_ERR_UNSUPPORTED;
  const uint32_t unorm = (ops & FSR1_POST_TEPD8) ? FSR1_FORMAT_RGBA8_UNORM : (ops & FSR1_POST_TEPD10) ? FSR1_FORMAT_RGB10A2_UNORM : 0;
  if (out_format != FSR1_FORMAT_RGBA16F && (!unorm || out_format != unorm)) return FSR1_ERR_UNSUPPORTED;
  // the half-arithmetic parity paths, fp32 EXACT/direct kernels and EASU-only frames keep the separate passes
  if (flags & (FSR1_FLAG_EXACT | FSR1_FLAG_FORCE_DIRECT | FSR1_FLAG_H_REFERENCE | FSR1_FLAG_RCAS_HX2 | FSR1_FLAG_NO_RCAS))
    return FSR1_ERR_UNSUPPORTED;
  return FSR1_OK;
}

}  // namespace

namespace fsr1 {

int easu(const fsr1_image* in, const fsr1_image* out, const uint32_t con[16], uint32_t y0, uint32_t y1, uint32_t flags, void* stream,
         const HaloSync* sync, bool* sync_taken) {
  NvtxRange range("EASU");
  int rc;
  const bool array_in = (flags & kArrayIn) != 0, tex_in = (flags & FSR1_FLAG_IN_TEXTURE) != 0;
  if ((rc = check_io(in, array_in)) != FSR1_OK || (rc = check_image(out)) != FSR1_OK) return rc;
  if (!con || bad_flags(flags)) return FSR1_ERR_INVALID_ARGUMENT;
  if (flags & FSR1_FLAG_OUT_SURFACE) return FSR1_ERR_UNSUPPORTED;  // EASU stores to linear images only
  if (array_in && (flags & kSurfRefused)) return FSR1_ERR_UNSUPPORTED;
  const bool r11 = in->format == FSR1_FORMAT_R11G11B10_FLOAT;
  if (array_in && ((in->format != FSR1_FORMAT_RGBA16F && !(tex_in && r11)) || !is_upscale(word_as_float(con[0]), word_as_float(con[1]))))
    return FSR1_ERR_UNSUPPORTED;
  if (out->format != easu_out_format(in->format)) return FSR1_ERR_UNSUPPORTED;
  if (r11 && (flags & kR11Refused)) return FSR1_ERR_UNSUPPORTED;
  if (y1 == 0) y1 = out->height;
  if (y0 >= y1 || y1 > out->height) return FSR1_ERR_INVALID_ARGUMENT;
  if (!window_holds(out, (int)y0, (int)y1 - 1)) return FSR1_ERR_WINDOW;
  uint32_t r0, r1;
  fsr1_easu_input_rows(con, in->height, y0, y1, &r0, &r1);
  if (!window_holds(in, (int)r0, (int)r1)) return FSR1_ERR_WINDOW;
  const bool srtm_in = (flags & FSR1_FLAG_SRTM_INPUT) != 0;
  if (srtm_in && (rc = srtm_input_check(in, out, con, flags)) != FSR1_OK) return rc;
  if (array_in && (rc = in_array_fits(in, flags)) != FSR1_OK) return rc;

  EasuParams p = easu_params(in, out, con, y0, y1);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool exact = (flags & FSR1_FLAG_EXACT) != 0;
  cudaError_t e = cudaErrorNotSupported;
  const char* name = "";
  // Which kernel runs may depend on the constants only through is_2x and is_upscale (fsr1_common.cuh).
  if (flags & FSR1_FLAG_H_REFERENCE) {
    if (in->format != FSR1_FORMAT_RGBA16F || exact) return FSR1_ERR_UNSUPPORTED;
    e = launch_easu_href(p, s, &name);
  } else if ((in->format == FSR1_FORMAT_RGBA16F || r11) && !exact && !(flags & FSR1_FLAG_FORCE_DIRECT)) {
    // the RGBA16F kernels, or their R11G11B10_FLOAT variants (which refused FSR1_FLAG_PRECISE above); else the direct kernel
    if (flags & FSR1_FLAG_PRECISE) e = launch_easu_h_precise(p, s, &name);
    if (e == cudaErrorNotSupported) {
      if (sync) p.sync = *sync;  // sharded frame: the neighbour hand-shake rides inside the kernel
      e = launch_easu_h_tiled(p, s, &name, srtm_in, r11, in_src(flags));
      if (e == cudaSuccess && sync) *sync_taken = true;
      p.sync = HaloSync{};
    }
    if (e == cudaErrorNotSupported && (srtm_in || array_in)) return FSR1_ERR_UNSUPPORTED;  // nothing launched; no other kernel applies the flag
  } else if (in->format == FSR1_FORMAT_RGBA32F && !exact && !(flags & FSR1_FLAG_FORCE_DIRECT)) {
    e = launch_easu_f32_tiled(p, s, &name);
  } else if ((in->format == FSR1_FORMAT_RGBA8_UNORM || in->format == FSR1_FORMAT_RGB10A2_UNORM) && !exact &&
             !(flags & (FSR1_FLAG_FORCE_DIRECT | FSR1_FLAG_PRECISE))) {
    e = launch_easu_u_tiled(p, (int)in->format, s, &name);  // half2 taps; FSR1_FLAG_PRECISE keeps the fp32 direct kernel
  }
  if (e == cudaErrorNotSupported) e = launch_easu_direct(p, (int)in->format, exact, s, &name);
  if (e != cudaSuccess) return cuda_fail(e);
  launched(name);
  if (flags & FSR1_FLAG_OUTPUT_SQUARE) return square_rows(out, y0, y1, s);
  return FSR1_OK;
}

int upscale(const fsr1_image* in, const fsr1_image* tmp, const fsr1_image* out, const uint32_t easu_con[16], const uint32_t rcas_con[4],
            uint32_t y0, uint32_t y1, uint32_t flags, void* stream, const HaloSync* sync, bool* sync_taken) {
  NvtxRange range("FSR1 upscale");
  if (!out) return FSR1_ERR_INVALID_ARGUMENT;
  if (y1 == 0) y1 = out->height;
  const bool r11 = in && in->format == FSR1_FORMAT_R11G11B10_FLOAT;
  if (r11) {  // every image after EASU is RGBA16F; refused here so that no EASU launch precedes a refusal of the RCAS pass
    if (out->format != FSR1_FORMAT_RGBA16F || (tmp && !(flags & FSR1_FLAG_NO_RCAS) && tmp->format != FSR1_FORMAT_RGBA16F))
      return FSR1_ERR_UNSUPPORTED;
    if (flags & kR11Refused) return FSR1_ERR_UNSUPPORTED;
  }
  const bool array_in = (flags & kArrayIn) != 0, surf_out = (flags & FSR1_FLAG_OUT_SURFACE) != 0;
  int rc;
  if (array_in || surf_out) {  // every refusal of the arrays before anything launches
    if ((rc = check_io(in, array_in)) != FSR1_OK || (rc = check_io(out, surf_out)) != FSR1_OK) return rc;
    if (!easu_con || bad_flags(flags)) return FSR1_ERR_INVALID_ARGUMENT;
    if ((rc = array_rules(in, out, easu_con, flags, false)) != FSR1_OK) return rc;
  }
  if (flags & FSR1_FLAG_NO_RCAS) return easu(in, out, easu_con, y0, y1, flags, stream, sync, sync_taken);
  const Rows e = easu_rows(y0, y1, out->height);
  if ((flags & FSR1_FLAG_FUSED) && in && easu_con && rcas_con && (in->format == FSR1_FORMAT_RGBA16F || r11) &&
      out->format == FSR1_FORMAT_RGBA16F && !(flags & kNotFused)) {
    if ((rc = check_io(in, array_in)) != FSR1_OK || (rc = check_io(out, surf_out)) != FSR1_OK) return rc;
    if (bad_flags(flags)) return FSR1_ERR_INVALID_ARGUMENT;
    if (y0 >= y1 || y1 > out->height) return FSR1_ERR_INVALID_ARGUMENT;
    if (!window_holds(out, (int)y0, (int)y1 - 1)) return FSR1_ERR_WINDOW;
    uint32_t r0, r1;
    fsr1_easu_input_rows(easu_con, in->height, e.a, e.b, &r0, &r1);
    if (!window_holds(in, (int)r0, (int)r1)) return FSR1_ERR_WINDOW;
    if ((flags & FSR1_FLAG_SRTM_INPUT) && (rc = srtm_input_check(in, nullptr, easu_con, flags)) != FSR1_OK) return rc;
    const cudaError_t err = launch_fused(in, out, easu_con, rcas_con, nullptr, y0, y1, flags, stream, sync, sync_taken);
    if (err == cudaSuccess) return FSR1_OK;
    if (err != cudaErrorNotSupported) return cuda_fail(err);
  }
  flags &= ~(uint32_t)FSR1_FLAG_FUSED;
  if (!tmp) return FSR1_ERR_INVALID_ARGUMENT;
  if (surf_out && (((uintptr_t)tmp->data & 15) || (tmp->pitch_bytes & 15))) return FSR1_ERR_UNSUPPORTED;  // the packed RCAS kernel's loads
  // the output square and OUT_SURFACE belong to the last pass, SRTM_INPUT, IN_SURFACE and IN_TEXTURE to EASU's load stage
  rc = easu(in, tmp, easu_con, e.a, e.b, flags & ~(uint32_t)(FSR1_FLAG_OUTPUT_SQUARE | FSR1_FLAG_OUT_SURFACE), stream, sync, sync_taken);
  if (rc != FSR1_OK) return rc;
  return fsr1_rcas(tmp, out, rcas_con, y0, y1, flags & ~(uint32_t)(FSR1_FLAG_SRTM_INPUT | kArrayIn), stream);
}

int upscale_post(const fsr1_image* in, const fsr1_image* tmp, const fsr1_image* out, const uint32_t easu_con[16],
                 const uint32_t rcas_con[4], const fsr1_post* post, uint32_t y0, uint32_t y1, uint32_t flags, void* stream,
                 const HaloSync* sync, bool* sync_taken) {
  if (!post || post->ops == 0) return upscale(in, tmp, out, easu_con, rcas_con, y0, y1, flags, stream, sync, sync_taken);
  NvtxRange range("FSR1 upscale post");
  int rc;
  const bool array_in = (flags & kArrayIn) != 0, surf_out = (flags & FSR1_FLAG_OUT_SURFACE) != 0;
  if ((rc = check_io(in, array_in)) != FSR1_OK || (rc = check_io(out, surf_out)) != FSR1_OK) return rc;
  if (!easu_con || !rcas_con) return FSR1_ERR_INVALID_ARGUMENT;
  PostParams q;
  if ((rc = post_params(post, in->format, out->format, flags, q)) != FSR1_OK) return rc;
  if ((flags & FSR1_FLAG_SRTM_INPUT) && (rc = srtm_input_check(in, nullptr, easu_con, flags)) != FSR1_OK) return rc;
  if (y1 == 0) y1 = out->height;
  if (y0 >= y1 || y1 > out->height) return FSR1_ERR_INVALID_ARGUMENT;
  if (!window_holds(out, (int)y0, (int)y1 - 1)) return FSR1_ERR_WINDOW;
  const Rows e = easu_rows(y0, y1, out->height);
  uint32_t r0, r1;
  fsr1_easu_input_rows(easu_con, in->height, e.a, e.b, &r0, &r1);
  if (!window_holds(in, (int)r0, (int)r1)) return FSR1_ERR_WINDOW;
  const int out_align = out->format == FSR1_FORMAT_RGBA16F ? 16 : 8;
  if (!surf_out && (((uintptr_t)out->data & (out_align - 1)) || (out->pitch_bytes & (out_align - 1)))) return FSR1_ERR_UNSUPPORTED;
  if (tmp) {  // the intermediate of the two-kernel path (unused by the fused kernel)
    if ((rc = check_image(tmp)) != FSR1_OK) return rc;
    if (tmp->format != FSR1_FORMAT_RGBA16F) return FSR1_ERR_UNSUPPORTED;
    if (tmp->width != out->width || tmp->height != out->height) return FSR1_ERR_INVALID_ARGUMENT;
    if (!window_holds(tmp, (int)e.a, (int)e.b - 1)) return FSR1_ERR_WINDOW;
    if (((uintptr_t)tmp->data & 15) || (tmp->pitch_bytes & 15)) return FSR1_ERR_UNSUPPORTED;
    if (!surf_out && overlaps(tmp, out)) return FSR1_ERR_INVALID_ARGUMENT;
  }
  if ((array_in || surf_out) && (rc = array_rules(in, out, easu_con, flags, true)) != FSR1_OK) return rc;
  if ((flags & FSR1_FLAG_FUSED) && !(flags & kNotFused)) {
    const cudaError_t err = launch_fused(in, out, easu_con, rcas_con, &q, y0, y1, flags, stream, sync, sync_taken);
    if (err == cudaSuccess) return FSR1_OK;
    if (err != cudaErrorNotSupported) return cuda_fail(err);
  }
  // EASU into tmp (as fsr1_upscale does), then RCAS with the epilogue in its store
  if (!tmp) return FSR1_ERR_INVALID_ARGUMENT;
  rc = easu(in, tmp, easu_con, e.a, e.b, flags & ~(uint32_t)(FSR1_FLAG_FUSED | FSR1_FLAG_OUTPUT_SQUARE | FSR1_FLAG_OUT_SURFACE), stream, sync,
            sync_taken);
  if (rc != FSR1_OK) return rc;
  RcasParams p = rcas_params(tmp, out, rcas_con, y0, y1, flags);
  p.options |= (flags & FSR1_FLAG_OUTPUT_SQUARE) ? 4 : 0;
  const char* name = "";
  const cudaError_t err = launch_rcas_h_post(p, q, (int)out->format, static_cast<cudaStream_t>(stream), &name, surf_out);
  if (err != cudaSuccess) return err == cudaErrorNotSupported ? FSR1_ERR_UNSUPPORTED : cuda_fail(err);
  launched(name);
  return FSR1_OK;
}

int post_rules(const fsr1_post* post, uint32_t in_format, uint32_t out_format, uint32_t flags) {
  if (!post) return FSR1_ERR_INVALID_ARGUMENT;
  PostParams q;
  return post_params(post, in_format, out_format, flags, q);
}

}  // namespace fsr1

extern "C" {

int fsr1_abi_version(void) { return FSR1_ABI_VERSION; }

const char* fsr1_error_string(int err) {
  switch (err) {
    case FSR1_OK: return "ok";
    case FSR1_ERR_INVALID_ARGUMENT: return "invalid argument";
    case FSR1_ERR_UNSUPPORTED: return "unsupported format combination";
    case FSR1_ERR_WINDOW: return "image window does not hold the rows this pass touches";
    case FSR1_ERR_CUDA: return "CUDA error (see fsr1_last_cuda_error)";
    case FSR1_ERR_NO_DEVICE: return "no usable CUDA device";
    case FSR1_ERR_TIMEOUT: return "a neighbouring rank's halo rows or credit did not arrive in time";
    default: return "unknown fsr1 error";
  }
}
int fsr1_last_cuda_error(void) { return t_last_cuda; }
uint64_t fsr1_launch_count(void) { return g_launches.load(); }
const char* fsr1_last_kernel_name(void) { return t_last_kernel; }

void fsr1_easu_con(uint32_t con[16], float vw, float vh, float sw, float sh, float ow, float oh) {
  FsrEasuCon(con, con + 4, con + 8, con + 12, vw, vh, sw, sh, ow, oh);
}
void fsr1_easu_con_offset(uint32_t con[16], float vw, float vh, float sw, float sh, float ow, float oh, float ox,
                          float oy) {
  FsrEasuConOffset(con, con + 4, con + 8, con + 12, vw, vh, sw, sh, ow, oh, ox, oy);
}
void fsr1_rcas_con(uint32_t con[4], float sharpness_stops) { FsrRcasCon(con, sharpness_stops); }

int fsr1_easu_input_rows(const uint32_t con[16], uint32_t in_height, uint32_t y0, uint32_t y1, uint32_t* first_row,
                         uint32_t* last_row) {
  if (!con || !first_row || !last_row || in_height == 0 || y1 <= y0) return FSR1_ERR_INVALID_ARGUMENT;
  const float sy = word_as_float(con[1]), oy = word_as_float(con[3]);
  int lo = host_cell(y0, sy, oy) - 1, hi = host_cell(y1 - 1, sy, oy) + 2;
  const int H = (int)in_height;
  lo = lo < 0 ? 0 : (lo > H - 1 ? H - 1 : lo);
  hi = hi < 0 ? 0 : (hi > H - 1 ? H - 1 : hi);
  *first_row = (uint32_t)lo;
  *last_row = (uint32_t)hi;
  return FSR1_OK;
}

int fsr1_easu(const fsr1_image* in, const fsr1_image* out, const uint32_t con[16], uint32_t y0, uint32_t y1,
              uint32_t flags, void* stream) {
  return easu(in, out, con, y0, y1, flags, stream, nullptr, nullptr);
}

int fsr1_rcas(const fsr1_image* in, const fsr1_image* out, const uint32_t con[4], uint32_t y0, uint32_t y1,
              uint32_t flags, void* stream) {
  NvtxRange range("RCAS");
  int rc;
  const bool surf_out = (flags & FSR1_FLAG_OUT_SURFACE) != 0;
  if ((rc = check_image(in)) != FSR1_OK || (rc = check_io(out, surf_out)) != FSR1_OK) return rc;
  if (!con || bad_flags(flags)) return FSR1_ERR_INVALID_ARGUMENT;
  if (flags & FSR1_FLAG_SRTM_INPUT) return FSR1_ERR_INVALID_ARGUMENT;  // RCAS has no input stage
  if (flags & kArrayIn) return FSR1_ERR_UNSUPPORTED;                   // RCAS reads the linear intermediate
  if (surf_out && ((flags & kSurfRefused) || out->format != FSR1_FORMAT_RGBA16F)) return FSR1_ERR_UNSUPPORTED;
  if (in->format != out->format || in->format == FSR1_FORMAT_R11G11B10_FLOAT) return FSR1_ERR_UNSUPPORTED;
  if ((rc = rcas_images(in, out, y0, y1, surf_out)) != FSR1_OK) return rc;

  RcasParams p = rcas_params(in, out, con, y0, y1, flags);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const bool exact = (flags & FSR1_FLAG_EXACT) != 0;
  cudaError_t e = cudaErrorNotSupported;
  const char* name = "";
  bool squared = false;  // the Sample.x hook folded into the kernel's store (c *= c before the one rounding)
  const int fused_square = (flags & FSR1_FLAG_OUTPUT_SQUARE) ? 4 : 0;
  if (flags & FSR1_FLAG_RCAS_HX2) {  // the packed calling convention: FsrRcasHx2 + FsrRcasDepackHx2
    if (in->format != FSR1_FORMAT_RGBA16F || exact) return FSR1_ERR_UNSUPPORTED;
    e = launch_rcas_hx2(p, s, &name);
  } else if (flags & FSR1_FLAG_H_REFERENCE) {
    if (in->format != FSR1_FORMAT_RGBA16F || exact) return FSR1_ERR_UNSUPPORTED;
    e = launch_rcas_href(p, s, &name);
  } else if (in->format == FSR1_FORMAT_RGBA16F && !exact && !(flags & FSR1_FLAG_FORCE_DIRECT)) {
    p.options |= fused_square;  // the reference's options are template bits of the packed kernels: no slower fallback
    e = launch_rcas_h_packed(p, s, &name, surf_out);
    squared = e == cudaSuccess;
    if (e == cudaErrorNotSupported && surf_out) return FSR1_ERR_UNSUPPORTED;  // nothing launched; no other kernel writes a surface
  } else if (in->format == FSR1_FORMAT_RGBA32F && !exact && !(flags & FSR1_FLAG_FORCE_DIRECT)) {
    p.options |= fused_square;
    e = launch_rcas_f32_packed(p, s, &name);
    squared = e == cudaSuccess;
  } else if ((in->format == FSR1_FORMAT_RGBA8_UNORM || in->format == FSR1_FORMAT_RGB10A2_UNORM) && !exact &&
             !(flags & (FSR1_FLAG_FORCE_DIRECT | FSR1_FLAG_PRECISE))) {
    p.options |= fused_square;
    e = launch_rcas_u_packed(p, (int)in->format, s, &name);
    squared = e == cudaSuccess;
  }
  if (e == cudaErrorNotSupported) p.options &= 3;
  if (e == cudaErrorNotSupported) e = launch_rcas_direct(p, (int)in->format, exact, s, &name);
  if (e != cudaSuccess) return cuda_fail(e);
  launched(name);
  if ((flags & FSR1_FLAG_OUTPUT_SQUARE) && !squared) return square_rows(out, y0, y1, s);  // direct / H-reference kernels: separate pass
  return FSR1_OK;
}

int fsr1_upscale(const fsr1_image* in, const fsr1_image* tmp, const fsr1_image* out, const uint32_t easu_con[16],
                 const uint32_t rcas_con[4], uint32_t y0, uint32_t y1, uint32_t flags, void* stream) {
  return upscale(in, tmp, out, easu_con, rcas_con, y0, y1, flags, stream, nullptr, nullptr);
}

int fsr1_upscale_post(const fsr1_image* in, const fsr1_image* tmp, const fsr1_image* out, const uint32_t easu_con[16],
                      const uint32_t rcas_con[4], const fsr1_post* post, uint32_t y0, uint32_t y1, uint32_t flags, void* stream) {
  return upscale_post(in, tmp, out, easu_con, rcas_con, post, y0, y1, flags, stream, nullptr, nullptr);
}

// A frame rendered at display size: one RCAS kernel with the input stage (R11G11B10F decode, FsrSrtmF) and the display epilogue.
// RGBA16F input without SRTM_INPUT runs the kernels of fsr1_rcas (no ops) and of fsr1_upscale_post's RCAS pass.
int fsr1_rcas_post(const fsr1_image* in, const fsr1_image* out, const uint32_t rcas_con[4], const fsr1_post* post, uint32_t y0, uint32_t y1,
                   uint32_t flags, void* stream) {
  NvtxRange range("RCAS post");
  // the other arithmetic paths, EASU-only frames and input surfaces: only the packed RGBA16F kernel has the input stage
  constexpr uint32_t kRefused = FSR1_FLAG_EXACT | FSR1_FLAG_FORCE_DIRECT | FSR1_FLAG_H_REFERENCE | FSR1_FLAG_PRECISE | FSR1_FLAG_RCAS_HX2 |
                                FSR1_FLAG_NO_RCAS | kArrayIn;
  int rc;
  const bool surf_out = (flags & FSR1_FLAG_OUT_SURFACE) != 0;
  if ((rc = check_image(in)) != FSR1_OK || (rc = check_io(out, surf_out)) != FSR1_OK) return rc;
  if (!rcas_con || bad_flags(flags)) return FSR1_ERR_INVALID_ARGUMENT;
  if (flags & kRefused) return FSR1_ERR_UNSUPPORTED;
  if (in->format != FSR1_FORMAT_RGBA16F && in->format != FSR1_FORMAT_R11G11B10_FLOAT) return FSR1_ERR_UNSUPPORTED;
  const bool ops = post && post->ops;
  PostParams q;
  if (ops && (rc = post_params(post, in->format, out->format, flags, q)) != FSR1_OK) return rc;
  if (!ops && out->format != FSR1_FORMAT_RGBA16F) return FSR1_ERR_UNSUPPORTED;
  const bool r11 = in->format == FSR1_FORMAT_R11G11B10_FLOAT, srtm = (flags & FSR1_FLAG_SRTM_INPUT) != 0;
  const uint64_t in_align = r11 ? 8 : 16, out_align = out->format == FSR1_FORMAT_RGBA16F ? 16 : 8;  // one vector access per pixel pair
  if (((uintptr_t)in->data & (in_align - 1)) || (in->pitch_bytes & (in_align - 1))) return FSR1_ERR_UNSUPPORTED;
  if (!surf_out && (((uintptr_t)out->data & (out_align - 1)) || (out->pitch_bytes & (out_align - 1)))) return FSR1_ERR_UNSUPPORTED;
  if ((rc = rcas_images(in, out, y0, y1, surf_out)) != FSR1_OK) return rc;

  RcasParams p = rcas_params(in, out, rcas_con, y0, y1, flags);
  p.options |= (flags & FSR1_FLAG_OUTPUT_SQUARE) ? 4 : 0;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const char* name = "";
  cudaError_t e;
  if (r11 || srtm) e = launch_rcas_h_in(p, ops ? &q : nullptr, (int)out->format, r11, srtm, s, &name, surf_out);
  else if (ops) e = launch_rcas_h_post(p, q, (int)out->format, s, &name, surf_out);
  else e = launch_rcas_h_packed(p, s, &name, surf_out);
  if (e != cudaSuccess) return e == cudaErrorNotSupported ? FSR1_ERR_UNSUPPORTED : cuda_fail(e);
  launched(name);
  return FSR1_OK;
}

// ---- pointwise companions ------------------------------------------------------------------------------
int fsr1_srtm(const fsr1_image* in, const fsr1_image* out, int inverse, uint32_t y0, uint32_t y1, void* stream) {
  return pointwise(inverse ? 2 : 1, false, in, nullptr, out, 0.0f, 0u, y0, y1, stream);
}

int fsr1_lfga(const fsr1_image* in, const fsr1_image* grain, const fsr1_image* out, float amount, uint32_t y0,
              uint32_t y1, void* stream) {
  if (!grain) return FSR1_ERR_INVALID_ARGUMENT;
  if (grain->format != FSR1_FORMAT_RGBA16F && grain->format != FSR1_FORMAT_RGBA32F) return FSR1_ERR_UNSUPPORTED;  // signed values
  return pointwise(3, false, in, grain, out, amount, 0u, y0, y1, stream);
}

int fsr1_tepd(const fsr1_image* in, const fsr1_image* dither, const fsr1_image* out, int bits, uint32_t frame,
              uint32_t y0, uint32_t y1, void* stream) {
  if (bits != 8 && bits != 10) return FSR1_ERR_INVALID_ARGUMENT;
  return pointwise(bits == 8 ? 4 : 5, false, in, dither, out, 0.0f, frame, y0, y1, stream);
}

int fsr1_srtm_h(const fsr1_image* in, const fsr1_image* out, int inverse, uint32_t y0, uint32_t y1, void* stream) {
  return pointwise(inverse ? 2 : 1, true, in, nullptr, out, 0.0f, 0u, y0, y1, stream);
}

int fsr1_lfga_h(const fsr1_image* in, const fsr1_image* grain, const fsr1_image* out, float amount, uint32_t y0, uint32_t y1,
                void* stream) {
  if (!grain) return FSR1_ERR_INVALID_ARGUMENT;
  return pointwise(3, true, in, grain, out, amount, 0u, y0, y1, stream);
}

int fsr1_tepd_h(const fsr1_image* in, const fsr1_image* dither, const fsr1_image* out, int bits, uint32_t frame, uint32_t y0,
                uint32_t y1, void* stream) {
  if (bits != 8 && bits != 10) return FSR1_ERR_INVALID_ARGUMENT;
  return pointwise(bits == 8 ? 4 : 5, true, in, dither, out, 0.0f, frame, y0, y1, stream);
}

// ---- context --------------------------------------------------------------------------------------
struct fsr1_context {
  uint32_t in_w, in_h, out_w, out_h, format;
  void* tmp;          // intermediate, out_w x out_h
  uint64_t tmp_pitch;
  void* dev_in;       // staging for the host-frame entry point (allocated on first use)
  void* dev_out;
  uint64_t in_pitch, out_pitch;
};

int fsr1_context_create(fsr1_context** ctx, uint32_t in_w, uint32_t in_h, uint32_t out_w, uint32_t out_h,
                        uint32_t format) {
  if (!ctx || !in_w || !in_h || !out_w || !out_h || !bytes_per_pixel(format)) return FSR1_ERR_INVALID_ARGUMENT;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return FSR1_ERR_NO_DEVICE;
  fsr1_context* c = new (std::nothrow) fsr1_context();
  if (!c) return FSR1_ERR_INVALID_ARGUMENT;
  memset(c, 0, sizeof *c);
  c->in_w = in_w; c->in_h = in_h; c->out_w = out_w; c->out_h = out_h; c->format = format;
  const uint64_t bpp = (uint64_t)bytes_per_pixel(easu_out_format(format));  // the intermediate
  c->tmp_pitch = ((uint64_t)out_w * bpp + 127) & ~(uint64_t)127;
  cudaError_t e = cudaMalloc(&c->tmp, c->tmp_pitch * out_h);
  if (e != cudaSuccess) { delete c; return cuda_fail(e); }
  *ctx = c;
  return FSR1_OK;
}

void fsr1_context_destroy(fsr1_context* c) {
  if (!c) return;
  cudaFree(c->tmp);
  cudaFree(c->dev_in);
  cudaFree(c->dev_out);
  delete c;
}

// One frame of the context: the caller's input is render_w x render_h (the top-left of the resource), the output follows the post
// ops: with TEPD the matching UNORM code values (the display image), otherwise EASU's output format.  The constants are exactly what
// FSR_Filter::Upscale passes (sample/src/DX12/FSR_Filter.cpp:106,124).  The context owns the intermediate, so a frame the fused
// kernel covers takes it; other render sizes, formats and options fall back to EASU + RCAS through c->tmp.
static int context_run(fsr1_context* c, void* in_dev, uint64_t in_pitch, uint32_t render_w, uint32_t render_h, void* out_dev,
                       uint64_t out_pitch, float sharpness, const fsr1_post* post, uint32_t flags, void* stream) {
  const uint32_t ops = post ? post->ops : 0u;
  uint32_t ofmt = easu_out_format(c->format);
  if ((ops & FSR1_POST_TEPD10) && !(ops & FSR1_POST_TEPD8)) ofmt = FSR1_FORMAT_RGB10A2_UNORM;
  if ((ops & FSR1_POST_TEPD8) && !(ops & FSR1_POST_TEPD10)) ofmt = FSR1_FORMAT_RGBA8_UNORM;
  fsr1_image in = {in_dev, in_pitch, render_w, render_h, 0, render_h, c->format, 0};
  fsr1_image tmp = {c->tmp, c->tmp_pitch, c->out_w, c->out_h, 0, c->out_h, easu_out_format(c->format), 0};
  fsr1_image out = {out_dev, out_pitch, c->out_w, c->out_h, 0, c->out_h, ofmt, 0};
  uint32_t econ[16], rcon[4];
  fsr1_easu_con(econ, (float)render_w, (float)render_h, (float)render_w, (float)render_h, (float)c->out_w, (float)c->out_h);
  fsr1_rcas_con(rcon, sharpness);
  return fsr1_upscale_post(&in, &tmp, &out, econ, rcon, post, 0, c->out_h, flags | FSR1_FLAG_FUSED, stream);
}

int fsr1_context_upscale_render(fsr1_context* c, const void* in_dev, uint64_t in_pitch, uint32_t render_w, uint32_t render_h,
                                void* out_dev, uint64_t out_pitch, float sharpness, uint32_t flags, void* stream) {
  if (!c || !in_dev || !out_dev || !render_w || !render_h) return FSR1_ERR_INVALID_ARGUMENT;
  if (render_w > c->in_w || render_h > c->in_h) return FSR1_ERR_INVALID_ARGUMENT;  // would read past the caller's input
  return context_run(c, const_cast<void*>(in_dev), in_pitch, render_w, render_h, out_dev, out_pitch, sharpness, nullptr, flags, stream);
}

int fsr1_context_upscale_post(fsr1_context* c, const void* in_dev, uint64_t in_pitch, uint32_t render_w, uint32_t render_h,
                              void* out_dev, uint64_t out_pitch, float sharpness, const fsr1_post* post, uint32_t flags, void* stream) {
  if (!c || !in_dev || !out_dev) return FSR1_ERR_INVALID_ARGUMENT;
  if (c->format != FSR1_FORMAT_RGBA16F && c->format != FSR1_FORMAT_R11G11B10_FLOAT) return FSR1_ERR_UNSUPPORTED;
  if (render_w == 0) render_w = c->in_w;
  if (render_h == 0) render_h = c->in_h;
  if (render_w > c->in_w || render_h > c->in_h) return FSR1_ERR_INVALID_ARGUMENT;  // would read past the caller's input
  return context_run(c, const_cast<void*>(in_dev), in_pitch, render_w, render_h, out_dev, out_pitch, sharpness, post, flags, stream);
}

int fsr1_context_upscale(fsr1_context* c, const void* in_dev, uint64_t in_pitch, void* out_dev, uint64_t out_pitch,
                         float sharpness, uint32_t flags, void* stream) {
  if (!c || !in_dev || !out_dev) return FSR1_ERR_INVALID_ARGUMENT;
  return context_run(c, const_cast<void*>(in_dev), in_pitch, c->in_w, c->in_h, out_dev, out_pitch, sharpness, nullptr, flags, stream);
}

int fsr1_context_upscale_host(fsr1_context* c, const void* in_host, uint64_t in_pitch, void* out_host,
                              uint64_t out_pitch, float sharpness, uint32_t flags, void* stream) {
  if (!c || !in_host || !out_host) return FSR1_ERR_INVALID_ARGUMENT;
  if (flags & kArrayFlags) return FSR1_ERR_UNSUPPORTED;  // its frames are host memory, staged through the context's linear buffers
  const uint64_t bpp = (uint64_t)bytes_per_pixel(c->format), obpp = (uint64_t)bytes_per_pixel(easu_out_format(c->format));
  if (in_pitch < c->in_w * bpp || out_pitch < c->out_w * obpp) return FSR1_ERR_INVALID_ARGUMENT;
  cudaError_t e;
  if (!c->dev_in || !c->dev_out) {  // both or neither: a failed second allocation leaves nothing half-initialised
    c->in_pitch = ((uint64_t)c->in_w * bpp + 127) & ~(uint64_t)127;
    c->out_pitch = ((uint64_t)c->out_w * obpp + 127) & ~(uint64_t)127;
    void *din = nullptr, *dout = nullptr;
    if ((e = cudaMalloc(&din, c->in_pitch * c->in_h)) != cudaSuccess) return cuda_fail(e);
    if ((e = cudaMalloc(&dout, c->out_pitch * c->out_h)) != cudaSuccess) { cudaFree(din); return cuda_fail(e); }
    c->dev_in = din;
    c->dev_out = dout;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  e = cudaMemcpy2DAsync(c->dev_in, c->in_pitch, in_host, in_pitch, c->in_w * bpp, c->in_h, cudaMemcpyHostToDevice, s);
  if (e != cudaSuccess) return cuda_fail(e);
  int rc = context_run(c, c->dev_in, c->in_pitch, c->in_w, c->in_h, c->dev_out, c->out_pitch, sharpness, nullptr, flags, stream);
  if (rc != FSR1_OK) return rc;
  e = cudaMemcpy2DAsync(out_host, out_pitch, c->dev_out, c->out_pitch, c->out_w * obpp, c->out_h, cudaMemcpyDeviceToHost, s);
  if (e != cudaSuccess) return cuda_fail(e);
  return FSR1_OK;
}

}  // extern "C"
