/* fsr1_b200.h — C ABI of the H100-native (sm_90a) FSR 1.0 hot path (EASU upsample + RCAS sharpen).
 *
 * Plain C, plain pointers and sizes; no CUDA or torch types appear in any signature (a stream is
 * passed as void* = cudaStream_t, NULL = the legacy default stream).  This is what a binding in
 * the reference's host code (or any FFI: ctypes, cgo, JNI ...) attaches to; see INTEGRATION.md.
 *
 * What each entry point replaces in the reference (GPUOpen-Effects/FidelityFX-FSR):
 *   fsr1_easu      the EASU dispatch: shader FsrEasuF/FsrEasuH (ffx-fsr/ffx_fsr1.h:315-437, 505-593)
 *                  entered from mainCS/CurrFilter (sample/src/DX12/FSR_Pass.hlsl:68-118), recorded by
 *                  FSR_Filter::Upscale -> m_easu.Draw (sample/src/DX12/FSR_Filter.cpp:121,135)
 *   fsr1_rcas      the RCAS dispatch: FsrRcasF/FsrRcasH (ffx-fsr/ffx_fsr1.h:684-769, 782-866),
 *                  m_rcas.Draw (sample/src/DX12/FSR_Filter.cpp:131)
 *   fsr1_upscale   the whole of FSR_Filter::Upscale (sample/src/DX12/FSR_Filter.cpp:101-141):
 *                  EASU -> (barrier) -> RCAS through a display-sized intermediate
 *   fsr1_context_* FSR_Filter::OnCreateWindowSizeDependentResources / OnDestroy... (FSR_Filter.cpp:70-99):
 *                  owns the intermediate image (and, for the *_host call, device staging buffers)
 *   fsr1_upscale_host  same as fsr1_upscale for callers whose frames live in HOST memory: copies the
 *                  input up, runs both passes, copies the result back, all on one stream
 * The constant blocks (con0..con3, rcas con) are EXACTLY the uint32[4] words FsrEasuCon /
 * FsrEasuConOffset / FsrRcasCon produce (include/fsr1_host.h, or the reference's own header).
 *
 * Semantics fixed by the reference and reproduced here:
 *   - images are row-major RGBA, 4 x fp16 (FSR1_FORMAT_RGBA16F, the reference's rgba16f path) or
 *     4 x fp32 (FSR1_FORMAT_RGBA32F, the SAMPLE_SLOW_FALLBACK path); EASU/RCAS read RGB, ignore A,
 *     and store A = 1 (FSR_Pass.hlsl:80,95)
 *   - EASU taps are clamped to the edge of the input RESOURCE (linear/clamp sampler, FSR_Filter.cpp:48-53)
 *   - RCAS taps outside the image read 0 (D3D12 Load); FSR1_FLAG_RCAS_CLAMP selects clamp instead
 *   - fp32 images run the F algorithm in fp32; fp16 images run a packed-half implementation whose
 *     results stay within 1e-2 of the fp32 algorithm on the same (quantised) input; UNORM images (the
 *     formats the sample renders into, FSR_Filter.cpp:72-73) run the F algorithm in fp32 on the D3D
 *     unorm<->float conversions (c/(2^n-1); clamp, scale, +0.5, truncate)
 * All launch calls are asynchronous with respect to the host and allocate nothing
 * (fsr1_context_create and fsr1_upscale_host's first use are the only allocating calls).
 * Thread-safe for distinct contexts/streams.  Every function returns FSR1_OK or a negative fsr1 error;
 * CUDA failures are reported as FSR1_ERR_CUDA and the CUDA error is kept for fsr1_last_cuda_error().
 */
#ifndef FSR1_B200_H
#define FSR1_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FSR1_ABI_VERSION 3  /* additions that leave existing callers untouched keep the number: FSR1_FLAG_RCAS_HX2, fsr1_srtm_h / fsr1_lfga_h / fsr1_tepd_h, fsr1_upscale_post, FSR1_FLAG_SRTM_INPUT, FSR1_SHARD_DYNAMIC / fsr1_shard_frame, fsr1_shard_create_post / fsr1_shard_post, FSR1_FORMAT_R11G11B10_FLOAT, FSR1_FLAG_IN_SURFACE / FSR1_FLAG_OUT_SURFACE, fsr1_rcas_post, FSR1_FLAG_IN_TEXTURE */

enum {
  FSR1_OK = 0,
  FSR1_ERR_INVALID_ARGUMENT = -1, /* null pointer, zero size, bad row range, unknown format/flag   */
  FSR1_ERR_UNSUPPORTED = -2,      /* format combination the kernels do not implement              */
  FSR1_ERR_WINDOW = -3,           /* an image window (row0/rows) does not hold the rows the pass reads/writes */
  FSR1_ERR_CUDA = -4,             /* a CUDA call failed; see fsr1_last_cuda_error()                */
  FSR1_ERR_NO_DEVICE = -5,        /* no usable sm_90 device / driver                               */
  FSR1_ERR_TIMEOUT = -6           /* fsr1_shard_*: a neighbour's halo or credit did not arrive in time */
};

enum {
  FSR1_FORMAT_RGBA16F = 1,
  FSR1_FORMAT_RGBA32F = 2,
  FSR1_FORMAT_RGBA8_UNORM = 3,    /* 4 B/px, byte order R,G,B,A (DXGI_FORMAT_R8G8B8A8_UNORM)                      */
  FSR1_FORMAT_RGB10A2_UNORM = 4,  /* 4 B/px, bits 0-9 R, 10-19 G, 20-29 B, 30-31 A (DXGI_FORMAT_R10G10B10A2_UNORM) */
  FSR1_FORMAT_R11G11B10_FLOAT = 5 /* 4 B/px, unsigned floats (DXGI_FORMAT_R11G11B10_FLOAT): bits 0-10 R and 11-21 G, each 6 mantissa
                                     bits below 5 exponent bits; bits 22-31 B, 5 mantissa bits below 5 exponent bits; exponent bias 15,
                                     no alpha.  An INPUT format only: every channel is a half without its sign and low mantissa bits,
                                     so the kernels decode each texel exactly to the RGBA16F texel (R, G, B, 1.0) as they load it
                                     (denormals, inf and NaN included), and every call is bit-identical to the same call on that RGBA16F
                                     image of the decoded values.  Where it is the input, EASU's output, the intermediate and the output
                                     are RGBA16F (with fsr1_upscale_post's TEPD, the UNORM format TEPD implies).  fsr1_easu,
                                     fsr1_upscale*, fsr1_context_* and fsr1_shard_* take it, on the RGBA16F kernels (tiled, fused, post,
                                     with FSR1_FLAG_SRTM_INPUT too) and, for the layouts, scales and FSR1_FLAG_FORCE_DIRECT those decline,
                                     the fp32 direct kernel.  FSR1_ERR_UNSUPPORTED, before any CUDA call: as any output, as RCAS input,
                                     as an image or tile of the pointwise passes, and combined with FSR1_FLAG_EXACT / H_REFERENCE /
                                     PRECISE / RCAS_HX2. */
};

enum {
  FSR1_FLAG_RCAS_CLAMP = 1u << 0,   /* RCAS out-of-image taps clamp instead of reading 0               */
  FSR1_FLAG_EXACT = 1u << 1,        /* fp32 images only: no FMA contraction, IEEE division — bit-identical
                                       to the reference source compiled with -ffp-contract=off          */
  FSR1_FLAG_FORCE_DIRECT = 1u << 2, /* skip the TMA/shared-memory kernels, use the direct-load kernels   */
  FSR1_FLAG_NO_RCAS = 1u << 3,      /* fsr1_upscale*: EASU straight to the output (bUseRcas == false)   */
  FSR1_FLAG_PRECISE = 1u << 5,      /* fp16 images: fp32 arithmetic on fp16 storage where a tiled kernel exists for it
                                       (EASU at exactly 2x: fp32 tap weights) ; ~10x closer to the fp32 algorithm */
  FSR1_FLAG_RCAS_DENOISE = 1u << 6, /* the reference's FSR_RCAS_DENOISE compile-time option (ffx_fsr1.h:651,731-763)      */
  FSR1_FLAG_RCAS_PASSTHROUGH_ALPHA = 1u << 7, /* FSR_RCAS_PASSTHROUGH_ALPHA (:648,688-702): output alpha = input alpha */
  FSR1_FLAG_OUTPUT_SQUARE = 1u << 8, /* the sample's Sample.x hook (sample/src/DX12/FSR_Pass.hlsl:78-79,93-94): `c *= c` on the
                                       output of the LAST pass (gamma 2.0, as produced by TEPD, back to linear)      */
  FSR1_FLAG_FUSED = 1u << 9,        /* fsr1_upscale*: EASU and RCAS in ONE kernel where one exists (RGBA16F, exactly 2x, out-of-image
                                       RCAS taps read 0, no RCAS options): the intermediate stays in shared memory, `tmp` is not
                                       touched, HBM traffic drops from 26 to 10 bytes per output pixel; results are bit-identical
                                       to the two-kernel path.  Falls back to the two kernels otherwise.  fsr1_shard_* and
                                       fsr1_context_* own their intermediate and take the fused kernel automatically; the flag
                                       only matters for fsr1_upscale, whose caller passes `tmp`. */
  FSR1_FLAG_RCAS_HX2 = 1u << 10,    /* fsr1_rcas, fp16 images only: the reference's PACKED calling convention FsrRcasHx2 +
                                       FsrRcasDepackHx2 (ffx_fsr1.h:880-984): each lane sharpens pixels ip and ip + (8,0) held as
                                       half2 structure-of-arrays registers, every operation a packed half operation with its own
                                       rounding.  Bit-identical to FSR1_FLAG_H_REFERENCE (the reference's Hx2 and H sources agree
                                       bit for bit); honours RCAS_CLAMP, RCAS_DENOISE, RCAS_PASSTHROUGH_ALPHA.  A parity path. */
  FSR1_FLAG_SRTM_INPUT = 1u << 11,  /* the input holds LINEAR HDR values: EASU reads FsrSrtmF(texel) (ffx_fsr1.h:1030-1046, the tonemap
                                       before the filter) for every input texel, applied as the kernel loads it, so the caller's input is
                                       never written and no extra pass runs.  On rows [y0, y1) the result is bit-identical to the
                                       flag-free call on the RGBA16F image I = fsr1_srtm(in, I, 0, ...) over the same window (each texel:
                                       half -> fp32 FsrSrtmF -> rounded once to half; EASU's luma comes from that half texel).  Undo it
                                       after RCAS with fsr1_upscale_post's FSR1_POST_SRTM_INVERSE: the full HDR round trip.
                                       fsr1_easu, fsr1_upscale*, fsr1_context_* and fsr1_shard_* take it (RCAS never sees it; the shard's
                                       halo carries raw input rows and fsr1_easu_input_rows is unchanged: SRTM is pointwise).  RGBA16F
                                       (or R11G11B10_FLOAT, decoded first) input on the TMA-tiled kernels only: FSR1_ERR_UNSUPPORTED, with nothing launched, for another input
                                       format, EXACT / FORCE_DIRECT / H_REFERENCE / PRECISE, an input (or EASU output) whose base or pitch
                                       is not 16-byte aligned, or constants that do not upscale (0 < con0.x, con0.y <= 1).
                                       fsr1_rcas: FSR1_ERR_INVALID_ARGUMENT. */
  FSR1_FLAG_IN_SURFACE = 1u << 12,  /* `in` is a CUDA surface object on a 2D CUDA array (EASU's load stage); see "surface images" */
  FSR1_FLAG_OUT_SURFACE = 1u << 13, /* `out` is a CUDA surface object on a 2D CUDA array (the store of the pass that writes `out`) */
  FSR1_FLAG_IN_TEXTURE = 1u << 14,  /* `in` is a CUDA texture object on a 2D CUDA array (EASU's load stage); see "texture images" */
  FSR1_FLAG_H_REFERENCE = 1u << 4  /* fp16 images only: the literal FsrEasuH / FsrRcasH arithmetic (packed-half
                                       algorithm, half magic numbers, per-operation half rounding), bit-identical
                                       to the reference's H source; a parity path, slower and LESS accurate than
                                       the default fp16 kernels (see DESIGN.md "numerics")                  */
};

/* A (window of a) device image.  `width`/`height` are the logical size of the whole image; `data`
 * points at logical row `row0` and holds `rows` rows (row0 = 0, rows = height for a whole image).
 * Windows exist for row-slab sharding: a GPU holds only the rows it needs (plus halo) but clamping and
 * out-of-image rules still refer to the whole image.  pitch_bytes >= width * bytes-per-pixel. */
typedef struct fsr1_image {
  void* data;
  uint64_t pitch_bytes;
  uint32_t width, height;
  uint32_t row0, rows;
  uint32_t format;
  uint32_t reserved;
} fsr1_image;

/* Surface images (FSR1_FLAG_IN_SURFACE, FSR1_FLAG_OUT_SURFACE): the render target and the display image of an engine, imported through
 * CUDA interop as CUDA arrays (cudaImportExternalMemory -> cudaExternalMemoryGetMappedMipmappedArray -> level 0), read and written in
 * place instead of through linear copies.  `data` holds the cudaSurfaceObject_t (cast to a pointer), pitch_bytes is 0, row0 = 0 and
 * rows = height: a surface image is never a window.  width x height is its logical size, the TOP-LEFT region of the array, which may be
 * larger; EASU clamps its taps at the logical edge and no kernel touches the array outside [0, width) x [0, height) (the surfaces are
 * accessed in zero / ignore mode, never trap).  The array must be 2D (not layered, not 3D), created with surface load/store
 * (cudaArraySurfaceLoadStore), with an element of the format's size: 8 bytes for RGBA16F, 4 for RGBA8_UNORM and RGB10A2_UNORM.  The
 * bytes stored are exactly those the call stores into a linear image, and every result is bit-identical to the same call on linear
 * images holding the same pixels; the channel description is the caller's business.
 *   FSR1_FLAG_IN_SURFACE   `in` is a surface image, RGBA16F only: EASU's load stage of fsr1_easu, fsr1_upscale (fused, or EASU -> tmp
 *                          -> RCAS), fsr1_upscale_post and fsr1_context_upscale / _render / _post (`in_dev` is the handle, `in_pitch`
 *                          0).  With FSR1_FLAG_SRTM_INPUT too.  fsr1_rcas: FSR1_ERR_UNSUPPORTED.
 *   FSR1_FLAG_OUT_SURFACE  `out` is a surface image written by the pass that writes `out`: fsr1_rcas, fsr1_upscale (not with
 *                          FSR1_FLAG_NO_RCAS), fsr1_upscale_post into RGBA16F, or with TEPD8 / TEPD10 RGBA8_UNORM / RGB10A2_UNORM, and the
 *                          context calls (`out_dev` is the handle, `out_pitch` 0).  With the RCAS options.  fsr1_easu:
 *                          FSR1_ERR_UNSUPPORTED.
 * Images the library owns, and `tmp`, stay linear.  A frame the linear call runs on the fused kernel runs on the fused kernel's surface
 * twin.  FSR1_ERR_UNSUPPORTED, with nothing launched: another input format, an output format the RGBA16F kernels do not write,
 * FSR1_FLAG_EXACT / FORCE_DIRECT / H_REFERENCE / PRECISE / RCAS_HX2, constants that do not upscale with FSR1_FLAG_IN_SURFACE, and
 * fsr1_context_upscale_host, fsr1_shard_create and fsr1_shard_create_post with either flag.  Validation, before any launch and
 * allocating nothing: first the flag, format and layout rules above (no CUDA call; FSR1_ERR_INVALID_ARGUMENT for a null handle, a
 * pitch other than 0 or a window), then the array behind each handle (cudaGetSurfaceObjectResourceDesc, cudaArrayGetInfo): an unknown
 * handle or an extent smaller than width x height returns FSR1_ERR_INVALID_ARGUMENT; a resource that is not a 2D array, or an element
 * size other than the format's, FSR1_ERR_UNSUPPORTED. */

/* Texture images (FSR1_FLAG_IN_TEXTURE): the render target read the way the reference reads it, by sampling (an SRV), so an array
 * mapped without surface load/store (a render target created without storage / UAV usage, or an R11G11B10_FLOAT one whose format has
 * no storage support) is read in place.  `data` holds the cudaTextureObject_t, pitch_bytes is 0, row0 = 0 and rows = height: never a
 * window.  width x height is the logical size, the TOP-LEFT region of the array; EASU clamps its taps at the logical edge and fetches
 * no texel outside it.  Formats: FSR1_FORMAT_RGBA16F and FSR1_FORMAT_R11G11B10_FLOAT.  The kernels use the raw texel bits, so every
 * result is bit-identical to the same call on a linear image holding the same pixels (NaN payloads, -0 and denormals included), and:
 *   - the array's channels are UNSIGNED INTEGERS of the texel's layout: map RGBA16F with
 *     cudaCreateChannelDesc(16, 16, 16, 16, cudaChannelFormatKindUnsigned) and R11G11B10_FLOAT with
 *     cudaCreateChannelDesc(32, 0, 0, 0, cudaChannelFormatKindUnsigned) (CU_AD_FORMAT_UNSIGNED_INT16 x 4 / UNSIGNED_INT32 x 1);
 *     a float channel kind would have the texture unit convert to fp32: FSR1_ERR_UNSUPPORTED;
 *   - the texture description: cudaReadModeElementType, normalizedCoords 0, cudaFilterModePoint, sRGB 0; any address mode (every
 *     fetch is inside the array);
 *   - the resource: cudaResourceTypeArray, a 2D array (not layered, not 3D) of at least width x height; a pitch2D, linear or
 *     mipmapped-array resource is refused (pass the level-0 array of a mipmapped one).
 * FSR1_FLAG_IN_TEXTURE is taken exactly where FSR1_FLAG_IN_SURFACE is, with the same rules otherwise: fsr1_easu, fsr1_upscale (fused,
 * or EASU -> tmp -> RCAS), fsr1_upscale_post (every output format, FSR1_FLAG_OUT_SURFACE too) and fsr1_context_upscale / _render /
 * _post (`in_dev` is the handle, `in_pitch` 0), with FSR1_FLAG_SRTM_INPUT too.  FSR1_ERR_UNSUPPORTED, with nothing launched: fsr1_rcas,
 * fsr1_rcas_post, fsr1_context_upscale_host, fsr1_shard_create and fsr1_shard_create_post with the flag, another input format,
 * FSR1_FLAG_EXACT / FORCE_DIRECT / H_REFERENCE / PRECISE / RCAS_HX2, and constants that do not upscale.  FSR1_FLAG_IN_TEXTURE together
 * with FSR1_FLAG_IN_SURFACE: FSR1_ERR_INVALID_ARGUMENT.  Validation, before any launch: first the flag, format and layout rules (no
 * CUDA call), then the handle (cudaGetTextureObjectResourceDesc, cudaGetTextureObjectTextureDesc, cudaArrayGetInfo): an unknown handle
 * or an extent smaller than width x height returns FSR1_ERR_INVALID_ARGUMENT; a wrong channel kind or size, texture description or
 * resource type, FSR1_ERR_UNSUPPORTED. */

/* EASU over output rows [y0, y1) (y1 == 0 means "to the last row").  con = con0..con3, 16 words.  in and out have the same format, but
 * for R11G11B10_FLOAT input, whose output is RGBA16F. */
int fsr1_easu(const fsr1_image* in, const fsr1_image* out, const uint32_t con[16], uint32_t y0, uint32_t y1,
              uint32_t flags, void* stream);

/* RCAS over rows [y0, y1); in and out have the same logical size and format.  con = 4 words. */
int fsr1_rcas(const fsr1_image* in, const fsr1_image* out, const uint32_t con[4], uint32_t y0, uint32_t y1,
              uint32_t flags, void* stream);

/* First and last input row EASU reads to produce output rows [y0,y1) (clamped to the image): what a
 * slab must hold, and what must be exchanged as halo when the output is sharded by rows. */
int fsr1_easu_input_rows(const uint32_t con[16], uint32_t in_height, uint32_t y0, uint32_t y1,
                         uint32_t* first_row, uint32_t* last_row);

/* EASU -> RCAS for output rows [y0,y1).  `tmp` is the display-sized intermediate (same format as out; both RGBA16F for
 * R11G11B10_FLOAT input);
 * it must hold rows [y0-1, y1+1) clipped to the image.  easu_con 16 words, rcas_con 4 words. */
int fsr1_upscale(const fsr1_image* in, const fsr1_image* tmp, const fsr1_image* out, const uint32_t easu_con[16],
                 const uint32_t rcas_con[4], uint32_t y0, uint32_t y1, uint32_t flags, void* stream);

/* ---- resource-owning context (the FSR_Filter object of the sample) ---------------------------- */
typedef struct fsr1_context fsr1_context;

/* Allocates the intermediate image for (out_width x out_height, format) on the current device.  `format` is the input's; the
 * intermediate and the output are in that format too, but RGBA16F for R11G11B10_FLOAT. */
int fsr1_context_create(fsr1_context** ctx, uint32_t in_width, uint32_t in_height, uint32_t out_width,
                        uint32_t out_height, uint32_t format);
void fsr1_context_destroy(fsr1_context* ctx);

/* Device-resident frames: constants are derived inside exactly as FSR_Filter::Upscale does
 * (FsrEasuCon(renderW,renderH,renderW,renderH,displayW,displayH); FsrRcasCon(sharpness_stops)). */
int fsr1_context_upscale(fsr1_context* ctx, const void* in_dev, uint64_t in_pitch, void* out_dev, uint64_t out_pitch,
                         float sharpness_stops, uint32_t flags, void* stream);

/* The same with the render size of THIS frame (dynamic resolution / a preset change without re-creating the resources):
 * FSR_Filter::Upscale rebuilds FsrEasuCon from pState->renderWidth/renderHeight on every call (FSR_Filter.cpp:106).
 * The render region is the top-left render_width x render_height of in_dev; taps clamp at its edge, never reading the
 * rest of the buffer.  A render size larger than the context's input size returns FSR1_ERR_INVALID_ARGUMENT. */
int fsr1_context_upscale_render(fsr1_context* ctx, const void* in_dev, uint64_t in_pitch, uint32_t render_width,
                                uint32_t render_height, void* out_dev, uint64_t out_pitch, float sharpness_stops,
                                uint32_t flags, void* stream);

/* Host-resident frames (pinned memory recommended): H2D copy, EASU, RCAS, D2H copy on `stream`. */
int fsr1_context_upscale_host(fsr1_context* ctx, const void* in_host, uint64_t in_pitch, void* out_host,
                              uint64_t out_pitch, float sharpness_stops, uint32_t flags, void* stream);

/* ---- row-slab sharding across the GPUs of one box (the reference has no multi-GPU path: new) ------
 * The output image is cut into `world` contiguous row slabs, one per rank (= per GPU).  Rank k owns input rows
 * [k*in_h/world, (k+1)*in_h/world) and needs 2-3 more rows each side: the EASU footprint of its slab plus the
 * one-row apron RCAS reads, so there is exactly ONE neighbour exchange per frame and no collective.
 * A fsr1_shard owns the rank's share of a ring of `slots` frames: input window (own rows + halo), output slab,
 * three internal streams, and an intermediate only when its frames cannot take the fused EASU->RCAS kernel (see
 * FSR1_FLAG_FUSED; decided at create time).  The halo moves by direct NVLink stores into the neighbour's window
 * (CUDA IPC between processes, peer access inside one process), flow-controlled by sequence numbers in device
 * memory: no NCCL call, no host synchronisation and no allocation per frame.  Per frame the caller writes its
 * input rows into fsr1_shard_input(slot) on `stream`, calls fsr1_shard_submit(slot, stream), and orders its
 * consumer after fsr1_shard_wait(slot, stream).  Consecutive frames run on two streams in turn and overlap.
 * All ranks must create shards with identical arguments (except rank) and submit slots in the same order.
 * Set-up between processes: every rank calls fsr1_shard_export, the 64-byte handles are gathered in rank order by
 * any means (torch.distributed all_gather, MPI, a pipe), every rank calls fsr1_shard_attach.  In one process
 * driving several devices: fsr1_shard_attach_local(shard, shard_of_rank-1, shard_of_rank+1). */
typedef struct fsr1_shard fsr1_shard;
#define FSR1_SHARD_HANDLE_BYTES 64
#define FSR1_SHARD_ONE_STREAM (1u << 16) /* fsr1_shard_create flag: every frame on one stream (no overlap of consecutive frames; default: two
                                            streams, whole frames in turn, so RCAS of frame i overlaps EASU of frame i+1)                  */
#define FSR1_SHARD_TRACE (1u << 18)      /* keep device timestamps of the last 256 frames (fsr1_shard_trace)                          */
#define FSR1_SHARD_SKIP_HALO (1u << 17)  /* MEASUREMENT ONLY: no halo exchange (slab borders are wrong); times the frame without it */
#define FSR1_SHARD_DYNAMIC (1u << 19)    /* dynamic resolution: in_width x in_height is the input RESOURCE, the largest render size a frame
                                            may use; fsr1_shard_frame gives each use of a slot its own render size and sharpness (the
                                            create-time sharpness_stops is the default).  Allocates the intermediate at create.     */

typedef struct fsr1_shard_info {   /* logical row ranges [row0, row1) of this rank */
  uint32_t out_row0, out_row1;       /* output slab                                                 */
  uint32_t easu_row0, easu_row1;     /* rows EASU produces (slab + RCAS apron)                      */
  uint32_t owned_row0, owned_row1;   /* input rows this rank owns (the caller writes them)          */
  uint32_t needed_row0, needed_row1; /* input rows EASU reads                                       */
  uint32_t window_row0, window_row1; /* input rows resident on this rank (owned + halo)             */
  uint32_t send_up_row0, send_up_row1, send_down_row0, send_down_row1; /* rows pushed to rank-1 / rank+1 */
  uint64_t halo_recv_bytes;          /* halo payload received per frame                             */
  uint64_t arena_bytes;
} fsr1_shard_info;

/* `flags`: FSR1_FLAG_* for the kernels, optionally FSR1_SHARD_ONE_STREAM / _DYNAMIC.  FSR1_ERR_UNSUPPORTED when a slab is
 * shorter than the halo it must supply (the halo would come from beyond the direct neighbours); with FSR1_SHARD_DYNAMIC this is
 * checked for the whole resource here and for each frame's render height in fsr1_shard_frame.  fsr1_shard_geometry always
 * describes the whole-resource frame. */
int fsr1_shard_create(fsr1_shard** shard, uint32_t in_width, uint32_t in_height, uint32_t out_width, uint32_t out_height,
                      uint32_t format, uint32_t world, uint32_t rank, uint32_t slots, float sharpness_stops, uint32_t flags);
void fsr1_shard_destroy(fsr1_shard* shard);
int fsr1_shard_geometry(const fsr1_shard* shard, fsr1_shard_info* info);
int fsr1_shard_export(const fsr1_shard* shard, void* handle /* FSR1_SHARD_HANDLE_BYTES */);
int fsr1_shard_attach(fsr1_shard* shard, const void* handles /* world x FSR1_SHARD_HANDLE_BYTES, rank order */, uint32_t count);
int fsr1_shard_attach_local(fsr1_shard* shard, fsr1_shard* up /* rank-1 or NULL */, fsr1_shard* down /* rank+1 or NULL */);
int fsr1_shard_input(const fsr1_shard* shard, uint32_t slot, fsr1_image* owned);   /* where the caller writes its rows */
int fsr1_shard_window(const fsr1_shard* shard, uint32_t slot, fsr1_image* window); /* owned rows + halo (read-only)     */
int fsr1_shard_output(const fsr1_shard* shard, uint32_t slot, fsr1_image* out);    /* the rank's output slab            */
void* fsr1_shard_arena(const fsr1_shard* shard);
/* FSR1_SHARD_DYNAMIC: describe the next use of `slot` (call it before writing the frame's input rows).  The input is the top-left
 * render_width x render_height of the resource, as in fsr1_context_upscale_render; the constants are
 * FsrEasuCon(rw, rh, rw, rh, out_w, out_h) and FsrRcasCon(sharpness_stops).  Afterwards fsr1_shard_input / fsr1_shard_window
 * describe that frame's rows (rank k owns input rows [k*rh/world, (k+1)*rh/world), logical width rw, the resource's pitch) and
 * fsr1_shard_submit runs it; the output slab does not change.  A slot keeps its last description; the first is the whole resource
 * at the create sharpness, so a dynamic shard that is never given one launches exactly what a static shard launches.  Every rank
 * must describe the same use of a slot with the same arguments.  Host-only: no CUDA call, nothing allocated.
 * FSR1_ERR_INVALID_ARGUMENT: a shard created without FSR1_SHARD_DYNAMIC, a bad slot, a zero render size, one larger than the
 * resource, or world > render_height.  FSR1_ERR_UNSUPPORTED: at that render height a rank's halo would have to come from beyond its
 * direct neighbours (the rule of fsr1_shard_create); a render height below the shard's minimum, a few rows per rank, where a
 * neighbour's rows for one frame could land on window rows a rank's push of the previous frame in the slot still reads (26 rows at
 * 8 ranks from a resource of half the output size); or the kernels refused a frame of its kind (2x / other upscale / downscale)
 * with the create flags when fsr1_shard_create tried one. */
int fsr1_shard_frame(fsr1_shard* shard, uint32_t slot, uint32_t render_width, uint32_t render_height, float sharpness_stops);
/* Upscale the frame in `slot`: ordered after everything already on `stream`; returns without waiting. */
int fsr1_shard_submit(fsr1_shard* shard, uint32_t slot, void* stream);
/* Orders `stream` after the slot's result (and after this rank's halo rows have left: the input may be rewritten). */
int fsr1_shard_wait(fsr1_shard* shard, uint32_t slot, void* stream);
/* FSR1_SHARD_TRACE: 8 GPU globaltimer stamps (ns) per frame, oldest first: [0] EASU began waiting for its halo, [1] halo present,
 * [2] last EASU CTA done (credit sent), [3]/[5] push up/down started, [4]/[6] push up/down published, [7] unused. */
int fsr1_shard_trace(fsr1_shard* shard, uint64_t* out /* max_frames x 8 */, uint32_t max_frames, uint32_t* n_frames);
int fsr1_shard_status(fsr1_shard* shard);  /* FSR1_OK, or FSR1_ERR_TIMEOUT if a neighbour never answered (call after a sync) */

/* ---- pointwise companions of the scaling path (ffx-fsr/ffx_fsr1.h:986-1199) ----------------------
 * The passes the sample runs either side of EASU/RCAS, as whole-image streaming kernels over rows [y0,y1)
 * (y1 == 0: to the last row).  `in` and `out` have the same logical size and may be the same image (in place).
 * Arithmetic is fp32 with separate roundings for every storage format: RGBA32F results are bit-identical to the
 * reference's F functions, other formats round that result once on store.  Alpha is carried through.
 *   fsr1_srtm   FsrSrtmF (inverse == 0) / FsrSrtmInvF (inverse != 0)   ffx_fsr1.h:1044,1046
 *   fsr1_lfga   FsrLfgaF: c += (grain * amount) * min(1 - c, c)         ffx_fsr1.h:1014
 *               `grain` = RGB image of {-0.5..0.5} values (float formats), tiled over the frame with wrap addressing
 *   fsr1_tepd   FsrTepdC8F (bits == 8) / FsrTepdC10F (bits == 10)       ffx_fsr1.h:1100-1126
 *               dither == NULL: FsrTepdDitF(pixel, frame) (ffx_fsr1.h:1086-1095); else the saturated .w channel of the
 *               tiled `dither` image (sample/src/DX12/FSR_Tonemapping.hlsl:87).  `out` may be the same format as `in`
 *               or, from a float image, RGBA8_UNORM (bits 8) / RGB10A2_UNORM (bits 10): the code values themselves. */
int fsr1_srtm(const fsr1_image* in, const fsr1_image* out, int inverse, uint32_t y0, uint32_t y1, void* stream);
int fsr1_lfga(const fsr1_image* in, const fsr1_image* grain, const fsr1_image* out, float amount, uint32_t y0,
              uint32_t y1, void* stream);
int fsr1_tepd(const fsr1_image* in, const fsr1_image* dither, const fsr1_image* out, int bits, uint32_t frame,
              uint32_t y0, uint32_t y1, void* stream);

/* The same passes in the reference's HALF arithmetic, through its packed calling convention (two pixels, p and p + (8,0), per lane
 * in half2 registers): RGBA16F images only (in, out, grain, dither), every operation rounded to half once, results bit-identical
 * to the reference's H and Hx2 functions (which agree with each other bit for bit).  Same arguments and rules as above.
 *   fsr1_srtm_h   FsrSrtmH / FsrSrtmHx2 (inverse == 0), FsrSrtmInvH / FsrSrtmInvHx2     ffx_fsr1.h:1049-1055
 *   fsr1_lfga_h   FsrLfgaH / FsrLfgaHx2; `amount` is converted to half once               ffx_fsr1.h:1019-1024
 *   fsr1_tepd_h   FsrTepdC8H / C8Hx2 (bits == 8), FsrTepdC10H / C10Hx2 (bits == 10)      ffx_fsr1.h:1137-1153,1166-1199
 *                 dither == NULL: FsrTepdDitH / FsrTepdDitHx2(pixel, frame) (:1129-1135,1156-1164); `out` is RGBA16F */
int fsr1_srtm_h(const fsr1_image* in, const fsr1_image* out, int inverse, uint32_t y0, uint32_t y1, void* stream);
int fsr1_lfga_h(const fsr1_image* in, const fsr1_image* grain, const fsr1_image* out, float amount, uint32_t y0,
                uint32_t y1, void* stream);
int fsr1_tepd_h(const fsr1_image* in, const fsr1_image* dither, const fsr1_image* out, int bits, uint32_t frame,
                uint32_t y0, uint32_t y1, void* stream);

/* ---- upscale straight to the display output (ffx_fsr1.h:1030-1040 usage notes) ------------------
 * fsr1_upscale followed by the passes an application runs after RCAS, applied inside RCAS's store instead of as whole-image passes:
 * the chain writes the output once and reads nothing extra but the small grain / dither tiles.  The result is bit-identical, on rows
 * [y0, y1), to
 *     fsr1_upscale(in, tmp, T, easu_con, rcas_con, y0, y1, flags)      T: an RGBA16F image of out's size
 *     FSR1_POST_SRTM_INVERSE:  fsr1_srtm(T, T, 1, ...)                 FsrSrtmInvF      ffx_fsr1.h:1046
 *     FSR1_POST_LFGA:          fsr1_lfga(T, grain, T, lfga_amount, ...) FsrLfgaF        ffx_fsr1.h:1014
 *     FSR1_POST_TEPD8 / 10:    fsr1_tepd(T, dither, out, 8 / 10, frame, ...)  FsrTepdC8F / C10F  ffx_fsr1.h:1100-1126
 * in that order (the last step writes `out`).  Alpha is what RCAS stores (1, or the input's with FSR1_FLAG_RCAS_PASSTHROUGH_ALPHA).
 *   in      RGBA16F or R11G11B10_FLOAT.
 *   out     RGBA16F; with TEPD also RGBA8_UNORM (TEPD8) or RGB10A2_UNORM (TEPD10): the code values, as fsr1_tepd writes them.
 *   tmp     the RGBA16F intermediate of the two-kernel path (as fsr1_upscale); NULL is accepted when the frame takes the fused
 *           kernel (FSR1_FLAG_FUSED, exactly 2x, no RCAS option, no OUTPUT_SQUARE, no PRECISE), which then is the only launch.
 *   post    NULL or ops == 0: exactly fsr1_upscale.  grain: an RGBA16F / RGBA32F tile (wrap addressing, as fsr1_lfga); dither:
 *           NULL = FsrTepdDitF(pixel, frame), else the saturated .w of a tile (as fsr1_tepd).  Tiles are whole images.
 * Every other scale, the RCAS options, OUTPUT_SQUARE and PRECISE run EASU into tmp and one RCAS kernel with the epilogue.
 * FSR1_ERR_UNSUPPORTED: another input/output format, FSR1_FLAG_EXACT / FORCE_DIRECT / H_REFERENCE / RCAS_HX2 / NO_RCAS, or a layout
 * the packed kernels cannot take (out and tmp 16-byte aligned, 8 for UNORM out); those callers keep using the separate passes.
 * FSR1_ERR_INVALID_ARGUMENT: unknown ops bits, both TEPD bits, LFGA without a grain tile, a tile that is a window.  All
 * validation happens before any CUDA call. */
enum { FSR1_POST_SRTM_INVERSE = 1u << 0, FSR1_POST_LFGA = 1u << 1, FSR1_POST_TEPD8 = 1u << 2, FSR1_POST_TEPD10 = 1u << 3 };
typedef struct fsr1_post {
  uint32_t ops;              /* FSR1_POST_*, applied in this order; TEPD8 and TEPD10 exclusive */
  float lfga_amount;
  const fsr1_image* grain;   /* LFGA tile */
  const fsr1_image* dither;  /* TEPD tile or NULL */
  uint32_t frame, reserved;  /* TEPD positional dither: FsrTepdDitF(pixel, frame) */
} fsr1_post;
int fsr1_upscale_post(const fsr1_image* in, const fsr1_image* tmp, const fsr1_image* out, const uint32_t easu_con[16],
                      const uint32_t rcas_con[4], const fsr1_post* post, uint32_t y0, uint32_t y1, uint32_t flags, void* stream);
/* The context form, as fsr1_context_upscale_render (render size 0 = the context's input size; always FSR1_FLAG_FUSED).  The context's
 * format must be RGBA16F or R11G11B10_FLOAT.  `out_dev` is RGBA8_UNORM with TEPD8, RGB10A2_UNORM with TEPD10, RGBA16F otherwise. */
int fsr1_context_upscale_post(fsr1_context* ctx, const void* in_dev, uint64_t in_pitch, uint32_t render_width,
                              uint32_t render_height, void* out_dev, uint64_t out_pitch, float sharpness_stops,
                              const fsr1_post* post, uint32_t flags, void* stream);

/* Sharpen a frame rendered at display resolution (render size = display size: a native / "sharpen only" setting, dynamic resolution
 * at 100 %) straight to the display output: the input stage, RCAS and the display steps of fsr1_upscale_post in ONE kernel, with no
 * EASU pass and no intermediate.  On rows [y0, y1) (y1 == 0: to the last row) the result is bit-identical to
 *     I = in (RGBA16F), or for R11G11B10_FLOAT the RGBA16F image (R, G, B, 1.0) of its codes
 *     FSR1_FLAG_SRTM_INPUT:  I = fsr1_srtm(I, ., 0) over the rows RCAS reads, [y0-1, y1+1) clipped to the image
 *     fsr1_rcas(I, T, rcas_con, y0, y1, the RCAS_CLAMP / RCAS_DENOISE / RCAS_PASSTHROUGH_ALPHA / OUTPUT_SQUARE bits of flags), T RGBA16F
 *     the steps of `post` on T as fsr1_upscale_post applies them (SRTM inverse, LFGA, TEPD8 / TEPD10), the last one writing `out`.
 * Out-of-image taps read 0 in the decoded domain (or clamp with RCAS_CLAMP); R11G11B10_FLOAT has no alpha, so PASSTHROUGH_ALPHA gives 1.0.
 * post == NULL or ops == 0 on RGBA16F input without SRTM_INPUT is exactly fsr1_rcas (the same kernel).
 *   in      RGBA16F (base and pitch 16-byte aligned) or R11G11B10_FLOAT (8-byte aligned), linear, possibly a row window holding rows
 *           [y0-1, y1+1) clipped to the image (the rule of fsr1_rcas).
 *   out     in's logical size; RGBA16F (16-byte aligned), or with TEPD the UNORM format it implies (8-byte aligned), as fsr1_upscale_post;
 *           a surface image with FSR1_FLAG_OUT_SURFACE.
 *   flags   RCAS_CLAMP, RCAS_DENOISE, RCAS_PASSTHROUGH_ALPHA, OUTPUT_SQUARE, SRTM_INPUT, OUT_SURFACE; FUSED is accepted and has no effect.
 * FSR1_ERR_INVALID_ARGUMENT: a null in, out or rcas_con, an unknown flag, a bad row range, in and out of different sizes, linear storage
 * of in and out that overlaps, and every refusal of fsr1_upscale_post's post description.  FSR1_ERR_UNSUPPORTED: another input or
 * output format, EXACT / FORCE_DIRECT / H_REFERENCE / PRECISE / RCAS_HX2 / NO_RCAS / IN_SURFACE, or an unaligned layout (there is no
 * fall-back kernel).  FSR1_ERR_WINDOW: a window that does not hold the rows.  All returned before any CUDA call but the array query of
 * FSR1_FLAG_OUT_SURFACE. */
int fsr1_rcas_post(const fsr1_image* in, const fsr1_image* out, const uint32_t rcas_con[4], const fsr1_post* post, uint32_t y0, uint32_t y1,
                   uint32_t flags, void* stream);

/* Display output from the sharded frame stream: every frame of the shard is fsr1_upscale_post with `post` instead of fsr1_upscale,
 * so each rank's output slab holds the display image's rows (for rows [out_row0, out_row1), bit-identical to the same rows of
 * fsr1_upscale_post / fsr1_context_upscale_post on the whole frame) and no pass runs over the slabs afterwards.  fsr1_shard_create is
 * fsr1_shard_create_post(..., format, format, NULL, ...).
 *   format      the input's format; with post ops RGBA16F or R11G11B10_FLOAT.  The windows and the halo are sized at its bytes per
 *               pixel (4 for R11G11B10_FLOAT); an intermediate, when there is one, is in EASU's output format (RGBA16F for it).
 *   out_format  the slabs' format: RGBA16F, or with TEPD the UNORM format it implies (RGBA8_UNORM for TEPD8, RGB10A2_UNORM for
 *               TEPD10, 4 B/px); without post ops it must equal `format`, but RGBA16F for R11G11B10_FLOAT input (fsr1_shard_create
 *               gives RGBA16F slabs then).  fsr1_shard_output describes slabs in this format.
 *   post        NULL or ops == 0: no display steps.  `post->ops` is fixed for the shard's life (it decides which kernels the create-time
 *               dry frames load); the rest is the first description of every slot (fsr1_shard_post).  The tiles (grain, dither) are
 *               whole device images on the rank's own device, read by every frame that uses them: the caller keeps them alive and
 *               unchanged until those frames have completed (fsr1_shard_wait); the shard copies the descriptors, not the pixels.
 * The rules are those of fsr1_upscale_post, all checked before any CUDA call: FSR1_ERR_INVALID_ARGUMENT for unknown ops bits, both TEPD
 * bits, LFGA without a grain tile, a tile that is a window; FSR1_ERR_UNSUPPORTED for another input / output format, FSR1_FLAG_EXACT /
 * FORCE_DIRECT / H_REFERENCE / RCAS_HX2 / NO_RCAS.  A static 2x shard whose frames take the fused post kernel allocates no intermediate;
 * every other shard allocates an RGBA16F one, as fsr1_shard_create does.  The halo hand-shake rides inside the post kernels exactly as
 * inside the plain ones (trace stamps [0]-[2]). */
int fsr1_shard_create_post(fsr1_shard** shard, uint32_t in_width, uint32_t in_height, uint32_t out_width, uint32_t out_height,
                           uint32_t format, uint32_t out_format, const fsr1_post* post, uint32_t world, uint32_t rank, uint32_t slots,
                           float sharpness_stops, uint32_t flags);
/* Describe the display steps of the next use of `slot`, as fsr1_shard_frame describes its render size: the TEPD `frame` of the
 * positional dither FsrTepdDitF(pixel, frame), the LFGA amount and the grain / dither tiles.  `post->ops` must equal the shard's.  A slot
 * keeps its last description; the first is the create-time `post`.  Host-only: no CUDA call, nothing allocated.
 * FSR1_ERR_INVALID_ARGUMENT: a shard created without post ops, ops other than the shard's, a bad slot, or a description
 * fsr1_upscale_post refuses (LFGA without a grain tile, a tile that is a window); FSR1_ERR_UNSUPPORTED: a grain tile that is not
 * RGBA16F / RGBA32F.  The slot keeps its previous description on any error. */
int fsr1_shard_post(fsr1_shard* shard, uint32_t slot, const fsr1_post* post);

/* ---- constants through the ABI (for FFIs that cannot include fsr1_host.h) ---------------------- */
void fsr1_easu_con(uint32_t con[16], float in_viewport_w, float in_viewport_h, float in_size_w, float in_size_h,
                   float out_w, float out_h);
void fsr1_easu_con_offset(uint32_t con[16], float in_viewport_w, float in_viewport_h, float in_size_w,
                          float in_size_h, float out_w, float out_h, float in_off_x, float in_off_y);
void fsr1_rcas_con(uint32_t con[4], float sharpness_stops);

/* ---- introspection ----------------------------------------------------------------------------- */
int fsr1_abi_version(void);
const char* fsr1_error_string(int err);
int fsr1_last_cuda_error(void);          /* cudaError_t of the last failed CUDA call on this thread   */
uint64_t fsr1_launch_count(void);        /* kernels launched by this library since load (all threads) */
const char* fsr1_last_kernel_name(void); /* which kernel variant the last launch on this thread used  */

#ifdef __cplusplus
}
#endif
#endif /* FSR1_B200_H */
