// fsr1_common.cuh — shared device-side definitions of the FSR1 kernels (sm_90a).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/fsr1_b200.h"

namespace fsr1 {

// Device view of an fsr1_image (include/fsr1_b200.h): logical size w x h, storage holds rows
// [row0, row0+rows).  `base` already points at logical row `row0`.
struct ImgView {
  unsigned char* base;
  long long pitch;  // bytes
  int w, h;         // logical size
  int row0, rows;   // stored window
};

// Logical row y is inside the image AND inside the stored window.  The checked load paths of the RCAS kernels test
// this (not just 0 <= y < h): a lane requests kRows+2 rows up front, and the last partial chunk of a row slab would
// otherwise read up to kRows-1 rows past the rows the window is required to hold.
__host__ __device__ __forceinline__ bool row_stored(const ImgView& im, int y) {
  return y >= im.row0 && y < im.row0 + im.rows && y >= 0 && y < im.h;
}

// Row-slab sharding (fsr1_shard.cu): the neighbour hand-shake of a frame folded INTO the kernel that reads the input window, so the
// frame costs no extra launch on the critical stream.  ready[side]: flags in this GPU's memory the neighbours set (release.sys) when
// the halo rows of use `seq` of this window are in place — every CTA's thread 0 acquires them before the CTA's first load.
// credit[side]: flags in the NEIGHBOURS' memory the last CTA to finish sets: "use `seq` of my window has been read, you may overwrite
// your rows in it".  All pointers null outside the sharded path.
struct HaloSync {
  const uint32_t* ready[2];
  uint32_t* credit[2];
  uint32_t* counter;  // CTAs finished (device memory, zero between launches)
  uint32_t* status;   // != 0: a wait timed out
  unsigned long long* trace;  // optional (fsr1_shard_trace): globaltimer at [0] wait begin, [1] wait end (CTA 0), [2] last CTA done
  uint32_t seq;
};

struct EasuParams {
  ImgView in, out;
  float c0x, c0y, c0z, c0w;  // con0 of FsrEasuCon: scale.xy, offset.zw
  int y0, y1;                // output rows [y0,y1)
  HaloSync sync = {};
};

// The two tests of the EASU constants every kernel choice depends on (con0 of FsrEasuCon: scale.xy, offset.zw): exactly 2x (the 2x
// kernels) and upscaling (the any-scale tiled kernels).  They are also the kinds of frame a dynamic fsr1_shard loads kernels for at
// create (frame_kind, fsr1_shard.cu), so a kernel choice on any other property of the constants needs a kind of its own there.
__host__ __device__ inline bool is_2x(float c0x, float c0y, float c0z, float c0w) {
  return c0x == 0.5f && c0y == 0.5f && c0z == -0.25f && c0w == -0.25f;
}
__host__ __device__ inline bool is_upscale(float c0x, float c0y) { return c0x > 0.0f && c0x <= 1.0f && c0y > 0.0f && c0y <= 1.0f; }

struct RcasParams {
  ImgView in, out;
  float sharp;      // con.x as float
  uint32_t sharp_h2;  // con.y: half2(sharp,sharp)
  int y0, y1;
  int clamp;        // 0: out-of-image taps read 0 (D3D12 Load), 1: clamp
  int options;      // bit 0: FSR_RCAS_DENOISE, bit 1: FSR_RCAS_PASSTHROUGH_ALPHA (direct / H-reference kernels)
};

// ---- the reference's bit-trick approximations (ffx-fsr/ffx_a.h:1843-1845), bit-exact ------------
__device__ __forceinline__ float prx_lo_rcp(float a) { return __uint_as_float(0x7ef07ebbu - __float_as_uint(a)); }
__device__ __forceinline__ float prx_lo_rsq(float a) { return __uint_as_float(0x5f347d74u - (__float_as_uint(a) >> 1)); }

// Arithmetic policy.  Exact: every product and sum rounds separately (no FMA contraction) and
// reciprocals are IEEE, so the result is bit-identical to the reference source compiled with
// -ffp-contract=off.  Fast: the compiler may contract a*b+c into FMA (what a shader compiler does).
template <bool kExact> struct Ar;
template <> struct Ar<true> {
  static __device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
  static __device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
  static __device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
  static __device__ __forceinline__ float mad(float a, float b, float c) { return __fadd_rn(__fmul_rn(a, b), c); }
  static __device__ __forceinline__ float rcp(float a) { return __fdiv_rn(1.0f, a); }
};
template <> struct Ar<false> {
  static __device__ __forceinline__ float mul(float a, float b) { return a * b; }
  static __device__ __forceinline__ float add(float a, float b) { return a + b; }
  static __device__ __forceinline__ float sub(float a, float b) { return a - b; }
  static __device__ __forceinline__ float mad(float a, float b, float c) { return fmaf(a, b, c); }
  static __device__ __forceinline__ float rcp(float a) { return __frcp_rn(a); }
};

__device__ __forceinline__ float sat(float x) { return __saturatef(x); }  // saturate(NaN) = 0

// Output pixel -> (cell origin, fraction).  Always mul then add (two roundings): this is what the
// oracle does, and the footprint computed on the host must agree with it for every pixel.
__device__ __forceinline__ void easu_pos(int o, float scale, float offset, int& fp, float& pp) {
  float p = __fadd_rn(__fmul_rn((float)o, scale), offset);
  float f = floorf(p);
  fp = (int)f;
  pp = __fsub_rn(p, f);
}

// ---- storage access ------------------------------------------------------------------------------
template <typename S> struct Px;
template <> struct Px<float> {
  static constexpr int kBytes = 16;
  static __device__ __forceinline__ float3 load(const ImgView& im, int x, int y) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(im.base + (long long)(y - im.row0) * im.pitch) + x);
    return make_float3(v.x, v.y, v.z);
  }
  static __device__ __forceinline__ void store(const ImgView& im, int x, int y, float r, float g, float b, float a = 1.0f) {
    reinterpret_cast<float4*>(im.base + (long long)(y - im.row0) * im.pitch)[x] = make_float4(r, g, b, a);
  }
  static __device__ __forceinline__ float alpha(const ImgView& im, int x, int y) {
    return __ldg(reinterpret_cast<const float4*>(im.base + (long long)(y - im.row0) * im.pitch) + x).w;
  }
};
template <> struct Px<__half> {
  static constexpr int kBytes = 8;
  static __device__ __forceinline__ float3 load(const ImgView& im, int x, int y) {
    const uint2 v = __ldg(reinterpret_cast<const uint2*>(im.base + (long long)(y - im.row0) * im.pitch) + x);
    const float2 rg = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
    const float2 ba = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
    return make_float3(rg.x, rg.y, ba.x);
  }
  static __device__ __forceinline__ float alpha(const ImgView& im, int x, int y) {
    const uint2 v = __ldg(reinterpret_cast<const uint2*>(im.base + (long long)(y - im.row0) * im.pitch) + x);
    return __high2float(*reinterpret_cast<const __half2*>(&v.y));
  }
  static __device__ __forceinline__ void store(const ImgView& im, int x, int y, float r, float g, float b, float a = 1.0f) {
    __half2 rg = __floats2half2_rn(r, g), ba = __floats2half2_rn(b, a);
    uint2 v;
    v.x = *reinterpret_cast<uint32_t*>(&rg);
    v.y = *reinterpret_cast<uint32_t*>(&ba);
    reinterpret_cast<uint2*>(im.base + (long long)(y - im.row0) * im.pitch)[x] = v;
  }
};

// UNORM storage (the formats the sample actually renders into: R8G8B8A8_UNORM, R10G10B10A2_UNORM,
// sample/src/DX12/FSR_Filter.cpp:72-73).  Conversions follow the D3D rules: unorm -> float is c / (2^n - 1),
// float -> unorm is clamp to [0,1] (NaN -> 0), scale by 2^n - 1, add 0.5, truncate.  4 bytes per pixel.
struct Unorm8 {};
struct Unorm10 {};
__device__ __forceinline__ uint32_t to_unorm(float v, float scale) {
  return (uint32_t)__fadd_rn(__fmul_rn(__saturatef(v), scale), 0.5f);
}
template <> struct Px<Unorm8> {
  static constexpr int kBytes = 4;
  static __device__ __forceinline__ float3 load(const ImgView& im, int x, int y) {
    const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(im.base + (long long)(y - im.row0) * im.pitch) + x);
    return make_float3(__fdiv_rn((float)(v & 255u), 255.0f), __fdiv_rn((float)((v >> 8) & 255u), 255.0f),
                       __fdiv_rn((float)((v >> 16) & 255u), 255.0f));
  }
  static __device__ __forceinline__ float alpha(const ImgView& im, int x, int y) {
    const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(im.base + (long long)(y - im.row0) * im.pitch) + x);
    return __fdiv_rn((float)(v >> 24), 255.0f);
  }
  static __device__ __forceinline__ void store(const ImgView& im, int x, int y, float r, float g, float b, float a = 1.0f) {
    reinterpret_cast<uint32_t*>(im.base + (long long)(y - im.row0) * im.pitch)[x] =
        to_unorm(r, 255.0f) | (to_unorm(g, 255.0f) << 8) | (to_unorm(b, 255.0f) << 16) | (to_unorm(a, 255.0f) << 24);
  }
};
template <> struct Px<Unorm10> {
  static constexpr int kBytes = 4;
  static __device__ __forceinline__ float3 load(const ImgView& im, int x, int y) {
    const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(im.base + (long long)(y - im.row0) * im.pitch) + x);
    return make_float3(__fdiv_rn((float)(v & 1023u), 1023.0f), __fdiv_rn((float)((v >> 10) & 1023u), 1023.0f),
                       __fdiv_rn((float)((v >> 20) & 1023u), 1023.0f));
  }
  static __device__ __forceinline__ float alpha(const ImgView& im, int x, int y) {
    const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(im.base + (long long)(y - im.row0) * im.pitch) + x);
    return __fdiv_rn((float)(v >> 30), 3.0f);
  }
  static __device__ __forceinline__ void store(const ImgView& im, int x, int y, float r, float g, float b, float a = 1.0f) {
    reinterpret_cast<uint32_t*>(im.base + (long long)(y - im.row0) * im.pitch)[x] =
        to_unorm(r, 1023.0f) | (to_unorm(g, 1023.0f) << 10) | (to_unorm(b, 1023.0f) << 20) | (to_unorm(a, 3.0f) << 30);
  }
};

// R11G11B10_FLOAT (DXGI_FORMAT_R11G11B10_FLOAT, 4 B/px): bits 0-10 R, 11-21 G (6 mantissa bits below 5 exponent bits), 22-31 B
// (5 mantissa bits below 5 exponent bits).  Each channel is a half without its sign bit and with the low mantissa bits cut off (same
// exponent and bias), so the texel decodes EXACTLY to the RGBA16F texel (R, G, B, 1.0) with shifts and masks: (e << 10) | (m << 4)
// for R and G, (e << 10) | (m << 5) for B; denormals, inf and NaN land on their half counterparts.  An input format only.
struct R11f {};
__host__ __device__ __forceinline__ uint2 r11_to_half(uint32_t v) {
  return make_uint2(((v & 0x7ffu) << 4) | ((v << 9) & 0x7ff00000u), ((v >> 17) & 0x7fe0u) | 0x3c000000u);
}
template <> struct Px<R11f> {
  static constexpr int kBytes = 4;
  static __device__ __forceinline__ float3 load(const ImgView& im, int x, int y) {
    const uint2 v = r11_to_half(__ldg(reinterpret_cast<const uint32_t*>(im.base + (long long)(y - im.row0) * im.pitch) + x));
    const float2 rg = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
    return make_float3(rg.x, rg.y, __low2float(*reinterpret_cast<const __half2*>(&v.y)));
  }
};

// c / (2^n - 1) CORRECTLY ROUNDED without a division: q = c * (1/s) is off by one ulp for half of the 8-bit codes, and an ulp of
// luma is enough to turn an exact tie between neighbouring texels (0/0 in FsrEasuSetF's length term, ffx_fsr1.h:298) into 1.0 instead
// of 0.0 — the filter of a whole 2x2 cell block changes.  One FMA refinement makes q exact for every 8- and 10-bit code
// (checked exhaustively, tests/test_constants.py).
__device__ __forceinline__ float unorm_to_float(uint32_t c, float s, float rs) {
  const float fc = __uint_as_float(0x4b000000u | c) - 8388608.0f;  // (float)c for c < 2^23 without the conversion pipe: 2^23 + c, minus 2^23
  const float q = fc * rs;
  return fmaf(fmaf(-q, s, fc), rs, q);
}

// ---- flags shared between GPUs (system scope) --------------------------------------------------------------------------
#ifdef FSR1_CPU_EMU
inline void halo_sync_begin(const HaloSync&) {}
inline void halo_sync_end(const HaloSync&) {}
#else
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
constexpr unsigned long long kSpinTimeoutNs = 4000000000ull;  // 4 s: a dead neighbour sets an error word instead of hanging the GPU
// wait until *flag >= want (sequence numbers, wrap-safe); false on timeout
__device__ __forceinline__ bool spin_until(const uint32_t* flag, uint32_t want) {
  if ((int32_t)(ld_acquire_sys(flag) - want) >= 0) return true;
  const unsigned long long t0 = global_ns();
  while ((int32_t)(ld_acquire_sys(flag) - want) < 0) {
    if (global_ns() - t0 > kSpinTimeoutNs) return false;
    __nanosleep(50);
  }
  return true;
}
// first thing a kernel does (all threads): the halo rows of this use of the window are in place
__device__ __forceinline__ void halo_sync_begin(const HaloSync& hs) {
  if (hs.ready[0] || hs.ready[1]) {
    if (threadIdx.x == 0) {
      const bool tr = hs.trace && blockIdx.x == 0 && blockIdx.y == 0;
      if (tr) hs.trace[0] = global_ns();
      if (hs.ready[0] && !spin_until(hs.ready[0], hs.seq)) atomicExch(hs.status, 3u);
      if (hs.ready[1] && !spin_until(hs.ready[1], hs.seq)) atomicExch(hs.status, 4u);
      if (tr) hs.trace[1] = global_ns();
    }
    __syncthreads();
  }
}
// last thing (all threads, after the CTA's last read of the window): the last CTA of the grid tells the neighbours
__device__ __forceinline__ void halo_sync_end(const HaloSync& hs) {
  if (hs.counter) {
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      if (atomicAdd(hs.counter, 1u) == gridDim.x * gridDim.y - 1) {
        atomicExch(hs.counter, 0u);
        __threadfence();
        if (hs.trace) hs.trace[2] = global_ns();
        if (hs.credit[0]) st_release_sys(hs.credit[0], hs.seq);
        if (hs.credit[1]) st_release_sys(hs.credit[1], hs.seq);
      }
    }
  }
}
#endif

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return min(max(v, lo), hi); }

// ---- surface access (FSR1_FLAG_IN_SURFACE / FSR1_FLAG_OUT_SURFACE) ---------------------------------------------------------
// A surface image's ImgView holds the cudaSurfaceObject_t in `base` (pitch 0, row0 0, rows = h).  x is a pixel index here and a byte
// offset in the instruction.  Zero mode: an access outside the array reads 0 and a store there is dropped; callers clamp to the
// LOGICAL image themselves and never rely on it (trap mode would turn a coordinate bug into a fault).  tests/emu supplies these
// wrappers under FSR1_CPU_EMU (fsr1_emu_surf.h), as it does the PTX wrappers of fsr1_easu_common.cuh.
#ifdef FSR1_CPU_EMU
}  // namespace fsr1
#include "fsr1_emu_surf.h"
namespace fsr1 {
#else
__device__ __forceinline__ unsigned long long surf_of(const ImgView& im) { return (unsigned long long)im.base; }
__device__ __forceinline__ uint2 surf_load8(unsigned long long s, int x, int y) {
  return surf2Dread<uint2>(s, x * 8, y, cudaBoundaryModeZero);
}
__device__ __forceinline__ void surf_store8(unsigned long long s, int x, int y, uint2 v) { surf2Dwrite(v, s, x * 8, y, cudaBoundaryModeZero); }
__device__ __forceinline__ void surf_store4(unsigned long long s, int x, int y, uint32_t v) {
  surf2Dwrite(v, s, x * 4, y, cudaBoundaryModeZero);
}
#endif

// ---- texture access (FSR1_FLAG_IN_TEXTURE) -----------------------------------------------------------------------------------
// A texture image's ImgView holds the cudaTextureObject_t in `base` (pitch 0, row0 0, rows = h).  The array's channels are unsigned
// integers (16,16,16,16 for RGBA16F, 32 for R11G11B10F) read in element mode with point filtering and unnormalized coordinates, so a
// fetch returns the texel's raw bits; the texel centre x + 0.5 is the sample position.  Callers clamp to the logical image, so the
// address mode never applies.  tests/emu supplies these under FSR1_CPU_EMU (fsr1_emu_tex.h).
#ifdef FSR1_CPU_EMU
}  // namespace fsr1
#include "fsr1_emu_tex.h"
namespace fsr1 {
#else
__device__ __forceinline__ uint2 tex_load8(unsigned long long t, int x, int y) {
  const ushort4 v = tex2D<ushort4>(t, (float)x + 0.5f, (float)y + 0.5f);
  return make_uint2((uint32_t)v.x | ((uint32_t)v.y << 16), (uint32_t)v.z | ((uint32_t)v.w << 16));
}
__device__ __forceinline__ uint32_t tex_load4(unsigned long long t, int x, int y) {
  return tex2D<unsigned int>(t, (float)x + 0.5f, (float)y + 0.5f);
}
#endif

// Where EASU's load stage reads the input from: a TMA tensor map over linear memory, or a CUDA array whose handle is ImgView::base,
// through a surface object (FSR1_FLAG_IN_SURFACE, RGBA16F) or a texture object (FSR1_FLAG_IN_TEXTURE, RGBA16F or R11G11B10F).
enum InSrc : int { kInTma = 0, kInSurf = 1, kInTex = 2 };
// The RGBA16F bits of an array input's texel at (x, y), which the caller clamped to the logical image: phase 1 of the array kernels.
template <int kIn, bool kR11>
__device__ __forceinline__ uint2 array_texel(unsigned long long h, int x, int y) {
  static_assert(kIn == kInTex || (kIn == kInSurf && !kR11), "surfaces carry RGBA16F only");
  if constexpr (kIn == kInSurf) return surf_load8(h, x, y);
  else if constexpr (kR11) return r11_to_half(tex_load4(h, x, y));
  else return tex_load8(h, x, y);
}

// ---- host helpers of the dispatch layer (fsr1_capi.cu, fsr1_shard.cu) -----------------------------------------------------
inline int bytes_per_pixel(uint32_t fmt) {  // 0: not a format include/fsr1_b200.h defines
  switch (fmt) {
    case FSR1_FORMAT_RGBA16F: return 8;
    case FSR1_FORMAT_RGBA32F: return 16;
    case FSR1_FORMAT_RGBA8_UNORM: case FSR1_FORMAT_RGB10A2_UNORM: case FSR1_FORMAT_R11G11B10_FLOAT: return 4;
    default: return 0;
  }
}
// The format of the image EASU writes from an input of format `fmt`: R11G11B10_FLOAT is an input format only, its EASU output (and
// every intermediate and output after it) is RGBA16F, the exact superset of its values.
inline uint32_t easu_out_format(uint32_t fmt) { return fmt == FSR1_FORMAT_R11G11B10_FLOAT ? (uint32_t)FSR1_FORMAT_RGBA16F : fmt; }
inline float word_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }  // a constant word of FsrEasuCon / FsrRcasCon
struct Rows { uint32_t a, b; };  // [a, b)
// The rows EASU writes for output rows [y0, y1) of an image out_h rows tall, and the rows RCAS reads for them: one more on each side
// inside the image.  So a row slab's EASU produces the apron its RCAS reads, and needs no second exchange.
inline Rows easu_rows(uint32_t y0, uint32_t y1, uint32_t out_h) { return Rows{y0 == 0 ? 0 : y0 - 1, y1 >= out_h ? out_h : y1 + 1}; }

void set_last_detail(int v);  // fsr1_capi.cu: detail word reported by fsr1_last_cuda_error()
// fsr1_capi.cu -> fsr1_shard.cu: the rules fsr1_upscale_post applies to the post description (ops, tiles), the formats and the flags,
// with the error it would return; no CUDA call.  The frame's images (sizes, windows, alignment) are checked by each launch.
int post_rules(const ::fsr1_post* post, uint32_t in_format, uint32_t out_format, uint32_t flags);
// fsr1_capi.cu -> fsr1_shard.cu: fsr1_easu, fsr1_upscale and fsr1_upscale_post (which call them with nulls) for a frame of a sharded
// stream.  `sync`: the neighbour hand-shake the EASU (or fused) kernel is to carry; null outside the sharded path.  *sync_taken is set
// to true when a kernel that carries it launched (the TMA-tiled fp16 and the fused kernels do), and left alone otherwise: the shard
// then runs its own tiny wait / signal kernels around the frame.  sync_taken may be null when sync is.
int easu(const ::fsr1_image* in, const ::fsr1_image* out, const uint32_t con[16], uint32_t y0, uint32_t y1, uint32_t flags, void* stream,
         const HaloSync* sync, bool* sync_taken);
int upscale(const ::fsr1_image* in, const ::fsr1_image* tmp, const ::fsr1_image* out, const uint32_t easu_con[16],
            const uint32_t rcas_con[4], uint32_t y0, uint32_t y1, uint32_t flags, void* stream, const HaloSync* sync, bool* sync_taken);
int upscale_post(const ::fsr1_image* in, const ::fsr1_image* tmp, const ::fsr1_image* out, const uint32_t easu_con[16],
                 const uint32_t rcas_con[4], const ::fsr1_post* post, uint32_t y0, uint32_t y1, uint32_t flags, void* stream,
                 const HaloSync* sync, bool* sync_taken);

// launchers (defined in the .cu files, called from fsr1_capi.cu)
cudaError_t launch_easu_direct(const EasuParams& p, int format, bool exact, cudaStream_t s, const char** name);
cudaError_t launch_rcas_direct(const RcasParams& p, int format, bool exact, cudaStream_t s, const char** name);
// Packed-half production kernels.  Return cudaErrorNotSupported when the image layout does not
// meet their alignment needs (the caller then falls back to the direct kernels).  srtm_in: FSR1_FLAG_SRTM_INPUT (the caller
// must not fall back then: no other kernel applies it).
// r11: the input is R11G11B10_FLOAT (the output RGBA16F); no fall-back either (launch_easu_direct decodes the format itself).
// in: kInSurf (FSR1_FLAG_IN_SURFACE), p.in.base is a surface object on an RGBA16F array; kInTex (FSR1_FLAG_IN_TEXTURE), a texture object
// on an RGBA16F or (r11) R11G11B10F array.  surf_out (FSR1_FLAG_OUT_SURFACE): p.out.base is a surface object.  No fall-back for any of
// them: no other kernel reads an array or writes a surface.
cudaError_t launch_easu_h_tiled(const EasuParams& p, cudaStream_t s, const char** name, bool srtm_in = false, bool r11 = false,
                                InSrc in = kInTma);
cudaError_t launch_rcas_h_packed(const RcasParams& p, cudaStream_t s, const char** name, bool surf_out = false);
// UNORM images through the TMA-tiled 2x EASU / packed RCAS kernels: cudaErrorNotSupported when not applicable
cudaError_t launch_easu_u_tiled(const EasuParams& p, int format, cudaStream_t s, const char** name);
cudaError_t launch_rcas_u_packed(const RcasParams& p, int format, cudaStream_t s, const char** name);
// EASU -> RCAS in one kernel (RGBA16F, exactly 2x, out-of-image taps read 0): e.in = input, e.out = final output, rows [e.y0, e.y1)
cudaError_t launch_fused_h(const EasuParams& e, uint32_t sharp_h2, int clamp, cudaStream_t s, const char** name, bool srtm_in = false,
                           bool r11 = false, InSrc in = kInTma, bool surf_out = false);
cudaError_t launch_easu_f32_tiled(const EasuParams& p, cudaStream_t s, const char** name);  // RGBA32F, exactly 2x
cudaError_t launch_easu_h_precise(const EasuParams& p, cudaStream_t s, const char** name);  // RGBA16F io, fp32 math, 2x
cudaError_t launch_rcas_f32_packed(const RcasParams& p, cudaStream_t s, const char** name);
// Literal FsrEasuH / FsrRcasH semantics, bit-identical to the reference's packed-half source (parity path).
cudaError_t launch_easu_href(const EasuParams& p, cudaStream_t s, const char** name);
cudaError_t launch_rcas_href(const RcasParams& p, cudaStream_t s, const char** name);
// The packed Hx2 calling convention (fsr1_hx2.cu): two pixels per lane in half2 SoA registers, bit-identical to the H source.
cudaError_t launch_rcas_hx2(const RcasParams& p, cudaStream_t s, const char** name);
cudaError_t launch_pointwise_hx2(int op, const ImgView& in, const ImgView& out, const ImgView* aux, float amount, uint32_t frame, int y0,
                                 int y1, cudaStream_t s, const char** name);

// Pointwise companions (fsr1_pointwise.cu): op 1 SRTM, 2 SRTM inverse, 3 LFGA, 4 TEPD 8 bit, 5 TEPD 10 bit, 6 square.
cudaError_t launch_pointwise(int op, const ImgView& in, int in_format, const ImgView& out, int out_format, const ImgView* aux,
                             int aux_format, float amount, uint32_t frame, int y0, int y1, cudaStream_t s, const char** name);

}  // namespace fsr1
