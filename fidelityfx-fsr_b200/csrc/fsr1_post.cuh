// fsr1_post.cuh — the fp32 arithmetic of the pointwise companions (SRTM / SRTM inverse, LFGA, TEPD; fsr1_pointwise.cu) and the
// display epilogue that applies them inside RCAS's store (fsr1_upscale_post: fsr1_fused.cu, fsr1_rcas_packed.cu).  The formulas
// exist only here, so the epilogue computes the bits the separate passes compute.
//
// Policy (EXACT): separate roundings, IEEE sqrt and division, bit-identical to the reference source compiled with
// -ffp-contract=off.  The epilogue rounds to half between steps, as the separate passes round on their RGBA16F store.
#pragma once
#include <type_traits>
#include "fsr1_common.cuh"

namespace fsr1 {

enum { kOpSrtm = 1, kOpSrtmInv = 2, kOpLfga = 3, kOpTepd8 = 4, kOpTepd10 = 5, kOpSquare = 6 };

template <typename S> __device__ __forceinline__ float4 load4(const ImgView& im, int x, int y);
template <> __device__ __forceinline__ float4 load4<float>(const ImgView& im, int x, int y) {
  return __ldg(reinterpret_cast<const float4*>(im.base + (long long)(y - im.row0) * im.pitch) + x);
}
template <> __device__ __forceinline__ float4 load4<__half>(const ImgView& im, int x, int y) {
  const uint2 v = __ldg(reinterpret_cast<const uint2*>(im.base + (long long)(y - im.row0) * im.pitch) + x);
  const float2 rg = __half22float2(*reinterpret_cast<const __half2*>(&v.x));
  const float2 ba = __half22float2(*reinterpret_cast<const __half2*>(&v.y));
  return make_float4(rg.x, rg.y, ba.x, ba.y);
}
template <> __device__ __forceinline__ float4 load4<Unorm8>(const ImgView& im, int x, int y) {
  const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(im.base + (long long)(y - im.row0) * im.pitch) + x);
  return make_float4(__fdiv_rn((float)(v & 255u), 255.0f), __fdiv_rn((float)((v >> 8) & 255u), 255.0f),
                     __fdiv_rn((float)((v >> 16) & 255u), 255.0f), __fdiv_rn((float)(v >> 24), 255.0f));
}
template <> __device__ __forceinline__ float4 load4<Unorm10>(const ImgView& im, int x, int y) {
  const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(im.base + (long long)(y - im.row0) * im.pitch) + x);
  return make_float4(__fdiv_rn((float)(v & 1023u), 1023.0f), __fdiv_rn((float)((v >> 10) & 1023u), 1023.0f),
                     __fdiv_rn((float)((v >> 20) & 1023u), 1023.0f), __fdiv_rn((float)(v >> 30), 3.0f));
}

// aux tiles (grain, dither) are small and L1/L2-resident: runtime format; (x, y) already wrapped into the tile
__device__ __forceinline__ float4 load_aux(const ImgView& im, int fmt, int x, int y) {
  switch (fmt) {
    case 1: return load4<__half>(im, x, y);
    case 2: return load4<float>(im, x, y);
    case 3: return load4<Unorm8>(im, x, y);
    default: return load4<Unorm10>(im, x, y);
  }
}

// APrxMedRcpF1 (ffx-fsr/ffx_a.h:1844), separate roundings; the integer subtract wraps for negative arguments
__device__ __forceinline__ float prx_med_rcp_exact(float a) {
  const float b = __uint_as_float(0x7ef19fffu - __float_as_uint(a));
  return __fmul_rn(b, __fadd_rn(__fmul_rn(-b, a), 2.0f));
}

__device__ __forceinline__ float tepd_dit(uint32_t px, uint32_t py, uint32_t frame) {
  const float x = (float)(px + frame), y = (float)py;
  const float a = 1.61803398874989484820f, b = (float)(1.0 / 3.69);
  const float v = __fadd_rn(__fmul_rn(x, a), __fmul_rn(y, b));
  return __fsub_rn(v, floorf(v));
}

__device__ __forceinline__ float tepd_channel(float c, float dit, float q, float rq) {
  float n = __fsqrt_rn(c);
  n = __fmul_rn(floorf(__fmul_rn(n, q)), rq);
  const float a = __fmul_rn(n, n);
  float b = __fadd_rn(n, rq);
  b = __fmul_rn(b, b);
  const float r = __fmul_rn(__fsub_rn(c, b), prx_med_rcp_exact(__fsub_rn(a, b)));
  // AGtZeroF1(m) = saturate(m * +INF): 1 for m > 0, else 0 (0 * INF = NaN saturates to 0)
  const float gt = sat(__fmul_rn(__fsub_rn(dit, r), __uint_as_float(0x7f800000u)));
  return sat(__fadd_rn(n, __fmul_rn(gt, rq)));
}

// One pointwise step on pixel (x, y).  (ax, ay) = (x mod aux width, y mod aux height), maintained by the caller.
__device__ __forceinline__ float4 apply_op(int op, float4 c, const ImgView& aux, int aux_format, float amount, uint32_t frame, int x,
                                           int y, int ax, int ay) {
  switch (op) {
    case kOpSrtm: {
      const float r = __fdiv_rn(1.0f, __fadd_rn(fmaxf(c.x, fmaxf(c.y, c.z)), 1.0f));
      return make_float4(__fmul_rn(c.x, r), __fmul_rn(c.y, r), __fmul_rn(c.z, r), c.w);
    }
    case kOpSrtmInv: {
      const float r = __fdiv_rn(1.0f, fmaxf((float)(1.0 / 32768.0), __fsub_rn(1.0f, fmaxf(c.x, fmaxf(c.y, c.z)))));
      return make_float4(__fmul_rn(c.x, r), __fmul_rn(c.y, r), __fmul_rn(c.z, r), c.w);
    }
    case kOpLfga: {
      const float4 t = load_aux(aux, aux_format, ax, ay);
      const float a = amount;
      return make_float4(__fadd_rn(c.x, __fmul_rn(__fmul_rn(t.x, a), fminf(__fsub_rn(1.0f, c.x), c.x))),
                         __fadd_rn(c.y, __fmul_rn(__fmul_rn(t.y, a), fminf(__fsub_rn(1.0f, c.y), c.y))),
                         __fadd_rn(c.z, __fmul_rn(__fmul_rn(t.z, a), fminf(__fsub_rn(1.0f, c.z), c.z))), c.w);
    }
    case kOpTepd8:
    case kOpTepd10: {
      const float q = op == kOpTepd8 ? 255.0f : 1023.0f;
      const float rq = op == kOpTepd8 ? (float)(1.0 / 255.0) : (float)(1.0 / 1023.0);
      const float dit = aux_format ? sat(load_aux(aux, aux_format, ax, ay).w) : tepd_dit((uint32_t)x, (uint32_t)y, frame);
      return make_float4(tepd_channel(c.x, dit, q, rq), tepd_channel(c.y, dit, q, rq), tepd_channel(c.z, dit, q, rq), c.w);
    }
    default:  // kOpSquare
      return make_float4(__fmul_rn(c.x, c.x), __fmul_rn(c.y, c.y), __fmul_rn(c.z, c.z), c.w);
  }
}

// ---- FSR1_FLAG_SRTM_INPUT: FsrSrtmF as the EASU kernels load each texel ------------------------------------------------------------
// One RGBA16F texel -> fp32 -> FsrSrtmF -> rounded once to half: the texel fsr1_srtm(in, I, 0) writes into an RGBA16F image I.
__device__ __forceinline__ uint2 srtm_texel(uint2 t) {
  const float2 rg = __half22float2(*reinterpret_cast<const __half2*>(&t.x));
  const float2 ba = __half22float2(*reinterpret_cast<const __half2*>(&t.y));
  const float4 c = apply_op(kOpSrtm, make_float4(rg.x, rg.y, ba.x, ba.y), ImgView{}, 0, 0.0f, 0u, 0, 0, 0, 0);
  const __half2 o0 = __floats2half2_rn(c.x, c.y), o1 = __floats2half2_rn(c.z, c.w);
  return make_uint2(*reinterpret_cast<const uint32_t*>(&o0), *reinterpret_cast<const uint32_t*>(&o1));
}

// ---- the display epilogue of fsr1_upscale_post ---------------------------------------------------------------------------
// ops bits: FSR1_POST_* of include/fsr1_b200.h, applied in this order
enum { kPostSrtmInv = 1, kPostLfga = 2, kPostTepd8 = 4, kPostTepd10 = 8 };

struct PostParams {
  ImgView grain, dither;  // whole tiles (row0 = 0); an unused tile is described as 1 x 1 so that its cursor wraps harmlessly
  int grain_fmt;
  int dither_fmt;         // 0: FsrTepdDitF(pixel, frame)
  int ops;
  float amount;
  uint32_t frame;
};

// A lane's pixel pair (x, x+1) inside the grain and dither tiles: columns fixed for the lane, the row advances by one per output
// row (two divisions when the lane starts a run of rows, none per pixel).
struct PostCursor {
  int gx0, gx1, gy, dx0, dx1, dy;
  __device__ __forceinline__ void init(const PostParams& q, int x, int y) {
    x = x < 0 ? 0 : x;  // lanes left of the image only feed their neighbours; they never store
    gx0 = x % q.grain.w;
    gx1 = gx0 + 1 == q.grain.w ? 0 : gx0 + 1;
    gy = y % q.grain.h;
    if (gy < 0) gy += q.grain.h;
    dx0 = x % q.dither.w;
    dx1 = dx0 + 1 == q.dither.w ? 0 : dx0 + 1;
    dy = y % q.dither.h;
    if (dy < 0) dy += q.dither.h;
  }
  __device__ __forceinline__ void next_row(const PostParams& q) {
    if (++gy == q.grain.h) gy = 0;
    if (++dy == q.dither.h) dy = 0;
  }
};

// the RGBA16F store of the separate passes: round (c0, c1) of one channel to half and back
__device__ __forceinline__ void round_half(float& a, float& b) {
  const float2 r = __half22float2(__floats2half2_rn(a, b));
  a = r.x;
  b = r.y;
}

__device__ __forceinline__ void post_steps(const PostParams& q, float4& c0, float4& c1, int x, int y, const PostCursor& k) {
  if (q.ops & kPostSrtmInv) {  // warp-uniform
    c0 = apply_op(kOpSrtmInv, c0, q.grain, 0, 0.0f, 0u, x, y, 0, 0);
    c1 = apply_op(kOpSrtmInv, c1, q.grain, 0, 0.0f, 0u, x + 1, y, 0, 0);
    round_half(c0.x, c1.x); round_half(c0.y, c1.y); round_half(c0.z, c1.z);
  }
  if (q.ops & kPostLfga) {
    c0 = apply_op(kOpLfga, c0, q.grain, q.grain_fmt, q.amount, 0u, x, y, k.gx0, k.gy);
    c1 = apply_op(kOpLfga, c1, q.grain, q.grain_fmt, q.amount, 0u, x + 1, y, k.gx1, k.gy);
    round_half(c0.x, c1.x); round_half(c0.y, c1.y); round_half(c0.z, c1.z);
  }
  if (q.ops & (kPostTepd8 | kPostTepd10)) {
    const int op = (q.ops & kPostTepd8) ? kOpTepd8 : kOpTepd10;
    c0 = apply_op(op, c0, q.dither, q.dither_fmt, 0.0f, q.frame, x, y, k.dx0, k.dy);
    c1 = apply_op(op, c1, q.dither, q.dither_fmt, 0.0f, q.frame, x + 1, y, k.dx1, k.dy);
  }
}

// Output store of the epilogue for the pixel pair (x, x+1): SO = __half (RGBA16F, 16 B), Unorm8 or Unorm10 (8 B).  `both`: x+1 is
// inside the image.  The encodings are Px<SO>::store's.  store_surf: the same bytes through a surface object, one store per pixel.
template <typename SO> struct PostStore;
template <> struct PostStore<void> { static constexpr int kBytes = 8; };  // no epilogue: the RGBA16F store of RCAS itself
template <> struct PostStore<__half> {
  static constexpr int kBytes = 8;
  static __device__ __forceinline__ void store(unsigned char* o, float4 c0, float4 c1, bool both) {
    const __half2 rg0 = __floats2half2_rn(c0.x, c0.y), ba0 = __floats2half2_rn(c0.z, c0.w);
    const __half2 rg1 = __floats2half2_rn(c1.x, c1.y), ba1 = __floats2half2_rn(c1.z, c1.w);
    const uint4 w = make_uint4(*reinterpret_cast<const uint32_t*>(&rg0), *reinterpret_cast<const uint32_t*>(&ba0),
                               *reinterpret_cast<const uint32_t*>(&rg1), *reinterpret_cast<const uint32_t*>(&ba1));
    if (both) *reinterpret_cast<uint4*>(o) = w;
    else *reinterpret_cast<uint2*>(o) = make_uint2(w.x, w.y);
  }
  static __device__ __forceinline__ void store_surf(unsigned long long s, int x, int y, float4 c0, float4 c1, bool both) {
    const __half2 rg0 = __floats2half2_rn(c0.x, c0.y), ba0 = __floats2half2_rn(c0.z, c0.w);
    surf_store8(s, x, y, make_uint2(*reinterpret_cast<const uint32_t*>(&rg0), *reinterpret_cast<const uint32_t*>(&ba0)));
    if (both) {
      const __half2 rg1 = __floats2half2_rn(c1.x, c1.y), ba1 = __floats2half2_rn(c1.z, c1.w);
      surf_store8(s, x + 1, y, make_uint2(*reinterpret_cast<const uint32_t*>(&rg1), *reinterpret_cast<const uint32_t*>(&ba1)));
    }
  }
};
template <> struct PostStore<Unorm8> {
  static constexpr int kBytes = 4;
  static __device__ __forceinline__ uint32_t enc(float4 c) {
    return to_unorm(c.x, 255.0f) | (to_unorm(c.y, 255.0f) << 8) | (to_unorm(c.z, 255.0f) << 16) | (to_unorm(c.w, 255.0f) << 24);
  }
  static __device__ __forceinline__ void store(unsigned char* o, float4 c0, float4 c1, bool both) {
    if (both) *reinterpret_cast<uint2*>(o) = make_uint2(enc(c0), enc(c1));
    else *reinterpret_cast<uint32_t*>(o) = enc(c0);
  }
  static __device__ __forceinline__ void store_surf(unsigned long long s, int x, int y, float4 c0, float4 c1, bool both) {
    surf_store4(s, x, y, enc(c0));
    if (both) surf_store4(s, x + 1, y, enc(c1));
  }
};
template <> struct PostStore<Unorm10> {
  static constexpr int kBytes = 4;
  static __device__ __forceinline__ uint32_t enc(float4 c) {
    return to_unorm(c.x, 1023.0f) | (to_unorm(c.y, 1023.0f) << 10) | (to_unorm(c.z, 1023.0f) << 20) | (to_unorm(c.w, 3.0f) << 30);
  }
  static __device__ __forceinline__ void store(unsigned char* o, float4 c0, float4 c1, bool both) {
    if (both) *reinterpret_cast<uint2*>(o) = make_uint2(enc(c0), enc(c1));
    else *reinterpret_cast<uint32_t*>(o) = enc(c0);
  }
  static __device__ __forceinline__ void store_surf(unsigned long long s, int x, int y, float4 c0, float4 c1, bool both) {
    surf_store4(s, x, y, enc(c0));
    if (both) surf_store4(s, x + 1, y, enc(c1));
  }
};

// RCAS result of the pair (SoA half2, alpha = (A0, A1) as half2 bits, exactly what the RGBA16F store would write) -> post steps ->
// the output store.  y: the logical output row; k: the pair's tile positions on that row.  o: the pair's address, or with kSurfOut
// the output's ImgView::base (the surface object), stored to at (x, y).
template <typename SO, bool kSurfOut = false>
__device__ __forceinline__ void post_pair(const PostParams& q, const PostCursor& k, unsigned char* o, int x, int y, __half2 oR, __half2 oG,
                                          __half2 oB, uint32_t alpha, bool both) {
  const float2 r = __half22float2(oR), g = __half22float2(oG), b = __half22float2(oB);
  const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&alpha));
  float4 c0 = make_float4(r.x, g.x, b.x, a.x), c1 = make_float4(r.y, g.y, b.y, a.y);
  post_steps(q, c0, c1, x, y, k);
  if constexpr (kSurfOut) PostStore<SO>::store_surf((unsigned long long)o, x, y, c0, c1, both);
  else PostStore<SO>::store(o, c0, c1, both);
}

// launchers (fsr1_fused.cu, fsr1_rcas_packed.cu); out_format 1 RGBA16F, 3 RGBA8_UNORM, 4 RGB10A2_UNORM.  cudaErrorNotSupported: the
// frame or layout is not one the kernel takes (nothing launched).
// in / surf_out: FSR1_FLAG_IN_SURFACE or IN_TEXTURE / OUT_SURFACE (e.in holds the array's surface or texture object, p.out a surface
// object; no fall-back when declined).
cudaError_t launch_fused_h_post(const EasuParams& e, uint32_t sharp_h2, const PostParams& q, int out_format, cudaStream_t s,
                                const char** name, bool srtm_in = false, bool r11 = false, InSrc in = kInTma, bool surf_out = false);
cudaError_t launch_rcas_h_post(const RcasParams& p, const PostParams& q, int out_format, cudaStream_t s, const char** name,
                               bool surf_out = false);
// fsr1_rcas_post's input stage: p.in is R11G11B10_FLOAT (r11, 8-byte aligned) or RGBA16F (16-byte aligned), read through FsrSrtmF with
// srtm; then RCAS and the RGBA16F store (q null) or the epilogue q into out_format.  The rest as launch_rcas_h_post.
cudaError_t launch_rcas_h_in(const RcasParams& p, const PostParams* q, int out_format, bool r11, bool srtm, cudaStream_t s, const char** name,
                             bool surf_out = false);

}  // namespace fsr1
