// fsr1_rcas_packed.cu — the production RCAS kernels for RGBA16F and UNORM images on sm_90a.
//
// RCAS is a 5-tap cross (b above, d left, e centre, f right, h below; ffx-fsr/ffx_fsr1.h:693-707) with 16
// bytes of compulsory traffic per pixel (8 for the UNORM formats): the HBM-bound half of the path.  The kernel is
// organised around the memory system and the issue slots, not shared memory:
//   * a lane owns TWO horizontally adjacent pixels (one 128-bit load and one 128-bit store per row; 64-bit for the
//     4-byte UNORM texels) and walks kRows rows downwards with a rolling 3-row register window;
//   * left/right neighbours (d, f) come from the adjacent lanes by warp shuffle.  A warp loads a 64-pixel
//     span but produces only its inner 60 pixels: lanes 0 and 31 exist to feed their neighbours, so there is
//     no per-row edge fetch and no divergence (spans overlap by 4 pixels; the re-read hits L1/L2);
//   * warps whose span and rows lie strictly inside the image take a path with no bounds checks at all;
//   * arithmetic is half2 over the lane's two pixels (fsr1_rcas_math.cuh), the reference's compile-time options
//     (FSR_RCAS_DENOISE, FSR_RCAS_PASSTHROUGH_ALPHA) and the sample's Sample.x output hook are template bits of THIS
//     kernel: no fallback to a slower kernel, no extra pass.
// UNORM texels are decoded to the same (pixel0, pixel1)-per-channel half2 form (c / (2^n - 1) in fp32, one rounding to
// half) and the saturated result is re-encoded in the half domain (x * (2^n - 1) + 1024 leaves round(x * (2^n - 1)) in the
// low mantissa bits).
#include "fsr1_post.cuh"
#include "fsr1_rcas_math.cuh"

namespace fsr1 {

constexpr int kNW = 4;     // warps per CTA, stacked vertically: CTA = 60 x (kNW*kRows) output pixels
constexpr int kRows = 4;   // rows walked by one lane
constexpr int kSpan = 60;  // output pixels per warp per row (lanes 1..30)

// ---- storage formats: how a lane's two pixels are fetched, decoded, encoded and stored --------------------------------
struct FmtHalf {  // RGBA16F, 8 B per pixel
  static constexpr int kBpp = 8;
  static constexpr bool kClampArg = false;  // RCAS_CLAMP is the kernel's template bit (InStage, fsr1_rcas_in.cu: p.clamp)
  typedef uint4 Raw;
  static __device__ __forceinline__ Raw zero() { return make_uint4(0u, 0u, 0u, 0u); }
  static __device__ __forceinline__ Raw load2(const unsigned char* a) { return __ldg(reinterpret_cast<const uint4*>(a)); }
  static __device__ __forceinline__ Raw load11(const unsigned char* a0, const unsigned char* a1) {  // either may be null (-> 0)
    uint4 v = zero();
    if (a0) { const uint2 t = __ldg(reinterpret_cast<const uint2*>(a0)); v.x = t.x; v.y = t.y; }
    if (a1) { const uint2 t = __ldg(reinterpret_cast<const uint2*>(a1)); v.z = t.x; v.w = t.y; }
    return v;
  }
  static __device__ __forceinline__ Row3 decode(Raw v) {  // AoS (RG0,BA0,RG1,BA1) -> SoA
    Row3 o;
    o.r = uh2(__byte_perm(v.x, v.z, 0x5410));
    o.g = uh2(__byte_perm(v.x, v.z, 0x7632));
    o.b = uh2(__byte_perm(v.y, v.w, 0x5410));
    return o;
  }
  static __device__ __forceinline__ uint32_t alpha(Raw v) { return __byte_perm(v.y, v.w, 0x7632); }  // (A0,A1) as half2 bits
  static __device__ __forceinline__ uint32_t opaque() { return 0x3c003c00u; }
  static __device__ __forceinline__ void store(unsigned char* o, __half2 oR, __half2 oG, __half2 oB, uint32_t a, bool both) {
    const uint4 w = pack_pair_half(oR, oG, oB, a);
    if (both) *reinterpret_cast<uint4*>(o) = w;
    else *reinterpret_cast<uint2*>(o) = make_uint2(w.x, w.y);
  }
  // FSR1_FLAG_OUT_SURFACE: the same bytes through the surface object s, one 8-byte store per pixel
  static __device__ __forceinline__ void store_surf(unsigned long long s, int x, int y, __half2 oR, __half2 oG, __half2 oB, uint32_t a,
                                                    bool both) {
    const uint4 w = pack_pair_half(oR, oG, oB, a);
    surf_store8(s, x, y, make_uint2(w.x, w.y));
    if (both) surf_store8(s, x + 1, y, make_uint2(w.z, w.w));
  }
};

template <int kBits> struct FmtUnorm {  // R8G8B8A8_UNORM (8) / R10G10B10A2_UNORM (10), 4 B per pixel
  static constexpr int kBpp = 4;
  static constexpr bool kClampArg = false;
  typedef uint2 Raw;
  static __device__ __forceinline__ Raw zero() { return make_uint2(0u, 0u); }
  static __device__ __forceinline__ Raw load2(const unsigned char* a) { return __ldg(reinterpret_cast<const uint2*>(a)); }
  static __device__ __forceinline__ Raw load11(const unsigned char* a0, const unsigned char* a1) {
    uint2 v = zero();
    if (a0) v.x = __ldg(reinterpret_cast<const uint32_t*>(a0));
    if (a1) v.y = __ldg(reinterpret_cast<const uint32_t*>(a1));
    return v;
  }
  static __device__ __forceinline__ Row3 decode(Raw v) {
    Row3 o;
    if (kBits == 8) {
      const float s = 255.0f, k = 1.0f / 255.0f;
      o.r = __floats2half2_rn(unorm_to_float(v.x & 255u, s, k), unorm_to_float(v.y & 255u, s, k));
      o.g = __floats2half2_rn(unorm_to_float((v.x >> 8) & 255u, s, k), unorm_to_float((v.y >> 8) & 255u, s, k));
      o.b = __floats2half2_rn(unorm_to_float((v.x >> 16) & 255u, s, k), unorm_to_float((v.y >> 16) & 255u, s, k));
    } else {
      const float s = 1023.0f, k = 1.0f / 1023.0f;
      o.r = __floats2half2_rn(unorm_to_float(v.x & 1023u, s, k), unorm_to_float(v.y & 1023u, s, k));
      o.g = __floats2half2_rn(unorm_to_float((v.x >> 10) & 1023u, s, k), unorm_to_float((v.y >> 10) & 1023u, s, k));
      o.b = __floats2half2_rn(unorm_to_float((v.x >> 20) & 1023u, s, k), unorm_to_float((v.y >> 20) & 1023u, s, k));
    }
    return o;
  }
  // alpha codes of the two pixels, passed through untouched: (A0 | A1 << 16)
  static __device__ __forceinline__ uint32_t alpha(Raw v) {
    return kBits == 8 ? ((v.x >> 24) | ((v.y >> 24) << 16)) : ((v.x >> 30) | ((v.y >> 30) << 16));
  }
  static __device__ __forceinline__ uint32_t opaque() { return kBits == 8 ? 0x00ff00ffu : 0x00030003u; }
  static __device__ __forceinline__ void store(unsigned char* o, __half2 r, __half2 g, __half2 b, uint32_t a, bool both) {
    const __half2 one = __float2half2_rn(1.0f), zero = __float2half2_rn(0.0f);
    r = __hmin2(one, __hmax2(zero, r));  // saturate to [0,1] for the encode (a UNORM store clamps anyway)
    g = __hmin2(one, __hmax2(zero, g));
    b = __hmin2(one, __hmax2(zero, b));
    const __half2 sc = __float2half2_rn(kBits == 8 ? 255.0f : 1023.0f), k1024 = __float2half2_rn(1024.0f);
    const uint32_t tr = hu2(__hfma2(r, sc, k1024)), tg = hu2(__hfma2(g, sc, k1024)), tb = hu2(__hfma2(b, sc, k1024));
    uint2 w;
    if (kBits == 8) {
      const uint32_t rg0 = __byte_perm(tr, tg, 0x0040), rg1 = __byte_perm(tr, tg, 0x0062);  // (R, G) of pixel 0 / pixel 1
      const uint32_t ba0 = __byte_perm(tb, a, 0x0040), ba1 = __byte_perm(tb, a, 0x0062);     // (B, A)
      w = make_uint2(__byte_perm(rg0, ba0, 0x5410), __byte_perm(rg1, ba1, 0x5410));
    } else {
      w = make_uint2((tr & 0x3ffu) | ((tg & 0x3ffu) << 10) | ((tb & 0x3ffu) << 20) | ((a & 3u) << 30),
                     ((tr >> 16) & 0x3ffu) | (((tg >> 16) & 0x3ffu) << 10) | (((tb >> 16) & 0x3ffu) << 20) | (((a >> 16) & 3u) << 30));
    }
    if (both) *reinterpret_cast<uint2*>(o) = w;
    else *reinterpret_cast<uint32_t*>(o) = w.x;
  }
};

// IN = FM: the pair as loaded; otherwise IN's input stage (InStage, fsr1_rcas_in.cu) turns it into FM's (FmtHalf's) texels
template <typename FM, typename IN>
__device__ __forceinline__ typename FM::Raw in_texels(typename IN::Raw v, bool srtm) {
  if constexpr (std::is_same<FM, IN>::value) return v;
  else return IN::texels(v, srtm);
}

// Pixels (x, x+1) of logical row y with the out-of-image rule applied (0, or clamp with kClamp, or with p.clamp for FM::kClampArg).
// Rows outside the STORED window are never used (they are prefetched past the row range of a slab) and read as 0.
template <typename FM, bool kClamp>
__device__ __forceinline__ typename FM::Raw load_checked(const RcasParams& p, int x, int y) {
  const bool clamp = kClamp || (FM::kClampArg && p.clamp);
  if (clamp) y = clampi(y, 0, p.in.h - 1);
  if (!row_stored(p.in, y)) return FM::zero();
  const unsigned char* row = p.in.base + (long long)(y - p.in.row0) * p.in.pitch;
  if (x >= 0 && x + 1 < p.in.w) return FM::load2(row + (long long)x * FM::kBpp);
  if (clamp) return FM::load11(row + (long long)clampi(x, 0, p.in.w - 1) * FM::kBpp, row + (long long)clampi(x + 1, 0, p.in.w - 1) * FM::kBpp);
  return FM::load11(x >= 0 && x < p.in.w ? row + (long long)x * FM::kBpp : nullptr,
                    x + 1 >= 0 && x + 1 < p.in.w ? row + (long long)(x + 1) * FM::kBpp : nullptr);
}

// SO: void = FM's own store; otherwise the display epilogue of fsr1_upscale_post (post_pair, fsr1_post.cuh) with its store.
// kSurfOut (FSR1_FLAG_OUT_SURFACE, FmtHalf only): p.out.base is a surface object; each pixel is one surface store at (x, y).
// IN (FM = FmtHalf only): the input stage of fsr1_rcas_post (InStage, fsr1_rcas_in.cu), which reads p.in in its own format; srtm is
// its argument.
template <typename FM, bool kChecked, bool kClamp, int kOpt, typename SO = void, bool kSurfOut = false, typename IN = FM>
__device__ __forceinline__ void rcas_rows(const RcasParams& p, int x, int ys, int lane, const PostParams* q = nullptr, bool srtm = false) {
  constexpr bool kPost = !std::is_void<SO>::value;
  constexpr int kOutBpp = kPost ? PostStore<SO>::kBytes : FM::kBpp;
  const __half2 sharp = uh2(p.sharp_h2);
  const bool writer = lane >= 1 && lane <= 30 && (!kChecked || x < p.out.w);
  // all kRows+2 rows are requested up front: kRows+2 independent vector loads in flight per lane
  Row3 rows[kRows + 2];
  uint32_t alphas[kRows];  // kRcasAlpha only: the centre pixels' alpha
  if (!kChecked) {  // one 64-bit address, then += pitch: no per-row address arithmetic
    const unsigned char* src = p.in.base + (long long)(ys - 1 - p.in.row0) * p.in.pitch + (long long)x * IN::kBpp;
#pragma unroll
    for (int r = 0; r < kRows + 2; r++) {
      const typename FM::Raw v = in_texels<FM, IN>(IN::load2(src + (long long)r * p.in.pitch), srtm);
      rows[r] = FM::decode(v);
      if ((kOpt & kRcasAlpha) && r >= 1 && r <= kRows) alphas[r - 1] = FM::alpha(v);
    }
  } else {
#pragma unroll
    for (int r = 0; r < kRows + 2; r++) {
      const typename FM::Raw v = in_texels<FM, IN>(load_checked<IN, kClamp>(p, x, ys - 1 + r), srtm);
      rows[r] = FM::decode(v);
      if ((kOpt & kRcasAlpha) && r >= 1 && r <= kRows) alphas[r - 1] = FM::alpha(v);
    }
  }
  unsigned char* dst = p.out.base + (long long)(ys - p.out.row0) * p.out.pitch + (long long)x * kOutBpp;
  PostCursor pc;
  if constexpr (kPost) pc.init(*q, x, ys);
#pragma unroll
  for (int r = 0; r < kRows; r++) {
    const int y = ys + r;
    if (kChecked && y >= p.y1) break;  // warp-uniform
    const Row3 prev = rows[r], cur = rows[r + 1], next = rows[r + 2];
    // d = (left lane's pixel1, my pixel0), f = (my pixel1, right lane's pixel0)
    Row3 d, f;
    d.r = uh2(__byte_perm(__shfl_up_sync(0xffffffffu, hu2(cur.r), 1), hu2(cur.r), 0x5432));
    d.g = uh2(__byte_perm(__shfl_up_sync(0xffffffffu, hu2(cur.g), 1), hu2(cur.g), 0x5432));
    d.b = uh2(__byte_perm(__shfl_up_sync(0xffffffffu, hu2(cur.b), 1), hu2(cur.b), 0x5432));
    f.r = uh2(__byte_perm(hu2(cur.r), __shfl_down_sync(0xffffffffu, hu2(cur.r), 1), 0x5432));
    f.g = uh2(__byte_perm(hu2(cur.g), __shfl_down_sync(0xffffffffu, hu2(cur.g), 1), 0x5432));
    f.b = uh2(__byte_perm(hu2(cur.b), __shfl_down_sync(0xffffffffu, hu2(cur.b), 1), 0x5432));
    __half2 oR, oG, oB;
    rcas_pair<kOpt>(prev, d, cur, f, next, sharp, oR, oG, oB);
    if constexpr (kPost) {
      if (writer)
        post_pair<SO, kSurfOut>(*q, pc, kSurfOut ? p.out.base : dst + (long long)r * p.out.pitch, x, y, oR, oG, oB,
                                (kOpt & kRcasAlpha) ? alphas[r] : FM::opaque(), !kChecked || x + 1 < p.out.w);
      pc.next_row(*q);
    } else if (writer) {
      if constexpr (kSurfOut)
        FM::store_surf(surf_of(p.out), x, y, oR, oG, oB, (kOpt & kRcasAlpha) ? alphas[r] : FM::opaque(), !kChecked || x + 1 < p.out.w);
      else
        FM::store(dst + (long long)r * p.out.pitch, oR, oG, oB, (kOpt & kRcasAlpha) ? alphas[r] : FM::opaque(), !kChecked || x + 1 < p.out.w);
    }
  }
}

template <typename FM, bool kClamp, int kOpt>
__global__ void __launch_bounds__(32 * kNW) rcas_packed_kernel(const RcasParams p) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int x0 = blockIdx.x * kSpan - 2;  // even -> every lane's pair is aligned for its vector access
  const int x = x0 + lane * 2;
  const int ys = p.y0 + (blockIdx.y * kNW + warp) * kRows;
  if (ys >= p.y1) return;  // whole warp
  const bool interior = x0 >= 0 && x0 + 64 <= p.in.w && ys >= 1 && ys + kRows < p.in.h && ys + kRows <= p.y1;
  if (interior)
    rcas_rows<FM, false, kClamp, kOpt>(p, x, ys, lane);
  else
    rcas_rows<FM, true, kClamp, kOpt>(p, x, ys, lane);
}

// fsr1_upscale_post: RCAS of an RGBA16F intermediate with the display epilogue in the store (SO: __half, Unorm8, Unorm10)
template <bool kClamp, int kOpt, typename SO>
__global__ void __launch_bounds__(32 * kNW) rcas_post_kernel(const RcasParams p, const __grid_constant__ PostParams q) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int x0 = blockIdx.x * kSpan - 2;
  const int x = x0 + lane * 2;
  const int ys = p.y0 + (blockIdx.y * kNW + warp) * kRows;
  if (ys >= p.y1) return;  // whole warp
  const bool interior = x0 >= 0 && x0 + 64 <= p.in.w && ys >= 1 && ys + kRows < p.in.h && ys + kRows <= p.y1;
  if (interior)
    rcas_rows<FmtHalf, false, kClamp, kOpt, SO>(p, x, ys, lane, &q);
  else
    rcas_rows<FmtHalf, true, kClamp, kOpt, SO>(p, x, ys, lane, &q);
}

// FSR1_FLAG_OUT_SURFACE: the two kernels above writing p.out through a surface object (SO = void: rcas_packed_kernel<FmtHalf, ...>)
template <bool kClamp, int kOpt, typename SO>
__global__ void __launch_bounds__(32 * kNW) rcas_surf_out_kernel(const RcasParams p, const __grid_constant__ PostParams q) {
  constexpr bool kPost = !std::is_void<SO>::value;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int x0 = blockIdx.x * kSpan - 2;
  const int x = x0 + lane * 2;
  const int ys = p.y0 + (blockIdx.y * kNW + warp) * kRows;
  if (ys >= p.y1) return;  // whole warp
  const bool interior = x0 >= 0 && x0 + 64 <= p.in.w && ys >= 1 && ys + kRows < p.in.h && ys + kRows <= p.y1;
  if (interior)
    rcas_rows<FmtHalf, false, kClamp, kOpt, SO, true>(p, x, ys, lane, kPost ? &q : nullptr);
  else
    rcas_rows<FmtHalf, true, kClamp, kOpt, SO, true>(p, x, ys, lane, kPost ? &q : nullptr);
}

// tests/emu compiles the device code above for the host and supplies its own launcher; fsr1_rcas_in.cu takes the templates only
#if !defined(FSR1_CPU_EMU) && !defined(FSR1_RCAS_PACKED_TEMPLATES_ONLY)
template <typename FM, bool kClamp>
static void launch_opt(const RcasParams& p, dim3 grid, cudaStream_t s) {
  switch (p.options & 7) {
    case 0: rcas_packed_kernel<FM, kClamp, 0><<<grid, 32 * kNW, 0, s>>>(p); break;
    case 1: rcas_packed_kernel<FM, kClamp, 1><<<grid, 32 * kNW, 0, s>>>(p); break;
    case 2: rcas_packed_kernel<FM, kClamp, 2><<<grid, 32 * kNW, 0, s>>>(p); break;
    case 3: rcas_packed_kernel<FM, kClamp, 3><<<grid, 32 * kNW, 0, s>>>(p); break;
    case 4: rcas_packed_kernel<FM, kClamp, 4><<<grid, 32 * kNW, 0, s>>>(p); break;
    case 5: rcas_packed_kernel<FM, kClamp, 5><<<grid, 32 * kNW, 0, s>>>(p); break;
    case 6: rcas_packed_kernel<FM, kClamp, 6><<<grid, 32 * kNW, 0, s>>>(p); break;
    default: rcas_packed_kernel<FM, kClamp, 7><<<grid, 32 * kNW, 0, s>>>(p); break;
  }
}
template <typename FM>
static cudaError_t launch_fmt(const RcasParams& p, cudaStream_t s) {
  // 4-warp CTAs (60 x 16 pixels), 4 rows per lane, MUFU reciprocals: same kernel time as 8-warp CTAs, but the smaller
  // CTA starts earlier in the tail of the preceding EASU and shares SMs with it when frames are pipelined
  // (round 1: 92.1 -> 90.7 us per frame back to back; the 8-row and Newton-reciprocal variants measured slower)
  const dim3 grid((p.out.w + kSpan - 1) / kSpan, (p.y1 - p.y0 + kNW * kRows - 1) / (kNW * kRows), 1);
  if (p.clamp) launch_opt<FM, true>(p, grid, s);
  else launch_opt<FM, false>(p, grid, s);
  return cudaGetLastError();
}
static bool aligned(const RcasParams& p, int a) {
  return !((reinterpret_cast<uintptr_t>(p.in.base) & (a - 1)) || (p.in.pitch & (a - 1)) || (reinterpret_cast<uintptr_t>(p.out.base) & (a - 1)) ||
           (p.out.pitch & (a - 1)));
}

cudaError_t launch_rcas_u_packed(const RcasParams& p, int format, cudaStream_t s, const char** name) {
  // R8G8B8A8 only: half arithmetic (11-bit significand) is coarser than the codes of R10G10B10A2 (measured 2-4 codes off),
  // which therefore stays on the fp32 direct kernel (<= 1 code)
  if (format != 3 || !aligned(p, 8)) return cudaErrorNotSupported;
  *name = "rcas_u8_packed<2px,4rows,shfl60>";
  return launch_fmt<FmtUnorm<8>>(p, s);
}

template <typename SO, bool kClamp>
static void launch_surf_opt(const RcasParams& p, const PostParams& q, dim3 grid, cudaStream_t s) {
  switch (p.options & 7) {
    case 0: rcas_surf_out_kernel<kClamp, 0, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    case 1: rcas_surf_out_kernel<kClamp, 1, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    case 2: rcas_surf_out_kernel<kClamp, 2, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    case 3: rcas_surf_out_kernel<kClamp, 3, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    case 4: rcas_surf_out_kernel<kClamp, 4, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    case 5: rcas_surf_out_kernel<kClamp, 5, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    case 6: rcas_surf_out_kernel<kClamp, 6, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    default: rcas_surf_out_kernel<kClamp, 7, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
  }
}
template <typename SO, bool kClamp>
static void launch_post_opt(const RcasParams& p, const PostParams& q, dim3 grid, cudaStream_t s) {
  switch (p.options & 7) {
    case 0: rcas_post_kernel<kClamp, 0, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    case 1: rcas_post_kernel<kClamp, 1, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    case 2: rcas_post_kernel<kClamp, 2, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    case 3: rcas_post_kernel<kClamp, 3, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    case 4: rcas_post_kernel<kClamp, 4, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    case 5: rcas_post_kernel<kClamp, 5, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    case 6: rcas_post_kernel<kClamp, 6, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
    default: rcas_post_kernel<kClamp, 7, SO><<<grid, 32 * kNW, 0, s>>>(p, q); break;
  }
}
template <typename SO>
static cudaError_t launch_post_fmt(const RcasParams& p, const PostParams& q, cudaStream_t s) {
  const dim3 grid((p.out.w + kSpan - 1) / kSpan, (p.y1 - p.y0 + kNW * kRows - 1) / (kNW * kRows), 1);
  if (p.clamp) launch_post_opt<SO, true>(p, q, grid, s);
  else launch_post_opt<SO, false>(p, q, grid, s);
  return cudaGetLastError();
}
template <typename SO>
static cudaError_t launch_surf_fmt(const RcasParams& p, const PostParams& q, cudaStream_t s) {
  const dim3 grid((p.out.w + kSpan - 1) / kSpan, (p.y1 - p.y0 + kNW * kRows - 1) / (kNW * kRows), 1);
  if (p.clamp) launch_surf_opt<SO, true>(p, q, grid, s);
  else launch_surf_opt<SO, false>(p, q, grid, s);
  return cudaGetLastError();
}
// 16-byte aligned input (and output, unless it is a surface): the 128-bit pair loads and stores
static bool aligned16(const RcasParams& p, bool surf_out, int out_align = 16) {
  return !((reinterpret_cast<uintptr_t>(p.in.base) & 15) || (p.in.pitch & 15) ||
           (!surf_out && ((reinterpret_cast<uintptr_t>(p.out.base) & (out_align - 1)) || (p.out.pitch & (out_align - 1)))));
}

// p.in: the RGBA16F intermediate; p.out: RGBA16F (out_format 1), RGBA8_UNORM (3) or RGB10A2_UNORM (4)
cudaError_t launch_rcas_h_post(const RcasParams& p, const PostParams& q, int out_format, cudaStream_t s, const char** name, bool surf_out) {
  if (!aligned16(p, surf_out, out_format == 1 ? 16 : 8)) return cudaErrorNotSupported;
  switch (out_format) {
    case 1:
      *name = surf_out ? "rcas_h_packed_post<2px,4rows,shfl60,rgba16f,surf_out>" : "rcas_h_packed_post<2px,4rows,shfl60,rgba16f>";
      return surf_out ? launch_surf_fmt<__half>(p, q, s) : launch_post_fmt<__half>(p, q, s);
    case 3:
      *name = surf_out ? "rcas_h_packed_post<2px,4rows,shfl60,rgba8,surf_out>" : "rcas_h_packed_post<2px,4rows,shfl60,rgba8>";
      return surf_out ? launch_surf_fmt<Unorm8>(p, q, s) : launch_post_fmt<Unorm8>(p, q, s);
    case 4:
      *name = surf_out ? "rcas_h_packed_post<2px,4rows,shfl60,rgb10a2,surf_out>" : "rcas_h_packed_post<2px,4rows,shfl60,rgb10a2>";
      return surf_out ? launch_surf_fmt<Unorm10>(p, q, s) : launch_post_fmt<Unorm10>(p, q, s);
  }
  return cudaErrorNotSupported;
}

cudaError_t launch_rcas_h_packed(const RcasParams& p, cudaStream_t s, const char** name, bool surf_out) {
  if (surf_out) {
    if (!aligned16(p, true)) return cudaErrorNotSupported;
    *name = "rcas_h_packed<2px,4rows,shfl60,surf_out>";
    return launch_surf_fmt<void>(p, PostParams{}, s);
  }
  if (!aligned(p, 16)) return cudaErrorNotSupported;
  *name = "rcas_h_packed<2px,4rows,shfl60>";
  return launch_fmt<FmtHalf>(p, s);
}

#endif  // FSR1_CPU_EMU

}  // namespace fsr1
