// fsr1_easu_f32.cu — tiled EASU for RGBA32F images at exactly 2x (the SAMPLE_SLOW_FALLBACK precision of
// BASELINE configs[3]).  Same structure as easu_h_quad2x_kernel (fsr1_easu_tiled.cu): persistent CTAs, TMA
// box load double-buffered on two mbarriers (here a 3-D tensor {4 floats, W, rows}), per-input-texel luma and
// FsrEasuSetF terms hoisted to shared memory, a lane owns the quad of output pixels (2k+1,2k+2)x(2m+1,2m+2)
// that shares one 4x4 tap window.  All arithmetic is fp32 (F path, ffx-fsr/ffx_fsr1.h:239-437); the tap weights of
// the two pixels of a row pair are computed as float2 pairs (ffma2 / fmul2 / fadd2, fsr1_easu_common.cuh), the colour
// accumulation with scalar FFMA.  The tap distance keeps the reference's own rotate-then-scale formulation (the expanded
// quadratic form used by the half kernels costs ~1e-6 in fp32, too close to the 1e-5 tolerance).  Tolerance
// against the oracle: 1e-5 (FMA contraction reorders roundings; FSR1_FLAG_EXACT = the bit-exact direct kernel).
#include "fsr1_easu_common.cuh"

namespace fsr1 {

constexpr int kFQCX = 32, kFQBW = kFQCX + 4, kFQSW = kFQBW - 2;

// storage of one texel in the tile / in the images: RGBA32F (float4) or RGBA16F (uint2); arithmetic is fp32 either way
template <typename S> struct Tex;
template <> struct Tex<float> {
  using T = float4;
  static constexpr int kBytes = 16;
  static __device__ __forceinline__ float4 rgb(const float4& t) { return t; }
  static __device__ __forceinline__ float4 pack(const float4& c) { return c; }
};
template <> struct Tex<__half> {
  using T = uint2;
  static constexpr int kBytes = 8;
  static __device__ __forceinline__ float4 rgb(const uint2& t) {
    const float2 rg = __half22float2(*reinterpret_cast<const __half2*>(&t.x));
    return make_float4(rg.x, rg.y, __low2float(*reinterpret_cast<const __half2*>(&t.y)), 1.0f);
  }
  static __device__ __forceinline__ uint2 pack(const float4& c) {
    const __half2 rg = __floats2half2_rn(c.x, c.y), ba = __floats2half2_rn(c.z, 1.0f);
    return make_uint2(*reinterpret_cast<const uint32_t*>(&rg), *reinterpret_cast<const uint32_t*>(&ba));
  }
};

template <typename S, int NW> struct FQuadCfg {
  static constexpr int kCY = 2 * NW, kBH = kCY + 3, kSH = kBH - 2, kElems = kFQBW * kBH;
  static constexpr int kPad = ((kElems * Tex<S>::kBytes + 127) / 128) * 128 / Tex<S>::kBytes;
};
template <typename S, int NW> struct __align__(128) FQuadSmem {
  typename Tex<S>::T tile[2][FQuadCfg<S, NW>::kPad];
  float4 S_[kFQSW * FQuadCfg<S, NW>::kSH];
  float L[FQuadCfg<S, NW>::kElems];
  uint64_t bar[2];
};

#ifdef FSR1_CPU_EMU
// the emulated 2-D copy is generic in the element size: a {4 floats, W, rows} box is a 2-D box of 16-byte elements
inline void tma_load_3d(void* dst, const CUtensorMap* map, int, int x, int y, uint64_t* bar) { tma_load_2d(dst, map, x, y, bar); }
#else
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, int c, int x, int y, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c), "r"(x), "r"(y), "r"(smem_u32(bar))
      : "memory");
}
#endif

__device__ __forceinline__ float2 f2(float a, float b) { return make_float2(a, b); }

// Per-pixel filter shape in the reference's own formulation (rotation * anisotropic scale), fp32:
//   v = (ox*cxx + oy*cxy, ox*cyx + oy*cyy),  cxx = dx*l2x, cxy = dy*l2x, cyx = -dy*l2y, cyy = dx*l2y
struct ShapeR { float cxx, cxy, cyx, cyy, lob, clp; };
__device__ __forceinline__ ShapeR pixel_shape_rot(float dx, float dy, float len) {
  const float dirR = fmaf(dx, dx, dy * dy);
  const bool zro = dirR < (1.0f / 32768.0f);
  const float rs = zro ? 1.0f : prx_lo_rsq(dirR);
  dx = (zro ? 1.0f : dx) * rs;
  dy *= rs;
  len *= 0.5f;
  len *= len;
  const float stretch = fmaf(dx, dx, dy * dy) * prx_lo_rcp(fmaxf(fabsf(dx), fabsf(dy)));
  const float l2x = fmaf(stretch - 1.0f, len, 1.0f), l2y = fmaf(-0.5f, len, 1.0f);
  ShapeR s;
  s.lob = fmaf((float)((1.0 / 4.0 - 0.04) - 0.5), len, 0.5f);
  s.clp = prx_lo_rcp(s.lob);
  s.cxx = dx * l2x; s.cxy = dy * l2x; s.cyx = -dy * l2y; s.cyy = dx * l2y;
  return s;
}

// One row pair (A: px=.25, B: px=.75) of the quad; kBottom selects py=.75.
template <bool kBottom>
__device__ __forceinline__ void fquad_pair(const float4 (&t)[4][4], const ShapeR& sA, const ShapeR& sB, float3 mn, float3 mx,
                                           float4& outA, float4& outB) {
  const float2 cxx = f2(sA.cxx, sB.cxx), cxy = f2(sA.cxy, sB.cxy), cyx = f2(sA.cyx, sB.cyx), cyy = f2(sA.cyy, sB.cyy);
  const float2 lob = f2(sA.lob, sB.lob);
  float3 aA = make_float3(0.f, 0.f, 0.f), aB = make_float3(0.f, 0.f, 0.f);
  float2 aW = f2(0.f, 0.f);
  constexpr float py = kBottom ? 0.75f : 0.25f;
#define FSR1_FQTAP(R, K)                                                                                      \
  {                                                                                                           \
    constexpr float oxA = (float)((K)-1) - 0.25f, oxB = (float)((K)-1) - 0.75f, oy = (float)((R)-1) - py;       \
    const float2 vx = ffma2(f2(oxA, oxB), cxx, fmul2(f2(oy, oy), cxy));                              \
    const float2 vy = ffma2(f2(oxA, oxB), cyx, fmul2(f2(oy, oy), cyy));                              \
    float2 d2 = ffma2(vx, vx, fmul2(vy, vy));                                                       \
    d2.x = fminf(d2.x, sA.clp);                                                                               \
    d2.y = fminf(d2.y, sB.clp);                                                                               \
    float2 wb = ffma2(f2(0.4f, 0.4f), d2, f2(-1.f, -1.f));                                                \
    float2 wa = ffma2(lob, d2, f2(-1.f, -1.f));                                                          \
    wb = fmul2(wb, wb);                                                                                  \
    wa = fmul2(wa, wa);                                                                                  \
    wb = ffma2(f2(1.5625f, 1.5625f), wb, f2(-0.5625f, -0.5625f));                                        \
    const float2 w = fmul2(wb, wa);                                                                      \
    const float4 c = t[R][K];                                                                                 \
    aA.x = fmaf(c.x, w.x, aA.x); aA.y = fmaf(c.y, w.x, aA.y); aA.z = fmaf(c.z, w.x, aA.z);                    \
    aB.x = fmaf(c.x, w.y, aB.x); aB.y = fmaf(c.y, w.y, aB.y); aB.z = fmaf(c.z, w.y, aB.z);                    \
    aW = fadd2(aW, w);                                                                                   \
  }
  FSR1_FQTAP(0, 1) FSR1_FQTAP(0, 2) FSR1_FQTAP(2, 0) FSR1_FQTAP(2, 1)   // the reference's order: b c i j f e k l h g o n
  FSR1_FQTAP(1, 1) FSR1_FQTAP(1, 0) FSR1_FQTAP(2, 2) FSR1_FQTAP(2, 3)
  FSR1_FQTAP(1, 3) FSR1_FQTAP(1, 2) FSR1_FQTAP(3, 2) FSR1_FQTAP(3, 1)
#undef FSR1_FQTAP
  const float rA = __frcp_rn(aW.x), rB = __frcp_rn(aW.y);
  outA = make_float4(fminf(mx.x, fmaxf(mn.x, aA.x * rA)), fminf(mx.y, fmaxf(mn.y, aA.y * rA)), fminf(mx.z, fmaxf(mn.z, aA.z * rA)), 1.0f);
  outB = make_float4(fminf(mx.x, fmaxf(mn.x, aB.x * rB)), fminf(mx.y, fmaxf(mn.y, aB.y * rB)), fminf(mx.z, fmaxf(mn.z, aB.z * rB)), 1.0f);
}

template <typename S, int NW, int MINB>
__global__ void __launch_bounds__(NW * 32, MINB)
easu_f32_quad2x_kernel(const EasuParams p, const __grid_constant__ CUtensorMap tmap, const int tiles_x,
                       const int n_tiles, const int mbase) {
  using C = FQuadCfg<S, NW>;
  using TT = typename Tex<S>::T;
  constexpr int NT = NW * 32, kB = Tex<S>::kBytes;
  __shared__ FQuadSmem<S, NW> sm;
  auto load_box = [&](TT* dst, int x, int y, uint64_t* bar) {
    if (kB == 16) tma_load_3d(dst, &tmap, 0, x, y, bar);
    else tma_load_2d(dst, &tmap, x, y, bar);
  };
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    mbar_init(&sm.bar[0], 1);
    mbar_init(&sm.bar[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  auto box_x = [&](int t) { return (t % tiles_x) * kFQCX - 2; };
  auto box_y = [&](int t) { return mbase + (t / tiles_x) * C::kCY - 1; };
  int t = blockIdx.x;
  if (tid == 0 && t < n_tiles) {
    mbar_expect_tx(&sm.bar[0], C::kElems * (uint32_t)kB);
    load_box(sm.tile[0], box_x(t), box_y(t) - p.in.row0, &sm.bar[0]);
  }
  for (int it = 0; t < n_tiles; t += gridDim.x, it++) {
    const int b = it & 1;
    const int tn = t + gridDim.x;
    if (tid == 0 && tn < n_tiles) {
      fence_proxy_async();
      mbar_expect_tx(&sm.bar[b ^ 1], C::kElems * (uint32_t)kB);
      load_box(sm.tile[b ^ 1], box_x(tn), box_y(tn) - p.in.row0, &sm.bar[b ^ 1]);
    }
    TT* tile = sm.tile[b];
    const int gx0 = box_x(t), gy0 = box_y(t);
    mbar_wait(&sm.bar[b], (it >> 1) & 1);
    if (gx0 < 0 || gy0 < 0 || gx0 + kFQBW > p.in.w || gy0 + C::kBH > p.in.h) {  // clamp-to-edge fix-up
      for (int j = warp; j < C::kBH; j += NW) {
        const int cy = clampi(gy0 + j, 0, p.in.h - 1) - gy0;
        for (int i = lane; i < kFQBW; i += 32) {
          const int cx = clampi(gx0 + i, 0, p.in.w - 1) - gx0;
          if ((cx != i || cy != j) && cx >= 0 && cx < kFQBW && cy >= 0 && cy < C::kBH) tile[j * kFQBW + i] = tile[cy * kFQBW + cx];
        }
      }
      fence_proxy_async();
      __syncthreads();
    }
    for (int i = tid; i < C::kElems; i += NT) {
      const float4 c = Tex<S>::rgb(tile[i]);
      sm.L[i] = fmaf(c.z, 0.5f, fmaf(c.x, 0.5f, c.y));
    }
    __syncthreads();
    for (int idx = tid; idx < kFQSW * C::kSH; idx += NT) {
      const int j = idx / kFQSW, i = idx - j * kFQSW;
      const float* c = sm.L + (j + 1) * kFQBW + (i + 1);
      sm.S_[idx] = texel_terms(c[-kFQBW], c[-1], c[0], c[1], c[kFQBW]);
    }
    __syncthreads();

    const int oxA = (gx0 + 1 + lane) * 2 + 1;
#pragma unroll 1
    for (int q = 0; q < 2; q++) {
      const int r = warp + q * NW;
      const int oyT = (gy0 + 1 + r) * 2 + 1;
      const bool rowT = oyT >= p.y0 && oyT < p.y1, rowB = oyT + 1 >= p.y0 && oyT + 1 < p.y1;
      if (oxA >= p.out.w || !(rowT || rowB)) continue;
      float4 tp[4][4];
      const TT* t0 = tile + r * kFQBW + lane;
#pragma unroll
      for (int R = 0; R < 4; R++)
#pragma unroll
        for (int K = 0; K < 4; K++)
          if (!((R == 0 || R == 3) && (K == 0 || K == 3))) tp[R][K] = Tex<S>::rgb(t0[R * kFQBW + K]);
      const float4* s0 = sm.S_ + r * kFQSW + lane;
      const float4 f = s0[0], g = s0[1], j = s0[kFQSW], k = s0[kFQSW + 1];
      const float3 mn = make_float3(fminf(fminf(tp[1][1].x, tp[1][2].x), fminf(tp[2][1].x, tp[2][2].x)),
                                    fminf(fminf(tp[1][1].y, tp[1][2].y), fminf(tp[2][1].y, tp[2][2].y)),
                                    fminf(fminf(tp[1][1].z, tp[1][2].z), fminf(tp[2][1].z, tp[2][2].z)));
      const float3 mx = make_float3(fmaxf(fmaxf(tp[1][1].x, tp[1][2].x), fmaxf(tp[2][1].x, tp[2][2].x)),
                                    fmaxf(fmaxf(tp[1][1].y, tp[1][2].y), fmaxf(tp[2][1].y, tp[2][2].y)),
                                    fmaxf(fmaxf(tp[1][1].z, tp[1][2].z), fmaxf(tp[2][1].z, tp[2][2].z)));
      // bilinear blends in the reference's f,g,j,k order with the constant weights of pp = .25 / .75
      auto blend = [&](float wf, float wg, float wj, float wk) {
        return pixel_shape_rot(fmaf(k.x, wk, fmaf(j.x, wj, fmaf(g.x, wg, f.x * wf))), fmaf(k.y, wk, fmaf(j.y, wj, fmaf(g.y, wg, f.y * wf))),
                           fmaf(k.z, wk, fmaf(j.z, wj, fmaf(g.z, wg, f.z * wf))));
      };
      unsigned char* orow = p.out.base + (long long)(oyT - p.out.row0) * p.out.pitch + (long long)oxA * kB;
      const bool okA = oxA >= 0, okB = oxA + 1 < p.out.w;
      float4 oA, oB;
      if (rowT) {
        fquad_pair<false>(tp, blend(0.5625f, 0.1875f, 0.1875f, 0.0625f), blend(0.1875f, 0.5625f, 0.0625f, 0.1875f), mn, mx, oA, oB);
        if (okA) *reinterpret_cast<TT*>(orow) = Tex<S>::pack(oA);
        if (okB) *reinterpret_cast<TT*>(orow + kB) = Tex<S>::pack(oB);
      }
      if (rowB) {
        fquad_pair<true>(tp, blend(0.1875f, 0.0625f, 0.5625f, 0.1875f), blend(0.0625f, 0.1875f, 0.1875f, 0.5625f), mn, mx, oA, oB);
        if (okA) *reinterpret_cast<TT*>(orow + p.out.pitch) = Tex<S>::pack(oA);
        if (okB) *reinterpret_cast<TT*>(orow + p.out.pitch + kB) = Tex<S>::pack(oB);
      }
    }
    __syncthreads();
  }
}

// =======================================================================================================
//  any scale >= 1: the structure of easu_h_pairs_kernel (fsr1_easu_tiled.cu) with fp32 arithmetic
// =======================================================================================================
// 64x32 output tile per CTA, persistent, double-buffered TMA box whose size is fixed per launch from the scale; a lane owns
// one output column and a VERTICAL pixel pair (A = row oy, B = row oy+1): whether the two rows share an input cell row is
// warp-uniform.  The tap weights of the pair are float2 pairs (.x = A, .y = B) in the reference's rotate-then-scale
// formulation; colours accumulate with scalar FFMA.  Presets 1.3x / 1.5x / 1.7x of RGBA32F images (sample/src/DX12/FSRSample.h:70-97
// with SAMPLE_SLOW_FALLBACK) and FSR1_FLAG_PRECISE on RGBA16F images at those scales run here instead of the direct kernel.
constexpr int kFTileW = 64, kFTileH = 32, kFThreads = 256;

template <typename S, int DR>
__device__ __forceinline__ void fvpair(const typename Tex<S>::T* __restrict__ t0, const float4* __restrict__ q0, int BW, int SW, float ppx,
                                       float ppyA, float ppyB, float4& outA, float4& outB) {
  const float4 f = q0[0], g = q0[1], j = q0[SW], k = q0[SW + 1];
  const float4 fB = DR ? j : f, gB = DR ? k : g, jB = DR ? q0[2 * SW] : j, kB = DR ? q0[2 * SW + 1] : k;
  const float ipx = 1.0f - ppx;
  ShapeR sA, sB;
  {
    const float ipy = 1.0f - ppyA, wf = ipx * ipy, wg = ppx * ipy, wj = ipx * ppyA, wk = ppx * ppyA;
    sA = pixel_shape_rot(fmaf(k.x, wk, fmaf(j.x, wj, fmaf(g.x, wg, f.x * wf))), fmaf(k.y, wk, fmaf(j.y, wj, fmaf(g.y, wg, f.y * wf))),
                         fmaf(k.z, wk, fmaf(j.z, wj, fmaf(g.z, wg, f.z * wf))));
  }
  {
    const float ipy = 1.0f - ppyB, wf = ipx * ipy, wg = ppx * ipy, wj = ipx * ppyB, wk = ppx * ppyB;
    sB = pixel_shape_rot(fmaf(kB.x, wk, fmaf(jB.x, wj, fmaf(gB.x, wg, fB.x * wf))), fmaf(kB.y, wk, fmaf(jB.y, wj, fmaf(gB.y, wg, fB.y * wf))),
                         fmaf(kB.z, wk, fmaf(jB.z, wj, fmaf(gB.z, wg, fB.z * wf))));
  }
  const float2 cxx = f2(sA.cxx, sB.cxx), cxy = f2(sA.cxy, sB.cxy), cyx = f2(sA.cyx, sB.cyx), cyy = f2(sA.cyy, sB.cyy);
  const float2 lob = f2(sA.lob, sB.lob);
  float3 aA = make_float3(0.f, 0.f, 0.f), aB = make_float3(0.f, 0.f, 0.f);
  float2 aW = f2(0.f, 0.f);
  float3 mnA, mxA, mnB, mxB;
#define FSR1_FVTAP(R, K)                                                                                       \
  {                                                                                                            \
    const float ox = (float)((K)-1) - ppx;                                                                     \
    const float2 oy = f2((float)((R)-1) - ppyA, (float)((R)-1) - ppyB);                                        \
    const float2 vx = ffma2(f2(ox, ox), cxx, fmul2(oy, cxy));                                        \
    const float2 vy = ffma2(f2(ox, ox), cyx, fmul2(oy, cyy));                                        \
    float2 d2 = ffma2(vx, vx, fmul2(vy, vy));                                                        \
    d2.x = fminf(d2.x, sA.clp);                                                                                \
    d2.y = fminf(d2.y, sB.clp);                                                                                \
    float2 wb = ffma2(f2(0.4f, 0.4f), d2, f2(-1.f, -1.f));                                                 \
    float2 wa = ffma2(lob, d2, f2(-1.f, -1.f));                                                           \
    wb = fmul2(wb, wb);                                                                                   \
    wa = fmul2(wa, wa);                                                                                   \
    wb = ffma2(f2(1.5625f, 1.5625f), wb, f2(-0.5625f, -0.5625f));                                         \
    const float2 w = fmul2(wb, wa);                                                                       \
    const float4 ca = Tex<S>::rgb(t0[(R) * BW + (K)]);                                                         \
    const float4 cb = DR ? Tex<S>::rgb(t0[((R) + 1) * BW + (K)]) : ca;                                         \
    aA.x = fmaf(ca.x, w.x, aA.x); aA.y = fmaf(ca.y, w.x, aA.y); aA.z = fmaf(ca.z, w.x, aA.z);                  \
    aB.x = fmaf(cb.x, w.y, aB.x); aB.y = fmaf(cb.y, w.y, aB.y); aB.z = fmaf(cb.z, w.y, aB.z);                  \
    aW = fadd2(aW, w);                                                                                    \
    if (((R) == 1 || (R) == 2) && ((K) == 1 || (K) == 2)) {                                                    \
      if ((R) == 1 && (K) == 1) { mnA = mxA = make_float3(ca.x, ca.y, ca.z); mnB = mxB = make_float3(cb.x, cb.y, cb.z); } \
      else {                                                                                                   \
        mnA = make_float3(fminf(mnA.x, ca.x), fminf(mnA.y, ca.y), fminf(mnA.z, ca.z));                         \
        mxA = make_float3(fmaxf(mxA.x, ca.x), fmaxf(mxA.y, ca.y), fmaxf(mxA.z, ca.z));                         \
        mnB = make_float3(fminf(mnB.x, cb.x), fminf(mnB.y, cb.y), fminf(mnB.z, cb.z));                         \
        mxB = make_float3(fmaxf(mxB.x, cb.x), fmaxf(mxB.y, cb.y), fmaxf(mxB.z, cb.z));                         \
      }                                                                                                        \
    }                                                                                                          \
  }
  // the reference's tap order: b c i j f e k l h g o n (ffx_fsr1.h:423-434); f is first among the four nearest
  FSR1_FVTAP(1, 1)
  FSR1_FVTAP(0, 1) FSR1_FVTAP(0, 2) FSR1_FVTAP(2, 0) FSR1_FVTAP(2, 1)
  FSR1_FVTAP(1, 0) FSR1_FVTAP(2, 2) FSR1_FVTAP(2, 3)
  FSR1_FVTAP(1, 3) FSR1_FVTAP(1, 2) FSR1_FVTAP(3, 2) FSR1_FVTAP(3, 1)
#undef FSR1_FVTAP
  const float rA = __frcp_rn(aW.x), rB = __frcp_rn(aW.y);
  outA = make_float4(fminf(mxA.x, fmaxf(mnA.x, aA.x * rA)), fminf(mxA.y, fmaxf(mnA.y, aA.y * rA)), fminf(mxA.z, fmaxf(mnA.z, aA.z * rA)), 1.0f);
  outB = make_float4(fminf(mxB.x, fmaxf(mnB.x, aB.x * rB)), fminf(mxB.y, fmaxf(mnB.y, aB.y * rB)), fminf(mxB.z, fmaxf(mnB.z, aB.z * rB)), 1.0f);
}

template <typename S> __host__ __device__ inline size_t fpairs_tile_stride(int BW, int BH) {
  return ((size_t)BW * BH * Tex<S>::kBytes + 127) & ~(size_t)127;
}
template <typename S> __host__ __device__ inline size_t fpairs_smem_bytes(int BW, int BH) {
  size_t off = 2 * fpairs_tile_stride<S>(BW, BH);
  off += ((size_t)BW * BH * 4 + 127) & ~(size_t)127;
  off += ((size_t)(BW - 2) * (BH - 2) * 16 + 127) & ~(size_t)127;
  return off + 16 + 128;
}

template <typename S>
__global__ void __launch_bounds__(kFThreads, 2)
easu_f32_pairs_kernel(const EasuParams p, const __grid_constant__ CUtensorMap tmap, const int BW, const int BH, const int tiles_x,
                      const int n_tiles) {
  using TT = typename Tex<S>::T;
  constexpr int kB = Tex<S>::kBytes;
#ifdef FSR1_CPU_EMU
  unsigned char* smem_raw = fsr1_emu_dynamic_smem();
#else
  extern __shared__ unsigned char smem_raw[];
#endif
  unsigned char* base = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
  const int n = BW * BH;
  const size_t tstride = fpairs_tile_stride<S>(BW, BH);
  float* L = reinterpret_cast<float*>(base + 2 * tstride);
  float4* Sm = reinterpret_cast<float4*>(base + 2 * tstride + (((size_t)n * 4 + 127) & ~(size_t)127));
  uint64_t* bar = reinterpret_cast<uint64_t*>(reinterpret_cast<unsigned char*>(Sm) + (((size_t)(BW - 2) * (BH - 2) * 16 + 127) & ~(size_t)127));
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  auto load_box = [&](void* dst, int x, int y, uint64_t* b) {
    if (kB == 16) tma_load_3d(dst, &tmap, 0, x, y, b);
    else tma_load_2d(dst, &tmap, x, y, b);
  };
  if (tid == 0) {
    mbar_init(&bar[0], 1);
    mbar_init(&bar[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  // box origin of tile t = first tap column/row of its first pixel (16-byte texels need no column rounding, 8-byte ones start even)
  auto origin = [&](int t, int& ox0, int& oy0, int& fx0, int& fy0) {
    ox0 = (t % tiles_x) * kFTileW;
    oy0 = p.y0 + (t / tiles_x) * kFTileH;
    float dummy;
    easu_pos(ox0, p.c0x, p.c0z, fx0, dummy);
    easu_pos(oy0, p.c0y, p.c0w, fy0, dummy);
    fx0 = kB == 16 ? fx0 - 1 : ((fx0 - 1) & ~1);
    fy0 -= 1;
  };
  int t = blockIdx.x;
  if (tid == 0 && t < n_tiles) {
    int a, b, fx, fy;
    origin(t, a, b, fx, fy);
    mbar_expect_tx(&bar[0], (uint32_t)n * (uint32_t)kB);
    load_box(base, fx, fy - p.in.row0, &bar[0]);
  }
  for (int it = 0; t < n_tiles; t += gridDim.x, it++) {
    const int bsel = it & 1;
    if (tid == 0 && t + (int)gridDim.x < n_tiles) {
      int a, b, fx, fy;
      origin(t + gridDim.x, a, b, fx, fy);
      fence_proxy_async();
      mbar_expect_tx(&bar[bsel ^ 1], (uint32_t)n * (uint32_t)kB);
      load_box(base + (bsel ^ 1) * tstride, fx, fy - p.in.row0, &bar[bsel ^ 1]);
    }
    TT* tile = reinterpret_cast<TT*>(base + bsel * tstride);
    int ox0, oy0, fx0, fy0;
    origin(t, ox0, oy0, fx0, fy0);
    mbar_wait(&bar[bsel], (it >> 1) & 1);
    if (fx0 < 0 || fy0 < 0 || fx0 + BW > p.in.w || fy0 + BH > p.in.h) {  // zero fill -> clamp-to-edge (border tiles, CTA-uniform)
      for (int j = warp; j < BH; j += kFThreads / 32) {
        const int cy = clampi(fy0 + j, 0, p.in.h - 1) - fy0;
        for (int i = lane; i < BW; i += 32) {
          const int cx = clampi(fx0 + i, 0, p.in.w - 1) - fx0;
          if ((cx != i || cy != j) && cx >= 0 && cx < BW && cy >= 0 && cy < BH) tile[j * BW + i] = tile[cy * BW + cx];
        }
      }
      fence_proxy_async();
      __syncthreads();
    }
    for (int i = tid; i < n; i += kFThreads) {
      const float4 c = Tex<S>::rgb(tile[i]);
      L[i] = fmaf(c.z, 0.5f, fmaf(c.x, 0.5f, c.y));
    }
    __syncthreads();
    const int SW = BW - 2, nS = SW * (BH - 2);
    {
      int j = tid / SW, i = tid - j * SW;
      const int dj = kFThreads / SW, di = kFThreads - dj * SW;
      for (int idx = tid; idx < nS; idx += kFThreads) {
        const float* c = L + (j + 1) * BW + (i + 1);
        Sm[idx] = texel_terms(c[-BW], c[-1], c[0], c[1], c[BW]);
        i += di; j += dj;
        if (i >= SW) { i -= SW; j += 1; }
      }
    }
    __syncthreads();
#pragma unroll 1
    for (int job = warp; job < (kFTileW / 32) * (kFTileH / 2); job += kFThreads / 32) {
      const int oyA = oy0 + (job >> 1) * 2;
      if (oyA >= p.y1) continue;  // warp-uniform
      const bool hasB = oyA + 1 < p.y1;
      const int oxr = ox0 + (job & 1) * 32 + lane;
      const bool active = oxr < p.out.w;
      const int ox = active ? oxr : p.out.w - 1;
      int fx, fyA, fyB;
      float ppx, ppyA, ppyB;
      easu_pos(ox, p.c0x, p.c0z, fx, ppx);
      easu_pos(oyA, p.c0y, p.c0w, fyA, ppyA);
      easu_pos(hasB ? oyA + 1 : oyA, p.c0y, p.c0w, fyB, ppyB);
      const TT* t0 = tile + (fyA - fy0 - 1) * BW + (fx - fx0 - 1);
      const float4* q0 = Sm + (fyA - fy0 - 1) * SW + (fx - fx0 - 1);
      float4 oA, oB;
      if (fyB == fyA) fvpair<S, 0>(t0, q0, BW, SW, ppx, ppyA, ppyB, oA, oB);
      else fvpair<S, 1>(t0, q0, BW, SW, ppx, ppyA, ppyB, oA, oB);
      if (active) {
        unsigned char* o = p.out.base + (long long)(oyA - p.out.row0) * p.out.pitch + (long long)ox * kB;
        *reinterpret_cast<TT*>(o) = Tex<S>::pack(oA);
        if (hasB) *reinterpret_cast<TT*>(o + p.out.pitch) = Tex<S>::pack(oB);
      }
    }
    __syncthreads();
  }
}

#ifndef FSR1_CPU_EMU
static int f_max_footprint(int n_out, int first, int tile, float scale, float offset, bool even_origin) {
  int best = 4;
  for (int o0 = first; o0 < n_out; o0 += tile) {
    const int o1 = (o0 + tile - 1 < n_out - 1) ? o0 + tile - 1 : n_out - 1;
    int origin = host_fp(o0, scale, offset) - 1;
    if (even_origin) origin &= ~1;
    const int span = host_fp(o1, scale, offset) + 2 - origin + 1;
    if (span > best) best = span;
  }
  return best;
}

template <typename S>
static cudaError_t launch_pairs_f32math(const EasuParams& p, cudaStream_t s, const char** name, const char* nm) {
  constexpr int kB = Tex<S>::kBytes;
  if ((reinterpret_cast<uintptr_t>(p.in.base) & 15) || (p.in.pitch & 15) || (reinterpret_cast<uintptr_t>(p.out.base) & 15) || (p.out.pitch & 15))
    return cudaErrorNotSupported;
  if (!is_upscale(p.c0x, p.c0y)) return cudaErrorNotSupported;
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) return cudaErrorNotSupported;
  int BW = f_max_footprint(p.out.w, 0, kFTileW, p.c0x, p.c0z, kB == 8);
  const int BH = f_max_footprint(p.y1, p.y0, kFTileH, p.c0y, p.c0w, false);
  if (kB == 8) BW = (BW + 1) & ~1;
  if (BW > 256 || BH > 256) return cudaErrorNotSupported;
  const size_t smem = fpairs_smem_bytes<S>(BW, BH);
  if (smem > 200 * 1024) return cudaErrorNotSupported;
  CUtensorMap tmap;
  CUresult r;
  if (kB == 16) {
    const cuuint64_t dims[3] = {4, (cuuint64_t)p.in.w, (cuuint64_t)p.in.rows};
    const cuuint64_t strides[2] = {16, (cuuint64_t)p.in.pitch};
    const cuuint32_t box[3] = {4, (cuuint32_t)BW, (cuuint32_t)BH};
    const cuuint32_t estr[3] = {1, 1, 1};
    r = encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, p.in.base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    const cuuint64_t dims[2] = {(cuuint64_t)p.in.w, (cuuint64_t)p.in.rows};
    const cuuint64_t strides[1] = {(cuuint64_t)p.in.pitch};
    const cuuint32_t box[2] = {(cuuint32_t)BW, (cuuint32_t)BH};
    const cuuint32_t estr[2] = {1, 1};
    r = encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, p.in.base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) return cudaErrorNotSupported;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(easu_f32_pairs_kernel<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  const int tiles_x = (p.out.w + kFTileW - 1) / kFTileW, n_tiles = tiles_x * ((p.y1 - p.y0 + kFTileH - 1) / kFTileH);
  const int per_sm = (size_t)2 * (smem + 1024) > 220 * 1024 ? 1 : 2;
  const int grid = n_tiles < per_sm * sm_count() ? n_tiles : per_sm * sm_count();
  easu_f32_pairs_kernel<S><<<grid, kFThreads, smem, s>>>(p, tmap, BW, BH, tiles_x, n_tiles);
  *name = nm;
  return cudaGetLastError();
}

template <typename S>
static cudaError_t launch_quad_f32math(const EasuParams& p, cudaStream_t s, const char** name, const char* nm) {
  if ((reinterpret_cast<uintptr_t>(p.in.base) & 15) || (p.in.pitch & 15) || (reinterpret_cast<uintptr_t>(p.out.base) & 15) ||
      (p.out.pitch & 15))
    return cudaErrorNotSupported;
  if (!is_2x(p.c0x, p.c0y, p.c0z, p.c0w)) return cudaErrorNotSupported;
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) return cudaErrorNotSupported;
  constexpr int NW = 4, per_sm = 4;
  using C = FQuadCfg<S, NW>;
  CUtensorMap tmap;
  CUresult r;
  if (Tex<S>::kBytes == 16) {
    const cuuint64_t dims[3] = {4, (cuuint64_t)p.in.w, (cuuint64_t)p.in.rows};
    const cuuint64_t strides[2] = {16, (cuuint64_t)p.in.pitch};
    const cuuint32_t box[3] = {4, (cuuint32_t)kFQBW, (cuuint32_t)C::kBH};
    const cuuint32_t estr[3] = {1, 1, 1};
    r = encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, p.in.base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    const cuuint64_t dims[2] = {(cuuint64_t)p.in.w, (cuuint64_t)p.in.rows};
    const cuuint64_t strides[1] = {(cuuint64_t)p.in.pitch};
    const cuuint32_t box[2] = {(cuuint32_t)kFQBW, (cuuint32_t)C::kBH};
    const cuuint32_t estr[2] = {1, 1};
    r = encode(&tmap, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, p.in.base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) return cudaErrorNotSupported;
  const int k_last = host_fp(p.out.w - 1, 0.5f, -0.25f);
  const int m_first = host_fp(p.y0, 0.5f, -0.25f), m_last = host_fp(p.y1 - 1, 0.5f, -0.25f);
  const int tiles_x = (k_last + 1 + 1 + kFQCX - 1) / kFQCX, tiles_y = (m_last - m_first + 1 + C::kCY - 1) / C::kCY;
  const int n_tiles = tiles_x * tiles_y;
  const int grid = n_tiles < per_sm * sm_count() ? n_tiles : per_sm * sm_count();
  easu_f32_quad2x_kernel<S, NW, per_sm><<<grid, NW * 32, 0, s>>>(p, tmap, tiles_x, n_tiles, m_first);
  *name = nm;
  return cudaGetLastError();
}

cudaError_t launch_easu_f32_tiled(const EasuParams& p, cudaStream_t s, const char** name) {
  const cudaError_t e = launch_quad_f32math<float>(p, s, name, "easu_f32_quad2x<4w,4/sm,tma2>");
  return e != cudaErrorNotSupported ? e : launch_pairs_f32math<float>(p, s, name, "easu_f32_vpairs<64x32,persistent,tma2>");
}
// RGBA16F storage, fp32 arithmetic (FSR1_FLAG_PRECISE): the accuracy of the fp32 path at fp16 bandwidth
cudaError_t launch_easu_h_precise(const EasuParams& p, cudaStream_t s, const char** name) {
  const cudaError_t e = launch_quad_f32math<__half>(p, s, name, "easu_h16io_f32math_quad2x<4w,4/sm,tma2>");
  return e != cudaErrorNotSupported ? e : launch_pairs_f32math<__half>(p, s, name, "easu_h16io_f32math_vpairs<64x32,persistent,tma2>");
}
#endif  // FSR1_CPU_EMU

}  // namespace fsr1
