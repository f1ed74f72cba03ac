// fsr1_easu_tiled.cu — the production EASU kernels for RGBA16F (and UNORM) images on sm_90a.
//
// Common structure.  A CTA produces a tile of the output.  The tile's input footprint (plus the 4x4
// tap window's halo) is fetched by ONE TMA 2D tile load (cp.async.bulk.tensor.2d, elected thread,
// mbarrier complete_tx) into shared memory; parts of the box outside the image arrive as zeros and are
// rewritten to clamp-to-edge (the reference samples through a CLAMP sampler,
// sample/src/DX12/FSR_Filter.cpp:48-53).  The arithmetic is then split the way it factors:
//
//   phase 1  per INPUT texel   2*luma, fp32                                         (ffx_fsr1.h:363-366)
//   phase 2  per INPUT texel   the FsrEasuSetF terms that do not depend on the output pixel:
//                              dirX, dirY, lenX^2+lenY^2 (fp32, F-path bit tricks)    (ffx_fsr1.h:295-313)
//   phase 3  per OUTPUT pixel  fp32 (float2 over a pixel pair): bilinear blend of the 4 nearest texels' terms
//                              (:383-386), normalise, stretch, lobe, clip (:389-409);  packed half2 over TWO output
//                              pixels: the 12 taps (:423-434) and the de-ringing clamp (:416-419,437).
//
// Precision split (DESIGN.md "numerics"): everything that decides the filter's ORIENTATION is fp32 — in
// half it is ill-conditioned where gradients nearly cancel and differs from the fp32 algorithm by up to
// 0.1; the taps (the bulk of the arithmetic) are half2 and stay within ~3e-3 of the fp32 oracle.
//
// Kernels:
//   easu_h_quad2x_kernel  exactly 2x (con0 = {.5,.5,-.25,-.25}, BASELINE configs[1]): a lane owns the quad of output
//                         pixels sharing one 4x4 window (fsr1_easu_quad.cuh).  Persistent CTAs, TMA double-buffered:
//                         tile i+1 loads while tile i computes; tiles strictly inside the image take a predicate-free
//                         copy of the per-quad body; tile coordinates advance incrementally.  7 CTAs x 4 warps per SM.
//   easu_u_quad2x_kernel  the same for R8G8B8A8_UNORM images (4-byte texels, decode pass, fused re-encode).
//   easu_h_pairs_kernel   any other scale >= 1; 64x32 output tile per CTA; lane = one output column and a VERTICAL
//                         pixel pair.
// Array inputs (FSR1_FLAG_IN_SURFACE / IN_TEXTURE): a TMA tensor map addresses global memory only, so the *_surf_in / *_tex_in twins
// fill the same half tile in phase 1 from the array (array_texel, fsr1_common.cuh); the rest of each kernel is the linear one.
// kSrtmIn (FSR1_FLAG_SRTM_INPUT, RGBA16F kernels): phase 1 first replaces each box texel by FsrSrtmF of it, rounded to half
// (srtm_texel, fsr1_post.cuh), and takes the luma from that half texel; the taps then read the transformed tile.  It runs after
// clamp_fixup, on the raw texels the fixup copied, so each texel is transformed once.  Its generic-proxy stores into the TMA buffer
// precede the barrier that closes the tile; the fence_proxy_async thread 0 issues before the next TMA load into that buffer orders
// them, as it does the tap loop's reads.
#include "fsr1_easu_quad.cuh"
#include "fsr1_post.cuh"
#include "fsr1_r11.cuh"

namespace fsr1 {

constexpr int kThreads = 256;

// =======================================================================================================
//  generic kernel: any scale, lane = one output column, vertical pixel pair (oy, oy+1), 64x32 tile
// =======================================================================================================
constexpr int kTileW = 64, kTileH = 32;

// One vertical pixel pair: pixel A (row oy) and B (row oy+1) in the same output column.  t0/q0 point at tap (0,0) /
// texel f of pixel A; DR = fy(B) - fy(A) in {0,1}.  Packed lanes are (A, B): the fp32 analysis of the pair as float2,
// the factored tap distance ox (qa ox + qb oy) + qc oy^2 and the integer distance clamp (tap_weight).
template <int DR>
__device__ __forceinline__ void vpair(const uint2* __restrict__ t0, const float4* __restrict__ q0, int BW, int SW, float ppx,
                                      float ppyA, float ppyB, uint2& outA, uint2& outB) {
  // fp32: blend of the f,g,j,k terms (reference order) and the filter shape, per pixel
  const float4 f = q0[0], g = q0[1], j = q0[SW], k = q0[SW + 1];
  const float ipx = 1.0f - ppx;
  const float4 f2 = DR ? j : f, g2 = DR ? k : g, j2 = DR ? q0[2 * SW] : j, k2 = DR ? q0[2 * SW + 1] : k;
  const float2 ppy = mk2(ppyA, ppyB), ipy = ffma2(ppy, bc2(-1.0f), bc2(1.0f));
  const float2 wf = fmul2(bc2(ipx), ipy), wg = fmul2(bc2(ppx), ipy);
  const float2 wj = fmul2(bc2(ipx), ppy), wk = fmul2(bc2(ppx), ppy);
#define FSR1_BLEND2(C)                                                                                                  \
  ffma2(mk2(k.C, k2.C), wk, ffma2(mk2(j.C, j2.C), wj, ffma2(mk2(g.C, g2.C), wg, fmul2(mk2(f.C, f2.C), wf))))
  const ShapeH sh = to_half(pixel_shape2(FSR1_BLEND2(x), FSR1_BLEND2(y), FSR1_BLEND2(z)));
#undef FSR1_BLEND2
  const __half2 qa = sh.qa, qb = sh.qb, qc = sh.qc, lob = sh.lob, clp = sh.clp;
  // d2(R,K) = ox_K (qa ox_K + qb oy_R) + qc oy_R^2; the column offset is the same for both pixels, the row offset is not
  const __half2 ppy2 = __floats2half2_rn(ppyA, ppyB), ppx2 = __float2half2_rn(ppx);
  __half2 OX[4], QY[4], OY[4];  // ox_K; qc oy_R^2; qb oy_R
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const __half2 oyr = __hsub2(h2c((float)(i - 1)), ppy2);
    OX[i] = __hsub2(h2c((float)(i - 1)), ppx2);
    OY[i] = __hmul2(qb, oyr);
    QY[i] = __hmul2(__hmul2(qc, oyr), oyr);
  }
  auto tapw = [&](int R, int K) -> __half2 { return tap_weight(__hfma2(__hfma2(qa, OX[K], OY[R]), OX[K], QY[R]), lob, clp); };
  const __half2 kZero = h2c(0.0f), one = h2c(1.0f);
  if (DR == 0) {
    // same window for both pixels: colour accumulators in structure-of-arrays form (A,B) per channel
    __half2 aR = kZero, aG = kZero, aB = kZero, aW = kZero;
#define FSR1_VTAP0(R, K)                                                                     \
    {                                                                                        \
      const uint2 c = t0[(R) * BW + (K)];                                                    \
      const __half2 w = tapw(R, K);                                                          \
      aR = __hfma2(__low2half2(u2h2(c.x)), w, aR);                                           \
      aG = __hfma2(__high2half2(u2h2(c.x)), w, aG);                                          \
      aB = __hfma2(__low2half2(u2h2(c.y)), w, aB);                                           \
      aW = __hadd2(aW, w);                                                                   \
    }
    FSR1_VTAP0(0, 1) FSR1_VTAP0(0, 2) FSR1_VTAP0(1, 0) FSR1_VTAP0(1, 3)   // far taps first (see quad_pair)
    FSR1_VTAP0(2, 0) FSR1_VTAP0(2, 3) FSR1_VTAP0(3, 1) FSR1_VTAP0(3, 2)
    FSR1_VTAP0(1, 1) FSR1_VTAP0(1, 2) FSR1_VTAP0(2, 1) FSR1_VTAP0(2, 2)
#undef FSR1_VTAP0
    const uint2 cf = t0[BW + 1], cg = t0[BW + 2], cj = t0[2 * BW + 1], ck = t0[2 * BW + 2];
    const __half2 mnRG = __hmin2(__hmin2(u2h2(cf.x), u2h2(cg.x)), __hmin2(u2h2(cj.x), u2h2(ck.x)));
    const __half2 mxRG = __hmax2(__hmax2(u2h2(cf.x), u2h2(cg.x)), __hmax2(u2h2(cj.x), u2h2(ck.x)));
    const __half2 mnBA = __hmin2(__hmin2(u2h2(cf.y), u2h2(cg.y)), __hmin2(u2h2(cj.y), u2h2(ck.y)));
    const __half2 mxBA = __hmax2(__hmax2(u2h2(cf.y), u2h2(cg.y)), __hmax2(u2h2(cj.y), u2h2(ck.y)));
    const float2 aWf = __half22float2(aW);
    const __half2 r = __floats2half2_rn(rcp_approx(aWf.x), rcp_approx(aWf.y));
    const __half2 oR = __hmin2(__low2half2(mxRG), __hmax2(__low2half2(mnRG), __hmul2(aR, r)));
    const __half2 oG = __hmin2(__high2half2(mxRG), __hmax2(__high2half2(mnRG), __hmul2(aG, r)));
    const __half2 oB = __hmin2(__low2half2(mxBA), __hmax2(__low2half2(mnBA), __hmul2(aB, r)));
    outA = make_uint2(h22u(__lows2half2(oR, oG)), h22u(__lows2half2(oB, one)));
    outB = make_uint2(h22u(__highs2half2(oR, oG)), h22u(__highs2half2(oB, one)));
  } else {
    // pixel B's window is one input row further down: tap (R,K) of A is texel row R, of B texel row R+1
    __half2 aRG_A = kZero, aBA_A = kZero, aRG_B = kZero, aBA_B = kZero, aW = kZero;
#define FSR1_VTAP1(R, K)                                                                     \
    {                                                                                        \
      const uint2 ca = t0[(R) * BW + (K)], cb = t0[((R) + 1) * BW + (K)];                    \
      const __half2 w = tapw(R, K);                                                          \
      const __half2 wA2 = __low2half2(w), wB2 = __high2half2(w);                             \
      aRG_A = __hfma2(u2h2(ca.x), wA2, aRG_A);                                               \
      aBA_A = __hfma2(u2h2(ca.y), wA2, aBA_A);                                               \
      aRG_B = __hfma2(u2h2(cb.x), wB2, aRG_B);                                               \
      aBA_B = __hfma2(u2h2(cb.y), wB2, aBA_B);                                               \
      aW = __hadd2(aW, w);                                                                   \
    }
    FSR1_VTAP1(0, 1) FSR1_VTAP1(0, 2) FSR1_VTAP1(1, 0) FSR1_VTAP1(1, 3)
    FSR1_VTAP1(2, 0) FSR1_VTAP1(2, 3) FSR1_VTAP1(3, 1) FSR1_VTAP1(3, 2)
    FSR1_VTAP1(1, 1) FSR1_VTAP1(1, 2) FSR1_VTAP1(2, 1) FSR1_VTAP1(2, 2)
#undef FSR1_VTAP1
    const uint2 r1a = t0[BW + 1], r1b = t0[BW + 2], r2a = t0[2 * BW + 1], r2b = t0[2 * BW + 2];
    const uint2 r3a = t0[3 * BW + 1], r3b = t0[3 * BW + 2];
    const __half2 midMnRG = __hmin2(u2h2(r2a.x), u2h2(r2b.x)), midMxRG = __hmax2(u2h2(r2a.x), u2h2(r2b.x));
    const __half2 midMnBA = __hmin2(u2h2(r2a.y), u2h2(r2b.y)), midMxBA = __hmax2(u2h2(r2a.y), u2h2(r2b.y));
    const __half2 mnRG_A = __hmin2(__hmin2(u2h2(r1a.x), u2h2(r1b.x)), midMnRG), mxRG_A = __hmax2(__hmax2(u2h2(r1a.x), u2h2(r1b.x)), midMxRG);
    const __half2 mnBA_A = __hmin2(__hmin2(u2h2(r1a.y), u2h2(r1b.y)), midMnBA), mxBA_A = __hmax2(__hmax2(u2h2(r1a.y), u2h2(r1b.y)), midMxBA);
    const __half2 mnRG_B = __hmin2(__hmin2(u2h2(r3a.x), u2h2(r3b.x)), midMnRG), mxRG_B = __hmax2(__hmax2(u2h2(r3a.x), u2h2(r3b.x)), midMxRG);
    const __half2 mnBA_B = __hmin2(__hmin2(u2h2(r3a.y), u2h2(r3b.y)), midMnBA), mxBA_B = __hmax2(__hmax2(u2h2(r3a.y), u2h2(r3b.y)), midMxBA);
    const float2 aWf = __half22float2(aW);
    const __half2 rA = __float2half2_rn(rcp_approx(aWf.x)), rB = __float2half2_rn(rcp_approx(aWf.y));
    const __half2 oRG_A = __hmin2(mxRG_A, __hmax2(mnRG_A, __hmul2(aRG_A, rA)));
    const __half2 oBA_A = __hmin2(mxBA_A, __hmax2(mnBA_A, __hmul2(aBA_A, rA)));
    const __half2 oRG_B = __hmin2(mxRG_B, __hmax2(mnRG_B, __hmul2(aRG_B, rB)));
    const __half2 oBA_B = __hmin2(mxBA_B, __hmax2(mnBA_B, __hmul2(aBA_B, rB)));
    outA = make_uint2(h22u(oRG_A), h22u(__lows2half2(oBA_A, one)));   // alpha = 1 (FSR_Pass.hlsl:95)
    outB = make_uint2(h22u(oRG_B), h22u(__lows2half2(oBA_B, one)));
  }
}

// dynamic shared memory: [tile0][tile1][luma][terms][2 mbarriers], every part 128-byte aligned
__host__ __device__ inline size_t pairs_tile_stride(int BW, int BH) { return ((size_t)BW * BH * 8 + 127) & ~(size_t)127; }
__host__ __device__ inline size_t pairs_smem_bytes(int BW, int BH) {
  size_t off = 2 * pairs_tile_stride(BW, BH);
  off += ((size_t)BW * BH * 4 + 127) & ~(size_t)127;
  off += ((size_t)(BW - 2) * (BH - 2) * 16 + 127) & ~(size_t)127;
  return off + 16 + 128;  // + barriers + slack for the manual 128B alignment
}

// kR11: R11G11B10_FLOAT input (fsr1_r11.cuh): the box is BW4 = BW + 2 or + 4 texels wide (a multiple of 4), from the multiple of 4 at or
// before the half tile's origin.  BW * BH <= kR11Per * kThreads holds for every upscale (BW <= 68, BH <= 35; the launcher checks).
constexpr int kR11Per = 10;
// kIn != kInTma (FSR1_FLAG_IN_SURFACE / IN_TEXTURE): p.in.base is a surface or texture object on a CUDA array and `tmap` is unused;
// phase 1 reads the box with surface loads or texture fetches (array_texel) at coordinates clamped to the logical image (the texels
// TMA + clamp_fixup leave in it) into tile buffer 0.  (kInSurf is 1: the surface twins are still easu_h_pairs_kernel<k, false, 1>.)
template <bool kSrtmIn = false, bool kR11 = false, int kIn = kInTma>
__global__ void __launch_bounds__(kThreads, 3)
easu_h_pairs_kernel(const EasuParams p, const __grid_constant__ CUtensorMap tmap, const int BW, const int BH,
                    const int tiles_x, const int n_tiles) {
  constexpr bool kArrayIn = kIn != kInTma;  // no TMA, no mbarrier, no prefetch
#ifdef FSR1_CPU_EMU
  unsigned char* smem_raw = fsr1_emu_dynamic_smem();
#else
  extern __shared__ unsigned char smem_raw[];
#endif
  // 128-byte align by OFFSET (pointer arithmetic on the shared array keeps the address space -> LDS/STS)
  unsigned char* base = smem_raw + ((128u - (smem_u32(smem_raw) & 127u)) & 127u);
  const int n = BW * BH;
  const size_t tstride = pairs_tile_stride(BW, BH);
  float* L = reinterpret_cast<float*>(base + 2 * tstride);
  float4* S = reinterpret_cast<float4*>(base + 2 * tstride + (((size_t)n * 4 + 127) & ~(size_t)127));
  uint64_t* bar = reinterpret_cast<uint64_t*>(reinterpret_cast<unsigned char*>(S) +
                                              (((size_t)(BW - 2) * (BH - 2) * 16 + 127) & ~(size_t)127));
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (!kArrayIn) {
    if (tid == 0) {
      mbar_init(&bar[0], 1);
      mbar_init(&bar[1], 1);
      mbar_fence_init();
    }
    __syncthreads();
  }
  halo_sync_begin(p.sync);
  // box origin of tile t = first tap column/row of its first pixel; the column is rounded down to even because
  // TMA traps unless the box starts on a 16-byte boundary (2 texels)
  auto origin = [&](int t, int& ox0, int& oy0, int& fx0, int& fy0) {
    ox0 = (t % tiles_x) * kTileW;
    oy0 = p.y0 + (t / tiles_x) * kTileH;
    float dummy;
    easu_pos(ox0, p.c0x, p.c0z, fx0, dummy);
    easu_pos(oy0, p.c0y, p.c0w, fy0, dummy);
    fx0 = (fx0 - 1) & ~1;
    fy0 -= 1;
  };
  int t = blockIdx.x;
  if (!kArrayIn && tid == 0 && t < n_tiles) {
    int a, b, fx, fy;
    origin(t, a, b, fx, fy);
    mbar_expect_tx(&bar[0], kR11 ? (uint32_t)(((BW + 5) & ~3) * BH) * 4u : (uint32_t)n * 8u);
    tma_load_2d(base, &tmap, kR11 ? fx & ~3 : fx, fy - p.in.row0, &bar[0]);
  }
  for (int it = 0; t < n_tiles; t += gridDim.x, it++) {
  const int bsel = kArrayIn ? 0 : it & 1;
  if (!kArrayIn && tid == 0 && t + (int)gridDim.x < n_tiles) {  // prefetch the next tile into the other buffer
    int a, b, fx, fy;
    origin(t + gridDim.x, a, b, fx, fy);
    fence_proxy_async();
    mbar_expect_tx(&bar[bsel ^ 1], kR11 ? (uint32_t)(((BW + 5) & ~3) * BH) * 4u : (uint32_t)n * 8u);
    tma_load_2d(base + (bsel ^ 1) * tstride, &tmap, kR11 ? fx & ~3 : fx, fy - p.in.row0, &bar[bsel ^ 1]);
  }
  uint2* tile = reinterpret_cast<uint2*>(base + bsel * tstride);
  int ox0, oy0, fx0, fy0;
  origin(t, ox0, oy0, fx0, fy0);
  if (!kArrayIn) {
    mbar_wait(&bar[bsel], (it >> 1) & 1);
    if (fx0 < 0 || fy0 < 0 || fx0 + BW > p.in.w || fy0 + BH > p.in.h) {  // border tiles only (CTA-uniform)
      if constexpr (kR11) clamp_fixup(reinterpret_cast<uint32_t*>(tile) + (fx0 & 3), (BW + 5) & ~3, BW, BH, fx0, fy0, p.in.w, p.in.h, lane, warp, kThreads / 32);
      else clamp_fixup(tile, BW, BW, BH, fx0, fy0, p.in.w, p.in.h, lane, warp, kThreads / 32);
      fence_proxy_async();
      __syncthreads();
    }
  }

  if constexpr (kArrayIn) {  // phase 1 from the array, row and column stepped as phase 2 steps them
    const unsigned long long src = surf_of(p.in);
    int j = tid / BW, c = tid - j * BW;
    const int dj = kThreads / BW, dc = kThreads - dj * BW;
    for (int i = tid; i < n; i += kThreads) {
      uint2 v = array_texel<kIn, kR11>(src, clampi(fx0 + c, 0, p.in.w - 1), clampi(fy0 + j, 0, p.in.h - 1));
      if (kSrtmIn) v = srtm_texel(v);
      tile[i] = v;
      L[i] = texel_luma(v);
      c += dc; j += dj;
      if (c >= BW) { c -= BW; j += 1; }
    }
  } else if constexpr (kR11) {
    r11_phase1_inplace<kSrtmIn, kThreads, kR11Per>(tile, L, n, BW, (BW + 5) & ~3, fx0 & 3, tid);
  } else {
    for (int i = tid; i < n; i += kThreads) {  // phase 1
      uint2 c = tile[i];
      if (kSrtmIn) tile[i] = c = srtm_texel(c);
      L[i] = texel_luma(c);
    }
  }
  __syncthreads();

  // phase 2 over the (BW-2)x(BH-2) inner texels, flattened so that all lanes stay busy
  const int SW = BW - 2, nS = SW * (BH - 2);
  {
    int j = tid / SW, i = tid - j * SW;
    const int dj = kThreads / SW, di = kThreads - dj * SW;
    for (int idx = tid; idx < nS; idx += kThreads) {
      const float* c = L + (j + 1) * BW + (i + 1);
      S[idx] = texel_terms(c[-BW], c[-1], c[0], c[1], c[BW]);
      i += di; j += dj;
      if (i >= SW) { i -= SW; j += 1; }
    }
  }
  __syncthreads();

  // phase 3: a lane owns one output column and the VERTICAL pixel pair (oy, oy+1).  Whether the two rows fall in
  // the same input cell row (DR = 0) or in consecutive ones (DR = 1) depends on oy only, so it is warp-uniform:
  // DR = 0 loads 12 taps + 4 term vectors once for both pixels, DR = 1 loads a 5-row window (16 + 6).  Lanes walk
  // the input row at < 1 texel per lane: shared-memory reads are (nearly) conflict-free, which the earlier
  // horizontal pairing (1.3-2 texels per lane, two windows per lane) was not — it was LSU-bound (ncu: 72 %).
#pragma unroll 1
  for (int job = warp; job < (kTileW / 32) * (kTileH / 2); job += kThreads / 32) {
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
    const uint2* t0 = tile + (fyA - fy0 - 1) * BW + (fx - fx0 - 1);       // window origin: tap (0,0) of pixel A
    const float4* q0 = S + (fyA - fy0 - 1) * SW + (fx - fx0 - 1);          // term vector of texel f of pixel A
    uint2 oA, oB;
    if (fyB == fyA) vpair<0>(t0, q0, BW, SW, ppx, ppyA, ppyB, oA, oB);
    else vpair<1>(t0, q0, BW, SW, ppx, ppyA, ppyB, oA, oB);
    if (active) {
      unsigned char* o = p.out.base + (long long)(oyA - p.out.row0) * p.out.pitch + (long long)ox * 8;
      *reinterpret_cast<uint2*>(o) = oA;
      if (hasB) *reinterpret_cast<uint2*>(o + p.out.pitch) = oB;
    }
  }
  __syncthreads();  // L, S and this tile buffer are free again
  }  // persistent tile loop
  halo_sync_end(p.sync);
}


// =======================================================================================================
//  2x kernel: lane = the quad of output pixels sharing input cell (k,m); persistent, double-buffered TMA
// =======================================================================================================
template <int NW> struct __align__(128) QuadSmem {
  uint2 tile[2][QuadCfg<NW>::kPad];
  float4 S[kQSW * QuadCfg<NW>::kSH];
  float L[QuadCfg<NW>::kElems];
  uint64_t bar[2];
};

// kR11: R11G11B10_FLOAT input (fsr1_r11.cuh): a kUBW = 40 texel box from 2 texels left of the half tile's origin (32 tx - 4: 16 bytes)
constexpr int kUBW = kQBW + 4;
// kIn != kInTma (FSR1_FLAG_IN_SURFACE / IN_TEXTURE): p.in.base is a surface or texture object on a CUDA array and `tmap` is unused;
// phase 1 reads the box with surface loads or texture fetches (array_texel) at coordinates clamped to the logical image (the texels
// TMA + clamp_fixup leave in it) into one tile buffer, which the previous tile's closing barrier frees: no TMA, no mbarrier, no prefetch.
template <int NW, bool kSrtmIn, bool kR11, int kIn = kInTma>
__device__ __forceinline__ void quad_body(const EasuParams p, const CUtensorMap& tmap, const int tiles_x, const int n_tiles,
                                          const int mbase) {
  constexpr bool kArrayIn = kIn != kInTma;
  using C = QuadCfg<NW>;
  constexpr int NT = NW * 32;
  constexpr uint32_t kBoxBytes = kR11 ? kUBW * C::kBH * 4u : C::kElems * 8u;
  constexpr int kShift = kR11 ? 2 : 0;
  constexpr int kStage = ((kUBW * C::kBH * 4 + 127) / 128) * 128 / 4;
  __shared__ QuadSmem<NW> sm;
  uint32_t* stage = nullptr;  // kR11 by TMA: where the boxes land (fsr1_r11.cuh)
  if constexpr (kR11 && !kArrayIn) {
    __shared__ R11Stage<kStage> r11_stage;
    stage = &r11_stage.w[0][0];
  }
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (!kArrayIn) {
    if (tid == 0) {
      mbar_init(&sm.bar[0], 1);
      mbar_init(&sm.bar[1], 1);
      mbar_fence_init();
    }
    __syncthreads();
  }
  halo_sync_begin(p.sync);
  // tile (tx, ty): cells k in [32 tx - 1, +32), m in [mbase + kCY ty, +kCY); box origin = (first cell) - 1.
  // Tile coordinates advance incrementally: one division per kernel instead of one per tile and thread.
  int t = blockIdx.x;
  int tx = t % tiles_x, ty = t / tiles_x;
  const int step_x = (int)gridDim.x % tiles_x, step_y = (int)gridDim.x / tiles_x;
  if (!kArrayIn && tid == 0 && t < n_tiles) {
    mbar_expect_tx(&sm.bar[0], kBoxBytes);
    tma_load_2d(kR11 ? (void*)stage : (void*)sm.tile[0], &tmap, tx * kQCX - 2 - kShift, mbase + ty * C::kCY - 1 - p.in.row0, &sm.bar[0]);
  }
  for (int it = 0; t < n_tiles; t += gridDim.x, it++) {
    const int b = it & 1;
    int txn = tx + step_x, tyn = ty + step_y;  // coordinates of the CTA's next tile
    if (txn >= tiles_x) { txn -= tiles_x; tyn++; }
    if (!kArrayIn && tid == 0 && t + (int)gridDim.x < n_tiles) {  // prefetch it into the other buffer (its readers all passed
      fence_proxy_async();                                       // the barrier that closed the previous iteration)
      mbar_expect_tx(&sm.bar[b ^ 1], kBoxBytes);
      tma_load_2d(kR11 ? (void*)(stage + (b ^ 1) * kStage) : (void*)sm.tile[b ^ 1], &tmap, txn * kQCX - 2 - kShift,
                  mbase + tyn * C::kCY - 1 - p.in.row0, &sm.bar[b ^ 1]);
    }
    uint2* tile = sm.tile[kR11 || kArrayIn ? 0 : b];  // kR11, kArrayIn: phase 1 writes the half tile after the previous tile's closing barrier
    const int gx0 = tx * kQCX - 2, gy0 = mbase + ty * C::kCY - 1;
    tx = txn;
    ty = tyn;
    if (!kArrayIn) {
      mbar_wait(&sm.bar[b], (it >> 1) & 1);
      if (gx0 < 0 || gy0 < 0 || gx0 + kQBW > p.in.w || gy0 + C::kBH > p.in.h) {
        if constexpr (kR11) clamp_fixup(stage + b * kStage + kShift, kUBW, kQBW, C::kBH, gx0, gy0, p.in.w, p.in.h, lane, warp, NW);
        else clamp_fixup(tile, kQBW, kQBW, C::kBH, gx0, gy0, p.in.w, p.in.h, lane, warp, NW);
        fence_proxy_async();  // these generic-proxy writes are later overwritten by a TMA (async proxy) load
        __syncthreads();
      }
    }
    if constexpr (kArrayIn) {
      const unsigned long long src = surf_of(p.in);
      for (int i = tid; i < C::kElems; i += NT) {
        const int j = i / kQBW, c = i - j * kQBW;
        uint2 v = array_texel<kIn, kR11>(src, clampi(gx0 + c, 0, p.in.w - 1), clampi(gy0 + j, 0, p.in.h - 1));
        if (kSrtmIn) v = srtm_texel(v);
        tile[i] = v;
        sm.L[i] = texel_luma(v);
      }
    } else if constexpr (kR11) {
      r11_phase1_staged<kSrtmIn, NT>(stage + b * kStage, tile, sm.L, C::kElems, kQBW, kUBW, kShift, tid);
    } else {
      for (int i = tid; i < C::kElems; i += NT) {
        uint2 c = tile[i];
        if (kSrtmIn) tile[i] = c = srtm_texel(c);
        sm.L[i] = texel_luma(c);
      }
    }
    __syncthreads();
    for (int idx = tid; idx < kQSW * C::kSH; idx += NT) {
      const int j = idx / kQSW, i = idx - j * kQSW;
      const float* c = sm.L + (j + 1) * kQBW + (i + 1);
      sm.S[idx] = texel_terms(c[-kQBW], c[-1], c[0], c[1], c[kQBW]);
    }
    __syncthreads();
    // every output pixel of the tile (columns 2(gx0+1)+1 .. 2(gx0+32)+2, rows 2(gy0+1)+1 .. 2(gy0+2NW)+2) in range?
    const bool inside = 2 * (gx0 + 1) + 1 >= 0 && 2 * (gx0 + 32) + 2 < p.out.w && 2 * (gy0 + 1) + 1 >= p.y0 &&
                        2 * (gy0 + C::kCY) + 2 < p.y1;
    if (inside) {
#pragma unroll 1
      for (int q = 0; q < 2; q++) quad_cell<true>(p, tile, sm.S, gx0, gy0, lane, warp + q * NW);
    } else {
#pragma unroll 1
      for (int q = 0; q < 2; q++) quad_cell<false>(p, tile, sm.S, gx0, gy0, lane, warp + q * NW);
    }
    __syncthreads();  // L, S and this tile buffer are free again
  }
  halo_sync_end(p.sync);
}

template <int NW, int MINB, bool kSrtmIn = false>
__global__ void __launch_bounds__(NW * 32, MINB)
easu_h_quad2x_kernel(const EasuParams p, const __grid_constant__ CUtensorMap tmap, const int tiles_x,
                     const int n_tiles, const int mbase) {
  quad_body<NW, kSrtmIn, false>(p, tmap, tiles_x, n_tiles, mbase);
}
// FSR1_FLAG_IN_SURFACE: the RGBA16F kernel reading its input through a surface object (`tmap` unused)
template <int NW, int MINB, bool kSrtmIn>
__global__ void __launch_bounds__(NW * 32, MINB)
easu_h_quad2x_surf_in_kernel(const EasuParams p, const __grid_constant__ CUtensorMap tmap, const int tiles_x, const int n_tiles,
                             const int mbase) {
  quad_body<NW, kSrtmIn, false, kInSurf>(p, tmap, tiles_x, n_tiles, mbase);
}
// FSR1_FLAG_IN_TEXTURE: the RGBA16F or (kR11) R11G11B10F kernel reading its input through a texture object (`tmap` unused)
template <int NW, int MINB, bool kSrtmIn, bool kR11>
__global__ void __launch_bounds__(NW * 32, MINB)
easu_h_quad2x_tex_in_kernel(const EasuParams p, const __grid_constant__ CUtensorMap tmap, const int tiles_x, const int n_tiles,
                            const int mbase) {
  quad_body<NW, kSrtmIn, kR11, kInTex>(p, tmap, tiles_x, n_tiles, mbase);
}
template <int NW, int MINB, bool kSrtmIn>
__global__ void __launch_bounds__(NW * 32, MINB)
easu_r11_quad2x_kernel(const EasuParams p, const __grid_constant__ CUtensorMap tmap, const int tiles_x,
                       const int n_tiles, const int mbase) {
  quad_body<NW, kSrtmIn, true>(p, tmap, tiles_x, n_tiles, mbase);
}

// ---- 2x EASU for the UNORM formats the sample renders into (sample/src/DX12/FSR_Filter.cpp:72-73) -------------------
// Same phases as easu_h_quad2x_kernel.  The TMA box holds 4-byte texels (origin rounded down to 4 texels = 16 bytes, so
// the box is 40 wide); one pass decodes it (c / (2^n - 1), fp32) into the half tile the tap loop reads and into the
// fp32 luma plane; the epilogue re-encodes in the half domain (StoreUnorm).
template <int NW> struct __align__(128) QuadSmemU {
  uint32_t stage[2][((kUBW * QuadCfg<NW>::kBH * 4 + 127) / 128) * 128 / 4];
  uint2 tile[QuadCfg<NW>::kPad];
  float4 S[kQSW * QuadCfg<NW>::kSH];
  float L[QuadCfg<NW>::kElems];
  uint64_t bar[2];
};

template <int kBits> __device__ __forceinline__ float3 unorm_decode(uint32_t u) {
  if (kBits == 8) {
    const float s = 255.0f, k = 1.0f / 255.0f;
    return make_float3(unorm_to_float(u & 255u, s, k), unorm_to_float((u >> 8) & 255u, s, k), unorm_to_float((u >> 16) & 255u, s, k));
  }
  const float s = 1023.0f, k = 1.0f / 1023.0f;
  return make_float3(unorm_to_float(u & 1023u, s, k), unorm_to_float((u >> 10) & 1023u, s, k), unorm_to_float((u >> 20) & 1023u, s, k));
}

template <int NW, int MINB, int kBits>
__global__ void __launch_bounds__(NW * 32, MINB)
easu_u_quad2x_kernel(const EasuParams p, const __grid_constant__ CUtensorMap tmap, const int tiles_x, const int n_tiles,
                     const int mbase) {
  using C = QuadCfg<NW>;
  constexpr int NT = NW * 32;
  constexpr uint32_t kBoxBytes = kUBW * C::kBH * 4u;
  __shared__ QuadSmemU<NW> sm;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) {
    mbar_init(&sm.bar[0], 1);
    mbar_init(&sm.bar[1], 1);
    mbar_fence_init();
  }
  __syncthreads();
  int t = blockIdx.x;
  int tx = t % tiles_x, ty = t / tiles_x;
  const int step_x = (int)gridDim.x % tiles_x, step_y = (int)gridDim.x / tiles_x;
  // tile (tx, ty): half tile origin gx0 = 32 tx - 2 (as in the half kernel); the staging box starts 2 texels further left
  if (tid == 0 && t < n_tiles) {
    mbar_expect_tx(&sm.bar[0], kBoxBytes);
    tma_load_2d(sm.stage[0], &tmap, tx * kQCX - 4, mbase + ty * C::kCY - 1 - p.in.row0, &sm.bar[0]);
  }
  for (int it = 0; t < n_tiles; t += gridDim.x, it++) {
    const int b = it & 1;
    int txn = tx + step_x, tyn = ty + step_y;
    if (txn >= tiles_x) { txn -= tiles_x; tyn++; }
    if (tid == 0 && t + (int)gridDim.x < n_tiles) {
      fence_proxy_async();
      mbar_expect_tx(&sm.bar[b ^ 1], kBoxBytes);
      tma_load_2d(sm.stage[b ^ 1], &tmap, txn * kQCX - 4, mbase + tyn * C::kCY - 1 - p.in.row0, &sm.bar[b ^ 1]);
    }
    const int gx0 = tx * kQCX - 2, gy0 = mbase + ty * C::kCY - 1;
    tx = txn;
    ty = tyn;
    uint32_t* stage = sm.stage[b];
    mbar_wait(&sm.bar[b], (it >> 1) & 1);
    if (gx0 < 0 || gy0 < 0 || gx0 + kQBW > p.in.w || gy0 + C::kBH > p.in.h) {  // zero fill -> clamp-to-edge, on the raw texels
      clamp_fixup(stage + 2, kUBW, kQBW, C::kBH, gx0, gy0, p.in.w, p.in.h, lane, warp, NW);
      fence_proxy_async();
      __syncthreads();
    }
    for (int i = tid; i < C::kElems; i += NT) {  // decode: half tile for the taps, fp32 luma for the analysis
      const int j = i / kQBW, c = i - j * kQBW;
      const float3 v = unorm_decode<kBits>(stage[j * kUBW + 2 + c]);
      sm.tile[i] = make_uint2(h22u(__floats2half2_rn(v.x, v.y)), h22u(__floats2half2_rn(v.z, 1.0f)));
      sm.L[i] = fmaf(v.z, 0.5f, fmaf(v.x, 0.5f, v.y));
    }
    __syncthreads();
    for (int idx = tid; idx < kQSW * C::kSH; idx += NT) {
      const int j = idx / kQSW, i = idx - j * kQSW;
      const float* c = sm.L + (j + 1) * kQBW + (i + 1);
      sm.S[idx] = texel_terms(c[-kQBW], c[-1], c[0], c[1], c[kQBW]);
    }
    __syncthreads();
    const bool inside = 2 * (gx0 + 1) + 1 >= 0 && 2 * (gx0 + 32) + 2 < p.out.w && 2 * (gy0 + 1) + 1 >= p.y0 &&
                        2 * (gy0 + C::kCY) + 2 < p.y1;
    if (inside) {
#pragma unroll 1
      for (int q = 0; q < 2; q++) quad_cell<true, StoreUnorm<kBits>>(p, sm.tile, sm.S, gx0, gy0, lane, warp + q * NW);
    } else {
#pragma unroll 1
      for (int q = 0; q < 2; q++) quad_cell<false, StoreUnorm<kBits>>(p, sm.tile, sm.S, gx0, gy0, lane, warp + q * NW);
    }
    __syncthreads();  // stage, tile, L and S are free again
  }
}

#ifndef FSR1_CPU_EMU
// ---- host side ----------------------------------------------------------------------------------------
// one texel = one TMA element (64-bit for RGBA16F, 32-bit for the UNORM formats); tensor = the stored window of the image
static bool make_tmap(CUtensorMap* tmap, const ImgView& in, int BW, int BH, CUtensorMapDataType type = CU_TENSOR_MAP_DATA_TYPE_UINT64) {
  EncodeTiledFn encode = get_encode_fn();
  if (!encode) return false;
  const cuuint64_t dims[2] = {(cuuint64_t)in.w, (cuuint64_t)in.rows};
  const cuuint64_t strides[1] = {(cuuint64_t)in.pitch};
  const cuuint32_t box[2] = {(cuuint32_t)BW, (cuuint32_t)BH};
  const cuuint32_t estr[2] = {1, 1};
  return encode(tmap, type, 2, in.base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// Largest footprint (in texels) any tile of `tile` output pixels needs along one axis; with even_origin the
// box starts at the even texel at or before the first tap (see the kernel).
static int max_footprint(int n_out, int first, int tile, float scale, float offset, bool even_origin) {
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

// tiles of the 2x kernels: cells k in [-1, k_last], rows of cells from the one holding output row y0
struct QuadGrid { int tiles_x, n_tiles, m_first, grid; };
static QuadGrid quad_grid(const EasuParams& p, int cy, int ctas_per_sm) {
  QuadGrid g;
  const int k_first = -1, k_last = host_fp(p.out.w - 1, 0.5f, -0.25f);
  const int m_last = host_fp(p.y1 - 1, 0.5f, -0.25f);
  g.m_first = host_fp(p.y0, 0.5f, -0.25f);
  g.tiles_x = (k_last - k_first + 1 + kQCX - 1) / kQCX;
  g.n_tiles = g.tiles_x * ((m_last - g.m_first + 1 + cy - 1) / cy);
  g.grid = g.n_tiles < ctas_per_sm * sm_count() ? g.n_tiles : ctas_per_sm * sm_count();
  return g;
}

// R8G8B8A8_UNORM images at exactly 2x.  (R10G10B10A2 stays on the fp32 direct kernel: half taps are coarser than its codes,
// 2-4 code values off where the 8-bit format is within one; the caller also routes FSR1_FLAG_PRECISE / _EXACT there.)
cudaError_t launch_easu_u_tiled(const EasuParams& p, int format, cudaStream_t s, const char** name) {
  if (format != 3) return cudaErrorNotSupported;
  if ((reinterpret_cast<uintptr_t>(p.in.base) & 15) || (p.in.pitch & 15) || !is_2x(p.c0x, p.c0y, p.c0z, p.c0w)) return cudaErrorNotSupported;  // TMA
  constexpr int NW = 4, CY = 2 * NW;
  CUtensorMap tmap;
  if (!make_tmap(&tmap, p.in, kUBW, CY + 3, CU_TENSOR_MAP_DATA_TYPE_UINT32)) return cudaErrorNotSupported;
  const QuadGrid g = quad_grid(p, CY, 6);
  easu_u_quad2x_kernel<NW, 6, 8><<<g.grid, NW * 32, 0, s>>>(p, tmap, g.tiles_x, g.n_tiles, g.m_first);
  *name = "easu_u8_quad2x<4w,6/sm,tma2>";
  return cudaGetLastError();
}

cudaError_t launch_easu_h_tiled(const EasuParams& p, cudaStream_t s, const char** name, bool srtm_in, bool r11, InSrc in) {
  const bool surf_in = in == kInSurf, tex_in = in == kInTex, array_in = in != kInTma;
  // layout requirements of TMA and of the vector stores
  if ((!array_in && ((reinterpret_cast<uintptr_t>(p.in.base) & 15) || (p.in.pitch & 15))) || (reinterpret_cast<uintptr_t>(p.out.base) & 15) ||
      (p.out.pitch & 15))
    return cudaErrorNotSupported;
  CUtensorMap tmap;
  if (array_in) memset(&tmap, 0, sizeof tmap);  // read by no kernel: the input is a surface or texture object
  const CUtensorMapDataType type = r11 ? CU_TENSOR_MAP_DATA_TYPE_UINT32 : CU_TENSOR_MAP_DATA_TYPE_UINT64;

  if (is_2x(p.c0x, p.c0y, p.c0z, p.c0w)) {
    // 4 warps x 7 CTAs per SM: the kernel needs 72 registers, exactly what 7 x 128 threads allow.  A launch that waits
    // for a neighbour's halo (p.sync, fsr1_shard.cu) is capped at 6 CTAs per SM: at 7 every warp scheduler's 16384
    // registers are taken but 256, so the one-warp halo_push_kernel that the wait depends on cannot be placed beside a
    // grid that fills every SM, and ranks sharing one GPU would wait for each other until the spin timeout.
    constexpr int NW = 4, CY = 2 * NW;
    if (!array_in && !make_tmap(&tmap, p.in, r11 ? kUBW : kQBW, CY + 3, type)) return cudaErrorNotSupported;
    const QuadGrid g = quad_grid(p, CY, (p.sync.ready[0] || p.sync.ready[1]) ? 6 : 7);
    if (tex_in) {
      if (r11 && srtm_in) easu_h_quad2x_tex_in_kernel<NW, 7, true, true><<<g.grid, NW * 32, 0, s>>>(p, tmap, g.tiles_x, g.n_tiles, g.m_first);
      else if (r11) easu_h_quad2x_tex_in_kernel<NW, 7, false, true><<<g.grid, NW * 32, 0, s>>>(p, tmap, g.tiles_x, g.n_tiles, g.m_first);
      else if (srtm_in) easu_h_quad2x_tex_in_kernel<NW, 7, true, false><<<g.grid, NW * 32, 0, s>>>(p, tmap, g.tiles_x, g.n_tiles, g.m_first);
      else easu_h_quad2x_tex_in_kernel<NW, 7, false, false><<<g.grid, NW * 32, 0, s>>>(p, tmap, g.tiles_x, g.n_tiles, g.m_first);
      *name = r11 ? (srtm_in ? "easu_h_quad2x<4w,7/sm,r11g11b10f_in,srtm_in,tex_in>" : "easu_h_quad2x<4w,7/sm,r11g11b10f_in,tex_in>")
                  : (srtm_in ? "easu_h_quad2x<4w,7/sm,srtm_in,tex_in>" : "easu_h_quad2x<4w,7/sm,tex_in>");
    } else if (surf_in) {
      if (srtm_in) easu_h_quad2x_surf_in_kernel<NW, 7, true><<<g.grid, NW * 32, 0, s>>>(p, tmap, g.tiles_x, g.n_tiles, g.m_first);
      else easu_h_quad2x_surf_in_kernel<NW, 7, false><<<g.grid, NW * 32, 0, s>>>(p, tmap, g.tiles_x, g.n_tiles, g.m_first);
      *name = srtm_in ? "easu_h_quad2x<4w,7/sm,srtm_in,surf_in>" : "easu_h_quad2x<4w,7/sm,surf_in>";
    } else if (r11 && srtm_in) {
      easu_r11_quad2x_kernel<NW, 7, true><<<g.grid, NW * 32, 0, s>>>(p, tmap, g.tiles_x, g.n_tiles, g.m_first);
      *name = "easu_h_quad2x<4w,7/sm,tma2,r11g11b10f_in,srtm_in>";
    } else if (r11) {
      easu_r11_quad2x_kernel<NW, 7, false><<<g.grid, NW * 32, 0, s>>>(p, tmap, g.tiles_x, g.n_tiles, g.m_first);
      *name = "easu_h_quad2x<4w,7/sm,tma2,r11g11b10f_in>";
    } else if (srtm_in) {
      easu_h_quad2x_kernel<NW, 7, true><<<g.grid, NW * 32, 0, s>>>(p, tmap, g.tiles_x, g.n_tiles, g.m_first);
      *name = "easu_h_quad2x<4w,7/sm,tma2,srtm_in>";
    } else {
      easu_h_quad2x_kernel<NW, 7><<<g.grid, NW * 32, 0, s>>>(p, tmap, g.tiles_x, g.n_tiles, g.m_first);
      *name = "easu_h_quad2x<4w,7/sm,tma2>";
    }
    return cudaGetLastError();
  }

  if (!is_upscale(p.c0x, p.c0y)) return cudaErrorNotSupported;
  int BW = max_footprint(p.out.w, 0, kTileW, p.c0x, p.c0z, true);
  int BH = max_footprint(p.y1, p.y0, kTileH, p.c0y, p.c0w, false);
  BW = (BW + 1) & ~1;  // inner box extent must be a multiple of 16 bytes
  if (BW > 256 || BH > 256) return cudaErrorNotSupported;
  if (r11 && BW * BH > kR11Per * kThreads) return cudaErrorNotSupported;  // cannot happen when upscaling (pairs_body)
  const size_t smem = pairs_smem_bytes(BW, BH);
  if (smem > 200 * 1024) return cudaErrorNotSupported;
  if (!array_in && !make_tmap(&tmap, p.in, r11 ? (BW + 5) & ~3 : BW, BH, type)) return cudaErrorNotSupported;
  void (*kernel)(const EasuParams, const CUtensorMap, const int, const int, const int, const int) =
      tex_in  ? (r11 ? (srtm_in ? easu_h_pairs_kernel<true, true, kInTex> : easu_h_pairs_kernel<false, true, kInTex>)
                     : (srtm_in ? easu_h_pairs_kernel<true, false, kInTex> : easu_h_pairs_kernel<false, false, kInTex>))
      : surf_in ? (srtm_in ? easu_h_pairs_kernel<true, false, kInSurf> : easu_h_pairs_kernel<false, false, kInSurf>)
      : r11   ? (srtm_in ? easu_h_pairs_kernel<true, true> : easu_h_pairs_kernel<false, true>)
              : (srtm_in ? easu_h_pairs_kernel<true, false> : easu_h_pairs_kernel<false, false>);
  if (smem > 48 * 1024) {  // per device and cheap: set on every launch that needs the opt-in
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  const int tiles_x = (p.out.w + kTileW - 1) / kTileW, n_tiles = tiles_x * ((p.y1 - p.y0 + kTileH - 1) / kTileH);
  int per_sm = 3;
  while (per_sm > 1 && (size_t)per_sm * (smem + 1024) > 220 * 1024) per_sm--;
  const int grid = n_tiles < per_sm * sm_count() ? n_tiles : per_sm * sm_count();
  kernel<<<grid, kThreads, smem, s>>>(p, tmap, BW, BH, tiles_x, n_tiles);
  *name = tex_in  ? (r11 ? (srtm_in ? "easu_h_vpairs<64x32,persistent,r11g11b10f_in,srtm_in,tex_in>" : "easu_h_vpairs<64x32,persistent,r11g11b10f_in,tex_in>")
                         : (srtm_in ? "easu_h_vpairs<64x32,persistent,srtm_in,tex_in>" : "easu_h_vpairs<64x32,persistent,tex_in>"))
          : surf_in ? (srtm_in ? "easu_h_vpairs<64x32,persistent,srtm_in,surf_in>" : "easu_h_vpairs<64x32,persistent,surf_in>")
          : r11   ? (srtm_in ? "easu_h_vpairs<64x32,persistent,tma2,r11g11b10f_in,srtm_in>" : "easu_h_vpairs<64x32,persistent,tma2,r11g11b10f_in>")
                  : (srtm_in ? "easu_h_vpairs<64x32,persistent,tma2,srtm_in>" : "easu_h_vpairs<64x32,persistent,tma2>");
  return cudaGetLastError();
}

#endif  // FSR1_CPU_EMU

}  // namespace fsr1
