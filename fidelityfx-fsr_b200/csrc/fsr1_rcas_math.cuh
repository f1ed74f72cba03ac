// fsr1_rcas_math.cuh — the RCAS arithmetic for TWO pixels in packed half2, shared by the packed RCAS kernels
// (fsr1_rcas_packed.cu: RGBA16F and UNORM images) and the fused EASU->RCAS kernel (fsr1_fused.cu).
//
// Structure-of-arrays like the reference's FsrRcasHx2 (ffx-fsr/ffx_fsr1.h:888-984): (R0,R1) (G0,G1) (B0,B1).
// Numerics: the six "high precision" reciprocals (ffx_fsr1.h:750-755) are rcp.approx.f32 on the unpacked halves
// (h2rcp, MUFU; a packed Newton iteration on the fp16 pipe measured slower); the resolve reciprocal is the packed
// APrxMedRcpH2 (ffx_a.h:1815).  Against the fp32 oracle on the same half input: <= 2e-3 (tolerance 1e-2).  min/max are
// the non-propagating half2 forms, so the 0*inf NaNs of flat black / white neighbourhoods drop out exactly as with
// HLSL min/max (:756-759).
// The reference's compile-time options are template bits here (no fallback to a slower kernel):
//   kRcasDenoise   FSR_RCAS_DENOISE           (ffx_fsr1.h:651,731-739,761-763)
//   kRcasAlpha     FSR_RCAS_PASSTHROUGH_ALPHA (:648,688-702): output alpha = the centre pixel's alpha (else 1)
//   kRcasSquare    the sample's Sample.x hook (sample/src/DX12/FSR_Pass.hlsl:93-94): c *= c before the store
#pragma once
#include "fsr1_common.cuh"

namespace fsr1 {

enum { kRcasDenoise = 1, kRcasAlpha = 2, kRcasSquare = 4 };

struct Row3 { __half2 r, g, b; };  // (pixel0, pixel1) per channel

__device__ __forceinline__ __half2 uh2(uint32_t u) { return *reinterpret_cast<__half2*>(&u); }
__device__ __forceinline__ uint32_t hu2(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }

// lobe of one channel for two pixels:  max(-hitMin, hitMax) = -min( min(mn4,e)/(4 mx4), (1-max(mx4,e))/(4-4 mn4) )
__device__ __forceinline__ __half2 lobe_channel(__half2 b, __half2 d, __half2 e, __half2 f, __half2 h) {
  const __half2 mn4 = __hmin2(__hmin2(b, d), __hmin2(f, h));
  const __half2 mx4 = __hmax2(__hmax2(b, d), __hmax2(f, h));
  const __half2 k4 = __float2half2_rn(4.0f), k1 = __float2half2_rn(1.0f), km4 = __float2half2_rn(-4.0f);
  const __half2 hitMin = __hmul2(__hmin2(mn4, e), h2rcp(__hmul2(k4, mx4)));
  const __half2 negHitMax = __hmul2(__hsub2(k1, __hmax2(mx4, e)), h2rcp(__hfma2(km4, mn4, k4)));
  return __hneg2(__hmin2(hitMin, negHitMax));  // __hmin2 drops the 0*inf NaN of a flat black / white ring
}

__device__ __forceinline__ __half2 resolve_channel(__half2 lobe, __half2 rcpL, __half2 b, __half2 d, __half2 e,
                                                   __half2 f, __half2 h) {
  const __half2 ring = __hadd2(__hadd2(b, d), __hadd2(h, f));
  return __hmul2(__hfma2(lobe, ring, e), rcpL);
}

__device__ __forceinline__ __half2 luma2x(const Row3& c) {  // bL = bB*0.5 + (bR*0.5 + bG)   (ffx_fsr1.h:725-729)
  const __half2 kHalf = __float2half2_rn(0.5f);
  return __hfma2(c.b, kHalf, __hfma2(c.r, kHalf, c.g));
}

// packed APrxMedRcpH2 (ffx_a.h:1815): 16-bit magic subtract + one Newton step.  The subtract wraps inside each 16-bit lane as the
// reference's does: a 32-bit 0x778d778d - a would let a low lane above 0x778d (the denoise range of overflowing content: >= 30928,
// inf or NaN) borrow from the other pixel's lane.  Per lane: (K | 0x8000) - (a & 0x7fff) cannot borrow across lanes, and the XOR
// restores bit 15 of K - a.
__device__ __forceinline__ __half2 prx_med_rcp_h2(__half2 a) {
  const uint32_t u = hu2(a);
  const __half2 s = uh2((0xf78df78du - (u & 0x7fff7fffu)) ^ (~(u ^ 0x778d778du) & 0x80008000u));
  return __hmul2(s, __hfma2(__hneg2(s), a, __float2half2_rn(2.0f)));
}

// b above, d left, e centre, f right, h below: each the pixel pair's taps per channel.  sharp = half2(con.y).
template <int kOpt>
__device__ __forceinline__ void rcas_pair(const Row3& b, const Row3& d, const Row3& e, const Row3& f, const Row3& h, __half2 sharp,
                                          __half2& oR, __half2& oG, __half2& oB) {
  const __half2 kLimit = __float2half2_rn(-0.1875f), kZero = __float2half2_rn(0.0f);
  const __half2 lR = lobe_channel(b.r, d.r, e.r, f.r, h.r);
  const __half2 lG = lobe_channel(b.g, d.g, e.g, f.g, h.g);
  const __half2 lB = lobe_channel(b.b, d.b, e.b, f.b, h.b);
  __half2 lobe = __hmul2(__hmax2(kLimit, __hmin2(__hmax2(lR, __hmax2(lG, lB)), kZero)), sharp);
  if (kOpt & kRcasDenoise) {
    const __half2 bL = luma2x(b), dL = luma2x(d), eL = luma2x(e), fL = luma2x(f), hL = luma2x(h);
    const __half2 q = __float2half2_rn(0.25f), one = __float2half2_rn(1.0f);
    // nz = 0.25 bL + 0.25 dL + 0.25 fL + 0.25 hL - eL, in the reference's order (ffx_fsr1.h:731)
    __half2 nz = __hsub2(__hfma2(q, hL, __hfma2(q, fL, __hfma2(q, dL, __hmul2(q, bL)))), eL);
    const __half2 mx = __hmax2(__hmax2(__hmax2(bL, dL), eL), __hmax2(fL, hL));
    const __half2 mn = __hmin2(__hmin2(__hmin2(bL, dL), eL), __hmin2(fL, hL));
    nz = __hmul2(__habs2(nz), prx_med_rcp_h2(__hsub2(mx, mn)));
    nz = __hmin2(one, __hmax2(nz, kZero));  // saturate; a flat neighbourhood's 0*inf NaN becomes 0 like HLSL saturate
    nz = __hfma2(__float2half2_rn(-0.5f), nz, one);
    lobe = __hmul2(lobe, nz);
  }
  const __half2 rcpL = prx_med_rcp_h2(__hfma2(__float2half2_rn(4.0f), lobe, __float2half2_rn(1.0f)));
  oR = resolve_channel(lobe, rcpL, b.r, d.r, e.r, f.r, h.r);
  oG = resolve_channel(lobe, rcpL, b.g, d.g, e.g, f.g, h.g);
  oB = resolve_channel(lobe, rcpL, b.b, d.b, e.b, f.b, h.b);
  if (kOpt & kRcasSquare) {
    oR = __hmul2(oR, oR);
    oG = __hmul2(oG, oG);
    oB = __hmul2(oB, oB);
  }
}

// SoA pair -> two RGBA16F pixels; alpha = (A0,A1) as half2
__device__ __forceinline__ uint4 pack_pair_half(__half2 oR, __half2 oG, __half2 oB, uint32_t alpha) {
  return make_uint4(__byte_perm(hu2(oR), hu2(oG), 0x5410), __byte_perm(hu2(oB), alpha, 0x5410), __byte_perm(hu2(oR), hu2(oG), 0x7632),
                    __byte_perm(hu2(oB), alpha, 0x7632));
}

}  // namespace fsr1
