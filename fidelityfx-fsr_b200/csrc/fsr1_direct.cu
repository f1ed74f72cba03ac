// fsr1_direct.cu — direct-load EASU and RCAS kernels in fp32 arithmetic.
//
// One thread per output pixel, taps fetched straight from global memory (read-only path, L1/L2
// absorb the 12x / 5x reuse).  These kernels are (a) the fp32-image path, (b) with kExact the
// bit-exact parity path (no FMA contraction), and (c) the fallback for fp16 images whose layout
// the TMA/vector kernels cannot take.  The packed-half production kernels are in
// fsr1_easu_tiled.cu and fsr1_rcas_packed.cu.
//
// Algorithm per pixel (what the reference's FsrEasuF / FsrRcasF compute, ffx-fsr/ffx_fsr1.h:315-437,
// 684-769):  EASU = luma of 12 taps -> per-texel edge direction/length for the 4 nearest texels,
// bilinearly blended -> normalise -> anisotropic rotated Lanczos-like window -> 12 weighted taps ->
// divide, clamp to min/max of the 4 nearest.  RCAS = 5-tap cross, solve the largest negative lobe
// that does not clip, limit, resolve with a medium-precision reciprocal.
#include "fsr1_common.cuh"

namespace fsr1 {

// Per-texel direction/length term, lA..lE = up, left, centre, right, down lumas.
template <bool kExact>
__device__ __forceinline__ void easu_set(float& dx, float& dy, float& len, float w, float lA, float lB, float lC,
                                         float lD, float lE) {
  using A = Ar<kExact>;
  const float dc = A::sub(lD, lC), cb = A::sub(lC, lB);
  float lenX = prx_lo_rcp(fmaxf(fabsf(dc), fabsf(cb)));
  const float dirX = A::sub(lD, lB);
  dx = A::mad(dirX, w, dx);
  lenX = sat(A::mul(fabsf(dirX), lenX));
  lenX = A::mul(lenX, lenX);
  len = A::mad(lenX, w, len);
  const float ec = A::sub(lE, lC), ca = A::sub(lC, lA);
  float lenY = prx_lo_rcp(fmaxf(fabsf(ec), fabsf(ca)));
  const float dirY = A::sub(lE, lA);
  dy = A::mad(dirY, w, dy);
  lenY = sat(A::mul(fabsf(dirY), lenY));
  lenY = A::mul(lenY, lenY);
  len = A::mad(lenY, w, len);
}

template <bool kExact>
__device__ __forceinline__ void easu_tap(float3& aC, float& aW, float ox, float oy, float dx, float dy, float l2x,
                                         float l2y, float lob, float clp, float3 c) {
  using A = Ar<kExact>;
  float vx = A::add(A::mul(ox, dx), A::mul(oy, dy));
  float vy = A::add(A::mul(ox, -dy), A::mul(oy, dx));
  vx = A::mul(vx, l2x);
  vy = A::mul(vy, l2y);
  float d2 = A::add(A::mul(vx, vx), A::mul(vy, vy));
  d2 = fminf(d2, clp);
  float wB = A::mad(0.4f, d2, -1.0f);
  float wA = A::mad(lob, d2, -1.0f);
  wB = A::mul(wB, wB);
  wA = A::mul(wA, wA);
  wB = A::mad(1.5625f, wB, -0.5625f);
  const float w = A::mul(wB, wA);
  aC.x = A::mad(c.x, w, aC.x);
  aC.y = A::mad(c.y, w, aC.y);
  aC.z = A::mad(c.z, w, aC.z);
  aW = A::add(aW, w);
}

template <bool kExact> __device__ __forceinline__ float luma(float3 c) {
  using A = Ar<kExact>;
  return A::add(A::mul(c.z, 0.5f), A::add(A::mul(c.x, 0.5f), c.y));  // 2*luma = 0.5B + (0.5R + G)
}

// S: the input's storage, SO: the output's (the same but for R11G11B10_FLOAT input, which writes RGBA16F)
template <typename S, typename SO, bool kExact>
__device__ __forceinline__ void easu_direct_body(const EasuParams& p) {
  using A = Ar<kExact>;
  const int ox = blockIdx.x * 32 + threadIdx.x;
  const int oy = p.y0 + blockIdx.y * 8 + threadIdx.y;
  if (ox >= p.out.w || oy >= p.y1) return;
  int fx, fy;
  float ppx, ppy;
  easu_pos(ox, p.c0x, p.c0z, fx, ppx);
  easu_pos(oy, p.c0y, p.c0w, fy, ppy);
  // 4x4 window, corners unused:   b c / e f g h / i j k l / n o
  const int x0 = clampi(fx - 1, 0, p.in.w - 1), x1 = clampi(fx, 0, p.in.w - 1);
  const int x2 = clampi(fx + 1, 0, p.in.w - 1), x3 = clampi(fx + 2, 0, p.in.w - 1);
  const int y0 = clampi(fy - 1, 0, p.in.h - 1), y1 = clampi(fy, 0, p.in.h - 1);
  const int y2 = clampi(fy + 1, 0, p.in.h - 1), y3 = clampi(fy + 2, 0, p.in.h - 1);
  const float3 b = Px<S>::load(p.in, x1, y0), c = Px<S>::load(p.in, x2, y0);
  const float3 e = Px<S>::load(p.in, x0, y1), f = Px<S>::load(p.in, x1, y1);
  const float3 g = Px<S>::load(p.in, x2, y1), h = Px<S>::load(p.in, x3, y1);
  const float3 i = Px<S>::load(p.in, x0, y2), j = Px<S>::load(p.in, x1, y2);
  const float3 k = Px<S>::load(p.in, x2, y2), l = Px<S>::load(p.in, x3, y2);
  const float3 n = Px<S>::load(p.in, x1, y3), o = Px<S>::load(p.in, x2, y3);
  const float bL = luma<kExact>(b), cL = luma<kExact>(c), eL = luma<kExact>(e), fL = luma<kExact>(f);
  const float gL = luma<kExact>(g), hL = luma<kExact>(h), iL = luma<kExact>(i), jL = luma<kExact>(j);
  const float kL = luma<kExact>(k), lL = luma<kExact>(l), nL = luma<kExact>(n), oL = luma<kExact>(o);
  float dx = 0.0f, dy = 0.0f, len = 0.0f;
  const float ipx = A::sub(1.0f, ppx), ipy = A::sub(1.0f, ppy);
  easu_set<kExact>(dx, dy, len, A::mul(ipx, ipy), bL, eL, fL, gL, jL);
  easu_set<kExact>(dx, dy, len, A::mul(ppx, ipy), cL, fL, gL, hL, kL);
  easu_set<kExact>(dx, dy, len, A::mul(ipx, ppy), fL, iL, jL, kL, nL);
  easu_set<kExact>(dx, dy, len, A::mul(ppx, ppy), gL, jL, kL, lL, oL);
  float dirR = A::add(A::mul(dx, dx), A::mul(dy, dy));
  const bool zro = dirR < (1.0f / 32768.0f);
  dirR = prx_lo_rsq(dirR);
  dirR = zro ? 1.0f : dirR;
  dx = zro ? 1.0f : dx;
  dx = A::mul(dx, dirR);
  dy = A::mul(dy, dirR);
  len = A::mul(len, 0.5f);
  len = A::mul(len, len);
  const float stretch = A::mul(A::add(A::mul(dx, dx), A::mul(dy, dy)), prx_lo_rcp(fmaxf(fabsf(dx), fabsf(dy))));
  const float l2x = A::mad(A::sub(stretch, 1.0f), len, 1.0f);
  const float l2y = A::mad(-0.5f, len, 1.0f);
  const float lob = A::mad((float)((1.0 / 4.0 - 0.04) - 0.5), len, 0.5f);
  const float clp = prx_lo_rcp(lob);
  float3 aC = make_float3(0.f, 0.f, 0.f);
  float aW = 0.0f;
  const float xm = A::sub(-1.0f, ppx), x0f = A::sub(0.0f, ppx), xp = A::sub(1.0f, ppx), xq = A::sub(2.0f, ppx);
  const float ym = A::sub(-1.0f, ppy), y0f = A::sub(0.0f, ppy), yp = A::sub(1.0f, ppy), yq = A::sub(2.0f, ppy);
  // the reference's accumulation order: b c i j f e k l h g o n
  easu_tap<kExact>(aC, aW, x0f, ym, dx, dy, l2x, l2y, lob, clp, b);
  easu_tap<kExact>(aC, aW, xp, ym, dx, dy, l2x, l2y, lob, clp, c);
  easu_tap<kExact>(aC, aW, xm, yp, dx, dy, l2x, l2y, lob, clp, i);
  easu_tap<kExact>(aC, aW, x0f, yp, dx, dy, l2x, l2y, lob, clp, j);
  easu_tap<kExact>(aC, aW, x0f, y0f, dx, dy, l2x, l2y, lob, clp, f);
  easu_tap<kExact>(aC, aW, xm, y0f, dx, dy, l2x, l2y, lob, clp, e);
  easu_tap<kExact>(aC, aW, xp, yp, dx, dy, l2x, l2y, lob, clp, k);
  easu_tap<kExact>(aC, aW, xq, yp, dx, dy, l2x, l2y, lob, clp, l);
  easu_tap<kExact>(aC, aW, xq, y0f, dx, dy, l2x, l2y, lob, clp, h);
  easu_tap<kExact>(aC, aW, xp, y0f, dx, dy, l2x, l2y, lob, clp, g);
  easu_tap<kExact>(aC, aW, xp, yq, dx, dy, l2x, l2y, lob, clp, o);
  easu_tap<kExact>(aC, aW, x0f, yq, dx, dy, l2x, l2y, lob, clp, n);
  const float rW = A::rcp(aW);
  const float mnR = fminf(fminf(f.x, fminf(g.x, j.x)), k.x), mxR = fmaxf(fmaxf(f.x, fmaxf(g.x, j.x)), k.x);
  const float mnG = fminf(fminf(f.y, fminf(g.y, j.y)), k.y), mxG = fmaxf(fmaxf(f.y, fmaxf(g.y, j.y)), k.y);
  const float mnB = fminf(fminf(f.z, fminf(g.z, j.z)), k.z), mxB = fmaxf(fmaxf(f.z, fmaxf(g.z, j.z)), k.z);
  Px<SO>::store(p.out, ox, oy, fminf(mxR, fmaxf(mnR, A::mul(aC.x, rW))), fminf(mxG, fmaxf(mnG, A::mul(aC.y, rW))),
                fminf(mxB, fmaxf(mnB, A::mul(aC.z, rW))));
}

template <typename S, bool kExact>
__global__ void __launch_bounds__(256) easu_direct_kernel(const EasuParams p) {
  easu_direct_body<S, S, kExact>(p);
}

// R11G11B10_FLOAT input: every texel decoded exactly (r11_to_half) to fp32; the output is RGBA16F
__global__ void __launch_bounds__(256) easu_direct_r11_kernel(const EasuParams p) { easu_direct_body<R11f, __half, false>(p); }

template <typename S>
__device__ __forceinline__ float3 rcas_fetch(const RcasParams& p, int x, int y) {
  if (p.clamp) {
    x = clampi(x, 0, p.in.w - 1);
    y = clampi(y, 0, p.in.h - 1);
  } else if (x < 0 || y < 0 || x >= p.in.w || y >= p.in.h) {
    return make_float3(0.f, 0.f, 0.f);
  }
  return Px<S>::load(p.in, x, y);
}

template <bool kExact>
__device__ __forceinline__ float rcas_lobe(float b, float d, float e, float f, float h) {
  using A = Ar<kExact>;
  const float mn4 = fminf(fminf(b, fminf(d, f)), h);
  const float mx4 = fmaxf(fmaxf(b, fmaxf(d, f)), h);
  const float hitMin = A::mul(fminf(mn4, e), A::rcp(A::mul(4.0f, mx4)));
  const float hitMax = A::mul(A::sub(1.0f, fmaxf(mx4, e)), A::rcp(A::mad(4.0f, mn4, -4.0f)));
  return fmaxf(-hitMin, hitMax);  // fmaxf drops the NaN of 0*inf, like HLSL max
}

template <bool kExact>
__device__ __forceinline__ float rcas_resolve(float lobe, float rcpL, float b, float d, float e, float f, float h) {
  using A = Ar<kExact>;
  // ((((lobe*b + lobe*d) + lobe*h) + lobe*f) + e) * rcpL
  float s = A::mul(lobe, b);
  s = A::mad(lobe, d, s);
  s = A::mad(lobe, h, s);
  s = A::mad(lobe, f, s);
  s = A::add(s, e);
  return A::mul(s, rcpL);
}

template <typename S, bool kExact>
__global__ void __launch_bounds__(256) rcas_direct_kernel(const RcasParams p) {
  using A = Ar<kExact>;
  const int x = blockIdx.x * 32 + threadIdx.x;
  const int y = p.y0 + blockIdx.y * 8 + threadIdx.y;
  if (x >= p.out.w || y >= p.y1) return;
  const float3 b = rcas_fetch<S>(p, x, y - 1), d = rcas_fetch<S>(p, x - 1, y), e = rcas_fetch<S>(p, x, y);
  const float3 f = rcas_fetch<S>(p, x + 1, y), h = rcas_fetch<S>(p, x, y + 1);
  const float lR = rcas_lobe<kExact>(b.x, d.x, e.x, f.x, h.x);
  const float lG = rcas_lobe<kExact>(b.y, d.y, e.y, f.y, h.y);
  const float lB = rcas_lobe<kExact>(b.z, d.z, e.z, f.z, h.z);
  float lobe = A::mul(fmaxf(-0.1875f, fminf(fmaxf(lR, fmaxf(lG, lB)), 0.0f)), p.sharp);
  if (p.options & 1) {  // FSR_RCAS_DENOISE (ffx_fsr1.h:731-739, 761-763)
    const float bL = luma<kExact>(b), dL = luma<kExact>(d), eL = luma<kExact>(e), fL = luma<kExact>(f), hL = luma<kExact>(h);
    float nz = A::sub(A::mad(0.25f, hL, A::mad(0.25f, fL, A::mad(0.25f, dL, A::mul(0.25f, bL)))), eL);
    const float mx = fmaxf(fmaxf(bL, fmaxf(dL, eL)), fmaxf(fL, hL)), mn = fminf(fminf(bL, fminf(dL, eL)), fminf(fL, hL));
    const float rng = A::sub(mx, mn);
    const float sd = __uint_as_float(0x7ef19fffu - __float_as_uint(rng));
    nz = sat(A::mul(fabsf(nz), A::mul(sd, A::mad(-sd, rng, 2.0f))));
    nz = A::mad(-0.5f, nz, 1.0f);
    lobe = A::mul(lobe, nz);
  }
  // APrxMedRcpF1 (ffx_a.h:1844): bit-trick seed + one Newton step
  const float a = A::mad(4.0f, lobe, 1.0f);
  const float s = __uint_as_float(0x7ef19fffu - __float_as_uint(a));
  const float rcpL = A::mul(s, A::mad(-s, a, 2.0f));
  const float alpha = (p.options & 2) ? Px<S>::alpha(p.in, x, y) : 1.0f;  // FSR_RCAS_PASSTHROUGH_ALPHA (:688-702)
  Px<S>::store(p.out, x, y, rcas_resolve<kExact>(lobe, rcpL, b.x, d.x, e.x, f.x, h.x),
               rcas_resolve<kExact>(lobe, rcpL, b.y, d.y, e.y, f.y, h.y),
               rcas_resolve<kExact>(lobe, rcpL, b.z, d.z, e.z, f.z, h.z), alpha);
}

static inline dim3 grid_for(int w, int rows) { return dim3((w + 31) / 32, (rows + 7) / 8, 1); }

template <typename S>
static void launch_easu_s(const EasuParams& p, bool exact, cudaStream_t s, dim3 grid, dim3 block) {
  if (exact) easu_direct_kernel<S, true><<<grid, block, 0, s>>>(p);
  else easu_direct_kernel<S, false><<<grid, block, 0, s>>>(p);
}
template <typename S>
static void launch_rcas_s(const RcasParams& p, bool exact, cudaStream_t s, dim3 grid, dim3 block) {
  if (exact) rcas_direct_kernel<S, true><<<grid, block, 0, s>>>(p);
  else rcas_direct_kernel<S, false><<<grid, block, 0, s>>>(p);
}
static const char* direct_name(const char* pass, int format, bool exact) {
  static const char* names[2][4][2] = {
      {{"easu_direct<f16io,fast>", "easu_direct<f16io,exact>"}, {"easu_direct<f32,fast>", "easu_direct<f32,exact>"},
       {"easu_direct<unorm8,fast>", "easu_direct<unorm8,exact>"}, {"easu_direct<unorm10,fast>", "easu_direct<unorm10,exact>"}},
      {{"rcas_direct<f16io,fast>", "rcas_direct<f16io,exact>"}, {"rcas_direct<f32,fast>", "rcas_direct<f32,exact>"},
       {"rcas_direct<unorm8,fast>", "rcas_direct<unorm8,exact>"}, {"rcas_direct<unorm10,fast>", "rcas_direct<unorm10,exact>"}}};
  return names[pass[0] == 'r'][format - 1][exact ? 1 : 0];
}

cudaError_t launch_easu_direct(const EasuParams& p, int format, bool exact, cudaStream_t s, const char** name) {
  const dim3 block(32, 8, 1), grid = grid_for(p.out.w, p.y1 - p.y0);
  switch (format) {
    case 1: launch_easu_s<__half>(p, exact, s, grid, block); break;
    case 2: launch_easu_s<float>(p, exact, s, grid, block); break;
    case 3: launch_easu_s<Unorm8>(p, exact, s, grid, block); break;
    case 4: launch_easu_s<Unorm10>(p, exact, s, grid, block); break;
    case 5:
      if (exact) return cudaErrorNotSupported;  // refused by the caller (FSR1_FLAG_EXACT is an fp32-image path)
      easu_direct_r11_kernel<<<grid, block, 0, s>>>(p);
      *name = "easu_direct<r11g11b10f_in,f16out,fast>";
      return cudaGetLastError();
    default: return cudaErrorInvalidValue;
  }
  *name = direct_name("easu", format, exact);
  return cudaGetLastError();
}

cudaError_t launch_rcas_direct(const RcasParams& p, int format, bool exact, cudaStream_t s, const char** name) {
  const dim3 block(32, 8, 1), grid = grid_for(p.out.w, p.y1 - p.y0);
  switch (format) {
    case 1: launch_rcas_s<__half>(p, exact, s, grid, block); break;
    case 2: launch_rcas_s<float>(p, exact, s, grid, block); break;
    case 3: launch_rcas_s<Unorm8>(p, exact, s, grid, block); break;
    case 4: launch_rcas_s<Unorm10>(p, exact, s, grid, block); break;
    default: return cudaErrorInvalidValue;
  }
  *name = direct_name("rcas", format, exact);
  return cudaGetLastError();
}

}  // namespace fsr1
