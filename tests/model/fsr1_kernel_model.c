// TEST INFRASTRUCTURE — a per-pixel model of the arithmetic of the production half-storage kernels, written to be compared
// with them bit for bit:
//   easu_h   RGBA16F EASU: easu_h_quad2x (exactly 2x) and easu_h_vpairs (any other upscale)
//   easu_u8  R8G8B8A8_UNORM EASU at exactly 2x (easu_u8_quad2x)
//   rcas_h   RGBA16F RCAS (rcas_h_packed, and the RCAS half of the fused kernel), every option set
//   rcas_u8  R8G8B8A8_UNORM RCAS (rcas_u8_packed)
// One output pixel at a time: no tiles, boxes, lanes or pixel pairs.  It restates ffx_fsr1.h (line numbers below refer to
// include/compat/ffx_fsr1.h) with the precision split of the kernels (DESIGN.md §4): everything that decides the filter's
// orientation is fp32, the taps and RCAS are half.
//
// Every half operation rounds exactly once.  A half is converted to double exactly; the product of two halves (22 significant
// bits) and the sum or difference of two halves (exponents 2^15 .. 2^-24, 40 bits) are exact in double, so rounding that double
// to half (h_round) is the one rounding.  a*b+c is not always exact in double (the span can reach 2^16 .. 2^-48), so hfma adds
// the tail of the sum by TwoSum and h_round breaks a tie with its sign: the double result s differs from the exact value only
// by that tail (|tail| <= half an ulp of s), half rounding boundaries are representable in double, so the exact value lies on
// the same side of every boundary as s except when s is itself a boundary.
//
// The two approximate instructions of the kernels both take a half and are rounded to half at once: rcp.approx.ftz.f32 on the
// EASU weight sum and h2rcp (cvt.f32.f16, rcp.approx.ftz.f32, cvt.rn.f16.f32) in the RCAS lobe.  For every finite half x, 1/x
// lies at least 2 fp32 ulps from every half rounding boundary (tests/test_kernel_model.py checks all of them exactly), and
// rcp.approx.f32 is within 1 ulp of 1/x, so its half rounding equals the correctly rounded half of 1/x: h_recip.
//
// min / max (HMNMX2) do not propagate NaN: a NaN operand yields the other one.  -0 orders below +0 (the CUDA __hmin2 / __hmax2
// rule), so min and max are a total order on the non-NaN halves and the order in which a kernel reduces does not matter.
// A NaN produced by arithmetic is the canonical 0x7fff.
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

typedef uint16_t h16;

// ---- half <-> double ---------------------------------------------------------------------------------------------------
static double g_h2d[65536];
__attribute__((constructor)) static void init_h2d(void) {
  for (int b = 0; b < 65536; b++) {
    const int s = b >> 15, e = (b >> 10) & 31, m = b & 1023;
    double v;
    if (e == 0) v = ldexp((double)m, -24);
    else if (e == 31) v = m ? NAN : INFINITY;
    else v = ldexp((double)(1024 + m), e - 25);
    g_h2d[b] = s ? -v : v;
  }
}
static inline double H(h16 a) { return g_h2d[a]; }

// Round v + tail to half, round-to-nearest-even.  tail: the sign (-1, 0, +1) of a remainder smaller than half an ulp of v.
static h16 h_round(double v, int tail) {
  uint64_t b;
  memcpy(&b, &v, 8);
  const h16 sign = (h16)((b >> 48) & 0x8000u);
  const uint64_t ab = b & 0x7fffffffffffffffull;
  if (ab >= 0x7ff0000000000000ull) return ab > 0x7ff0000000000000ull ? 0x7fff : (h16)(sign | 0x7c00);
  if (ab == 0) return sign;
  if (sign) tail = -tail;  // tail of the magnitude
  const int e = (int)(ab >> 52) - 1023;
  if (e > 15) return (h16)(sign | 0x7c00);
  if (e < -40) return sign;  // below a quarter of the smallest subnormal
  const uint64_t m = (ab & 0xfffffffffffffull) | (1ull << 52);  // magnitude = m 2^(e-52)
  const int q = (e < -14 ? -14 : e) - 10;                          // exponent of the half ulp at this magnitude
  const int s = q - (e - 52);                                      // 42 .. 64: bits below the half ulp
  uint64_t n, rem, half;
  if (s >= 64) { n = 0; rem = m; half = 1ull << 63; }
  else { n = m >> s; rem = m & ((1ull << s) - 1); half = 1ull << (s - 1); }
  if (rem > half || (rem == half && (tail > 0 || (tail == 0 && (n & 1))))) n++;
  uint32_t r;
  if (e < -14) r = (uint32_t)n;  // subnormal (n = 1024 is the smallest normal, whose bits are 0x400)
  else r = ((uint32_t)(e + 15) << 10) + (uint32_t)n - 1024u;
  if (r >= 0x7c00u) r = 0x7c00u;
  return (h16)(sign | r);
}
static inline h16 h_of_float(float f) { return h_round((double)f, 0); }

// ---- half arithmetic: one rounding each ----------------------------------------------------------------------------------
static inline h16 hmul(h16 a, h16 b) { return h_round(H(a) * H(b), 0); }
static inline h16 hadd(h16 a, h16 b) { return h_round(H(a) + H(b), 0); }
static inline h16 hsub(h16 a, h16 b) { return h_round(H(a) - H(b), 0); }
static inline h16 hfma(h16 a, h16 b, h16 c) {
  const double p = H(a) * H(b), cc = H(c), s = p + cc;
  if (!isfinite(s)) return h_round(s, 0);
  const double bp = s - p, t = (p - (s - bp)) + (cc - bp);  // TwoSum: s + t == p + c exactly
  return h_round(s, t > 0 ? 1 : t < 0 ? -1 : 0);
}
static inline int h_isnan(h16 a) { return (a & 0x7fff) > 0x7c00; }
static inline int h_less(h16 a, h16 b) {  // total order on non-NaN halves with -0 < +0
  const int ka = (a & 0x8000) ? -(int)(a & 0x7fff) - 1 : (int)a, kb = (b & 0x8000) ? -(int)(b & 0x7fff) - 1 : (int)b;
  return ka < kb;
}
static inline h16 hmin(h16 a, h16 b) {
  if (h_isnan(a)) return h_isnan(b) ? 0x7fff : b;
  if (h_isnan(b)) return a;
  return h_less(b, a) ? b : a;
}
static inline h16 hmax(h16 a, h16 b) {
  if (h_isnan(a)) return h_isnan(b) ? 0x7fff : b;
  if (h_isnan(b)) return a;
  return h_less(a, b) ? b : a;
}
static inline h16 hneg(h16 a) { return a ^ 0x8000; }
static inline h16 habs(h16 a) { return a & 0x7fff; }
static inline h16 h_recip(h16 a) { return h_round(1.0 / H(a), 0); }  // see the header: exact for every half
static inline h16 hc(float f) { return h_of_float(f); }

// ---- fp32 helpers (ffx_a.h:1843-1845 bit tricks) -------------------------------------------------------------------------
static inline float u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float prx_lo_rcp(float a) { return u2f(0x7ef07ebbu - f2u(a)); }
static inline float prx_lo_rsq(float a) { return u2f(0x5f347d74u - (f2u(a) >> 1)); }
static inline float sat(float x) { return x != x ? 0.0f : x < 0.0f ? 0.0f : x > 1.0f ? 1.0f : x; }
static inline int clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

// ---- EASU ----------------------------------------------------------------------------------------------------------------
// The source image as the kernels see it: per texel the three half colour values the taps read and the fp32 luma.
typedef struct {
  int w, h;
  const h16* rgb;  // [h][w][3]
  const float* L;  // [h][w]: 2 luma = 0.5 B + (0.5 R + G) (ffx_fsr1.h:363-366), fp32
} Src;

static inline float luma_at(const Src* s, int x, int y) { return s->L[(long long)clampi(y, 0, s->h - 1) * s->w + clampi(x, 0, s->w - 1)]; }
static inline const h16* rgb_at(const Src* s, int x, int y) { return s->rgb + ((long long)clampi(y, 0, s->h - 1) * s->w + clampi(x, 0, s->w - 1)) * 3; }

// FsrEasuSetF without the bilinear weight (ffx_fsr1.h:295-313): (dirX, dirY, lenX^2 + lenY^2) of texel (x, y), every luma read
// through the clamp-to-edge sampler.
static void texel_terms(const Src* s, int x, int y, float t[3]) {
  const float lA = luma_at(s, x, y - 1), lB = luma_at(s, x - 1, y), lC = luma_at(s, x, y), lD = luma_at(s, x + 1, y), lE = luma_at(s, x, y + 1);
  const float dirX = lD - lB, dirY = lE - lA;
  const float lenX = sat(fabsf(dirX) * prx_lo_rcp(fmaxf(fabsf(lD - lC), fabsf(lC - lB))));
  const float lenY = sat(fabsf(dirY) * prx_lo_rcp(fmaxf(fabsf(lE - lC), fabsf(lC - lA))));
  t[0] = dirX;
  t[1] = dirY;
  t[2] = fmaf(lenX, lenX, lenY * lenY);
}

typedef struct { h16 qa, qb, qc, lob, clp; } Shape;

// Normalise, stretch, lobe, clip (ffx_fsr1.h:389-409) in fp32, then the quadratic form of the rotated, anisotropically scaled
// distance d2 = qa ox^2 + qb ox oy + qc oy^2, each coefficient rounded once to half.
static Shape pixel_shape(float dx, float dy, float len) {
  const float dirR = fmaf(dx, dx, dy * dy);
  const int zro = dirR < (1.0f / 32768.0f);
  const float rs = zro ? 1.0f : prx_lo_rsq(dirR);
  dx = (zro ? 1.0f : dx) * rs;
  dy = dy * rs;
  len = len * 0.5f;
  len = len * len;
  const float dx2 = dx * dx, dy2 = dy * dy;
  const float rmax = prx_lo_rcp(fmaxf(fabsf(dx), fabsf(dy)));
  const float stretch = (dx2 + dy2) * rmax;
  const float l2x = fmaf(stretch + -1.0f, len, 1.0f), l2y = fmaf(-0.5f, len, 1.0f);
  const float lob = fmaf((float)((1.0 / 4.0 - 0.04) - 0.5), len, 0.5f);
  const float clp = prx_lo_rcp(lob);
  const float X2 = l2x * l2x, Y2 = l2y * l2y;
  Shape h;
  h.qa = h_of_float(fmaf(X2, dx2, Y2 * dy2));
  h.qc = h_of_float(fmaf(X2, dy2, Y2 * dx2));
  h.qb = h_of_float(((dx * dy) * 2.0f) * fmaf(Y2, -1.0f, X2));
  h.lob = h_of_float(lob);
  h.clp = h_of_float(clp);
  return h;
}

// Window weight at squared distance d2 (ffx_fsr1.h:255-270) in Horner form: ((d2/4 - 5/4) d2 + 1)(lob d2 - 1)^2.
static h16 weight_unclamped(h16 d2, h16 lob) {
  const h16 wb = hfma(hfma(hc(0.25f), d2, hc(-1.25f)), d2, hc(1.0f));
  h16 wa = hfma(lob, d2, hc(-1.0f));
  wa = hmul(wa, wa);
  return hmul(wb, wa);
}
// min(d2, clp) compares the bit patterns as signed 16-bit integers: d2 itself when rounding made it slightly negative
static h16 weight(h16 d2, h16 lob, h16 clp) {
  return weight_unclamped((int16_t)d2 < (int16_t)clp ? d2 : clp, lob);
}

// The 12 taps in accumulation order: the eight far taps first, the four nearest (f g j k) last.  (row R, column K) of the 4x4
// window whose texel (1,1) is f.
static const int kTaps[12][2] = {{0, 1}, {0, 2}, {1, 0}, {1, 3}, {2, 0}, {2, 3}, {3, 1}, {3, 2}, {1, 1}, {1, 2}, {2, 1}, {2, 2}};

// Output pixel -> cell and fraction, mul then add (two roundings), as the kernels and the oracle do
static void easu_pos(int o, float scale, float offset, int* fp, float* pp) {
  const float p = (float)o * scale + offset;
  const float f = floorf(p);
  *fp = (int)f;
  *pp = p - f;
}

// One output pixel (x, y): out[3] = R, G, B.  quad: the exactly-2x form (easu_h_quad2x, easu_u8_quad2x); else the any-scale
// form (easu_h_vpairs).
static void easu_pixel(const Src* s, const float c0[4], int quad, int x, int y, h16 out[3]) {
  int fx, fy;
  float ppx, ppy;
  easu_pos(x, c0[0], c0[2], &fx, &ppx);
  easu_pos(y, c0[1], c0[3], &fy, &ppy);
  float f[3], g[3], j[3], k[3], b[3];
  texel_terms(s, fx, fy, f);
  texel_terms(s, fx + 1, fy, g);
  texel_terms(s, fx, fy + 1, j);
  texel_terms(s, fx + 1, fy + 1, k);
  // bilinear blend of the f g j k terms, in the reference's order f, g, j, k (ffx_fsr1.h:383-386)
  if (quad) {  // at 2x, ppx and ppy are 0.25 or 0.75: the horizontal blend of each texel row, then the vertical one
    const float wG = ppx, wF = 1.0f - ppx;
    for (int c = 0; c < 3; c++) {
      const float T = fmaf(g[c], wG, f[c] * wF), B = fmaf(k[c], wG, j[c] * wF);
      b[c] = fmaf(B, ppy, T * (1.0f - ppy));
    }
  } else {
    const float ipx = 1.0f - ppx, ipy = fmaf(ppy, -1.0f, 1.0f);
    const float wf = ipx * ipy, wg = ppx * ipy, wj = ipx * ppy, wk = ppx * ppy;
    for (int c = 0; c < 3; c++) b[c] = fmaf(k[c], wk, fmaf(j[c], wj, fmaf(g[c], wg, f[c] * wf)));
  }
  const Shape sh = pixel_shape(b[0], b[1], b[2]);
  // the taps (ffx_fsr1.h:423-434): d2 in half, every offset an fp32 value rounded to half
  h16 acc[3] = {0, 0, 0}, aw = 0;
  for (int i = 0; i < 12; i++) {
    const int R = kTaps[i][0], K = kTaps[i][1];
    h16 d2;
    int clamp = 1;
    if (quad) {
      const float ox = (float)(K - 1) - ppx, oy = (float)(R - 1) - ppy;
      if (R == 0 || R == 3) {  // two taps per row: the unfactored distance
        d2 = hfma(sh.qa, hc(ox * ox), hfma(sh.qc, hc(oy * oy), hmul(sh.qb, hc(ox * oy))));
      } else {                 // four taps per row: ox (qa ox + qb oy) + qc oy^2 with the row terms qb oy, qc oy^2 hoisted
        const h16 rowB = hmul(sh.qb, hc(oy)), rowC = hmul(sh.qc, hc(oy * oy)), hox = hc(ox);
        d2 = hfma(hfma(sh.qa, hox, rowB), hox, rowC);
        clamp = !(K == 1 || K == 2);  // the four nearest taps skip min(d2, clp): their d2 < clp at 2x (fsr1_easu_quad.cuh)
      }
    } else {  // offsets in half: OX = h(K-1) - h(ppx), OY = qb oyr, QY = (qc oyr) oyr with oyr = h(R-1) - h(ppy)
      const h16 OX = hsub(hc((float)(K - 1)), hc(ppx)), oyr = hsub(hc((float)(R - 1)), hc(ppy));
      const h16 OY = hmul(sh.qb, oyr), QY = hmul(hmul(sh.qc, oyr), oyr);
      d2 = hfma(hfma(sh.qa, OX, OY), OX, QY);
    }
    const h16 w = clamp ? weight(d2, sh.lob, sh.clp) : weight_unclamped(d2, sh.lob);
    const h16* t = rgb_at(s, fx - 1 + K, fy - 1 + R);
    for (int c = 0; c < 3; c++) acc[c] = hfma(t[c], w, acc[c]);
    aw = hadd(aw, w);
  }
  // normalise by the half reciprocal of the weight sum, then the de-ringing clamp to the f g j k texels (ffx_fsr1.h:416-419,437)
  const h16 r = h_recip(aw);
  const h16 *tf = rgb_at(s, fx, fy), *tg = rgb_at(s, fx + 1, fy), *tj = rgb_at(s, fx, fy + 1), *tk = rgb_at(s, fx + 1, fy + 1);
  for (int c = 0; c < 3; c++) {
    const h16 mn = hmin(hmin(tf[c], tg[c]), hmin(tj[c], tk[c])), mx = hmax(hmax(tf[c], tg[c]), hmax(tj[c], tk[c]));
    out[c] = hmin(mx, hmax(mn, hmul(acc[c], r)));
  }
}

static int is_2x(const float c0[4]) { return c0[0] == 0.5f && c0[1] == 0.5f && c0[2] == -0.25f && c0[3] == -0.25f; }

// x in [0, 1] -> round(255 x): one half FMA x 255 + 1024 lands where the ulp of a half is 1 (StoreUnorm<8>).  255 is odd, so the
// only half x in [0, 1] for which 255 x is a tie is 1/2: the FMA rounds 1151.5 to the even 1152, code 128.  (The float -> UNORM
// rule of the direct kernels, to_unorm in csrc/fsr1_common.cuh: scale, add 0.5, truncate, gives 128 there too.)
static int unorm8_of(h16 x) {
  const h16 t = hfma(x, hc(255.0f), hc(1024.0f));
  return (int)(H(t) - 1024.0) & 255;
}

// RGBA16F EASU of output rows [y0, y1).  Pitches in elements.  The constants select the form as the launcher does (exactly 2x:
// easu_h_quad2x, else easu_h_vpairs); any_scale forces the any-scale form.  Returns 0, or -1 for a downscaled axis (the direct kernels).
int fkm_easu_h(const h16* in, int iw, int ih, long long in_pitch, h16* out, int ow, int oh, long long out_pitch, const uint32_t* con,
               int y0, int y1, int any_scale) {
  float c0[4];
  memcpy(c0, con, 16);
  const int quad = is_2x(c0) && !any_scale;
  if (!quad && !(c0[0] > 0.0f && c0[0] <= 1.0f && c0[1] > 0.0f && c0[1] <= 1.0f)) return -1;
  (void)oh;
  h16* rgb = malloc(sizeof(h16) * 3 * (size_t)iw * ih);
  float* L = malloc(sizeof(float) * (size_t)iw * ih);
  for (int y = 0; y < ih; y++)
    for (int x = 0; x < iw; x++) {
      const h16* p = in + y * in_pitch + 4LL * x;
      h16* q = rgb + ((size_t)y * iw + x) * 3;
      q[0] = p[0]; q[1] = p[1]; q[2] = p[2];
      L[(size_t)y * iw + x] = fmaf((float)H(p[2]), 0.5f, fmaf((float)H(p[0]), 0.5f, (float)H(p[1])));
    }
  const Src s = {iw, ih, rgb, L};
#pragma omp parallel for schedule(dynamic, 2)
  for (int y = y0; y < y1; y++)
    for (int x = 0; x < ow; x++) {
      h16* o = out + y * out_pitch + 4LL * x;
      easu_pixel(&s, c0, quad, x, y, o);
      o[3] = 0x3c00;  // alpha = 1 (FSR_Pass.hlsl:80)
    }
  free(rgb);
  free(L);
  return 0;
}

// c / 255 correctly rounded in fp32 (what unorm_to_float computes)
static inline float unorm8_to_float(uint32_t c) { return (float)c / 255.0f; }

// R8G8B8A8_UNORM EASU at exactly 2x: the taps read each decoded value rounded to half, the luma is taken from the fp32 values;
// the result is stored as round(255 x), alpha 255.  Pitches in pixels.  Returns 0, or -1 unless exactly 2x.
int fkm_easu_u8(const uint32_t* in, int iw, int ih, long long in_pitch, uint32_t* out, int ow, int oh, long long out_pitch,
                const uint32_t* con, int y0, int y1) {
  float c0[4];
  memcpy(c0, con, 16);
  if (!is_2x(c0)) return -1;
  (void)oh;
  h16* rgb = malloc(sizeof(h16) * 3 * (size_t)iw * ih);
  float* L = malloc(sizeof(float) * (size_t)iw * ih);
  for (int y = 0; y < ih; y++)
    for (int x = 0; x < iw; x++) {
      const uint32_t u = in[y * in_pitch + x];
      const float r = unorm8_to_float(u & 255u), g = unorm8_to_float((u >> 8) & 255u), b = unorm8_to_float((u >> 16) & 255u);
      h16* q = rgb + ((size_t)y * iw + x) * 3;
      q[0] = h_of_float(r); q[1] = h_of_float(g); q[2] = h_of_float(b);
      L[(size_t)y * iw + x] = fmaf(b, 0.5f, fmaf(r, 0.5f, g));
    }
  const Src s = {iw, ih, rgb, L};
#pragma omp parallel for schedule(dynamic, 2)
  for (int y = y0; y < y1; y++)
    for (int x = 0; x < ow; x++) {
      h16 o[3];
      easu_pixel(&s, c0, 1, x, y, o);
      out[y * out_pitch + x] = (uint32_t)unorm8_of(o[0]) | ((uint32_t)unorm8_of(o[1]) << 8) |
                               ((uint32_t)unorm8_of(o[2]) << 16) | 0xff000000u;
    }
  free(rgb);
  free(L);
  return 0;
}

// ---- RCAS ------------------------------------------------------------------------------------------------------------------
enum { kDenoise = 1, kAlpha = 2, kSquare = 4 };

typedef struct {
  int w, h, clamp;
  const h16* rgb;  // [h][w][3], the half values the kernel computes with
} RSrc;

// tap (x, y): clamp-to-edge, or 0 outside the image (a D3D12 Load; ffx_fsr1.h:693-707)
static void rtap(const RSrc* s, int x, int y, h16 o[3]) {
  if (s->clamp) { x = clampi(x, 0, s->w - 1); y = clampi(y, 0, s->h - 1); }
  if (x < 0 || x >= s->w || y < 0 || y >= s->h) { o[0] = o[1] = o[2] = 0; return; }
  memcpy(o, s->rgb + ((size_t)y * s->w + x) * 3, 6);
}

// lobe of one channel: max(-hitMin, hitMax) = -min(min(mn4, e) / (4 mx4), (1 - max(mx4, e)) / (4 - 4 mn4))  (ffx_fsr1.h:750-759)
static h16 lobe_channel(h16 b, h16 d, h16 e, h16 f, h16 h) {
  const h16 mn4 = hmin(hmin(b, d), hmin(f, h)), mx4 = hmax(hmax(b, d), hmax(f, h));
  const h16 hitMin = hmul(hmin(mn4, e), h_recip(hmul(hc(4.0f), mx4)));
  const h16 negHitMax = hmul(hsub(hc(1.0f), hmax(mx4, e)), h_recip(hfma(hc(-4.0f), mn4, hc(4.0f))));
  return hneg(hmin(hitMin, negHitMax));
}
static h16 luma2x(const h16 c[3]) { return hfma(c[2], hc(0.5f), hfma(c[0], hc(0.5f), c[1])); }  // ffx_fsr1.h:725-729

// APrxMedRcpH1 (ffx_a.h:1814): 16-bit magic subtract (wrapping in 16 bits) and one Newton step
static h16 prx_med_rcp(h16 a) {
  const h16 s = (h16)(0x778du - a);
  return hmul(s, hfma(hneg(s), a, hc(2.0f)));
}

// max - min of the five lumas: the denominator of the noise measure (ffx_fsr1.h:731-739)
static h16 luma_range(const RSrc* s, int x, int y, h16 L[5]) {
  h16 t[3];
  const int dx[5] = {0, -1, 0, 1, 0}, dy[5] = {-1, 0, 0, 0, 1};
  for (int i = 0; i < 5; i++) { rtap(s, x + dx[i], y + dy[i], t); L[i] = luma2x(t); }
  const h16 mx = hmax(hmax(hmax(L[0], L[1]), L[2]), hmax(L[3], L[4])), mn = hmin(hmin(hmin(L[0], L[1]), L[2]), hmin(L[3], L[4]));
  return hsub(mx, mn);
}

// One output pixel (x, y) of RCAS (ffx_fsr1.h:684-769): out[3] = R, G, B.
static void rcas_pixel(const RSrc* s, h16 sharp, int opts, int x, int y, h16 out[3]) {
  h16 b[3], d[3], e[3], f[3], h[3];
  rtap(s, x, y - 1, b);
  rtap(s, x - 1, y, d);
  rtap(s, x, y, e);
  rtap(s, x + 1, y, f);
  rtap(s, x, y + 1, h);
  h16 l = hmax(lobe_channel(b[0], d[0], e[0], f[0], h[0]), hmax(lobe_channel(b[1], d[1], e[1], f[1], h[1]), lobe_channel(b[2], d[2], e[2], f[2], h[2])));
  h16 lobe = hmul(hmax(hc(-0.1875f), hmin(l, 0)), sharp);
  if (opts & kDenoise) {
    h16 L[5];
    const h16 range = luma_range(s, x, y, L);
    const h16 q = hc(0.25f);
    h16 nz = hsub(hfma(q, L[4], hfma(q, L[3], hfma(q, L[1], hmul(q, L[0])))), L[2]);
    nz = hmul(habs(nz), prx_med_rcp(range));
    nz = hmin(hc(1.0f), hmax(nz, 0));
    nz = hfma(hc(-0.5f), nz, hc(1.0f));
    lobe = hmul(lobe, nz);
  }
  const h16 rcpL = prx_med_rcp(hfma(hc(4.0f), lobe, hc(1.0f)));
  for (int c = 0; c < 3; c++) {
    const h16 ring = hadd(hadd(b[c], d[c]), hadd(h[c], f[c]));
    out[c] = hmul(hfma(lobe, ring, e[c]), rcpL);
    if (opts & kSquare) out[c] = hmul(out[c], out[c]);
  }
}

// RGBA16F RCAS of rows [y0, y1).  con[1] = sharpness as half2.  opts: bit 0 FSR_RCAS_DENOISE, bit 1 FSR_RCAS_PASSTHROUGH_ALPHA
// (alpha = the centre pixel's), bit 2 the output square of the sample's Sample.x hook.  Pitches in elements.
int fkm_rcas_h(const h16* in, int w, int h, long long in_pitch, h16* out, long long out_pitch, const uint32_t* con, int clamp, int y0,
               int y1, int opts) {
  h16* rgb = malloc(sizeof(h16) * 3 * (size_t)w * h);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) memcpy(rgb + ((size_t)y * w + x) * 3, in + y * in_pitch + 4LL * x, 6);
  const RSrc s = {w, h, clamp, rgb};
  const h16 sharp = (h16)(con[1] & 0xffffu);
#pragma omp parallel for schedule(dynamic, 4)
  for (int y = y0; y < y1; y++)
    for (int x = 0; x < w; x++) {
      h16* o = out + y * out_pitch + 4LL * x;
      rcas_pixel(&s, sharp, opts, x, y, o);
      o[3] = (opts & kAlpha) ? in[y * in_pitch + 4LL * x + 3] : 0x3c00;
    }
  free(rgb);
  return 0;
}

// R8G8B8A8_UNORM RCAS: each code decodes to half through fp32 (c / 255, one rounding to half); the result saturates to [0, 1]
// before the encode; alpha is the centre pixel's code or 255.  Pitches in pixels.
int fkm_rcas_u8(const uint32_t* in, int w, int h, long long in_pitch, uint32_t* out, long long out_pitch, const uint32_t* con, int clamp,
                int y0, int y1, int opts) {
  h16* rgb = malloc(sizeof(h16) * 3 * (size_t)w * h);
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      const uint32_t u = in[y * in_pitch + x];
      for (int c = 0; c < 3; c++) rgb[((size_t)y * w + x) * 3 + c] = h_of_float(unorm8_to_float((u >> (8 * c)) & 255u));
    }
  const RSrc s = {w, h, clamp, rgb};
  const h16 sharp = (h16)(con[1] & 0xffffu);
#pragma omp parallel for schedule(dynamic, 4)
  for (int y = y0; y < y1; y++)
    for (int x = 0; x < w; x++) {
      h16 o[3];
      rcas_pixel(&s, sharp, opts, x, y, o);
      uint32_t v = (opts & kAlpha) ? (in[y * in_pitch + x] & 0xff000000u) : 0xff000000u;
      for (int c = 0; c < 3; c++) v |= (uint32_t)unorm8_of(hmin(hc(1.0f), hmax(0, o[c]))) << (8 * c);
      out[y * out_pitch + x] = v;
    }
  free(rgb);
  return 0;
}

// Correctly rounded half of 1/x for half bits x (what the kernels' rcp.approx + cvt.rn.f16 compute; see the header)
h16 fkm_h_recip(h16 x) { return h_recip(x); }
h16 fkm_hfma(h16 a, h16 b, h16 c) { return hfma(a, b, c); }
