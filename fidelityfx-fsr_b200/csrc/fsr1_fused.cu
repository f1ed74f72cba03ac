// fsr1_fused.cu — EASU -> RCAS in ONE kernel for RGBA16F images at exactly 2x (SURVEY.md §8(f).2).
//
// The reference runs two dispatches through a display-sized intermediate texture (sample/src/DX12/FSR_Filter.cpp:121-131,
// intermediate at :72-73).  Here the intermediate never leaves the SM: a CTA walks DOWN a column strip of the output,
// step by step; each step
//   1. takes a TMA box of the input (double-buffered, the next step's box is in flight),
//   2. runs EASU phases 1-3 exactly as easu_h_quad2x_kernel does (same device functions, fsr1_easu_quad.cuh) but stores
//      the 64 x 2n pixels into a shared-memory "mid" tile — rounded to fp16, i.e. the very bits the intermediate image
//      would hold — in the (pixel0, pixel1)-per-channel half2 layout RCAS wants,
//   3. runs RCAS (fsr1_rcas_math.cuh, the arithmetic of rcas_packed_kernel) on the rows of the mid tile whose upper and
//      lower neighbours are present and stores the result with 128-bit stores.
// The last two mid rows of a step stay in shared memory for the next step, so nothing is recomputed vertically inside a
// strip run; horizontally a strip is 31 cells (62 output pixels) of the 32 a warp computes (the 1-pixel apron RCAS needs).
// The result is bit-identical to fsr1_easu + fsr1_rcas (tests/test_gpu_parity.py::test_fused_*): same operations on the same
// rounded intermediate.  Compulsory HBM traffic: bpp (Pin + Pout) = 10 B per output pixel instead of 26.
//
// Work distribution (FusedIter): the CTAs of a strip split it into "runs" (strip, [ya, yb)) of whole steps.  A run starts like
// a row slab: its first step also computes the cell row above ya (RCAS's upper neighbour), which is the only vertical
// redundancy (~1 cell row per ~73 at 1080p->4K).  Only a strip's last run may end with a partial step.
//
// Geometry of a step with cell rows m0 .. m0+n-1 (n <= CY) of strip tx (cells k0 .. k0+31, k0 = 31 tx - 1):
//   mid row index i  <->  pixel row 2 m0 - 1 + i   (i = 0, 1: kept from the previous step; cell row r -> i = 2r+2, 2r+3)
//   mid pair k (lane) <-> pixels (2k+1, 2k+2)
//   RCAS output pair of lane l >= 1: pixels (2k, 2k+1), k = k0 + l:  e = (P[k-1].hi, P[k].lo), d = P[k-1], f = P[k]
//   output rows o in [2 m0, 2 m0 + 2n - 1] ∩ [ya, yb): mid index o - 2 m0 + 1, needs indices -1/+1 around it.
// Out-of-image mid pixels hold 0 (D3D12 Load semantics, ffx_fsr1.h:698-707 through FSR_Pass.hlsl:61); FSR1_FLAG_RCAS_CLAMP is not
// implemented here (the caller falls back to the two-kernel path).
// kSrtmIn (FSR1_FLAG_SRTM_INPUT): phase 1 of a step first replaces each texel it covers by FsrSrtmF of it, rounded to half, as
// easu_h_quad2x_kernel does (fsr1_easu_tiled.cu: after clamp_fixup, luma from the half texel; the fence_proxy_async before the next
// TMA load into the buffer orders the stores).  Those kFBW (n + 3) texels are exactly the ones the step's taps read.
// kR11 (R11G11B10_FLOAT input, fsr1_r11.cuh): a kRBW = 40 texel box of 4-byte texels from the multiple of 4 at or before box_x (38
// texels are 152 bytes: TMA boxes are multiples of 16 bytes), expanded in phase 1 into the same half tile, the step's kFBW (n + 3) texels.
// Array inputs (FSR1_FLAG_IN_SURFACE: RGBA16F; FSR1_FLAG_IN_TEXTURE: RGBA16F or R11G11B10F): phase 1 fetches the step's texels from the
// CUDA array at clamped coordinates instead (fused_body's kIn); the *_surf and *_tex kernels below.
#include "fsr1_easu_quad.cuh"
#include "fsr1_post.cuh"
#include "fsr1_r11.cuh"
#include "fsr1_rcas_math.cuh"

namespace fsr1 {

constexpr int kFBW = kQBW + 2;   // box width 38: the strip origin 31 tx - 2 is odd for odd tx and TMA boxes start on 16 bytes
constexpr int kFSW = kFBW - 2;   // texels carrying terms per row
constexpr int kStripCells = 31;  // cells per strip (lanes 1..31 produce RCAS output; lane 0 only feeds its right neighbour)
constexpr int kRBW = kFBW + 2;   // kR11: box width in 4-byte texels

struct FusedParams {
  ImgView in, out;
  int y0, y1;          // output rows
  uint32_t sharp_h2;   // RCAS con.y
  int n_strips;
  HaloSync sync = {};
};

template <int NW> struct FusedCfg {
  static constexpr int kCY = 2 * NW, kBH = kCY + 3, kSH = kCY + 1, kElems = kFBW * kBH;
  static constexpr int kPad = ((kElems * 8 + 127) / 128) * 128 / 8;
  static constexpr int kMidRows = 2 * kCY + 2;
};

template <int NW> struct __align__(128) FusedSmem {
  uint2 tile[2][FusedCfg<NW>::kPad];
  float4 S[kFSW * FusedCfg<NW>::kSH];
  uint4 mid[FusedCfg<NW>::kMidRows][32];  // (R0R1, G0G1, B0B1, -) of pixel pair (2k+1, 2k+2)
  float L[FusedCfg<NW>::kElems];
  uint64_t bar[2];
};

// EASU output of a quad into the mid tile; pixels outside the image become 0 (what an out-of-image Load returns).
// kIn: every pixel of the step is inside the image, so nothing is masked.
template <bool kIn> struct MidSink {
  uint4* top;          // &mid[2r+2][lane]
  bool zT, zB;         // pixel row outside the image
  uint32_t keep;       // per-half mask of the pair: 0xffff low = pixel 2k+1 inside, high = pixel 2k+2 inside
  __device__ __forceinline__ void put(bool bottom, __half2 oR, __half2 oG, __half2 oB) const {
    if (kIn) {
      top[bottom ? 32 : 0] = make_uint4(h22u(oR), h22u(oG), h22u(oB), 0u);
      return;
    }
    const uint32_t m = (bottom ? zB : zT) ? 0u : keep;
    top[bottom ? 32 : 0] = make_uint4(h22u(oR) & m, h22u(oG) & m, h22u(oB) & m, 0u);
  }
};

struct FusedStep { int tx, m0, n, ya, yb; };

// The CTA's share of the work, in whole steps of CY cell rows of one strip.  A strip needs cell rows mfirst .. mlast (pixel rows
// y0 - 1 .. y1).  With at least as many CTAs as strips, strip s goes to the g CTAs [ctas s / S, ctas (s+1) / S); they split it into
// runs of whole steps, and a run's first cell row is the last one of the run above (the upper neighbour of its first output row),
// so g runs cover the C = mlast - mfirst + 1 cell rows in T = ceil((C + g - 1) / CY) steps and CTA i of the g takes steps
// [T i / g, T (i+1) / g).  Only the strip's last run may end with a partial step, at y1.  (When T < g, some CTAs take no step and
// the T runs of one step each overlap T - 1 times: T = ceil((C - 1) / (CY - 1)).)  With fewer CTAs than strips a CTA takes whole
// strips.  A run's first step produces the output rows of its last CY - 1 cell rows, every later step those of all CY.
template <int CY> struct FusedIter {
  int y0, y1, mfirst, mlast;
  int strip, strip_end, ma, mb, m;
  __device__ void init(const FusedParams& p, int cta, int ctas) {
    y0 = p.y0; y1 = p.y1;
    mfirst = (y0 - 2) >> 1;  // cell row holding pixel row y0-1 (arithmetic shift = floor)
    mlast = (y1 - 1) >> 1;   // cell row holding pixel row y1
    const int S = p.n_strips, C = mlast - mfirst + 1;
    strip = strip_end = 0; ma = 0; mb = -1; m = 1;
    if (y1 <= y0) return;
    if (ctas < S) {
      strip = (int)((long long)S * cta / ctas);
      strip_end = (int)((long long)S * (cta + 1) / ctas);
      ma = mfirst; mb = mlast; m = ma;
      return;
    }
    const int s = (int)(((long long)(cta + 1) * S - 1) / ctas);
    const int g0 = (int)((long long)ctas * s / S), g = (int)((long long)ctas * (s + 1) / S) - g0, i = cta - g0;
    int T = (C + g - 1 + CY - 1) / CY;
    if (T < g) T = (C - 1 + CY - 2) / (CY - 1);
    const int a = (int)((long long)T * i / g), k = (int)((long long)T * (i + 1) / g) - a;
    const int ra = mfirst + CY * a - (i < a ? i : a);  // each run above this one (min(i, a) of them) shares a cell row with the next
    if (k == 0 || 2 * ra + 2 >= y1) return;            // no step, or the runs above already cover the strip
    ma = ra;
    mb = ma + CY * k - 1 < mlast ? ma + CY * k - 1 : mlast;
    strip = s; strip_end = s + 1; m = ma;
  }
  __device__ bool next(FusedStep& s) {
    if (m > mb) {  // next strip (fewer CTAs than strips)
      if (++strip >= strip_end) return false;
      m = ma;
    }
    s.tx = strip; s.m0 = m;
    s.ya = 2 * ma + 2 > y0 ? 2 * ma + 2 : y0;
    s.yb = 2 * mb + 2 < y1 ? 2 * mb + 2 : y1;
    s.n = mb - m + 1 < CY ? mb - m + 1 : CY;
    m += s.n;
    return true;
  }
};

// Phase 3 (EASU of the step's cells into the mid tile), a barrier, then RCAS of the step's output rows.  kIn: an interior step
// (see the caller): no pixel masked, every store a full pair, no row skipped but the first two of a run's first step — a
// predicate-free copy of the body, as easu_h_quad2x_kernel takes for interior tiles.
// SO: void = RCAS's own RGBA16F store; otherwise the display epilogue of fsr1_upscale_post (post_pair, fsr1_post.cuh) with its store.
// kSurfOut (FSR1_FLAG_OUT_SURFACE): p.out.base is a surface object; each output pixel is one surface store of its element at (x, row).
template <bool kIn, int NW, typename SO, bool kSurfOut = false>
__device__ __forceinline__ void fused_step(FusedSmem<NW>& sm, const FusedParams& p, const FusedStep& cur, const uint2* tile, int dx,
                                           int k0, __half2 sharp, int lane, int warp, const PostParams* q) {
  constexpr int CY = FusedCfg<NW>::kCY;
  constexpr bool kPost = !std::is_void<SO>::value;
  const int n = cur.n;
#pragma unroll 1
  for (int q = 0; q < 2; q++) {
    const int r = warp + q * NW;
    if (!kIn && r >= n) break;  // warp-uniform
    const int pyT = 2 * (cur.m0 + r) + 1, pxA = 2 * (k0 + lane) + 1;
    MidSink<kIn> sink;
    sink.top = &sm.mid[2 * r + 2][lane];
    sink.zT = !kIn && (pyT < 0 || pyT >= p.out.h);
    sink.zB = !kIn && (pyT + 1 < 0 || pyT + 1 >= p.out.h);
    sink.keep = kIn ? 0xffffffffu
                    : ((pxA >= 0 && pxA < p.out.w) ? 0x0000ffffu : 0u) | ((pxA + 1 >= 0 && pxA + 1 < p.out.w) ? 0xffff0000u : 0u);
    quad_compute<MidSink<kIn>, kFBW, kFSW>(tile + dx, sm.S + dx, lane, r, true, true, sink);
  }
  __syncthreads();
  // RCAS on the rows whose neighbours are in the mid tile: warp w takes output rows 2 m0 + 4w .. + 3 (mid index 4w+1 ..)
  constexpr int kR = 2 * CY / NW;  // rows per warp
  const int o_first = 2 * cur.m0 + warp * kR;
  const int i0 = warp * kR;        // mid index of the row above the warp's first output row
  const int lm = lane > 0 ? lane - 1 : 0;
  const int ox = 2 * (k0 + lane);  // first pixel of the lane's output pair
  const bool writer = lane >= 1 && (kIn || ox < p.out.w);
  // kIn: only the first two rows of a run's first step (warp 0) lie above ya; they are computed like the others, not stored
  const bool wtop = writer && (!kIn || o_first >= cur.ya);
  if constexpr (kPost || kSurfOut) {
    // the epilogue needs registers: a rolling window of three mid rows instead of all kR + 2 up front (no spills at 6 CTAs per SM);
    // the surface stores take the same window (surf_per_sm)
    auto mid_row = [&](int i, Row3& e, Row3& d, Row3& f) {
      const uint4 a = sm.mid[i][lm], c = sm.mid[i][lane];
      e.r = uh2(__byte_perm(a.x, c.x, 0x5432));
      e.g = uh2(__byte_perm(a.y, c.y, 0x5432));
      e.b = uh2(__byte_perm(a.z, c.z, 0x5432));
      d.r = uh2(a.x); d.g = uh2(a.y); d.b = uh2(a.z);
      f.r = uh2(c.x); f.g = uh2(c.y); f.b = uh2(c.z);
    };
    Row3 ea, eb, db, fb, ec, dc, fc;
    mid_row(i0, ea, dc, fc);
    mid_row(i0 + 1, eb, db, fb);
    unsigned char* dst = p.out.base + (long long)(o_first - p.out.row0) * p.out.pitch + (long long)ox * PostStore<SO>::kBytes;
    PostCursor pc;
    if constexpr (kPost) pc.init(*q, ox, o_first);
#pragma unroll
    for (int r = 0; r < kR; r++) {
      const int o = o_first + r;
      mid_row(i0 + r + 2, ec, dc, fc);
      if (kIn || (o >= cur.ya && o < cur.yb && o < 2 * cur.m0 + 2 * n)) {  // warp-uniform
        __half2 oR, oG, oB;
        rcas_pair<0>(ea, db, eb, fb, ec, sharp, oR, oG, oB);
        if (r >= 2 ? writer : wtop) {
          if constexpr (kPost) {
            post_pair<SO, kSurfOut>(*q, pc, kSurfOut ? p.out.base : dst + (long long)r * p.out.pitch, ox, o, oR, oG, oB, 0x3c003c00u,
                                    kIn || ox + 1 < p.out.w);
          } else {
            const uint4 w = pack_pair_half(oR, oG, oB, 0x3c003c00u);
            surf_store8(surf_of(p.out), ox, o, make_uint2(w.x, w.y));
            if (kIn || ox + 1 < p.out.w) surf_store8(surf_of(p.out), ox + 1, o, make_uint2(w.z, w.w));
          }
        }
      }
      if constexpr (kPost) pc.next_row(*q);
      ea = eb; eb = ec; db = dc; fb = fc;
    }
  } else {
    Row3 E[kR + 2], D[kR], Fv[kR];
#pragma unroll
    for (int r = 0; r < kR + 2; r++) {
      const uint4 a = sm.mid[i0 + r][lm], c = sm.mid[i0 + r][lane];
      E[r].r = uh2(__byte_perm(a.x, c.x, 0x5432));
      E[r].g = uh2(__byte_perm(a.y, c.y, 0x5432));
      E[r].b = uh2(__byte_perm(a.z, c.z, 0x5432));
      if (r >= 1 && r <= kR) {
        D[r - 1].r = uh2(a.x); D[r - 1].g = uh2(a.y); D[r - 1].b = uh2(a.z);
        Fv[r - 1].r = uh2(c.x); Fv[r - 1].g = uh2(c.y); Fv[r - 1].b = uh2(c.z);
      }
    }
    unsigned char* dst = p.out.base + (long long)(o_first - p.out.row0) * p.out.pitch + (long long)ox * 8;
#pragma unroll
    for (int r = 0; r < kR; r++) {
      const int o = o_first + r;
      if (kIn || (o >= cur.ya && o < cur.yb && o < 2 * cur.m0 + 2 * n)) {  // warp-uniform
        __half2 oR, oG, oB;
        rcas_pair<0>(E[r], D[r], E[r + 1], Fv[r], E[r + 2], sharp, oR, oG, oB);
        if (r >= 2 ? writer : wtop) {
          const uint4 w = pack_pair_half(oR, oG, oB, 0x3c003c00u);
          unsigned char* o8 = dst + (long long)r * p.out.pitch;
          if (kIn || ox + 1 < p.out.w) *reinterpret_cast<uint4*>(o8) = w;
          else *reinterpret_cast<uint2*>(o8) = make_uint2(w.x, w.y);
        }
      }
    }
  }
}

// kIn != kInTma (FSR1_FLAG_IN_SURFACE / IN_TEXTURE): p.in.base is a surface or texture object on a CUDA array and `tmap` is unused.
// Phase 1 reads the step's kFBW (n + 3) texels with surface loads or texture fetches (array_texel) at coordinates clamped to the
// logical image (the texels TMA + clamp_fixup would leave in the tile), into one tile buffer: no TMA, no mbarrier, no prefetch.  The
// previous step's closing barrier frees the buffer.  (kInSurf is 1, so the surface twins' bool kSurfIn selects it.)
template <int NW, typename SO, bool kSrtmIn, bool kR11 = false, int kIn = kInTma, bool kSurfOut = false>
__device__ __forceinline__ void fused_body(const FusedParams p, const CUtensorMap& tmap, const PostParams* q) {
  constexpr bool kArrayIn = kIn != kInTma;
  using C = FusedCfg<NW>;
  constexpr int NT = NW * 32, CY = C::kCY;
  constexpr uint32_t kBoxBytes = kR11 ? kRBW * C::kBH * 4u : C::kElems * 8u;
  constexpr int kStage = ((kRBW * C::kBH * 4 + 127) / 128) * 128 / 4;
  __shared__ FusedSmem<NW> sm;
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
  FusedIter<CY> iter;
  iter.init(p, blockIdx.x, gridDim.x);
  FusedStep cur, nxt;
  bool has = iter.next(cur);
  auto box_x = [](const FusedStep& s) { return (kStripCells * s.tx - 2) & ~1; };  // even texel at or before the first tap column
  auto tma_x = [&](const FusedStep& s) { return kR11 ? box_x(s) & ~3 : box_x(s); };
  if (!kArrayIn && tid == 0 && has) {
    mbar_expect_tx(&sm.bar[0], kBoxBytes);
    tma_load_2d(kR11 ? (void*)stage : (void*)sm.tile[0], &tmap, tma_x(cur), cur.m0 - 1 - p.in.row0, &sm.bar[0]);
  }
  const __half2 sharp = uh2(p.sharp_h2);
  for (int it = 0; has; it++) {
    const int b = it & 1;
    const bool hasn = iter.next(nxt);
    if (!kArrayIn && tid == 0 && hasn) {  // prefetch the next step's box into the other buffer (its readers passed the closing barrier)
      fence_proxy_async();
      mbar_expect_tx(&sm.bar[b ^ 1], kBoxBytes);
      tma_load_2d(kR11 ? (void*)(stage + (b ^ 1) * kStage) : (void*)sm.tile[b ^ 1], &tmap, tma_x(nxt), nxt.m0 - 1 - p.in.row0,
                  &sm.bar[b ^ 1]);
    }
    uint2* tile = sm.tile[kR11 || kArrayIn ? 0 : b];  // kR11, kArrayIn: phase 1 writes the half tile after the previous step's closing barrier
    const int k0 = kStripCells * cur.tx - 1;       // first cell of the strip (lane 0)
    const int gxe = box_x(cur), dx = (k0 - 1) - gxe;  // box origin; offset of tap column 0 of lane 0 inside it (0 or 1)
    const int gy0 = cur.m0 - 1, n = cur.n;
    if (!kArrayIn) {
      mbar_wait(&sm.bar[b], (it >> 1) & 1);
      if (gxe < 0 || gy0 < 0 || gxe + kFBW > p.in.w || gy0 + C::kBH > p.in.h) {
        if constexpr (kR11) clamp_fixup(stage + b * kStage + (gxe & 3), kRBW, kFBW, C::kBH, gxe, gy0, p.in.w, p.in.h, lane, warp, NW);
        else clamp_fixup(tile, kFBW, kFBW, C::kBH, gxe, gy0, p.in.w, p.in.h, lane, warp, NW);
        fence_proxy_async();
        __syncthreads();
      }
    }
    // phases 1 and 2 on the rows this step needs (n + 3 texel rows, n + 1 rows of terms)
    if constexpr (kArrayIn) {
      const unsigned long long src = surf_of(p.in);
      for (int i = tid; i < kFBW * (n + 3); i += NT) {
        const int j = i / kFBW, c = i - j * kFBW;
        uint2 t = array_texel<kIn, kR11>(src, clampi(gxe + c, 0, p.in.w - 1), clampi(gy0 + j, 0, p.in.h - 1));
        if (kSrtmIn) t = srtm_texel(t);
        tile[i] = t;
        sm.L[i] = texel_luma(t);
      }
    } else if constexpr (kR11) {
      r11_phase1_staged<kSrtmIn, NT>(stage + b * kStage, tile, sm.L, kFBW * (n + 3), kFBW, kRBW, gxe & 3, tid);
    } else {
      for (int i = tid; i < kFBW * (n + 3); i += NT) {
        uint2 c = tile[i];
        if (kSrtmIn) tile[i] = c = srtm_texel(c);
        sm.L[i] = texel_luma(c);
      }
    }
    __syncthreads();
    for (int idx = tid; idx < kFSW * (n + 1); idx += NT) {
      const int j = idx / kFSW, i = idx - j * kFSW;
      const float* c = sm.L + (j + 1) * kFBW + (i + 1);
      sm.S[idx] = texel_terms(c[-kFBW], c[-1], c[0], c[1], c[kFBW]);
    }
    __syncthreads();
    // interior step: the strip's cells and pixels are in the image (k0 >= 0, m0 >= 0, last pixel column and row inside), the step
    // is full (n = CY) and every output row it produces lies in [ya, yb), but for the first two of a run's first step, which lie
    // above ya (fused_step skips them)
    const bool inside = k0 >= 0 && 2 * (k0 + 31) + 2 < p.out.w && cur.m0 >= 0 && 2 * (cur.m0 + CY) < p.out.h && n == CY &&
                        2 * cur.m0 + 2 >= cur.ya && 2 * (cur.m0 + CY) <= cur.yb;
    if (inside) fused_step<true, NW, SO, kSurfOut>(sm, p, cur, tile, dx, k0, sharp, lane, warp, q);
    else fused_step<false, NW, SO, kSurfOut>(sm, p, cur, tile, dx, k0, sharp, lane, warp, q);
    __syncthreads();
    if (n == CY && tid < 64) {  // the run may continue: its last two mid rows become rows 0, 1 of the next step
      const int rr = tid >> 5;
      sm.mid[rr][lane] = sm.mid[2 * CY + rr][lane];
    }
    // (no barrier needed here: the next writers of mid rows >= 2 and the next readers of rows 0, 1 are both behind the
    //  two __syncthreads of the next iteration's phases 1 and 2)
    cur = nxt;
    has = hasn;
  }
  halo_sync_end(p.sync);
}

template <int NW, int MINB, bool kSrtmIn = false>
__global__ void __launch_bounds__(NW * 32, MINB)
fused_h_quad2x_kernel(const FusedParams p, const __grid_constant__ CUtensorMap tmap) {
  fused_body<NW, void, kSrtmIn>(p, tmap, nullptr);
}

// fsr1_upscale_post: the same kernel with the display epilogue in RCAS's store (SO: __half, Unorm8, Unorm10)
template <int NW, int MINB, typename SO, bool kSrtmIn = false>
__global__ void __launch_bounds__(NW * 32, MINB)
fused_h_quad2x_post_kernel(const FusedParams p, const __grid_constant__ CUtensorMap tmap, const __grid_constant__ PostParams q) {
  fused_body<NW, SO, kSrtmIn>(p, tmap, &q);
}

// R11G11B10_FLOAT input: the same two kernels on the kR11 box
template <int NW, int MINB, bool kSrtmIn>
__global__ void __launch_bounds__(NW * 32, MINB)
fused_r11_quad2x_kernel(const FusedParams p, const __grid_constant__ CUtensorMap tmap) {
  fused_body<NW, void, kSrtmIn, true>(p, tmap, nullptr);
}
template <int NW, int MINB, typename SO, bool kSrtmIn>
__global__ void __launch_bounds__(NW * 32, MINB)
fused_r11_quad2x_post_kernel(const FusedParams p, const __grid_constant__ CUtensorMap tmap, const __grid_constant__ PostParams q) {
  fused_body<NW, SO, kSrtmIn, true>(p, tmap, &q);
}

// FSR1_FLAG_IN_SURFACE / OUT_SURFACE: the same two kernels reading the input and / or writing the output through surface objects
// (RGBA16F input; `tmap` is unused with kSurfIn)
template <int NW, int MINB, bool kSrtmIn, bool kSurfIn, bool kSurfOut>
__global__ void __launch_bounds__(NW * 32, MINB)
fused_h_quad2x_surf_kernel(const FusedParams p, const __grid_constant__ CUtensorMap tmap) {
  fused_body<NW, void, kSrtmIn, false, kSurfIn, kSurfOut>(p, tmap, nullptr);
}
template <int NW, int MINB, typename SO, bool kSrtmIn, bool kSurfIn, bool kSurfOut>
__global__ void __launch_bounds__(NW * 32, MINB)
fused_h_quad2x_post_surf_kernel(const FusedParams p, const __grid_constant__ CUtensorMap tmap, const __grid_constant__ PostParams q) {
  fused_body<NW, SO, kSrtmIn, false, kSurfIn, kSurfOut>(p, tmap, &q);
}

// FSR1_FLAG_IN_TEXTURE: the same two kernels reading their RGBA16F or (kR11) R11G11B10F input through a texture object (`tmap` unused),
// writing a linear output or with kSurfOut a surface
template <int NW, int MINB, bool kSrtmIn, bool kR11, bool kSurfOut>
__global__ void __launch_bounds__(NW * 32, MINB)
fused_h_quad2x_tex_kernel(const FusedParams p, const __grid_constant__ CUtensorMap tmap) {
  fused_body<NW, void, kSrtmIn, kR11, kInTex, kSurfOut>(p, tmap, nullptr);
}
template <int NW, int MINB, typename SO, bool kSrtmIn, bool kR11, bool kSurfOut>
__global__ void __launch_bounds__(NW * 32, MINB)
fused_h_quad2x_post_tex_kernel(const FusedParams p, const __grid_constant__ CUtensorMap tmap, const __grid_constant__ PostParams q) {
  fused_body<NW, SO, kSrtmIn, kR11, kInTex, kSurfOut>(p, tmap, &q);
}

#ifndef FSR1_CPU_EMU
// tensor map, parameters and grid of a fused launch; cudaErrorNotSupported when the frame is not one the kernel takes.
// out_align: the alignment the output store needs (16 for RGBA16F pairs, 8 for UNORM pairs).  array_in / surf_out: the input is a
// surface or texture object, the output a surface object (no alignment rule; no tensor map for an array input: `tmap` is zeroed).
static cudaError_t fused_setup(const EasuParams& e, uint32_t sharp_h2, int out_align, bool r11, CUtensorMap& tmap, FusedParams& p,
                               int& per_sm, long long& grid, bool array_in = false, bool surf_out = false) {
  if (!is_2x(e.c0x, e.c0y, e.c0z, e.c0w)) return cudaErrorNotSupported;
  if ((!array_in && ((reinterpret_cast<uintptr_t>(e.in.base) & 15) || (e.in.pitch & 15))) ||
      (!surf_out && ((reinterpret_cast<uintptr_t>(e.out.base) & (out_align - 1)) || (e.out.pitch & (out_align - 1)))))
    return cudaErrorNotSupported;
  constexpr int NW = 4;
  using C = FusedCfg<NW>;
  EncodeTiledFn encode = get_encode_fn();
  if (array_in) memset(&tmap, 0, sizeof tmap);
  else if (!encode) return cudaErrorNotSupported;
  const cuuint64_t dims[2] = {(cuuint64_t)e.in.w, (cuuint64_t)e.in.rows};
  const cuuint64_t strides[1] = {(cuuint64_t)e.in.pitch};
  const cuuint32_t box[2] = {(cuuint32_t)(r11 ? kRBW : kFBW), (cuuint32_t)C::kBH};
  const cuuint32_t estr[2] = {1, 1};
  if (!array_in &&
      encode(&tmap, r11 ? CU_TENSOR_MAP_DATA_TYPE_UINT32 : CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, e.in.base, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return cudaErrorNotSupported;
  p.in = e.in; p.out = e.out; p.y0 = e.y0; p.y1 = e.y1; p.sharp_h2 = sharp_h2; p.sync = e.sync;
  // output pairs (2k, 2k+1), k = 0 .. (w-1)/2, 31 per strip
  p.n_strips = ((e.out.w + 1) / 2 + kStripCells - 1) / kStripCells;
  const long long units = (long long)p.n_strips * ((e.y1 - e.y0 + 1) / 2);
  // 72 registers = 7 CTAs per SM, as easu_h_quad2x; a launch that waits for a neighbour's halo (p.sync) takes 6 so that the
  // one-warp halo_push_kernel it waits for still fits beside it (launch_easu_h_tiled, DESIGN.md §6)
  if (p.sync.ready[0] || p.sync.ready[1]) per_sm = 6;
  grid = (long long)per_sm * sm_count();
  if (grid > (units + 7) / 8) grid = (units + 7) / 8;  // at least ~16 rows of a strip per CTA
  if (grid < 1) grid = 1;
  return cudaSuccess;
}

// The display epilogue needs more registers than the 72 of 7 CTAs per SM (-Xptxas -v: DESIGN.md §4): 6 per SM.
constexpr int kPostPerSm = 6;

// FSR1_FLAG_IN_SURFACE / OUT_SURFACE: the surface twin of the plain (SO = void) or post kernel for the flag combination.  The plain twin
// that takes its input by TMA and stores through a surface spills 4-8 B at the 72 registers of 7 CTAs per SM (-Xptxas -v, rolled or
// unrolled row loop), so it runs at 6 per SM; the others keep 7.
constexpr int surf_per_sm(bool surf_in, bool surf_out) { return surf_out && !surf_in ? 6 : 7; }
template <typename SO, bool kSrtmIn, bool kSurfIn, bool kSurfOut>
static void surf_kernel(const FusedParams& p, const CUtensorMap& tmap, const PostParams* q, long long grid, cudaStream_t s) {
  if constexpr (std::is_void<SO>::value)
    fused_h_quad2x_surf_kernel<4, surf_per_sm(kSurfIn, kSurfOut), kSrtmIn, kSurfIn, kSurfOut><<<(int)grid, 4 * 32, 0, s>>>(p, tmap);
  else fused_h_quad2x_post_surf_kernel<4, kPostPerSm, SO, kSrtmIn, kSurfIn, kSurfOut><<<(int)grid, 4 * 32, 0, s>>>(p, tmap, *q);
}
// names[0]: plain; [1..3]: post into RGBA16F, RGBA8, RGB10A2.  Index within a row: the combination (srtm_in, surf_in, surf_out) in the
// order of the switch below.
static const char* const kSurfNames[4][6] = {
    {"fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,7/sm,strips,surf_in>",
      "fused_easu_rcas_h_quad2x<4w,7/sm,strips,surf_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,srtm_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,7/sm,strips,srtm_in,surf_in>",
      "fused_easu_rcas_h_quad2x<4w,7/sm,strips,srtm_in,surf_in,surf_out>"},
    {"fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba16f,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba16f,surf_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba16f,surf_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba16f,srtm_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba16f,srtm_in,surf_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba16f,srtm_in,surf_in,surf_out>"},
    {"fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba8,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba8,surf_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba8,surf_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba8,srtm_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba8,srtm_in,surf_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba8,srtm_in,surf_in,surf_out>"},
    {"fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgb10a2,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgb10a2,surf_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgb10a2,surf_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgb10a2,srtm_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgb10a2,srtm_in,surf_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgb10a2,srtm_in,surf_in,surf_out>"}};
template <typename SO>
static cudaError_t launch_surf(const FusedParams& p, const CUtensorMap& tmap, const PostParams* q, long long grid, bool srtm_in, bool surf_in,
                               bool surf_out, cudaStream_t s, const char** name, int names_row) {
  int v = 0;
  switch ((srtm_in ? 4 : 0) | (surf_in ? 2 : 0) | (surf_out ? 1 : 0)) {
    case 1: surf_kernel<SO, false, false, true>(p, tmap, q, grid, s); v = 0; break;
    case 2: surf_kernel<SO, false, true, false>(p, tmap, q, grid, s); v = 1; break;
    case 3: surf_kernel<SO, false, true, true>(p, tmap, q, grid, s); v = 2; break;
    case 5: surf_kernel<SO, true, false, true>(p, tmap, q, grid, s); v = 3; break;
    case 6: surf_kernel<SO, true, true, false>(p, tmap, q, grid, s); v = 4; break;
    case 7: surf_kernel<SO, true, true, true>(p, tmap, q, grid, s); v = 5; break;
    default: return cudaErrorNotSupported;
  }
  *name = kSurfNames[names_row][v];
  return cudaGetLastError();
}

// FSR1_FLAG_IN_TEXTURE: the texture twin of the plain or post kernel, at the CTAs per SM of its surface-input twin
template <typename SO, bool kSrtmIn, bool kR11, bool kSurfOut>
static void tex_kernel(const FusedParams& p, const CUtensorMap& tmap, const PostParams* q, long long grid, cudaStream_t s) {
  if constexpr (std::is_void<SO>::value)
    fused_h_quad2x_tex_kernel<4, surf_per_sm(true, kSurfOut), kSrtmIn, kR11, kSurfOut><<<(int)grid, 4 * 32, 0, s>>>(p, tmap);
  else fused_h_quad2x_post_tex_kernel<4, kPostPerSm, SO, kSrtmIn, kR11, kSurfOut><<<(int)grid, 4 * 32, 0, s>>>(p, tmap, *q);
}
// rows as kSurfNames; index within a row: (r11 ? 4 : 0) | (srtm_in ? 2 : 0) | (surf_out ? 1 : 0)
static const char* const kTexNames[4][8] = {
    {"fused_easu_rcas_h_quad2x<4w,7/sm,strips,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,7/sm,strips,tex_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,7/sm,strips,srtm_in,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,7/sm,strips,srtm_in,tex_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,7/sm,strips,r11g11b10f_in,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,7/sm,strips,r11g11b10f_in,tex_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,7/sm,strips,r11g11b10f_in,srtm_in,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,7/sm,strips,r11g11b10f_in,srtm_in,tex_in,surf_out>"},
    {"fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba16f,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba16f,tex_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba16f,srtm_in,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba16f,srtm_in,tex_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba16f,r11g11b10f_in,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba16f,r11g11b10f_in,tex_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba16f,r11g11b10f_in,srtm_in,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba16f,r11g11b10f_in,srtm_in,tex_in,surf_out>"},
    {"fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba8,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba8,tex_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba8,srtm_in,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba8,srtm_in,tex_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba8,r11g11b10f_in,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba8,r11g11b10f_in,tex_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba8,r11g11b10f_in,srtm_in,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgba8,r11g11b10f_in,srtm_in,tex_in,surf_out>"},
    {"fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgb10a2,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgb10a2,tex_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgb10a2,srtm_in,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgb10a2,srtm_in,tex_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgb10a2,r11g11b10f_in,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgb10a2,r11g11b10f_in,tex_in,surf_out>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgb10a2,r11g11b10f_in,srtm_in,tex_in>",
      "fused_easu_rcas_h_quad2x<4w,6/sm,strips,post,rgb10a2,r11g11b10f_in,srtm_in,tex_in,surf_out>"}};
template <typename SO>
static cudaError_t launch_tex(const FusedParams& p, const CUtensorMap& tmap, const PostParams* q, long long grid, bool srtm_in, bool r11,
                              bool surf_out, cudaStream_t s, const char** name, int names_row) {
  const int v = (r11 ? 4 : 0) | (srtm_in ? 2 : 0) | (surf_out ? 1 : 0);
  switch (v) {
    case 0: tex_kernel<SO, false, false, false>(p, tmap, q, grid, s); break;
    case 1: tex_kernel<SO, false, false, true>(p, tmap, q, grid, s); break;
    case 2: tex_kernel<SO, true, false, false>(p, tmap, q, grid, s); break;
    case 3: tex_kernel<SO, true, false, true>(p, tmap, q, grid, s); break;
    case 4: tex_kernel<SO, false, true, false>(p, tmap, q, grid, s); break;
    case 5: tex_kernel<SO, false, true, true>(p, tmap, q, grid, s); break;
    case 6: tex_kernel<SO, true, true, false>(p, tmap, q, grid, s); break;
    default: tex_kernel<SO, true, true, true>(p, tmap, q, grid, s); break;
  }
  *name = kTexNames[names_row][v];
  return cudaGetLastError();
}

cudaError_t launch_fused_h(const EasuParams& e, uint32_t sharp_h2, int clamp, cudaStream_t s, const char** name, bool srtm_in, bool r11,
                           InSrc in, bool surf_out) {
  if (clamp) return cudaErrorNotSupported;
  const bool surf_in = in == kInSurf;
  CUtensorMap tmap;
  FusedParams p;
  int per_sm = surf_per_sm(in != kInTma, surf_out);
  long long grid = 0;
  const cudaError_t err = fused_setup(e, sharp_h2, 16, r11, tmap, p, per_sm, grid, in != kInTma, surf_out);
  if (err != cudaSuccess) return err;
  if (in == kInTex) return launch_tex<void>(p, tmap, nullptr, grid, srtm_in, r11, surf_out, s, name, 0);
  if (surf_in || surf_out) return launch_surf<void>(p, tmap, nullptr, grid, srtm_in, surf_in, surf_out, s, name, 0);  // RGBA16F input
  if (r11 && srtm_in) {
    fused_r11_quad2x_kernel<4, 7, true><<<(int)grid, 4 * 32, 0, s>>>(p, tmap);
    *name = per_sm == 7 ? "fused_easu_rcas_h_quad2x<4w,7/sm,tma2,strips,r11g11b10f_in,srtm_in>"
                        : "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,r11g11b10f_in,srtm_in>";
  } else if (r11) {
    fused_r11_quad2x_kernel<4, 7, false><<<(int)grid, 4 * 32, 0, s>>>(p, tmap);
    *name = per_sm == 7 ? "fused_easu_rcas_h_quad2x<4w,7/sm,tma2,strips,r11g11b10f_in>" : "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,r11g11b10f_in>";
  } else if (srtm_in) {
    fused_h_quad2x_kernel<4, 7, true><<<(int)grid, 4 * 32, 0, s>>>(p, tmap);
    *name = per_sm == 7 ? "fused_easu_rcas_h_quad2x<4w,7/sm,tma2,strips,srtm_in>" : "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,srtm_in>";
  } else {
    fused_h_quad2x_kernel<4, 7><<<(int)grid, 4 * 32, 0, s>>>(p, tmap);
    *name = per_sm == 7 ? "fused_easu_rcas_h_quad2x<4w,7/sm,tma2,strips>" : "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips>";
  }
  return cudaGetLastError();
}

// the post kernel for out_format (1 RGBA16F, 3 RGBA8_UNORM, 4 RGB10A2_UNORM) and input kind; its name through *name
template <bool kSrtmIn, bool kR11>
static cudaError_t launch_post_kernel(const FusedParams& p, const CUtensorMap& tmap, const PostParams& q, int out_format, long long grid,
                                      cudaStream_t s, const char** name) {
  static const char* const names[3][4] = {
      {"fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba16f>", "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba16f,srtm_in>",
       "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba16f,r11g11b10f_in>",
       "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba16f,r11g11b10f_in,srtm_in>"},
      {"fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba8>", "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba8,srtm_in>",
       "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba8,r11g11b10f_in>",
       "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgba8,r11g11b10f_in,srtm_in>"},
      {"fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgb10a2>", "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgb10a2,srtm_in>",
       "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgb10a2,r11g11b10f_in>",
       "fused_easu_rcas_h_quad2x<4w,6/sm,tma2,strips,post,rgb10a2,r11g11b10f_in,srtm_in>"}};
  const int v = (kSrtmIn ? 1 : 0) + (kR11 ? 2 : 0);
  switch (out_format) {
    case 1:
      if constexpr (kR11) fused_r11_quad2x_post_kernel<4, kPostPerSm, __half, kSrtmIn><<<(int)grid, 4 * 32, 0, s>>>(p, tmap, q);
      else fused_h_quad2x_post_kernel<4, kPostPerSm, __half, kSrtmIn><<<(int)grid, 4 * 32, 0, s>>>(p, tmap, q);
      *name = names[0][v];
      break;
    case 3:
      if constexpr (kR11) fused_r11_quad2x_post_kernel<4, kPostPerSm, Unorm8, kSrtmIn><<<(int)grid, 4 * 32, 0, s>>>(p, tmap, q);
      else fused_h_quad2x_post_kernel<4, kPostPerSm, Unorm8, kSrtmIn><<<(int)grid, 4 * 32, 0, s>>>(p, tmap, q);
      *name = names[1][v];
      break;
    case 4:
      if constexpr (kR11) fused_r11_quad2x_post_kernel<4, kPostPerSm, Unorm10, kSrtmIn><<<(int)grid, 4 * 32, 0, s>>>(p, tmap, q);
      else fused_h_quad2x_post_kernel<4, kPostPerSm, Unorm10, kSrtmIn><<<(int)grid, 4 * 32, 0, s>>>(p, tmap, q);
      *name = names[2][v];
      break;
    default: return cudaErrorNotSupported;
  }
  return cudaGetLastError();
}

cudaError_t launch_fused_h_post(const EasuParams& e, uint32_t sharp_h2, const PostParams& q, int out_format, cudaStream_t s,
                                const char** name, bool srtm_in, bool r11, InSrc in, bool surf_out) {
  if (out_format != 1 && out_format != 3 && out_format != 4) return cudaErrorNotSupported;
  const bool surf_in = in == kInSurf;
  CUtensorMap tmap;
  FusedParams p;
  int per_sm = kPostPerSm;
  long long grid = 0;
  const cudaError_t err = fused_setup(e, sharp_h2, out_format == 1 ? 16 : 8, r11, tmap, p, per_sm, grid, in != kInTma, surf_out);
  if (err != cudaSuccess) return err;
  if (in == kInTex) {
    switch (out_format) {
      case 1: return launch_tex<__half>(p, tmap, &q, grid, srtm_in, r11, surf_out, s, name, 1);
      case 3: return launch_tex<Unorm8>(p, tmap, &q, grid, srtm_in, r11, surf_out, s, name, 2);
      default: return launch_tex<Unorm10>(p, tmap, &q, grid, srtm_in, r11, surf_out, s, name, 3);
    }
  }
  if (surf_in || surf_out) {  // RGBA16F input
    switch (out_format) {
      case 1: return launch_surf<__half>(p, tmap, &q, grid, srtm_in, surf_in, surf_out, s, name, 1);
      case 3: return launch_surf<Unorm8>(p, tmap, &q, grid, srtm_in, surf_in, surf_out, s, name, 2);
      default: return launch_surf<Unorm10>(p, tmap, &q, grid, srtm_in, surf_in, surf_out, s, name, 3);
    }
  }
  if (r11) return srtm_in ? launch_post_kernel<true, true>(p, tmap, q, out_format, grid, s, name)
                          : launch_post_kernel<false, true>(p, tmap, q, out_format, grid, s, name);
  return srtm_in ? launch_post_kernel<true, false>(p, tmap, q, out_format, grid, s, name)
                 : launch_post_kernel<false, false>(p, tmap, q, out_format, grid, s, name);
}
#endif

}  // namespace fsr1
