// fsr1_pointwise.cu — the pointwise companions of the scaling path (SURVEY.md §8(f).4): the steps the sample runs
// directly before EASU and after RCAS, as image-level passes on sm_90a.
//
//   SRTM / SRTM-inverse   FsrSrtmF / FsrSrtmInvF      ffx-fsr/ffx_fsr1.h:1044,1046   reversible tone-mapper around the filter
//   LFGA                  FsrLfgaF                     ffx-fsr/ffx_fsr1.h:1014        film grain after scaling
//   TEPD 8 / 10 bit       FsrTepdC8F / FsrTepdC10F     ffx-fsr/ffx_fsr1.h:1100-1126   dithered linear -> gamma 2.0
//                         FsrTepdDitF                  ffx-fsr/ffx_fsr1.h:1086-1095   positional dither value
//   SQUARE                `c *= c`                     sample/src/DX12/FSR_Pass.hlsl:78-79,84-85,93-94,99-100
//                                                      (the Sample.x hook: gamma 2.0 back to linear on the last pass)
//
// These are streaming passes: 2 x bytes-per-pixel of compulsory traffic and a few dozen flops per pixel, i.e.
// HBM-bound by a wide margin.  One thread = kRowsPerThread pixels of ONE row, 256 apart (a CTA covers a contiguous
// 1024-pixel stretch of a row): the loads of all of them are issued before any arithmetic (memory-level
// parallelism), every warp access is one fully coalesced 128/256/512-byte segment, and there is no shared memory.  Because the arithmetic is free here, it is always the
// EXACT policy: separate roundings, IEEE sqrt and division — the fp32 results are bit-identical to the reference
// source compiled with -ffp-contract=off, for every storage format (fp16/unorm storage rounds that fp32 result once).
// Alpha is carried through unchanged (the reference functions take RGB).
#include <stdlib.h>
#include "fsr1_post.cuh"  // the arithmetic (apply_op), shared with the display epilogue of fsr1_upscale_post

namespace fsr1 {

constexpr int kRowsPerThread = 4;
constexpr int kPointThreads = 256;

struct PointParams {
  ImgView in, out, aux;
  int aux_format;  // 0: no aux image
  int op;
  float amount;    // LFGA
  uint32_t frame;  // TEPD positional dither
  int y0, y1;
};

// kCols = false: a thread owns one column position and kRowsPerThread rows (CTA = 256 x 4 pixels);
// kCols = true : a thread owns kRowsPerThread positions 256 apart in ONE row (CTA = 1024 x 1 pixels: one contiguous
//               8-16 KB stretch of a row per CTA).  Same arithmetic, different DRAM access shape (FSR1_POINT_LAYOUT).
template <typename SI, typename SO, bool kCols, int N>
__global__ void __launch_bounds__(kPointThreads) pointwise_kernel(const PointParams p, const int aux_step) {
  int xs[N], ys[N];
#pragma unroll
  for (int r = 0; r < N; r++) {
    xs[r] = kCols ? blockIdx.x * (kPointThreads * N) + threadIdx.x + kPointThreads * r : blockIdx.x * kPointThreads + threadIdx.x;
    ys[r] = kCols ? p.y0 + (int)blockIdx.y : p.y0 + (int)blockIdx.y * N + r;
  }
  float4 c[N];
#pragma unroll
  for (int r = 0; r < N; r++)
    if (xs[r] < p.out.w && ys[r] < p.y1) c[r] = load4<SI>(p.in, xs[r], ys[r]);
  // position inside the aux tile: one division per thread, then incremental with wrap
  int ax = 0, ay = 0;
  if (p.aux_format) {
    ax = xs[0] % p.aux.w;
    ay = ys[0] % p.aux.h;
  }
#pragma unroll
  for (int r = 0; r < N; r++) {
    if (xs[r] < p.out.w && ys[r] < p.y1) {
      const float4 o = apply_op(p.op, c[r], p.aux, p.aux_format, p.amount, p.frame, xs[r], ys[r], ax, ay);
      Px<SO>::store(p.out, xs[r], ys[r], o.x, o.y, o.z, o.w);
    }
    if (kCols) {
      ax += aux_step;  // aux_step = 256 mod aux width (host)
      if (ax >= p.aux.w) ax -= p.aux.w;
    } else if (++ay >= p.aux.h) {
      ay = 0;
    }
  }
}

template <typename SI, typename SO>
static cudaError_t launch_one(const PointParams& p, cudaStream_t s) {
  // a CTA covers a contiguous stretch of one row (measured: +8 % over a 256x4-pixel CTA on RGBA16F; 8 pixels per thread
  // is slower: registers)
  const int aux_step = p.aux_format ? kPointThreads % p.aux.w : 0;
  const int per_cta = kPointThreads * kRowsPerThread;
  const dim3 grid((p.out.w + per_cta - 1) / per_cta, p.y1 - p.y0, 1);
  pointwise_kernel<SI, SO, true, kRowsPerThread><<<grid, kPointThreads, 0, s>>>(p, aux_step);
  return cudaGetLastError();
}

// in_format == out_format for every op; TEPD may also write its 8/10-bit code values straight into a UNORM image
// from a float image (the conversion it exists for).
cudaError_t launch_pointwise(int op, const ImgView& in, int in_format, const ImgView& out, int out_format, const ImgView* aux,
                             int aux_format, float amount, uint32_t frame, int y0, int y1, cudaStream_t s, const char** name) {
  PointParams p;
  p.in = in;
  p.out = out;
  p.aux_format = aux ? aux_format : 0;
  if (aux) p.aux = *aux; else p.aux = in;
  p.op = op;
  p.amount = amount;
  p.frame = frame;
  p.y0 = y0;
  p.y1 = y1;
  static const char* const names[] = {"", "pointwise<srtm>", "pointwise<srtm_inv>", "pointwise<lfga>", "pointwise<tepd8>",
                                      "pointwise<tepd10>", "pointwise<square>"};
  if (op < kOpSrtm || op > kOpSquare) return cudaErrorInvalidValue;
  *name = names[op];
  if (in_format == out_format) {
    switch (in_format) {
      case 1: return launch_one<__half, __half>(p, s);
      case 2: return launch_one<float, float>(p, s);
      case 3: return launch_one<Unorm8, Unorm8>(p, s);
      case 4: return launch_one<Unorm10, Unorm10>(p, s);
    }
    return cudaErrorNotSupported;
  }
  if (op == kOpTepd8 && out_format == 3) {
    if (in_format == 1) return launch_one<__half, Unorm8>(p, s);
    if (in_format == 2) return launch_one<float, Unorm8>(p, s);
  }
  if (op == kOpTepd10 && out_format == 4) {
    if (in_format == 1) return launch_one<__half, Unorm10>(p, s);
    if (in_format == 2) return launch_one<float, Unorm10>(p, s);
  }
  return cudaErrorNotSupported;
}

}  // namespace fsr1
