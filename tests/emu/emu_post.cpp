// TEST INFRASTRUCTURE — runs the display epilogues of fsr1_upscale_post (fused_h_quad2x_post_kernel in csrc/fsr1_fused.cu,
// rcas_post_kernel in csrc/fsr1_rcas_packed.cu, the arithmetic in csrc/fsr1_post.cuh) on CPU threads, like emu_easu.cpp does for the
// other kernels (see include/cuda_emu.h).  A library of its own (post.mk): the .cu files are compiled AS IS with -DFSR1_CPU_EMU, and
// this harness re-creates the launchers' geometry and the CTA/thread structure.
#include <pthread.h>
#include <thread>
#include <vector>

#include "cuda_emu.h"

thread_local uint3 threadIdx, blockIdx;
thread_local dim3 gridDim, blockDim;
static pthread_barrier_t g_cta_barrier;
void __syncthreads() { pthread_barrier_wait(&g_cta_barrier); }
// warp shuffles: per-warp exchange buffer between two warp-wide barriers (initialised per CTA by the runners below)
static pthread_barrier_t g_warp_barrier[32];
static uint32_t g_shfl_buf[32][32];
uint32_t fsr1_emu_shfl(uint32_t v, int src) {
  const int w = (int)(threadIdx.x >> 5), lane = (int)(threadIdx.x & 31);
  g_shfl_buf[w][lane] = v;
  pthread_barrier_wait(&g_warp_barrier[w]);
  const uint32_t r = src < 0 ? v : g_shfl_buf[w][src];
  pthread_barrier_wait(&g_warp_barrier[w]);
  return r;
}
alignas(128) static unsigned char g_dynamic_smem[232448];
unsigned char* fsr1_emu_dynamic_smem() { return g_dynamic_smem; }

#include "../../fidelityfx-fsr_b200/csrc/fsr1_easu_tiled.cu"
#include "../../fidelityfx-fsr_b200/csrc/fsr1_rcas_packed.cu"
#include "../../fidelityfx-fsr_b200/csrc/fsr1_fused.cu"

using namespace fsr1;

// ---- the display epilogue of fsr1_upscale_post (csrc/fsr1_post.cuh) ------------------------------------------------------------------
// ops: FSR1_POST_* bits; tiles: whole images (format 1 RGBA16F, 2 RGBA32F, 3 RGBA8, 4 RGB10A2), dither_fmt 0 = positional dither
struct EmuPost {
  int ops;
  float amount;
  uint32_t frame;
  const void* grain;
  int gw, gh;
  long long gpitch;
  int gfmt;
  const void* dither;
  int dw, dh;
  long long dpitch;
  int dfmt;
};
static PostParams post_params(const EmuPost& e) {
  PostParams q;
  q.grain = e.grain ? ImgView{(unsigned char*)e.grain, e.gpitch, e.gw, e.gh, 0, e.gh} : ImgView{nullptr, 0, 1, 1, 0, 1};
  q.dither = e.dither ? ImgView{(unsigned char*)e.dither, e.dpitch, e.dw, e.dh, 0, e.dh} : ImgView{nullptr, 0, 1, 1, 0, 1};
  q.grain_fmt = e.grain ? e.gfmt : 0;
  q.dither_fmt = e.dither ? e.dfmt : 0;
  q.ops = e.ops; q.amount = e.amount; q.frame = e.frame;
  return q;
}

// fused_h_quad2x_post_kernel: launch geometry of launch_fused_h_post with `ctas` CTAs; out_format 1 RGBA16F, 3 RGBA8, 4 RGB10A2
extern "C" int emu_fused_h_post(const void* in, int iw, int ih, long long in_pitch, void* out, int ow, int oh, long long out_pitch,
                                int out_format, const uint32_t* rcon, int y0, int y1, int ctas, const EmuPost* post) {
  constexpr int NW = 4;
  using C = FusedCfg<NW>;
  FusedParams p;
  p.in = ImgView{(unsigned char*)in, in_pitch, iw, ih, 0, ih};
  p.out = ImgView{(unsigned char*)out, out_pitch, ow, oh, 0, oh};
  p.y0 = y0; p.y1 = y1; p.sharp_h2 = rcon[1];
  p.n_strips = ((ow + 1) / 2 + kStripCells - 1) / kStripCells;
  const PostParams q = post_params(*post);
  if (out_format != 1 && out_format != 3 && out_format != 4) return -1;
  CUtensorMap tmap{(const unsigned char*)in, iw, ih, in_pitch, kFBW, C::kBH, 8};
  const int threads = NW * 32;
  for (int b = 0; b < ctas; b++) {
    pthread_barrier_init(&g_cta_barrier, nullptr, (unsigned)threads);
    std::vector<std::thread> ts;
    for (int t = 0; t < threads; t++)
      ts.emplace_back([=, &p, &tmap, &q]() {
        threadIdx = uint3{(unsigned)t, 0, 0};
        blockIdx = uint3{(unsigned)b, 0, 0};
        gridDim.x = (unsigned)ctas;
        blockDim.x = (unsigned)threads;
        if (out_format == 1) fused_h_quad2x_post_kernel<NW, 6, __half>(p, tmap, q);
        else if (out_format == 3) fused_h_quad2x_post_kernel<NW, 6, Unorm8>(p, tmap, q);
        else fused_h_quad2x_post_kernel<NW, 6, Unorm10>(p, tmap, q);
      });
    for (auto& th : ts) th.join();
    pthread_barrier_destroy(&g_cta_barrier);
  }
  return 0;
}

// rcas_post_kernel: RCAS of an RGBA16F image with the epilogue; opts as emu_rcas_h_packed_opt, out_format as emu_fused_h_post
template <typename SO, bool kClamp> static void emu_rcas_post_dispatch(const RcasParams& p, const PostParams& q, int opts) {
  switch (opts & 7) {
    case 0: rcas_post_kernel<kClamp, 0, SO>(p, q); break;
    case 1: rcas_post_kernel<kClamp, 1, SO>(p, q); break;
    case 2: rcas_post_kernel<kClamp, 2, SO>(p, q); break;
    case 3: rcas_post_kernel<kClamp, 3, SO>(p, q); break;
    case 4: rcas_post_kernel<kClamp, 4, SO>(p, q); break;
    case 5: rcas_post_kernel<kClamp, 5, SO>(p, q); break;
    case 6: rcas_post_kernel<kClamp, 6, SO>(p, q); break;
    default: rcas_post_kernel<kClamp, 7, SO>(p, q); break;
  }
}
template <typename SO> static void emu_rcas_post_clamp(const RcasParams& p, const PostParams& q, int opts) {
  if (p.clamp) emu_rcas_post_dispatch<SO, true>(p, q, opts);
  else emu_rcas_post_dispatch<SO, false>(p, q, opts);
}
extern "C" int emu_rcas_h_packed_post(const void* in, void* out, int w, int h, long long in_pitch, long long out_pitch, int out_format,
                                      const uint32_t* con, int clamp, int y0, int y1, int opts, const EmuPost* post) {
  if (out_format != 1 && out_format != 3 && out_format != 4) return -1;
  RcasParams p;
  p.in = ImgView{(unsigned char*)in, in_pitch, w, h, 0, h};
  p.out = ImgView{(unsigned char*)out, out_pitch, w, h, 0, h};
  memcpy(&p.sharp, &con[0], 4);
  p.sharp_h2 = con[1];
  p.y0 = y0; p.y1 = y1; p.clamp = clamp; p.options = opts;
  const PostParams q = post_params(*post);
  constexpr int NWARP = 4, ROWS = 4, threads = 32 * NWARP;
  const int gx = (w + kSpan - 1) / kSpan, gy = (y1 - y0 + NWARP * ROWS - 1) / (NWARP * ROWS);
  for (int by = 0; by < gy; by++)
    for (int bx = 0; bx < gx; bx++) {
      for (int i = 0; i < NWARP; i++) pthread_barrier_init(&g_warp_barrier[i], nullptr, 32);
      std::vector<std::thread> ts;
      for (int t = 0; t < threads; t++)
        ts.emplace_back([=, &p, &q]() {
          threadIdx = uint3{(unsigned)t, 0, 0};
          blockIdx = uint3{(unsigned)bx, (unsigned)by, 0};
          gridDim.x = (unsigned)gx; gridDim.y = (unsigned)gy;
          blockDim.x = (unsigned)threads;
          if (out_format == 1) emu_rcas_post_clamp<__half>(p, q, opts);
          else if (out_format == 3) emu_rcas_post_clamp<Unorm8>(p, q, opts);
          else emu_rcas_post_clamp<Unorm10>(p, q, opts);
        });
      for (auto& th : ts) th.join();
      for (int i = 0; i < NWARP; i++) pthread_barrier_destroy(&g_warp_barrier[i]);
    }
  return 0;
}

