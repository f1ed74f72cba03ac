// TEST INFRASTRUCTURE — runs the input-stage RCAS kernels of fsr1_rcas_post (rcas_in_kernel in csrc/fsr1_rcas_in.cu: R11G11B10_FLOAT
// or RGBA16F input, with or without SRTM, into the RGBA16F store or the display epilogue) on CPU threads.  A library of its own
// (rcas_in.mk), built on emu_post.cpp: the .cu files compiled AS IS with -DFSR1_CPU_EMU; the runner re-creates the launcher's geometry.
#include "emu_post.cpp"
#include "../../fidelityfx-fsr_b200/csrc/fsr1_rcas_in.cu"

template <bool kR11, typename SO> static void rcas_in_opt(const RcasParams& p, const PostParams& q, int opts, int srtm) {
  switch (opts & 7) {
    case 0: rcas_in_kernel<kR11, 0, SO, false>(p, q, srtm); break;
    case 1: rcas_in_kernel<kR11, 1, SO, false>(p, q, srtm); break;
    case 2: rcas_in_kernel<kR11, 2, SO, false>(p, q, srtm); break;
    case 3: rcas_in_kernel<kR11, 3, SO, false>(p, q, srtm); break;
    case 4: rcas_in_kernel<kR11, 4, SO, false>(p, q, srtm); break;
    case 5: rcas_in_kernel<kR11, 5, SO, false>(p, q, srtm); break;
    case 6: rcas_in_kernel<kR11, 6, SO, false>(p, q, srtm); break;
    default: rcas_in_kernel<kR11, 7, SO, false>(p, q, srtm); break;
  }
}
template <bool kR11> static void rcas_in_any(const RcasParams& p, const PostParams* q, int out_format, int opts, int srtm) {
  if (!q) rcas_in_opt<kR11, void>(p, PostParams{}, opts, srtm);
  else if (out_format == 1) rcas_in_opt<kR11, __half>(p, *q, opts, srtm);
  else if (out_format == 3) rcas_in_opt<kR11, Unorm8>(p, *q, opts, srtm);
  else rcas_in_opt<kR11, Unorm10>(p, *q, opts, srtm);
}

// launch_rcas_h_in over rows [y0, y1) of a w x h image: `in` (R11G11B10F codes with r11, else RGBA16F) points at logical row in_row0
// and holds in_rows rows; post == null: the RGBA16F store (out_format 1), else the epilogue into out_format (1 RGBA16F, 3 RGBA8,
// 4 RGB10A2).  opts: bit 0 denoise, 1 passthrough alpha, 2 output square.
extern "C" int emu_rcas_in(const void* in, int in_row0, int in_rows, long long in_pitch, void* out, long long out_pitch, int w, int h,
                           int out_format, const uint32_t* con, int clamp, int y0, int y1, int opts, const EmuPost* post, int r11,
                           int srtm) {
  if (out_format != 1 && (!post || (out_format != 3 && out_format != 4))) return -1;
  RcasParams p;
  p.in = ImgView{(unsigned char*)in, in_pitch, w, h, in_row0, in_rows};
  p.out = ImgView{(unsigned char*)out, out_pitch, w, h, 0, h};
  memcpy(&p.sharp, &con[0], 4);
  p.sharp_h2 = con[1];
  p.y0 = y0; p.y1 = y1; p.clamp = clamp; p.options = opts;
  PostParams q{};
  if (post) q = post_params(*post);
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
          if (r11) rcas_in_any<true>(p, post ? &q : nullptr, out_format, opts, srtm);
          else rcas_in_any<false>(p, post ? &q : nullptr, out_format, opts, srtm);
        });
      for (auto& th : ts) th.join();
      for (int i = 0; i < NWARP; i++) pthread_barrier_destroy(&g_warp_barrier[i]);
    }
  return 0;
}
