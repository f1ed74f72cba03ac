// TEST INFRASTRUCTURE — runs the FSR1_FLAG_SRTM_INPUT variants of the RGBA16F EASU kernels (easu_h_quad2x_kernel and easu_h_pairs_kernel
// in csrc/fsr1_easu_tiled.cu, fused_h_quad2x_kernel and fused_h_quad2x_post_kernel in csrc/fsr1_fused.cu, kSrtmIn = true) on CPU threads.
// A library of its own (srtm_in.mk).  It builds on emu_post.cpp, which supplies the CTA/thread plumbing, the epilogue parameters and
// the .cu files compiled AS IS with -DFSR1_CPU_EMU; the runners below re-create the launchers' geometry as emu_easu.cpp does for the
// flag-free kernels.
#include "emu_post.cpp"

static int cell_of(int o, float scale, float offset) {  // = host_fp of the launcher = easu_pos on the device
  volatile float m = (float)o * scale;
  volatile float s = m + offset;
  return (int)floorf(s);
}

static int max_footprint(int n_out, int first, int tile, float scale, float offset, bool even_origin) {
  int best = 4;
  for (int o0 = first; o0 < n_out; o0 += tile) {
    const int o1 = (o0 + tile - 1 < n_out - 1) ? o0 + tile - 1 : n_out - 1;
    int origin = cell_of(o0, scale, offset) - 1;
    if (even_origin) origin &= ~1;
    const int span = cell_of(o1, scale, offset) + 2 - origin + 1;
    if (span > best) best = span;
  }
  return best;
}

// `ctas` CTAs of `threads` threads, one after the other; body() is the kernel call of one thread
template <typename Body> static void run_ctas(int ctas, int threads, Body body) {
  for (int b = 0; b < ctas; b++) {
    pthread_barrier_init(&g_cta_barrier, nullptr, (unsigned)threads);
    std::vector<std::thread> ts;
    for (int t = 0; t < threads; t++)
      ts.emplace_back([=, &body]() {
        threadIdx = uint3{(unsigned)t, 0, 0};
        blockIdx = uint3{(unsigned)b, 0, 0};
        gridDim.x = (unsigned)ctas;
        blockDim.x = (unsigned)threads;
        body();
      });
    for (auto& th : ts) th.join();
    pthread_barrier_destroy(&g_cta_barrier);
  }
}

static EasuParams easu_params(const void* in, int iw, int ih, long long in_pitch, void* out, int ow, int oh, long long out_pitch,
                              const uint32_t* con, int y0, int y1) {
  EasuParams p;
  p.in = ImgView{(unsigned char*)in, in_pitch, iw, ih, 0, ih};
  p.out = ImgView{(unsigned char*)out, out_pitch, ow, oh, 0, oh};
  memcpy(&p.c0x, &con[0], 4); memcpy(&p.c0y, &con[1], 4); memcpy(&p.c0z, &con[2], 4); memcpy(&p.c0w, &con[3], 4);
  p.y0 = y0; p.y1 = y1;
  return p;
}

// easu_h_quad2x_kernel<4, 7, true>: launch_easu_h_tiled's 2x branch.  Arguments as emu_easu_h_quad2x (without the variant).
extern "C" int emu_easu_h_quad2x_srtm_in(const void* in, int iw, int ih, long long in_pitch, void* out, int ow, int oh, long long out_pitch,
                                         const uint32_t* con, int y0, int y1, int max_ctas) {
  const EasuParams p = easu_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, con, y0, y1);
  if (!(p.c0x == 0.5f && p.c0y == 0.5f && p.c0z == -0.25f && p.c0w == -0.25f)) return -1;
  constexpr int NW = 4, CY = 2 * NW;
  const int k_first = -1, k_last = cell_of(ow - 1, 0.5f, -0.25f);
  const int m_first = cell_of(y0, 0.5f, -0.25f), m_last = cell_of(y1 - 1, 0.5f, -0.25f);
  const int tiles_x = (k_last - k_first + 1 + kQCX - 1) / kQCX;
  const int n_tiles = tiles_x * ((m_last - m_first + 1 + CY - 1) / CY);
  const int grid = n_tiles < max_ctas ? n_tiles : max_ctas;
  const CUtensorMap tmap{(const unsigned char*)in, iw, ih, in_pitch, kQBW, CY + 3, 8};
  run_ctas(grid, NW * 32, [&]() { easu_h_quad2x_kernel<NW, 7, true>(p, tmap, tiles_x, n_tiles, m_first); });
  return 0;
}

// easu_h_pairs_kernel<true>: launch_easu_h_tiled's any-scale branch.  Arguments as emu_easu_h_pairs (without the variant).
extern "C" int emu_easu_h_pairs_srtm_in(const void* in, int iw, int ih, long long in_pitch, void* out, int ow, int oh, long long out_pitch,
                                        const uint32_t* con, int y0, int y1, int max_ctas) {
  const EasuParams p = easu_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, con, y0, y1);
  if (!(p.c0x > 0.0f && p.c0x <= 1.0f && p.c0y > 0.0f && p.c0y <= 1.0f)) return -1;
  int BW = max_footprint(ow, 0, kTileW, p.c0x, p.c0z, true);
  const int BH = max_footprint(y1, y0, kTileH, p.c0y, p.c0w, false);
  BW = (BW + 1) & ~1;
  if (BW > 256 || BH > 256 || pairs_smem_bytes(BW, BH) > sizeof g_dynamic_smem) return -1;
  const int tiles_x = (ow + kTileW - 1) / kTileW, n_tiles = tiles_x * ((y1 - y0 + kTileH - 1) / kTileH);
  const int grid = n_tiles < max_ctas ? n_tiles : max_ctas;
  const CUtensorMap tmap{(const unsigned char*)in, iw, ih, in_pitch, BW, BH, 8};
  run_ctas(grid, kThreads, [&]() { easu_h_pairs_kernel<true>(p, tmap, BW, BH, tiles_x, n_tiles); });
  return 0;
}

static FusedParams fused_params(const void* in, int iw, int ih, long long in_pitch, void* out, int ow, int oh, long long out_pitch,
                                const uint32_t* rcon, int y0, int y1) {
  FusedParams p;
  p.in = ImgView{(unsigned char*)in, in_pitch, iw, ih, 0, ih};
  p.out = ImgView{(unsigned char*)out, out_pitch, ow, oh, 0, oh};
  p.y0 = y0; p.y1 = y1; p.sharp_h2 = rcon[1];
  p.n_strips = ((ow + 1) / 2 + kStripCells - 1) / kStripCells;
  return p;
}

// fused_h_quad2x_kernel<4, 7, true>: launch_fused_h with `ctas` CTAs.  Arguments as emu_fused_h.
extern "C" int emu_fused_h_srtm_in(const void* in, int iw, int ih, long long in_pitch, void* out, int ow, int oh, long long out_pitch,
                                   const uint32_t* rcon, int y0, int y1, int ctas) {
  constexpr int NW = 4;
  const FusedParams p = fused_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, rcon, y0, y1);
  const CUtensorMap tmap{(const unsigned char*)in, iw, ih, in_pitch, kFBW, FusedCfg<NW>::kBH, 8};
  run_ctas(ctas, NW * 32, [&]() { fused_h_quad2x_kernel<NW, 7, true>(p, tmap); });
  return 0;
}

// fused_h_quad2x_post_kernel<4, 6, SO, true>: launch_fused_h_post with `ctas` CTAs.  Arguments as emu_fused_h_post.
extern "C" int emu_fused_h_post_srtm_in(const void* in, int iw, int ih, long long in_pitch, void* out, int ow, int oh, long long out_pitch,
                                        int out_format, const uint32_t* rcon, int y0, int y1, int ctas, const EmuPost* post) {
  constexpr int NW = 4;
  if (out_format != 1 && out_format != 3 && out_format != 4) return -1;
  const FusedParams p = fused_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, rcon, y0, y1);
  const PostParams q = post_params(*post);
  const CUtensorMap tmap{(const unsigned char*)in, iw, ih, in_pitch, kFBW, FusedCfg<NW>::kBH, 8};
  run_ctas(ctas, NW * 32, [&]() {
    if (out_format == 1) fused_h_quad2x_post_kernel<NW, 6, __half, true>(p, tmap, q);
    else if (out_format == 3) fused_h_quad2x_post_kernel<NW, 6, Unorm8, true>(p, tmap, q);
    else fused_h_quad2x_post_kernel<NW, 6, Unorm10, true>(p, tmap, q);
  });
  return 0;
}
