// TEST INFRASTRUCTURE — runs the R11G11B10_FLOAT-input variants of the RGBA16F EASU kernels (easu_r11_quad2x_kernel and
// easu_h_pairs_kernel<kSrtmIn, true> in csrc/fsr1_easu_tiled.cu, fused_r11_quad2x_kernel and fused_r11_quad2x_post_kernel in
// csrc/fsr1_fused.cu) on CPU threads.  A library of its own (r11.mk), built on emu_srtm_in.cpp (and through it emu_post.cpp): the .cu
// files compiled AS IS with -DFSR1_CPU_EMU; the runners re-create the launchers' geometry with the R11G11B10F boxes (4-byte texels).
#include "emu_srtm_in.cpp"

// easu_r11_quad2x_kernel<4, 7, srtm>: launch_easu_h_tiled's 2x branch with r11.  Arguments as emu_easu_h_quad2x_srtm_in, plus srtm.
extern "C" int emu_easu_r11_quad2x(const void* in, int iw, int ih, long long in_pitch, void* out, int ow, int oh, long long out_pitch,
                                   const uint32_t* con, int y0, int y1, int max_ctas, int srtm) {
  const EasuParams p = easu_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, con, y0, y1);
  if (!(p.c0x == 0.5f && p.c0y == 0.5f && p.c0z == -0.25f && p.c0w == -0.25f)) return -1;
  constexpr int NW = 4, CY = 2 * NW;
  const int k_first = -1, k_last = cell_of(ow - 1, 0.5f, -0.25f);
  const int m_first = cell_of(y0, 0.5f, -0.25f), m_last = cell_of(y1 - 1, 0.5f, -0.25f);
  const int tiles_x = (k_last - k_first + 1 + kQCX - 1) / kQCX;
  const int n_tiles = tiles_x * ((m_last - m_first + 1 + CY - 1) / CY);
  const int grid = n_tiles < max_ctas ? n_tiles : max_ctas;
  const CUtensorMap tmap{(const unsigned char*)in, iw, ih, in_pitch, kUBW, CY + 3, 4};
  run_ctas(grid, NW * 32, [&]() {
    if (srtm) easu_r11_quad2x_kernel<NW, 7, true>(p, tmap, tiles_x, n_tiles, m_first);
    else easu_r11_quad2x_kernel<NW, 7, false>(p, tmap, tiles_x, n_tiles, m_first);
  });
  return 0;
}

// easu_h_pairs_kernel<srtm, true>: launch_easu_h_tiled's any-scale branch with r11
extern "C" int emu_easu_r11_pairs(const void* in, int iw, int ih, long long in_pitch, void* out, int ow, int oh, long long out_pitch,
                                  const uint32_t* con, int y0, int y1, int max_ctas, int srtm) {
  const EasuParams p = easu_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, con, y0, y1);
  if (!(p.c0x > 0.0f && p.c0x <= 1.0f && p.c0y > 0.0f && p.c0y <= 1.0f)) return -1;
  int BW = max_footprint(ow, 0, kTileW, p.c0x, p.c0z, true);
  const int BH = max_footprint(y1, y0, kTileH, p.c0y, p.c0w, false);
  BW = (BW + 1) & ~1;
  if (BW > 256 || BH > 256 || BW * BH > kR11Per * kThreads || pairs_smem_bytes(BW, BH) > sizeof g_dynamic_smem) return -1;
  const int tiles_x = (ow + kTileW - 1) / kTileW, n_tiles = tiles_x * ((y1 - y0 + kTileH - 1) / kTileH);
  const int grid = n_tiles < max_ctas ? n_tiles : max_ctas;
  const CUtensorMap tmap{(const unsigned char*)in, iw, ih, in_pitch, (BW + 5) & ~3, BH, 4};
  run_ctas(grid, kThreads, [&]() {
    if (srtm) easu_h_pairs_kernel<true, true>(p, tmap, BW, BH, tiles_x, n_tiles);
    else easu_h_pairs_kernel<false, true>(p, tmap, BW, BH, tiles_x, n_tiles);
  });
  return 0;
}

// fused_r11_quad2x_kernel<4, 7, srtm>: launch_fused_h with r11 and `ctas` CTAs
extern "C" int emu_fused_r11(const void* in, int iw, int ih, long long in_pitch, void* out, int ow, int oh, long long out_pitch,
                             const uint32_t* rcon, int y0, int y1, int ctas, int srtm) {
  constexpr int NW = 4;
  const FusedParams p = fused_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, rcon, y0, y1);
  const CUtensorMap tmap{(const unsigned char*)in, iw, ih, in_pitch, kRBW, FusedCfg<NW>::kBH, 4};
  run_ctas(ctas, NW * 32, [&]() {
    if (srtm) fused_r11_quad2x_kernel<NW, 7, true>(p, tmap);
    else fused_r11_quad2x_kernel<NW, 7, false>(p, tmap);
  });
  return 0;
}

template <bool kSrtm> static void fused_r11_post(const FusedParams& p, const CUtensorMap& tmap, const PostParams& q, int out_format) {
  if (out_format == 1) fused_r11_quad2x_post_kernel<4, 6, __half, kSrtm>(p, tmap, q);
  else if (out_format == 3) fused_r11_quad2x_post_kernel<4, 6, Unorm8, kSrtm>(p, tmap, q);
  else fused_r11_quad2x_post_kernel<4, 6, Unorm10, kSrtm>(p, tmap, q);
}

// fused_r11_quad2x_post_kernel<4, 6, SO, srtm>: launch_fused_h_post with r11 and `ctas` CTAs
extern "C" int emu_fused_r11_post(const void* in, int iw, int ih, long long in_pitch, void* out, int ow, int oh, long long out_pitch,
                                  int out_format, const uint32_t* rcon, int y0, int y1, int ctas, const EmuPost* post, int srtm) {
  constexpr int NW = 4;
  if (out_format != 1 && out_format != 3 && out_format != 4) return -1;
  const FusedParams p = fused_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, rcon, y0, y1);
  const PostParams q = post_params(*post);
  const CUtensorMap tmap{(const unsigned char*)in, iw, ih, in_pitch, kRBW, FusedCfg<NW>::kBH, 4};
  run_ctas(ctas, NW * 32, [&]() {
    if (srtm) fused_r11_post<true>(p, tmap, q, out_format);
    else fused_r11_post<false>(p, tmap, q, out_format);
  });
  return 0;
}
