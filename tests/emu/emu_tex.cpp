// TEST INFRASTRUCTURE — runs the texture twins of the RGBA16F production kernels and of their R11G11B10_FLOAT variants
// (FSR1_FLAG_IN_TEXTURE: easu_h_quad2x_tex_in_kernel and easu_h_pairs_kernel<kSrtmIn, kR11, kInTex> in csrc/fsr1_easu_tiled.cu,
// fused_h_quad2x_tex_kernel and fused_h_quad2x_post_tex_kernel in csrc/fsr1_fused.cu) and their linear twins on CPU threads.  A library
// of its own (tex.mk), built on emu_srtm_in.cpp (and through it emu_post.cpp): the .cu files compiled AS IS with -DFSR1_CPU_EMU.  Textures
// are entries of the handle table of include/fsr1_emu_tex.h over caller memory (emu_texture), output surfaces entries of the table of
// include/fsr1_emu_surf.h (emu_tex_surface); each runner takes the linear kernel or its texture twin by the `tex` argument, with the
// launchers' geometry.  r11: the input holds R11G11B10F codes (4 bytes per texel), else RGBA16F texels.
#include "emu_srtm_in.cpp"

// an emulated 2D CUDA array of w x h elements of `elem` bytes over `base` (row pitch in bytes), read through a texture: its handle
extern "C" unsigned long long emu_texture(int slot, const void* base, long long pitch, int w, int h, int elem) {
  if (slot < 0 || slot >= 64) return 0;
  emu_tex_table()[slot] = EmuTex{(const unsigned char*)base, pitch, w, h, elem};
  return (unsigned long long)slot + 1;
}
// the same for a surface the fused kernels store into (FSR1_FLAG_OUT_SURFACE)
extern "C" unsigned long long emu_tex_surface(int slot, void* base, long long pitch, int w, int h, int elem) {
  if (slot < 0 || slot >= 64) return 0;
  emu_surf_table()[slot] = EmuSurf{(unsigned char*)base, pitch, w, h, elem};
  return (unsigned long long)slot + 1;
}
// texture fetches outside an array or of the wrong element size since the library was loaded (the kernels must make none)
extern "C" long long emu_tex_faults() { return emu_tex_fault_count().load(); }

// an input or output image: the linear image at `p` (pitch bytes), or with `handle` the array object whose handle is `p`
static ImgView view(const void* p, long long pitch, int w, int h, bool handle) {
  return handle ? ImgView{(unsigned char*)p, 0, w, h, 0, h} : ImgView{(unsigned char*)p, pitch, w, h, 0, h};
}

// fsr1_easu at 2x: easu_h_quad2x_tex_in_kernel<4, 7, srtm, r11>, or the linear easu_h_quad2x_kernel / easu_r11_quad2x_kernel
extern "C" int emu_easu_quad2x_tex(const void* in, long long in_pitch, int iw, int ih, void* out, int ow, int oh, long long out_pitch,
                                   const uint32_t* con, int y0, int y1, int max_ctas, int srtm, int r11, int tex) {
  EasuParams p = easu_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, con, y0, y1);
  p.in = view(in, in_pitch, iw, ih, tex);
  if (!(p.c0x == 0.5f && p.c0y == 0.5f && p.c0z == -0.25f && p.c0w == -0.25f)) return -1;
  constexpr int NW = 4, CY = 2 * NW;
  const int k_first = -1, k_last = cell_of(ow - 1, 0.5f, -0.25f);
  const int m_first = cell_of(y0, 0.5f, -0.25f), m_last = cell_of(y1 - 1, 0.5f, -0.25f);
  const int tiles_x = (k_last - k_first + 1 + kQCX - 1) / kQCX;
  const int n_tiles = tiles_x * ((m_last - m_first + 1 + CY - 1) / CY);
  const int grid = n_tiles < max_ctas ? n_tiles : max_ctas;
  const CUtensorMap tmap{tex ? nullptr : (const unsigned char*)in, iw, ih, in_pitch, r11 ? kUBW : kQBW, CY + 3, r11 ? 4 : 8};
  run_ctas(grid, NW * 32, [&]() {
    const int v = (tex ? 4 : 0) | (r11 ? 2 : 0) | (srtm ? 1 : 0);
    switch (v) {
      case 0: easu_h_quad2x_kernel<NW, 7, false>(p, tmap, tiles_x, n_tiles, m_first); break;
      case 1: easu_h_quad2x_kernel<NW, 7, true>(p, tmap, tiles_x, n_tiles, m_first); break;
      case 2: easu_r11_quad2x_kernel<NW, 7, false>(p, tmap, tiles_x, n_tiles, m_first); break;
      case 3: easu_r11_quad2x_kernel<NW, 7, true>(p, tmap, tiles_x, n_tiles, m_first); break;
      case 4: easu_h_quad2x_tex_in_kernel<NW, 7, false, false>(p, tmap, tiles_x, n_tiles, m_first); break;
      case 5: easu_h_quad2x_tex_in_kernel<NW, 7, true, false>(p, tmap, tiles_x, n_tiles, m_first); break;
      case 6: easu_h_quad2x_tex_in_kernel<NW, 7, false, true>(p, tmap, tiles_x, n_tiles, m_first); break;
      default: easu_h_quad2x_tex_in_kernel<NW, 7, true, true>(p, tmap, tiles_x, n_tiles, m_first); break;
    }
  });
  return 0;
}

// fsr1_easu at any other upscale: easu_h_pairs_kernel<srtm, r11, kInTex>, or the linear easu_h_pairs_kernel<srtm, r11>
extern "C" int emu_easu_pairs_tex(const void* in, long long in_pitch, int iw, int ih, void* out, int ow, int oh, long long out_pitch,
                                  const uint32_t* con, int y0, int y1, int max_ctas, int srtm, int r11, int tex) {
  EasuParams p = easu_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, con, y0, y1);
  p.in = view(in, in_pitch, iw, ih, tex);
  if (!(p.c0x > 0.0f && p.c0x <= 1.0f && p.c0y > 0.0f && p.c0y <= 1.0f)) return -1;
  int BW = max_footprint(ow, 0, kTileW, p.c0x, p.c0z, true);
  const int BH = max_footprint(y1, y0, kTileH, p.c0y, p.c0w, false);
  BW = (BW + 1) & ~1;
  if (BW > 256 || BH > 256 || pairs_smem_bytes(BW, BH) > sizeof g_dynamic_smem) return -1;
  if (r11 && BW * BH > kR11Per * kThreads) return -1;
  const int tiles_x = (ow + kTileW - 1) / kTileW, n_tiles = tiles_x * ((y1 - y0 + kTileH - 1) / kTileH);
  const int grid = n_tiles < max_ctas ? n_tiles : max_ctas;
  const CUtensorMap tmap{tex ? nullptr : (const unsigned char*)in, iw, ih, in_pitch, r11 ? (BW + 5) & ~3 : BW, BH, r11 ? 4 : 8};
  run_ctas(grid, kThreads, [&]() {
    const int v = (tex ? 4 : 0) | (r11 ? 2 : 0) | (srtm ? 1 : 0);
    switch (v) {
      case 0: easu_h_pairs_kernel<false, false>(p, tmap, BW, BH, tiles_x, n_tiles); break;
      case 1: easu_h_pairs_kernel<true, false>(p, tmap, BW, BH, tiles_x, n_tiles); break;
      case 2: easu_h_pairs_kernel<false, true>(p, tmap, BW, BH, tiles_x, n_tiles); break;
      case 3: easu_h_pairs_kernel<true, true>(p, tmap, BW, BH, tiles_x, n_tiles); break;
      case 4: easu_h_pairs_kernel<false, false, kInTex>(p, tmap, BW, BH, tiles_x, n_tiles); break;
      case 5: easu_h_pairs_kernel<true, false, kInTex>(p, tmap, BW, BH, tiles_x, n_tiles); break;
      case 6: easu_h_pairs_kernel<false, true, kInTex>(p, tmap, BW, BH, tiles_x, n_tiles); break;
      default: easu_h_pairs_kernel<true, true, kInTex>(p, tmap, BW, BH, tiles_x, n_tiles); break;
    }
  });
  return 0;
}

// the fused kernel for (SO, srtm, r11): its texture twin (storing through a surface with kOut), or the linear kernel
template <typename SO, bool kSrtm, bool kR11>
static void fused_one(const FusedParams& p, const CUtensorMap& tmap, const PostParams* q, int tex, int surf_out) {
  if constexpr (std::is_void<SO>::value) {
    if (tex && surf_out) fused_h_quad2x_tex_kernel<4, 7, kSrtm, kR11, true>(p, tmap);
    else if (tex) fused_h_quad2x_tex_kernel<4, 7, kSrtm, kR11, false>(p, tmap);
    else if constexpr (kR11) fused_r11_quad2x_kernel<4, 7, kSrtm>(p, tmap);
    else fused_h_quad2x_kernel<4, 7, kSrtm>(p, tmap);
  } else {
    if (tex && surf_out) fused_h_quad2x_post_tex_kernel<4, 6, SO, kSrtm, kR11, true>(p, tmap, *q);
    else if (tex) fused_h_quad2x_post_tex_kernel<4, 6, SO, kSrtm, kR11, false>(p, tmap, *q);
    else if constexpr (kR11) fused_r11_quad2x_post_kernel<4, 6, SO, kSrtm>(p, tmap, *q);
    else fused_h_quad2x_post_kernel<4, 6, SO, kSrtm>(p, tmap, *q);
  }
}
template <typename SO>
static void fused_any(const FusedParams& p, const CUtensorMap& tmap, const PostParams* q, int srtm, int r11, int tex, int surf_out) {
  if (srtm && r11) fused_one<SO, true, true>(p, tmap, q, tex, surf_out);
  else if (srtm) fused_one<SO, true, false>(p, tmap, q, tex, surf_out);
  else if (r11) fused_one<SO, false, true>(p, tmap, q, tex, surf_out);
  else fused_one<SO, false, false>(p, tmap, q, tex, surf_out);
}

// fsr1_upscale / fsr1_upscale_post on the fused kernel with `ctas` CTAs: post == null the plain kernel (RGBA16F out), else the post
// kernel into out_format (1 RGBA16F, 3 RGBA8, 4 RGB10A2).  surf_out (texture input only): `out` is a surface handle.
extern "C" int emu_fused_tex(const void* in, long long in_pitch, int iw, int ih, void* out, long long out_pitch, int ow, int oh,
                             int out_format, const uint32_t* rcon, int y0, int y1, int ctas, const EmuPost* post, int srtm, int r11, int tex,
                             int surf_out) {
  constexpr int NW = 4;
  if ((!post && out_format != 1) || (surf_out && !tex)) return -1;
  FusedParams p = fused_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, rcon, y0, y1);
  p.in = view(in, in_pitch, iw, ih, tex);
  p.out = view(out, out_pitch, ow, oh, surf_out);
  PostParams q;
  if (post) q = post_params(*post);
  const CUtensorMap tmap{tex ? nullptr : (const unsigned char*)in, iw, ih, in_pitch, r11 ? kRBW : kFBW, FusedCfg<NW>::kBH, r11 ? 4 : 8};
  run_ctas(ctas, NW * 32, [&]() {
    if (!post) fused_any<void>(p, tmap, nullptr, srtm, r11, tex, surf_out);
    else if (out_format == 1) fused_any<__half>(p, tmap, &q, srtm, r11, tex, surf_out);
    else if (out_format == 3) fused_any<Unorm8>(p, tmap, &q, srtm, r11, tex, surf_out);
    else fused_any<Unorm10>(p, tmap, &q, srtm, r11, tex, surf_out);
  });
  return 0;
}
