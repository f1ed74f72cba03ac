// TEST INFRASTRUCTURE — runs the surface twins of the RGBA16F production kernels (FSR1_FLAG_IN_SURFACE / FSR1_FLAG_OUT_SURFACE:
// easu_h_quad2x_surf_in_kernel and easu_h_pairs_kernel<kSrtmIn, false, true> in csrc/fsr1_easu_tiled.cu, fused_h_quad2x_surf_kernel and
// fused_h_quad2x_post_surf_kernel in csrc/fsr1_fused.cu, rcas_surf_out_kernel in csrc/fsr1_rcas_packed.cu) and their linear twins on CPU
// threads.  A library of its own (surf.mk), built on emu_srtm_in.cpp (and through it emu_post.cpp): the .cu files compiled AS IS with
// -DFSR1_CPU_EMU.  Surfaces are entries of the handle table of include/fsr1_emu_surf.h over caller memory (emu_surface); each runner
// takes the linear kernel or its surface twin by the surf_in / surf_out arguments, with the launchers' geometry.
#include "emu_srtm_in.cpp"

// an emulated 2D CUDA array of w x h elements of `elem` bytes over `base` (row pitch in bytes): its handle (1 + the table slot)
extern "C" unsigned long long emu_surface(int slot, void* base, long long pitch, int w, int h, int elem) {
  if (slot < 0 || slot >= 64) return 0;
  emu_surf_table()[slot] = EmuSurf{(unsigned char*)base, pitch, w, h, elem};
  return (unsigned long long)slot + 1;
}

// an input or output image: the linear image at `p` (pitch bytes), or with `surf` the surface object whose handle is `p`
static ImgView view(const void* p, long long pitch, int w, int h, bool surf) {
  return surf ? ImgView{(unsigned char*)p, 0, w, h, 0, h} : ImgView{(unsigned char*)p, pitch, w, h, 0, h};
}

// fsr1_easu at 2x: easu_h_quad2x_kernel<4, 7, srtm> or easu_h_quad2x_surf_in_kernel<4, 7, srtm>
extern "C" int emu_easu_quad2x_surf(const void* in, long long in_pitch, int iw, int ih, void* out, int ow, int oh, long long out_pitch,
                                    const uint32_t* con, int y0, int y1, int max_ctas, int srtm, int surf_in) {
  EasuParams p = easu_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, con, y0, y1);
  p.in = view(in, in_pitch, iw, ih, surf_in);
  if (!(p.c0x == 0.5f && p.c0y == 0.5f && p.c0z == -0.25f && p.c0w == -0.25f)) return -1;
  constexpr int NW = 4, CY = 2 * NW;
  const int k_first = -1, k_last = cell_of(ow - 1, 0.5f, -0.25f);
  const int m_first = cell_of(y0, 0.5f, -0.25f), m_last = cell_of(y1 - 1, 0.5f, -0.25f);
  const int tiles_x = (k_last - k_first + 1 + kQCX - 1) / kQCX;
  const int n_tiles = tiles_x * ((m_last - m_first + 1 + CY - 1) / CY);
  const int grid = n_tiles < max_ctas ? n_tiles : max_ctas;
  const CUtensorMap tmap{surf_in ? nullptr : (const unsigned char*)in, iw, ih, in_pitch, kQBW, CY + 3, 8};
  run_ctas(grid, NW * 32, [&]() {
    if (surf_in && srtm) easu_h_quad2x_surf_in_kernel<NW, 7, true>(p, tmap, tiles_x, n_tiles, m_first);
    else if (surf_in) easu_h_quad2x_surf_in_kernel<NW, 7, false>(p, tmap, tiles_x, n_tiles, m_first);
    else if (srtm) easu_h_quad2x_kernel<NW, 7, true>(p, tmap, tiles_x, n_tiles, m_first);
    else easu_h_quad2x_kernel<NW, 7, false>(p, tmap, tiles_x, n_tiles, m_first);
  });
  return 0;
}

// fsr1_easu at any other upscale: easu_h_pairs_kernel<srtm, false, surf_in>
extern "C" int emu_easu_pairs_surf(const void* in, long long in_pitch, int iw, int ih, void* out, int ow, int oh, long long out_pitch,
                                   const uint32_t* con, int y0, int y1, int max_ctas, int srtm, int surf_in) {
  EasuParams p = easu_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, con, y0, y1);
  p.in = view(in, in_pitch, iw, ih, surf_in);
  if (!(p.c0x > 0.0f && p.c0x <= 1.0f && p.c0y > 0.0f && p.c0y <= 1.0f)) return -1;
  int BW = max_footprint(ow, 0, kTileW, p.c0x, p.c0z, true);
  const int BH = max_footprint(y1, y0, kTileH, p.c0y, p.c0w, false);
  BW = (BW + 1) & ~1;
  if (BW > 256 || BH > 256 || pairs_smem_bytes(BW, BH) > sizeof g_dynamic_smem) return -1;
  const int tiles_x = (ow + kTileW - 1) / kTileW, n_tiles = tiles_x * ((y1 - y0 + kTileH - 1) / kTileH);
  const int grid = n_tiles < max_ctas ? n_tiles : max_ctas;
  const CUtensorMap tmap{surf_in ? nullptr : (const unsigned char*)in, iw, ih, in_pitch, BW, BH, 8};
  run_ctas(grid, kThreads, [&]() {
    if (surf_in && srtm) easu_h_pairs_kernel<true, false, true>(p, tmap, BW, BH, tiles_x, n_tiles);
    else if (surf_in) easu_h_pairs_kernel<false, false, true>(p, tmap, BW, BH, tiles_x, n_tiles);
    else if (srtm) easu_h_pairs_kernel<true>(p, tmap, BW, BH, tiles_x, n_tiles);
    else easu_h_pairs_kernel<false>(p, tmap, BW, BH, tiles_x, n_tiles);
  });
  return 0;
}

template <typename SO, bool kSrtm, bool kIn, bool kOut>
static void fused_one(const FusedParams& p, const CUtensorMap& tmap, const PostParams* q) {
  if constexpr (std::is_void<SO>::value) {
    if constexpr (kIn || kOut) fused_h_quad2x_surf_kernel<4, 7, kSrtm, kIn, kOut>(p, tmap);
    else fused_h_quad2x_kernel<4, 7, kSrtm>(p, tmap);
  } else {
    if constexpr (kIn || kOut) fused_h_quad2x_post_surf_kernel<4, 6, SO, kSrtm, kIn, kOut>(p, tmap, *q);
    else fused_h_quad2x_post_kernel<4, 6, SO, kSrtm>(p, tmap, *q);
  }
}
template <typename SO, bool kSrtm>
static void fused_flags(const FusedParams& p, const CUtensorMap& tmap, const PostParams* q, int surf_in, int surf_out) {
  if (surf_in && surf_out) fused_one<SO, kSrtm, true, true>(p, tmap, q);
  else if (surf_in) fused_one<SO, kSrtm, true, false>(p, tmap, q);
  else if (surf_out) fused_one<SO, kSrtm, false, true>(p, tmap, q);
  else fused_one<SO, kSrtm, false, false>(p, tmap, q);
}
template <typename SO>
static void fused_any(const FusedParams& p, const CUtensorMap& tmap, const PostParams* q, int srtm, int surf_in, int surf_out) {
  if (srtm) fused_flags<SO, true>(p, tmap, q, surf_in, surf_out);
  else fused_flags<SO, false>(p, tmap, q, surf_in, surf_out);
}

// fsr1_upscale / fsr1_upscale_post on the fused kernel with `ctas` CTAs: post == null the plain kernel (RGBA16F out), else the post
// kernel into out_format (1 RGBA16F, 3 RGBA8, 4 RGB10A2)
extern "C" int emu_fused_surf(const void* in, long long in_pitch, int iw, int ih, void* out, long long out_pitch, int ow, int oh,
                              int out_format, const uint32_t* rcon, int y0, int y1, int ctas, const EmuPost* post, int srtm, int surf_in,
                              int surf_out) {
  constexpr int NW = 4;
  FusedParams p = fused_params(in, iw, ih, in_pitch, out, ow, oh, out_pitch, rcon, y0, y1);
  p.in = view(in, in_pitch, iw, ih, surf_in);
  p.out = view(out, out_pitch, ow, oh, surf_out);
  PostParams q;
  if (post) q = post_params(*post);
  const CUtensorMap tmap{surf_in ? nullptr : (const unsigned char*)in, iw, ih, in_pitch, kFBW, FusedCfg<NW>::kBH, 8};
  if (!post && out_format != 1) return -1;
  run_ctas(ctas, NW * 32, [&]() {
    if (!post) fused_any<void>(p, tmap, nullptr, srtm, surf_in, surf_out);
    else if (out_format == 1) fused_any<__half>(p, tmap, &q, srtm, surf_in, surf_out);
    else if (out_format == 3) fused_any<Unorm8>(p, tmap, &q, srtm, surf_in, surf_out);
    else fused_any<Unorm10>(p, tmap, &q, srtm, surf_in, surf_out);
  });
  return 0;
}

template <bool kClamp, int kOpt, typename SO>
static void rcas_one(const RcasParams& p, const PostParams& q, bool surf_out) {
  if (surf_out) rcas_surf_out_kernel<kClamp, kOpt, SO>(p, q);
  else if constexpr (std::is_void<SO>::value) rcas_packed_kernel<FmtHalf, kClamp, kOpt>(p);
  else rcas_post_kernel<kClamp, kOpt, SO>(p, q);
}
template <bool kClamp, typename SO> static void rcas_opt(const RcasParams& p, const PostParams& q, int opts, bool surf_out) {
  switch (opts & 7) {
    case 0: rcas_one<kClamp, 0, SO>(p, q, surf_out); break;
    case 1: rcas_one<kClamp, 1, SO>(p, q, surf_out); break;
    case 2: rcas_one<kClamp, 2, SO>(p, q, surf_out); break;
    case 3: rcas_one<kClamp, 3, SO>(p, q, surf_out); break;
    case 4: rcas_one<kClamp, 4, SO>(p, q, surf_out); break;
    case 5: rcas_one<kClamp, 5, SO>(p, q, surf_out); break;
    case 6: rcas_one<kClamp, 6, SO>(p, q, surf_out); break;
    default: rcas_one<kClamp, 7, SO>(p, q, surf_out); break;
  }
}
template <typename SO> static void rcas_any(const RcasParams& p, const PostParams& q, int opts, bool surf_out) {
  if (p.clamp) rcas_opt<true, SO>(p, q, opts, surf_out);
  else rcas_opt<false, SO>(p, q, opts, surf_out);
}

// fsr1_rcas (post == null, RGBA16F out) or the RCAS kernel of fsr1_upscale_post (out_format as emu_fused_surf) over rows [y0, y1) of an
// RGBA16F image; opts: bit 0 denoise, 1 passthrough alpha, 2 output square
extern "C" int emu_rcas_surf(const void* in, long long in_pitch, void* out, long long out_pitch, int w, int h, int out_format,
                             const uint32_t* con, int clamp, int y0, int y1, int opts, const EmuPost* post, int surf_out) {
  if (!post && out_format != 1) return -1;
  RcasParams p;
  p.in = ImgView{(unsigned char*)in, in_pitch, w, h, 0, h};
  p.out = view(out, out_pitch, w, h, surf_out);
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
          if (!post) rcas_any<void>(p, q, opts, surf_out);
          else if (out_format == 1) rcas_any<__half>(p, q, opts, surf_out);
          else if (out_format == 3) rcas_any<Unorm8>(p, q, opts, surf_out);
          else rcas_any<Unorm10>(p, q, opts, surf_out);
        });
      for (auto& th : ts) th.join();
      for (int i = 0; i < NWARP; i++) pthread_barrier_destroy(&g_warp_barrier[i]);
    }
  return 0;
}
