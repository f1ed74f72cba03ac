// fsr1_rcas_in.cu — the input-stage RCAS kernels of fsr1_rcas_post on sm_90a: the packed RCAS kernel of fsr1_rcas_packed.cu (its
// templates, included below) reading R11G11B10_FLOAT input and / or applying FsrSrtmF as it loads each texel.
// A translation unit of its own, so the module that holds the production RCAS kernels (fsr1_rcas_packed.cu) holds exactly those: loading
// it (on first use, or eagerly) costs what it did before these 128 kernels existed.
#include <stdio.h>

#ifndef FSR1_CPU_EMU  // tests/emu has included fsr1_rcas_packed.cu already
#define FSR1_RCAS_PACKED_TEMPLATES_ONLY
#include "fsr1_rcas_packed.cu"
#endif
#include "fsr1_post.cuh"

namespace fsr1 {

// ---- the input stage of fsr1_rcas_post: R11G11B10_FLOAT or RGBA16F input, with or without FSR1_FLAG_SRTM_INPUT -----------------------
// A lane's pair is fetched with the base format's loads (one 64-bit load of two R11G11B10F texels, as FmtUnorm's, or one 128-bit load
// of two RGBA16F texels) and turned into the RGBA16F texels FmtHalf::decode / FmtHalf::alpha take: r11_to_half on each R11G11B10F texel
// (exact, alpha 1.0), then with `srtm` srtm_texel on each texel, the bits fsr1_srtm writes.  `srtm` is a kernel argument (warp-uniform),
// so one kernel serves both, and so is RCAS_CLAMP (p.clamp, read by load_checked only).  An out-of-image pair (zero()) decodes to RGB 0
// either way: r11_to_half(0) and srtm_texel(0) are RGB 0.
template <bool kR11> struct InStage : std::conditional<kR11, FmtUnorm<8>, FmtHalf>::type {
  typedef typename std::conditional<kR11, FmtUnorm<8>, FmtHalf>::type::Raw Raw;
  static constexpr bool kClampArg = true;
  static __device__ __forceinline__ uint4 texels(Raw v, bool srtm) {
    uint2 t0, t1;
    if constexpr (kR11) {
      t0 = r11_to_half(v.x);
      t1 = r11_to_half(v.y);
    } else {
      t0 = make_uint2(v.x, v.y);
      t1 = make_uint2(v.z, v.w);
    }
    if (srtm) {
      t0 = srtm_texel(t0);
      t1 = srtm_texel(t1);
    }
    return make_uint4(t0.x, t0.y, t1.x, t1.y);
  }
};

// fsr1_rcas_post from R11G11B10F input (kR11) or with SRTM (srtm != 0), through InStage: rcas_packed_kernel, rcas_post_kernel and
// rcas_surf_out_kernel of fsr1_rcas_packed.cu with an input stage.
// SO = void: the RGBA16F store of RCAS itself; kSurfOut: p.out is a surface object.  RCAS_CLAMP: p.clamp (InStage::kClampArg).
// At most 96 registers instead of __launch_bounds__: srtm_texel's IEEE division calls its slow path, and at the 48-56 registers ptxas
// picks under the launch bound the registers live across that call spill (4-24 B).  Under 96 none spills (54-94 registers).
#ifdef FSR1_CPU_EMU
#define FSR1_RCAS_IN_REGS
#else
#define FSR1_RCAS_IN_REGS __maxnreg__(96)
#endif
template <bool kR11, int kOpt, typename SO, bool kSurfOut>
__global__ void FSR1_RCAS_IN_REGS rcas_in_kernel(const RcasParams p, const __grid_constant__ PostParams q, const int srtm) {
  constexpr bool kPost = !std::is_void<SO>::value;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int x0 = blockIdx.x * kSpan - 2;
  const int x = x0 + lane * 2;
  const int ys = p.y0 + (blockIdx.y * kNW + warp) * kRows;
  if (ys >= p.y1) return;  // whole warp
  const bool interior = x0 >= 0 && x0 + 64 <= p.in.w && ys >= 1 && ys + kRows < p.in.h && ys + kRows <= p.y1;
  if (interior)
    rcas_rows<FmtHalf, false, false, kOpt, SO, kSurfOut, InStage<kR11>>(p, x, ys, lane, kPost ? &q : nullptr, srtm != 0);
  else
    rcas_rows<FmtHalf, true, false, kOpt, SO, kSurfOut, InStage<kR11>>(p, x, ys, lane, kPost ? &q : nullptr, srtm != 0);
}

#ifndef FSR1_CPU_EMU  // tests/emu supplies its own launcher
template <bool kR11, typename SO, bool kSurfOut>
static void launch_in_opt(const RcasParams& p, const PostParams& q, int srtm, cudaStream_t s) {
  const dim3 grid((p.out.w + kSpan - 1) / kSpan, (p.y1 - p.y0 + kNW * kRows - 1) / (kNW * kRows), 1);
  switch (p.options & 7) {
    case 0: rcas_in_kernel<kR11, 0, SO, kSurfOut><<<grid, 32 * kNW, 0, s>>>(p, q, srtm); break;
    case 1: rcas_in_kernel<kR11, 1, SO, kSurfOut><<<grid, 32 * kNW, 0, s>>>(p, q, srtm); break;
    case 2: rcas_in_kernel<kR11, 2, SO, kSurfOut><<<grid, 32 * kNW, 0, s>>>(p, q, srtm); break;
    case 3: rcas_in_kernel<kR11, 3, SO, kSurfOut><<<grid, 32 * kNW, 0, s>>>(p, q, srtm); break;
    case 4: rcas_in_kernel<kR11, 4, SO, kSurfOut><<<grid, 32 * kNW, 0, s>>>(p, q, srtm); break;
    case 5: rcas_in_kernel<kR11, 5, SO, kSurfOut><<<grid, 32 * kNW, 0, s>>>(p, q, srtm); break;
    case 6: rcas_in_kernel<kR11, 6, SO, kSurfOut><<<grid, 32 * kNW, 0, s>>>(p, q, srtm); break;
    default: rcas_in_kernel<kR11, 7, SO, kSurfOut><<<grid, 32 * kNW, 0, s>>>(p, q, srtm); break;
  }
}
template <bool kR11, typename SO>
static void launch_in_store(const RcasParams& p, const PostParams& q, int srtm, bool surf_out, cudaStream_t s) {
  if (surf_out) launch_in_opt<kR11, SO, true>(p, q, srtm, s);
  else launch_in_opt<kR11, SO, false>(p, q, srtm, s);
}
template <bool kR11>
static void launch_in_out(const RcasParams& p, const PostParams* q, int out_format, int srtm, bool surf_out, cudaStream_t s) {
  if (!q) launch_in_store<kR11, void>(p, PostParams{}, srtm, surf_out, s);
  else if (out_format == 1) launch_in_store<kR11, __half>(p, *q, srtm, surf_out, s);
  else if (out_format == 3) launch_in_store<kR11, Unorm8>(p, *q, srtm, surf_out, s);
  else launch_in_store<kR11, Unorm10>(p, *q, srtm, surf_out, s);
}

// "rcas_h_packed[_post]<2px,4rows,shfl60[,r11g11b10f_in][,srtm_in][,rgba16f|rgba8|rgb10a2][,surf_out]>": [r11][srtm][store][surf_out]
static const char* in_kernel_name(bool r11, bool srtm, int store, bool surf_out) {
  static const struct Names {
    char s[2][2][4][2][96];
    Names() {
      static const char* const kStore[4] = {"", ",rgba16f", ",rgba8", ",rgb10a2"};
      for (int a = 0; a < 2; a++)
        for (int b = 0; b < 2; b++)
          for (int c = 0; c < 4; c++)
            for (int d = 0; d < 2; d++)
              snprintf(s[a][b][c][d], sizeof s[a][b][c][d], "rcas_h_packed%s<2px,4rows,shfl60%s%s%s%s>", c ? "_post" : "",
                       a ? ",r11g11b10f_in" : "", b ? ",srtm_in" : "", kStore[c], d ? ",surf_out" : "");
    }
  } names;
  return names.s[r11][srtm][store][surf_out];
}

cudaError_t launch_rcas_h_in(const RcasParams& p, const PostParams* q, int out_format, bool r11, bool srtm, cudaStream_t s, const char** name,
                             bool surf_out) {
  const int in_align = r11 ? 8 : 16, out_align = !q || out_format == 1 ? 16 : 8;
  if ((reinterpret_cast<uintptr_t>(p.in.base) & (in_align - 1)) || (p.in.pitch & (in_align - 1))) return cudaErrorNotSupported;
  if (!surf_out && ((reinterpret_cast<uintptr_t>(p.out.base) & (out_align - 1)) || (p.out.pitch & (out_align - 1))))
    return cudaErrorNotSupported;
  if (q && out_format != 1 && out_format != 3 && out_format != 4) return cudaErrorNotSupported;
  *name = in_kernel_name(r11, srtm, !q ? 0 : out_format == 1 ? 1 : out_format == 3 ? 2 : 3, surf_out);
  if (r11) launch_in_out<true>(p, q, out_format, srtm ? 1 : 0, surf_out, s);
  else launch_in_out<false>(p, q, out_format, srtm ? 1 : 0, surf_out, s);
  return cudaGetLastError();
}

#endif  // FSR1_CPU_EMU

}  // namespace fsr1
