// fsr1_r11.cuh — phase 1 of the TMA-tiled EASU kernels for R11G11B10_FLOAT input (FSR1_FORMAT_R11G11B10_FLOAT; fsr1_easu_tiled.cu,
// fsr1_fused.cu).
//
// The TMA box holds 4-byte texels.  It starts on a 16-byte boundary (a multiple of 4 texels, 0 or 2 texels left of the half tile's own
// origin) and is a multiple of 4 texels wide.  clamp_fixup runs on the packed texels.  Phase 1 then decodes each packed texel the
// step needs into the half tile the rest of the kernel reads: its exact RGBA16F texel (r11_to_half), through srtm_texel with kSrtmIn
// (the order of the RGBA16F kernels' prologue), and the luma of that half texel (texel_luma, so the bits match the RGBA16F kernels').
// Every later step is the RGBA16F kernel's, so each variant is bit-identical to its RGBA16F twin on the decoded image.
// Where the box lands:
//   - the 2x and fused kernels (static shared memory, 72 registers at 7 CTAs per SM): a double-buffered staging area of their own
//     (2 x 1792 bytes; 7 CTAs per SM still fit), as easu_u8_quad2x's; phase 1 reads it and needs no barrier of its own;
//   - the any-scale kernel (dynamic shared memory, whose size sets its CTAs per SM): the start of the half tile's own buffer (the
//     packed box is about half its size), expanded IN PLACE: every thread reads its packed texels into registers, a barrier, then it
//     writes them back expanded.
#pragma once
#include "fsr1_easu_quad.cuh"
#include "fsr1_post.cuh"

namespace fsr1 {

// the staging area: two boxes of kWords 4-byte texels, each 128-byte aligned (kWords a multiple of 32)
template <int kWords> struct __align__(128) R11Stage { uint32_t w[2][kWords]; };

template <bool kSrtmIn> __device__ __forceinline__ uint2 r11_texel(uint32_t v) {
  const uint2 c = r11_to_half(v);
  return kSrtmIn ? srtm_texel(c) : c;
}

// half texel i = j bw + c (i < n) from packed texel (j, c + shift) of `stage` (row pitch `ppitch` texels)
template <bool kSrtmIn, int NT>
__device__ __forceinline__ void r11_phase1_staged(const uint32_t* stage, uint2* tile, float* L, int n, int bw, int ppitch, int shift,
                                                  int tid) {
  for (int i = tid; i < n; i += NT) {
    const int j = i / bw;
    const uint2 c = r11_texel<kSrtmIn>(stage[j * ppitch + shift + (i - j * bw)]);
    tile[i] = c;
    L[i] = texel_luma(c);
  }
}

// The same with the packed box at the start of `tile` itself.  kPer >= ceil(n / NT): the packed texels a thread holds across the barrier.
template <bool kSrtmIn, int NT, int kPer>
__device__ __forceinline__ void r11_phase1_inplace(uint2* tile, float* L, int n, int bw, int ppitch, int shift, int tid) {
  const uint32_t* packed = reinterpret_cast<const uint32_t*>(tile);
  uint32_t v[kPer];
#pragma unroll
  for (int k = 0; k < kPer; k++) {
    const int i = tid + k * NT;
    if (i < n) {
      const int j = i / bw;
      v[k] = packed[j * ppitch + shift + (i - j * bw)];
    }
  }
  __syncthreads();  // every packed texel is in a register before an expanded one overwrites it
#pragma unroll
  for (int k = 0; k < kPer; k++) {
    const int i = tid + k * NT;
    if (i < n) {
      const uint2 c = r11_texel<kSrtmIn>(v[k]);
      tile[i] = c;
      L[i] = texel_luma(c);
    }
  }
}

}  // namespace fsr1
