// TEST INFRASTRUCTURE — host emulation of the texture wrappers of csrc/fsr1_common.cuh (tex2D in element mode with point filtering at
// unnormalized coordinates, used by FSR1_FLAG_IN_TEXTURE).  A handle is 1 + an index into a table of emulated 2D CUDA arrays over caller
// memory (tests/emu/emu_tex.cpp fills it).  The kernels clamp every fetch to the logical image, so a fetch outside the array, or of an
// element of the wrong size, is a kernel bug: it is counted (emu_tex_faults) and reads the clamped element, as a clamp-mode texture would.
#pragma once
#include "cuda_emu.h"

#include <atomic>

namespace fsr1 {

struct EmuTex {
  const unsigned char* base;
  long long pitch;  // bytes
  int w, h;         // extent in elements
  int elem;         // bytes per element: 8 (16,16,16,16) or 4 (32)
};
inline EmuTex* emu_tex_table() {
  static EmuTex table[64];
  return table;
}
inline std::atomic<long long>& emu_tex_fault_count() {
  static std::atomic<long long> n{0};
  return n;
}
inline const unsigned char* emu_tex_at(unsigned long long t, int x, int y, int bytes) {
  const EmuTex& a = emu_tex_table()[t - 1];
  if (bytes != a.elem || x < 0 || x >= a.w || y < 0 || y >= a.h) emu_tex_fault_count()++;
  x = x < 0 ? 0 : (x >= a.w ? a.w - 1 : x);
  y = y < 0 ? 0 : (y >= a.h ? a.h - 1 : y);
  return a.base + (long long)y * a.pitch + (long long)x * a.elem;
}
inline uint2 tex_load8(unsigned long long t, int x, int y) {
  uint2 v;
  memcpy(&v, emu_tex_at(t, x, y, 8), 8);
  return v;
}
inline uint32_t tex_load4(unsigned long long t, int x, int y) {
  uint32_t v;
  memcpy(&v, emu_tex_at(t, x, y, 4), 4);
  return v;
}

}  // namespace fsr1
