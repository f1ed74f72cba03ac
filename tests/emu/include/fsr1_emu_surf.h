// TEST INFRASTRUCTURE — host emulation of the surface wrappers of csrc/fsr1_common.cuh (surf2Dread / surf2Dwrite in zero mode, used by
// FSR1_FLAG_IN_SURFACE / FSR1_FLAG_OUT_SURFACE).  A handle is 1 + an index into a table of emulated 2D CUDA arrays over caller memory
// (tests/emu/emu_surf.cpp fills it).  An element outside the array's extent reads 0; a store there is dropped.
#pragma once
#include "cuda_emu.h"

namespace fsr1 {

struct EmuSurf {
  unsigned char* base;
  long long pitch;  // bytes
  int w, h;         // extent in elements
  int elem;         // bytes per element
};
inline EmuSurf* emu_surf_table() {
  static EmuSurf table[64];
  return table;
}
inline unsigned char* emu_surf_at(unsigned long long s, int xb, int y, int bytes) {
  const EmuSurf& a = emu_surf_table()[s - 1];
  if (bytes != a.elem || xb < 0 || xb % bytes || xb / bytes >= a.w || y < 0 || y >= a.h) return nullptr;
  return a.base + (long long)y * a.pitch + xb;
}
inline unsigned long long surf_of(const ImgView& im) { return (unsigned long long)im.base; }
inline uint2 surf_load8(unsigned long long s, int x, int y) {
  uint2 v{0u, 0u};
  if (const unsigned char* p = emu_surf_at(s, x * 8, y, 8)) memcpy(&v, p, 8);
  return v;
}
inline void surf_store8(unsigned long long s, int x, int y, uint2 v) {
  if (unsigned char* p = emu_surf_at(s, x * 8, y, 8)) memcpy(p, &v, 8);
}
inline void surf_store4(unsigned long long s, int x, int y, uint32_t v) {
  if (unsigned char* p = emu_surf_at(s, x * 4, y, 4)) memcpy(p, &v, 4);
}

}  // namespace fsr1
