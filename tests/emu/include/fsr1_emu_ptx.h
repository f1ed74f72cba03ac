// TEST INFRASTRUCTURE — host emulation of the PTX wrappers of csrc/fsr1_easu_common.cuh (mbarrier + TMA + rcp.approx).
#pragma once
#include <sched.h>
#include "cuda_emu.h"

namespace fsr1 {

inline uint32_t smem_u32(const void* p) { return (uint32_t)reinterpret_cast<uintptr_t>(p); }  // only its low bits are used

// mbarrier: the 64-bit word counts completed phases; try_wait.parity(p) succeeds once the phase of parity p is complete
inline std::atomic<uint64_t>* emu_bar(uint64_t* bar) { return reinterpret_cast<std::atomic<uint64_t>*>(bar); }
inline void mbar_init(uint64_t* bar, uint32_t) { emu_bar(bar)->store(0); }
inline void mbar_fence_init() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline void fence_proxy_async() { std::atomic_thread_fence(std::memory_order_seq_cst); }
inline void mbar_expect_tx(uint64_t*, uint32_t) {}
inline void mbar_wait(uint64_t* bar, uint32_t phase) {
  while ((emu_bar(bar)->load(std::memory_order_acquire) & 1u) == phase) sched_yield();
}
// cp.async.bulk.tensor.2d: copy the box whose origin is element (x, y); out-of-tensor elements arrive as zeros
inline void tma_load_2d(void* dst, const CUtensorMap* map, int x, int y, uint64_t* bar) {
  unsigned char* d = static_cast<unsigned char*>(dst);
  const int eb = map->elem_bytes;
  for (int j = 0; j < map->box_h; j++)
    for (int i = 0; i < map->box_w; i++) {
      const int gx = x + i, gy = y + j;
      unsigned char* o = d + ((size_t)j * map->box_w + i) * eb;
      if (gx >= 0 && gx < map->w && gy >= 0 && gy < map->rows) memcpy(o, map->base + (long long)gy * map->pitch + (long long)gx * eb, eb);
      else memset(o, 0, eb);
    }
  emu_bar(bar)->fetch_add(1, std::memory_order_release);
}
inline void mbar_arrive(uint64_t* bar) { emu_bar(bar)->fetch_add(1, std::memory_order_release); }
// MUFU.RCP is within 1 ulp of this, and that does not change a result: every caller passes a half and rounds the reciprocal to
// half at once, and for every half x, 1/x lies at least 2 fp32 ulps from every half rounding boundary (tests/test_kernel_model.py)
inline float rcp_approx(float a) { return 1.0f / a; }
// min.s16x2
inline uint32_t emu_min_s16x2(uint32_t a, uint32_t b) {
  const int16_t al = (int16_t)(a & 0xffff), ah = (int16_t)(a >> 16), bl = (int16_t)(b & 0xffff), bh = (int16_t)(b >> 16);
  return (uint32_t)(uint16_t)std::min(al, bl) | ((uint32_t)(uint16_t)std::min(ah, bh) << 16);
}

}  // namespace fsr1
