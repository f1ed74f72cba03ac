// TEST INFRASTRUCTURE — a minimal "CUDA on the host" shim so that the device code of csrc/*.cu can be compiled with
// g++ and run on CPU threads (tests/emu/).  It exists to debug kernels without spending GPU time: one OS thread per
// CUDA thread of a CTA, __syncthreads() = a barrier, CTAs run one after the other, TMA = a synchronous copy with zero
// fill that flips an emulated mbarrier.  Half arithmetic is emulated with one IEEE rounding per operation (what HFMA2,
// HMUL2, HADD2 do).  Not a product path: nothing under fidelityfx-fsr_b200/ uses it unless FSR1_CPU_EMU is defined.
#pragma once
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <atomic>

#define __device__
#define __host__
#define __global__
#define __forceinline__ inline
#define __restrict__
#define __grid_constant__
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) alignas(n)

struct uint3 { unsigned x, y, z; };
struct dim3 { unsigned x = 1, y = 1, z = 1; };
extern thread_local uint3 threadIdx, blockIdx;
extern thread_local dim3 gridDim, blockDim;
void __syncthreads();
inline void __syncwarp() {}

struct float2 { float x, y; };
struct float3 { float x, y, z; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) uint2 { uint32_t x, y; };
struct alignas(16) uint4 { uint32_t x, y, z, w; };
inline float2 make_float2(float a, float b) { return float2{a, b}; }
inline float3 make_float3(float a, float b, float c) { return float3{a, b, c}; }
inline float4 make_float4(float a, float b, float c, float d) { return float4{a, b, c, d}; }
inline uint2 make_uint2(uint32_t a, uint32_t b) { return uint2{a, b}; }
inline uint4 make_uint4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) { return uint4{a, b, c, d}; }

typedef struct CUstream_st* cudaStream_t;
typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorNotSupported = 801 };
inline cudaError_t cudaGetLastError() { return cudaSuccess; }

using std::max;
using std::min;

// ---- scalar fp32 intrinsics ------------------------------------------------------------------------
inline uint32_t __float_as_uint(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
inline float __fmul_rn(float a, float b) { volatile float r = a * b; return r; }
inline float __fadd_rn(float a, float b) { volatile float r = a + b; return r; }
inline float __fsub_rn(float a, float b) { volatile float r = a - b; return r; }
inline float __fdiv_rn(float a, float b) { volatile float r = a / b; return r; }
inline float __frcp_rn(float a) { volatile float r = 1.0f / a; return r; }
inline float __fsqrt_rn(float a) { volatile float r = sqrtf(a); return r; }
inline float __saturatef(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }  // NaN -> 0
template <typename T> inline T __ldg(const T* p) { return *p; }

// ---- half ----------------------------------------------------------------------------------------------
struct __half { uint16_t b; };
struct alignas(4) __half2 { __half x, y; };
inline float h2f(__half h) { _Float16 v; memcpy(&v, &h.b, 2); return (float)v; }
// one rounding (RNE); a NaN result is the canonical 0x7fff the GPU's half arithmetic and conversions produce (the host's is 0xfe00)
inline __half d2h(double d) { _Float16 v = (_Float16)d; __half h; memcpy(&h.b, &v, 2); if (d != d) h.b = 0x7fff; return h; }
inline __half f2h(float f) { _Float16 v = (_Float16)f; __half h; memcpy(&h.b, &v, 2); if (f != f) h.b = 0x7fff; return h; }
inline __half2 mkh2(__half a, __half b) { __half2 r; r.x = a; r.y = b; return r; }
inline __half2 __floats2half2_rn(float a, float b) { return mkh2(f2h(a), f2h(b)); }
inline __half2 __float2half2_rn(float a) { return mkh2(f2h(a), f2h(a)); }
inline float2 __half22float2(__half2 a) { return float2{h2f(a.x), h2f(a.y)}; }
inline float __low2float(__half2 a) { return h2f(a.x); }
inline float __high2float(__half2 a) { return h2f(a.y); }
inline __half2 __low2half2(__half2 a) { return mkh2(a.x, a.x); }
inline __half2 __high2half2(__half2 a) { return mkh2(a.y, a.y); }
inline __half2 __lows2half2(__half2 a, __half2 b) { return mkh2(a.x, b.x); }
inline __half2 __highs2half2(__half2 a, __half2 b) { return mkh2(a.y, b.y); }
// products of two halves are exact in double, and so is the sum with a third: a single rounding to half at the end
inline __half hfma1(__half a, __half b, __half c) { return d2h((double)h2f(a) * (double)h2f(b) + (double)h2f(c)); }
inline __half2 __hfma2(__half2 a, __half2 b, __half2 c) { return mkh2(hfma1(a.x, b.x, c.x), hfma1(a.y, b.y, c.y)); }
inline __half2 __hfma2_relu(__half2 a, __half2 b, __half2 c) { __half2 r = mkh2(hfma1(a.x, b.x, c.x), hfma1(a.y, b.y, c.y)); if (!(h2f(r.x) > 0.0f)) r.x.b = 0; if (!(h2f(r.y) > 0.0f)) r.y.b = 0; return r; }
inline __half2 __hmul2(__half2 a, __half2 b) { return mkh2(d2h((double)h2f(a.x) * h2f(b.x)), d2h((double)h2f(a.y) * h2f(b.y))); }
inline __half2 __hadd2(__half2 a, __half2 b) { return mkh2(d2h((double)h2f(a.x) + h2f(b.x)), d2h((double)h2f(a.y) + h2f(b.y))); }
inline __half2 __hsub2(__half2 a, __half2 b) { return mkh2(d2h((double)h2f(a.x) - h2f(b.x)), d2h((double)h2f(a.y) - h2f(b.y))); }
// the .rn forms that forbid contraction: one IEEE rounding per lane, as above
inline __half2 __hadd2_rn(__half2 a, __half2 b) { return __hadd2(a, b); }
inline __half2 __hsub2_rn(__half2 a, __half2 b) { return __hsub2(a, b); }
inline __half2 __hmul2_rn(__half2 a, __half2 b) { return __hmul2(a, b); }
inline __half2 __hmul2_sat(__half2 a, __half2 b) { return mkh2(f2h(__saturatef((float)((double)h2f(a.x) * h2f(b.x)))), f2h(__saturatef((float)((double)h2f(a.y) * h2f(b.y))))); }
inline __half2 __hneg2(__half2 a) { a.x.b ^= 0x8000; a.y.b ^= 0x8000; return a; }
inline __half2 __habs2(__half2 a) { a.x.b &= 0x7fff; a.y.b &= 0x7fff; return a; }
// non-propagating, like HMNMX2: a NaN operand yields the other one; -0 < +0 (fminf / fmaxf leave the sign of a zero result
// unspecified, and glibc's depends on the operand order)
inline bool hless1(__half a, __half b) {
  const int ka = (a.b & 0x8000) ? -(int)(a.b & 0x7fff) - 1 : (int)a.b, kb = (b.b & 0x8000) ? -(int)(b.b & 0x7fff) - 1 : (int)b.b;
  return ka < kb;
}
inline bool hnan1(__half a) { return (a.b & 0x7fff) > 0x7c00; }
inline __half hmin1(__half a, __half b) { return hnan1(a) ? (hnan1(b) ? __half{0x7fff} : b) : hnan1(b) ? a : hless1(b, a) ? b : a; }
inline __half hmax1(__half a, __half b) { return hnan1(a) ? (hnan1(b) ? __half{0x7fff} : b) : hnan1(b) ? a : hless1(a, b) ? b : a; }
inline __half2 __hmin2(__half2 a, __half2 b) { return mkh2(hmin1(a.x, b.x), hmin1(a.y, b.y)); }
inline __half2 __hmax2(__half2 a, __half2 b) { return mkh2(hmax1(a.x, b.x), hmax1(a.y, b.y)); }

inline __half2 h2rcp(__half2 a) { return mkh2(f2h(1.0f / h2f(a.x)), f2h(1.0f / h2f(a.y))); }

// ---- integer / warp intrinsics ---------------------------------------------------------------------------
inline uint32_t __byte_perm(uint32_t x, uint32_t y, uint32_t s) {
  const uint64_t v = ((uint64_t)y << 32) | x;
  uint32_t r = 0;
  for (int i = 0; i < 4; i++) r |= (uint32_t)((v >> (8 * ((s >> (4 * i)) & 7))) & 0xff) << (8 * i);
  return r;
}
// All 32 lanes of a warp must call these together (true for the kernels emulated here): exchange through a per-warp
// buffer between two warp-wide barriers.
uint32_t fsr1_emu_shfl(uint32_t v, int src_lane_or_negative_for_self);
inline uint32_t __shfl_up_sync(unsigned, uint32_t v, unsigned delta) {
  const int lane = (int)(threadIdx.x & 31);
  return fsr1_emu_shfl(v, lane >= (int)delta ? lane - (int)delta : -1);
}
inline uint32_t __shfl_down_sync(unsigned, uint32_t v, unsigned delta) {
  const int lane = (int)(threadIdx.x & 31);
  return fsr1_emu_shfl(v, lane + (int)delta < 32 ? lane + (int)delta : -1);
}
inline float __shfl_up_sync(unsigned m, float v, unsigned delta) { return __uint_as_float(__shfl_up_sync(m, __float_as_uint(v), delta)); }
inline float __shfl_down_sync(unsigned m, float v, unsigned delta) { return __uint_as_float(__shfl_down_sync(m, __float_as_uint(v), delta)); }

// ---- emulated TMA descriptor + mbarrier (see fsr1_emu_ptx.h) ----------------------------------------------
struct CUtensorMap {
  const unsigned char* base;
  int w, rows;          // tensor extent in elements / rows
  long long pitch;      // bytes
  int box_w, box_h;     // box extent
  int elem_bytes;
};
unsigned char* fsr1_emu_dynamic_smem();
