// br_port.h -- thin layer that lets the warp-task device code (br_lz77.h, br_entropy.h)
// also be compiled by g++ for the CPU "sim" harness under tests/sim/ (test infrastructure,
// never shipped).  In the product build (nvcc, sm_90a) every BR_DEV function is
// __device__-only: there is no host implementation of the hot path in the library.
//
// Programming model: "one warp = one task".  Scalar control flow is executed redundantly by
// all 32 lanes (warp-uniform); data-parallel steps spread over lanes and fold with
// ballot / shuffle.  Under BR_SIM the warp has a single lane and the folds degenerate.
#pragma once
#include <stdint.h>
#include <string.h>

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

#if defined(__CUDACC__) && !defined(BR_SIM)
#define BR_GPU 1
#define BR_DEV __device__ __forceinline__
#define BR_DEV_M __device__ __forceinline__   /* for static member functions */
#define BR_HD __host__ __device__ __forceinline__
#define BR_DEV_NOINLINE __device__ __noinline__
#define BR_WARP 32
BR_DEV int br_lane() { return (int)(threadIdx.x & 31u); }
BR_DEV u32 br_ballot(int p) { return __ballot_sync(0xffffffffu, p); }
template <class T> BR_DEV T br_shfl(T v, int src) { return __shfl_sync(0xffffffffu, v, src); }
BR_DEV void br_syncwarp() { __syncwarp(); }
BR_DEV int br_popc(u32 x) { return __popc(x); }
BR_DEV int br_ffs(u32 x) { return __ffs((int)x); }  // 1-based, 0 if none
BR_DEV int br_clz(u32 x) { return __clz((int)x); }
BR_DEV int br_ctz64(u64 x) {   // x != 0
  u32 lo = (u32)x;
  return lo ? __ffs((int)lo) - 1 : 31 + __ffs((int)(u32)(x >> 32));
}
BR_DEV u32 br_lanemask_lt() { u32 m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }
BR_DEV u32 br_match_any(u32 v) { return __match_any_sync(0xffffffffu, v); }
BR_DEV void br_prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); }
BR_DEV u32 br_atomic_or(u32* p, u32 v) { return atomicOr(p, v); }
BR_DEV u32 br_atomic_and(u32* p, u32 v) { return atomicAnd(p, v); }
BR_DEV u32 br_atomic_add(u32* p, u32 v) { return atomicAdd(p, v); }
BR_DEV int br_atomic_max(int* p, int v) { return atomicMax(p, v); }
BR_DEV u32 br_atomic_min(u32* p, u32 v) { return atomicMin(p, v); }
// Bit-exact IEEE double ops: never contracted into FMA (the reference is built without
// -march, so x86-64 emits separate mul/add; SURVEY.md section 0, T5).
BR_DEV double br_dmul(double a, double b) { return __dmul_rn(a, b); }
BR_DEV double br_dadd(double a, double b) { return __dadd_rn(a, b); }
BR_DEV double br_dsub(double a, double b) { return __dsub_rn(a, b); }
BR_DEV double br_ddiv(double a, double b) { return __ddiv_rn(a, b); }
template <class T> BR_DEV T br_ldg(const T* p) { return __ldg(p); }
BR_DEV u32 br_warp_sum(u32 v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// exclusive prefix sum across lanes; *total = sum over the warp
BR_DEV u32 br_warp_excl_scan(u32 v, u32* total) {
  u32 x = v;
  for (int o = 1; o < 32; o <<= 1) { u32 t = __shfl_up_sync(0xffffffffu, x, o); if ((threadIdx.x & 31) >= (unsigned)o) x += t; }
  *total = __shfl_sync(0xffffffffu, x, 31);
  return x - v;
}
BR_DEV u32 br_warp_min(u32 v) {
  for (int o = 16; o > 0; o >>= 1) { u32 t = __shfl_xor_sync(0xffffffffu, v, o); v = t < v ? t : v; }
  return v;
}
BR_DEV u32 br_warp_max(u32 v) {
  for (int o = 16; o > 0; o >>= 1) { u32 t = __shfl_xor_sync(0xffffffffu, v, o); v = t > v ? t : v; }
  return v;
}
#else
#define BR_GPU 0
#define BR_DEV static inline
#define BR_DEV_M inline
#define BR_HD static inline
#define BR_DEV_NOINLINE static
#define BR_WARP 1
BR_DEV int br_lane() { return 0; }
BR_DEV u32 br_ballot(int p) { return p ? 1u : 0u; }
template <class T> BR_DEV T br_shfl(T v, int) { return v; }
BR_DEV void br_syncwarp() {}
BR_DEV int br_popc(u32 x) { return __builtin_popcount(x); }
BR_DEV int br_ffs(u32 x) { return __builtin_ffs((int)x); }
BR_DEV int br_clz(u32 x) { return x ? __builtin_clz(x) : 32; }
BR_DEV int br_ctz64(u64 x) { return __builtin_ctzll(x); }
BR_DEV u32 br_lanemask_lt() { return 0; }
BR_DEV u32 br_match_any(u32) { return 1u; }
BR_DEV void br_prefetch_l2(const void*) {}
BR_DEV u32 br_atomic_or(u32* p, u32 v) { u32 o = *p; *p = o | v; return o; }
BR_DEV u32 br_atomic_and(u32* p, u32 v) { u32 o = *p; *p = o & v; return o; }
BR_DEV u32 br_atomic_add(u32* p, u32 v) { u32 o = *p; *p = o + v; return o; }
BR_DEV int br_atomic_max(int* p, int v) { int o = *p; if (v > o) *p = v; return o; }
BR_DEV u32 br_atomic_min(u32* p, u32 v) { u32 o = *p; if (v < o) *p = v; return o; }
BR_DEV double br_dmul(double a, double b) { volatile double r = a * b; return r; }
BR_DEV double br_dadd(double a, double b) { volatile double r = a + b; return r; }
BR_DEV double br_dsub(double a, double b) { volatile double r = a - b; return r; }
BR_DEV double br_ddiv(double a, double b) { volatile double r = a / b; return r; }
template <class T> BR_DEV T br_ldg(const T* p) { return *p; }
BR_DEV u32 br_warp_sum(u32 v) { return v; }
BR_DEV u32 br_warp_excl_scan(u32 v, u32* total) { *total = v; return 0; }
BR_DEV u32 br_warp_min(u32 v) { return v; }
BR_DEV u32 br_warp_max(u32 v) { return v; }
#endif

BR_DEV u32 br_log2floor(u32 n) { return 31u - (u32)br_clz(n); }  // n != 0
BR_DEV u32 br_min(u32 a, u32 b) { return a < b ? a : b; }
BR_DEV u32 br_max(u32 a, u32 b) { return a > b ? a : b; }

// Unaligned little-endian loads from a 4-byte aligned base (cudaMalloc'ed buffers are; the
// buffer carries >= 16 bytes of zero padding behind the last input byte).
BR_DEV u32 br_ld32u(const u8* base, u32 pos) {
#if BR_GPU
  const u32* w = (const u32*)base;
  u32 i = pos >> 2, sh = (pos & 3u) * 8u;
  u32 lo = br_ldg(w + i), hi = br_ldg(w + i + 1);
  return __funnelshift_r(lo, hi, sh);
#else
  u32 v; memcpy(&v, base + pos, 4); return v;
#endif
}
BR_DEV u64 br_ld64u(const u8* base, u32 pos) {
#if BR_GPU
  const u32* w = (const u32*)base;
  u32 i = pos >> 2, sh = (pos & 3u) * 8u;
  u32 a = br_ldg(w + i), b = br_ldg(w + i + 1), c = br_ldg(w + i + 2);
  u32 lo = __funnelshift_r(a, b, sh), hi = __funnelshift_r(b, c, sh);
  return ((u64)hi << 32) | lo;
#else
  u64 v; memcpy(&v, base + pos, 8); return v;
#endif
}
