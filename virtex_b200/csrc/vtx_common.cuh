// Shared host/device helpers for the virtex_b200 kernels.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <string.h>

// Programmatic dependent launch.  Every kernel of the library signals at
// its first instruction that dependents may be scheduled; the GEMM (the only kernel launched with the
// programmatic-serialisation attribute) runs its prologue -- barrier init, tensor-map prefetch --
// while the previous kernel drains, then waits for it to complete and flush before its first global access.
// Kernels launched without the attribute keep plain stream order, so nothing else changes semantics.
#define VTX_PDL_TRIGGER() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")
#define VTX_PDL_WAIT() asm volatile("griddepcontrol.wait;" ::: "memory")

namespace vtx {
// printf-style error recording; returns `code` so call sites can `return set_error(...)`.
int set_error(int code, const char* fmt, ...);
int check_launch(const char* what);

__device__ __forceinline__ float bf2f(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ __nv_bfloat16 f2bf(float x) { return __float2bfloat16_rn(x); }

// 8 x bf16 <-> 8 x float through one 16-byte vector
struct alignas(16) bf16x8 { __nv_bfloat162 h[4]; };
__device__ __forceinline__ void unpack8(const bf16x8& u, float* f) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    // bf16 -> fp32 is a 16-bit shift: one shift + one mask per pair (cuda_bf16's __bfloat1622float2 compiles to a
    // shift plus permute + shift, 3 instructions per pair; the GEMM's statistics pass is instruction-bound)
    const uint32_t w = *reinterpret_cast<const uint32_t*>(&u.h[j]);
    f[2 * j] = __uint_as_float(w << 16);
    f[2 * j + 1] = __uint_as_float(w & 0xffff0000u);
  }
}
__device__ __forceinline__ bf16x8 pack8(const float* f) {
  bf16x8 u;
#pragma unroll
  for (int j = 0; j < 4; ++j) u.h[j] = __floats2bfloat162_rn(f[2 * j], f[2 * j + 1]);
  return u;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Counter-based RNG for dropout (masks are recomputed in backward, never stored).  One 64-bit hash (murmur3-style
// finaliser) of (step seed, dropout site, element index / 4) serves FOUR consecutive elements, 16 bits each: a
// per-element hash (three 64-bit multiplies) would dominate the attention and GELU kernels.
// Drop probability = round(p * 65536) / 65536 (p = 0.1: 0.100006), kept elements are scaled by 1 / (1 - p).
__device__ __forceinline__ uint64_t hash_u64(uint64_t seed, uint32_t site, uint64_t ctr) {
  uint64_t x = seed ^ (0x9E3779B97F4A7C15ull * (uint64_t)(site + 1)) ^ (ctr * 0xD6E8FEB86659FD93ull);
  x ^= x >> 32; x *= 0xD6E8FEB86659FD93ull;
  x ^= x >> 32; x *= 0xD6E8FEB86659FD93ull;
  x ^= x >> 32;
  return x;
}
struct Drop4 {
  uint64_t h;
  uint32_t thr;
  float inv_keep;
  // scale of element `lane` (0..3) of the group: 0 if dropped, 1/(1-p) if kept; p == 0 -> thr == 0 -> always 1
  __device__ __forceinline__ float scale(int lane) const {
    return (((uint32_t)(h >> (16 * lane)) & 0xffffu) < thr) ? 0.f : inv_keep;
  }
};
// idx4 = (index of the group's first element) / 4; the group's elements are 4*idx4 .. 4*idx4 + 3
__device__ __forceinline__ Drop4 drop4(float p, float inv_keep, uint64_t seed, uint32_t site, uint64_t idx4) {
  Drop4 d;
  d.thr = p > 0.f ? (uint32_t)(p * 65536.f + 0.5f) : 0u;
  d.inv_keep = p > 0.f ? inv_keep : 1.f;
  d.h = p > 0.f ? hash_u64(seed, site, idx4) : 0ull;
  return d;
}
// single-element form (same mask as the grouped form for the same element index)
__device__ __forceinline__ float dropout_scale(float p, float inv_keep, uint64_t seed, uint32_t site, uint64_t idx) {
  if (p <= 0.f) return 1.f;
  return drop4(p, inv_keep, seed, site, idx >> 2).scale((int)(idx & 3));
}
}  // namespace vtx
