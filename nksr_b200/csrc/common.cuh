// Shared device helpers for the nksr_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/nksr_b200.h"

#define NKSR_CHECK_LAUNCH()                         \
  do {                                              \
    cudaError_t _e = cudaGetLastError();            \
    if (_e != cudaSuccess) return NKSR_E_CUDA;      \
  } while (0)

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

static inline int grid_for(int64_t n, int block) {
  int64_t g = (n + block - 1) / block;
  if (g < 1) g = 1;
  return (int)g;
}

// ---------------------------------------------------------------- Morton keys (SPEC S1)
// 21 bits per axis, x most significant: key bit 3b+2 = x bit b, 3b+1 = y, 3b = z.
__host__ __device__ __forceinline__ uint64_t part1by2(uint64_t v) {
  v &= 0x1FFFFFull;
  v = (v | (v << 32)) & 0x1F00000000FFFFull;
  v = (v | (v << 16)) & 0x1F0000FF0000FFull;
  v = (v | (v << 8)) & 0x100F00F00F00F00Full;
  v = (v | (v << 4)) & 0x10C30C30C30C30C3ull;
  v = (v | (v << 2)) & 0x1249249249249249ull;
  return v;
}
__host__ __device__ __forceinline__ uint32_t compact1by2(uint64_t v) {
  v &= 0x1249249249249249ull;
  v = (v | (v >> 2)) & 0x10C30C30C30C30C3ull;
  v = (v | (v >> 4)) & 0x100F00F00F00F00Full;
  v = (v | (v >> 8)) & 0x1F0000FF0000FFull;
  v = (v | (v >> 16)) & 0x1F00000000FFFFull;
  v = (v | (v >> 32)) & 0x1FFFFFull;
  return (uint32_t)v;
}
// u: offset (non-negative) coordinates
__host__ __device__ __forceinline__ int64_t morton3(int ux, int uy, int uz) {
  return (int64_t)((part1by2((uint64_t)(uint32_t)ux) << 2) | (part1by2((uint64_t)(uint32_t)uy) << 1) |
                   part1by2((uint64_t)(uint32_t)uz));
}
__host__ __device__ __forceinline__ void morton3_decode(int64_t k, int& ux, int& uy, int& uz) {
  ux = (int)compact1by2((uint64_t)k >> 2);
  uy = (int)compact1by2((uint64_t)k >> 1);
  uz = (int)compact1by2((uint64_t)k);
}
// offset of level-l voxel coordinates inside the key (SPEC S1): 2^(19-l); half-voxels: 2^20
__host__ __device__ __forceinline__ int level_offset(int level) { return 1 << (19 - level); }
#define NKSR_HALF_OFFSET (1 << 20)
#define NKSR_KEY_LIMIT (1 << 21)

// The one device definition of the half-voxel quantisation (SPEC S1): h = floor(p / half_w) + 2^20 per axis, with
// IEEE division.  p is relative to the keys' origin (callers with an origin subtract it first).  Returns false when an
// axis is outside (-(2^20 - 16), 2^20 - 16) or NaN; that axis then gets h = 2^20.  The containing voxel on level l is
// h >> (l+1).
__device__ __forceinline__ bool half_voxel(float px, float py, float pz, float half_w, int3& h) {
  const float p[3] = {px, py, pz};
  int u[3];
  bool bad = false;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    float q = floorf(__fdiv_rn(p[a], half_w));
    if (!(q > -(float)(NKSR_HALF_OFFSET - 16) && q < (float)(NKSR_HALF_OFFSET - 16))) { bad = true; q = 0.f; }
    u[a] = (int)q + NKSR_HALF_OFFSET;
  }
  h = make_int3(u[0], u[1], u[2]);
  return !bad;
}

// slot in child8[s] (the table of level s) of the level-(s-1) voxel that contains half-voxel coordinates h
__device__ __forceinline__ int child_octant(const int3& h, int s) {
  return (((h.x >> s) & 1) << 2) | (((h.y >> s) & 1) << 1) | ((h.z >> s) & 1);
}

// lower_bound over sorted keys; returns index or -1 when absent
__device__ __forceinline__ int find_key(const int64_t* __restrict__ keys, int64_t n, int64_t k) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    int64_t mid = (lo + hi) >> 1;
    if (__ldg(keys + mid) < k) lo = mid + 1; else hi = mid;
  }
  return (lo < n && __ldg(keys + lo) == k) ? (int)lo : -1;
}

// first index whose key is >= k (n when none)
__device__ __forceinline__ int64_t lower_bound_key(const int64_t* __restrict__ keys, int64_t n, int64_t k) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    int64_t mid = (lo + hi) >> 1;
    if (__ldg(keys + mid) < k) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// c + a * b on a pair of fp32 values, each an IEEE fma (sm_90 has no packed fp32 FMA)
__device__ __forceinline__ float2 ffma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// slot s in 0..26 <-> offset d in {-1,0,1}^3 with s = (dx+1)*9 + (dy+1)*3 + (dz+1)
__device__ __forceinline__ void slot_to_d(int s, int& dx, int& dy, int& dz) {
  dx = s / 9 - 1;
  dy = (s / 3) % 3 - 1;
  dz = s % 3 - 1;
}
