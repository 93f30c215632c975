// Exact nearest data point of one query on the multi-level voxel hash of a Morton-sorted cloud, one warp per query:
// shared by the PCNNField texture lookup (nearest.cu) and the mesh-metric nearest neighbours (metrics.cu).
//
// On level l (cell size h_l = h_0 2^l) the 27 cells around the query's cell are found by 27 lane-parallel binary
// searches of the level's sorted keys (the query's own cell need not hold a point), their contiguous point ranges are
// scanned cooperatively, and the minimum is EXACT as soon as it does not exceed h_l (every point closer than that lies
// inside the block); otherwise the search moves one level up.
#pragma once
#include "common.cuh"

namespace {

constexpr unsigned long long kNearNone = 0xffffffffffffffffull;

// packed (squared distance bits << 32) | index: ties go to the lower index
__device__ __forceinline__ unsigned long long near_key(float d2, unsigned q) {
  return ((unsigned long long)__float_as_uint(d2) << 32) | q;
}

__device__ __forceinline__ unsigned long long warp_min_key(unsigned long long best) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
    best = other < best ? other : best;
  }
  return best;
}

// the lane's minimum over its share (q = sb + lane, step 32) of the sorted points [sb, se), folded into `best`
__device__ __forceinline__ unsigned long long near_scan_range(const float* __restrict__ xyz, const int sb, const int se,
                                                              const float qx, const float qy, const float qz,
                                                              const int lane, unsigned long long best) {
  for (int q = sb + lane; q < se; q += 32) {
    const float ex = __ldg(xyz + 3 * (int64_t)q) - qx, ey = __ldg(xyz + 3 * (int64_t)q + 1) - qy,
                ez = __ldg(xyz + 3 * (int64_t)q + 2) - qz;
    const float d2 = fmaf(ex, ex, fmaf(ey, ey, ez * ez));
    const unsigned long long key = near_key(d2, (unsigned)q);
    best = key < best ? key : best;
  }
  return best;
}

// The hierarchy search from `start_level` up.  Returns the warp-uniform packed key of the nearest point found on the
// last level searched; `exact` tells whether a level proved it (false for a query outside the key frame or further
// than the coarsest cell size from every point: the caller resolves those).  (ox, oy, oz): the shift applied to the
// cloud before keying.
__device__ __forceinline__ unsigned long long nearest_on_levels(const nksr_svh_t& svh, const float* __restrict__ xyz,
                                                                const int32_t* __restrict__ range, const float qx,
                                                                const float qy, const float qz, const float ox,
                                                                const float oy, const float oz, const int start_level,
                                                                const int lane, bool& exact) {
  // half-voxel coordinates in the frame of the keys
  int3 h;
  const bool bad = !half_voxel(qx - ox, qy - oy, qz - oz, svh.voxel_size * 0.5f, h);
  const int L = svh.depth;
  int dx, dy, dz;
  slot_to_d(lane < 27 ? lane : 13, dx, dy, dz);
  unsigned long long best = kNearNone;
  exact = false;
  for (int l = start_level < L ? start_level : L - 1; l < L; ++l) {
    int rb = 0, re = 0;
    if (lane < 27 && !bad) {
      const int cx = (h.x >> (l + 1)) + dx, cy = (h.y >> (l + 1)) + dy, cz = (h.z >> (l + 1)) + dz;
      if (cx >= 0 && cy >= 0 && cz >= 0) {
        const int v = find_key(svh.keys[l], svh.n[l], morton3(cx, cy, cz));
        if (v >= 0) {
          const int2 r = __ldg(reinterpret_cast<const int2*>(range) + svh.offset[l] + v);
          rb = r.x; re = r.y;
        }
      }
    }
    best = kNearNone;
    for (int s = 0; s < 27; ++s) {
      const int sb = __shfl_sync(0xffffffffu, rb, s), se = __shfl_sync(0xffffffffu, re, s);
      best = near_scan_range(xyz, sb, se, qx, qy, qz, lane, best);
    }
    best = warp_min_key(best);
    const float hl = svh.voxel_size * (float)(1 << l) * 0.999f;
    if (best != kNearNone && __uint_as_float((unsigned)(best >> 32)) <= hl * hl) { exact = true; break; }
  }
  return best;
}

}  // namespace
