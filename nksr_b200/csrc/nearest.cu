// Nearest data point of arbitrary query positions on the multi-level voxel hash of a Morton-sorted cloud
// (SURVEY section 8(f) row 3: nksr.fields.PCNNField(xyz, color), the nearest-neighbour colour texture of
// examples/recons_colored_mesh.py:28-31, evaluated at every mesh vertex).
//
// One warp per query.  On level l (cell size h_l = h_0 2^l) the 27 cells around the query's cell are found by 27
// lane-parallel binary searches of the level's sorted keys (the query's own cell need not hold a point), their
// contiguous point ranges are scanned cooperatively, and the minimum is EXACT as soon as it does not exceed h_l
// (every point closer than that lies inside the block); otherwise the search moves one level up.
#include "common.cuh"

namespace {

constexpr int kNearWarps = 8;

__global__ void __launch_bounds__(kNearWarps * 32)
k_nearest_point(const nksr_svh_t svh, const float* __restrict__ xyz, const int32_t* __restrict__ range,
                const int64_t n_pts, const float* __restrict__ query, const int64_t m, const float ox, const float oy,
                const float oz, const int start_level, int32_t* __restrict__ out_idx, float* __restrict__ out_d2) {
  const int lane = threadIdx.x & 31;
  const int64_t i = blockIdx.x * (int64_t)kNearWarps + (threadIdx.x >> 5);
  if (i >= m) return;
  const float qx = __ldg(query + 3 * i), qy = __ldg(query + 3 * i + 1), qz = __ldg(query + 3 * i + 2);
  // half-voxel coordinates in the frame of the keys (cloud shifted to its bounding-box corner)
  int3 h;
  const bool bad = !half_voxel(qx - ox, qy - oy, qz - oz, svh.voxel_size * 0.5f, h);
  const int L = svh.depth;
  int dx, dy, dz;
  slot_to_d(lane < 27 ? lane : 13, dx, dy, dz);
  unsigned long long best = 0xffffffffffffffffull;   // (distance bits << 32) | index: ties go to the lower index
  bool exact = false;
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
    best = 0xffffffffffffffffull;
    for (int s = 0; s < 27; ++s) {
      const int sb = __shfl_sync(0xffffffffu, rb, s), se = __shfl_sync(0xffffffffu, re, s);
      for (int q = sb + lane; q < se; q += 32) {
        const float ex = __ldg(xyz + 3 * (int64_t)q) - qx, ey = __ldg(xyz + 3 * (int64_t)q + 1) - qy,
                    ez = __ldg(xyz + 3 * (int64_t)q + 2) - qz;
        const float d2 = fmaf(ex, ex, fmaf(ey, ey, ez * ez));
        const unsigned long long key = ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned)q;
        best = key < best ? key : best;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
      best = other < best ? other : best;
    }
    const float hl = svh.voxel_size * (float)(1 << l) * 0.999f;
    if (best != 0xffffffffffffffffull && __uint_as_float((unsigned)(best >> 32)) <= hl * hl) { exact = true; break; }
  }
  if (!exact) {
    // a query further from the data than the coarsest cell size (never a mesh vertex): scan the whole cloud
    best = 0xffffffffffffffffull;
    for (int64_t q = lane; q < n_pts; q += 32) {
      const float ex = __ldg(xyz + 3 * q) - qx, ey = __ldg(xyz + 3 * q + 1) - qy, ez = __ldg(xyz + 3 * q + 2) - qz;
      const float d2 = fmaf(ex, ex, fmaf(ey, ey, ez * ez));
      const unsigned long long key = ((unsigned long long)__float_as_uint(d2) << 32) | (unsigned)q;
      best = key < best ? key : best;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
      best = other < best ? other : best;
    }
  }
  if (lane == 0) {
    const bool found = best != 0xffffffffffffffffull;
    out_idx[i] = found ? (int32_t)(unsigned)(best & 0xffffffffull) : -1;
    if (out_d2) out_d2[i] = found ? __uint_as_float((unsigned)(best >> 32)) : 3.0e38f;
  }
}

}  // namespace

extern "C" {

int nksr_nearest_point(const nksr_svh_t* svh, const float* xyz, const int32_t* range, int64_t n_pts, const float* query,
                       int64_t m, const float* origin3, int start_level, int32_t* out_idx, float* out_d2,
                       void* stream) {
  if (!svh || !xyz || !range || !query || !origin3 || !out_idx || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH ||
      start_level < 0 || n_pts < 0)
    return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  k_nearest_point<<<grid_for(m, kNearWarps), kNearWarps * 32, 0, as_stream(stream)>>>(
      *svh, xyz, range, n_pts, query, m, origin3[0], origin3[1], origin3[2], start_level, out_idx, out_d2);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
