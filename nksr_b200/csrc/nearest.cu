// Nearest data point of arbitrary query positions on the multi-level voxel hash of a Morton-sorted cloud
// (SURVEY section 8(f) row 3: nksr.fields.PCNNField(xyz, color), the nearest-neighbour colour texture of
// examples/recons_colored_mesh.py:28-31, evaluated at every mesh vertex).  The per-level search is
// nearest_on_levels (nearest_common.cuh).
#include "nearest_common.cuh"

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
  bool exact;
  unsigned long long best = nearest_on_levels(svh, xyz, range, qx, qy, qz, ox, oy, oz, start_level, lane, exact);
  if (!exact) {
    // a query further from the data than the coarsest cell size (never a mesh vertex): scan the whole cloud
    best = kNearNone;
    for (int64_t q = lane; q < n_pts; q += 32) {
      const float ex = __ldg(xyz + 3 * q) - qx, ey = __ldg(xyz + 3 * q + 1) - qy, ez = __ldg(xyz + 3 * q + 2) - qz;
      const float d2 = fmaf(ex, ex, fmaf(ey, ey, ez * ez));
      const unsigned long long key = near_key(d2, (unsigned)q);
      best = key < best ? key : best;
    }
    best = warp_min_key(best);
  }
  if (lane == 0) {
    const bool found = best != kNearNone;
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
