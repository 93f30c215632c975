// Ground-truth SDF from an oriented point cloud (SURVEY section 8(f) row 4): a from-scratch sm_90a replacement of the
// reference's only native code, ext/sdfgen/sdf_from_points.cu + the tinyflann kd-tree ext/common/kdtree_cuda.cu
// (built by ext/__init__.py:18-23; call sites dataset/av_gt_geometry.py:63-78, models/loss.py:85).
//
// The reference builds a kd-tree level by level with a host synchronisation per level (kdtree_cuda.cu:762-790), writes
// the k-NN indices and distances of every query to global memory, and votes in a second kernel.  Here the reference
// points are Morton-sorted once into the multi-level voxel hash that also serves the normal estimation and the colour
// texture, and ONE kernel does the search and the vote: a warp per query selects its nb_points nearest points (exact:
// the answer of a level is accepted when the k-th distance does not exceed the cell size, otherwise one level coarser,
// finally a scan of the whole cloud) and evaluates the reference's rule (sdf_from_points.cu:92-147, or the IMLS variant
// :33-90) from registers -- no index / distance arrays.
#include "knn_common.cuh"

namespace {

constexpr int kSdfWarps = 8;

// k nearest points of (qx,qy,qz) in key[0..got): exact (see above)
__device__ __forceinline__ int knn_query(const nksr_svh_t& svh, const float* __restrict__ xyz,
                                         const int32_t* __restrict__ range, const int64_t n_pts, const float ox,
                                         const float oy, const float oz, const int start_level, const int k,
                                         const float qx, const float qy, const float qz,
                                         unsigned long long* __restrict__ key, const int lane) {
  int3 h;
  const bool bad = !half_voxel(qx - ox, qy - oy, qz - oz, svh.voxel_size * 0.5f, h);
  const int L = svh.depth;
  int dx, dy, dz;
  slot_to_d(lane < 27 ? lane : 13, dx, dy, dz);
  int fill = 0, got = 0;
  float bound = 3.0e38f, dk2 = 0.f;
  bool exact = false;
  // out of range: no level search, only the scan of the whole cloud below
  for (int l = bad ? L : (start_level < L ? start_level : L - 1); l < L; ++l) {
    int rb = 0, re = 0;
    if (lane < 27) {
      const int cx = (h.x >> (l + 1)) + dx, cy = (h.y >> (l + 1)) + dy, cz = (h.z >> (l + 1)) + dz;
      if (cx >= 0 && cy >= 0 && cz >= 0) {
        const int v = find_key(svh.keys[l], svh.n[l], morton3(cx, cy, cz));
        if (v >= 0) {
          const int2 r = __ldg(reinterpret_cast<const int2*>(range) + svh.offset[l] + v);
          rb = r.x; re = r.y;
        }
      }
    }
    int total = re - rb;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
    if (total < k) continue;
    const float hl = svh.voxel_size * (float)(1 << l) * 0.999f;
    knn_reset(key, fill, bound, lane, hl * hl * 1.0000005f);   // further neighbours cannot make this level acceptable
    for (int s = 0; s < 27; ++s) {
      const int sb = __shfl_sync(0xffffffffu, rb, s), se = __shfl_sync(0xffffffffu, re, s);
      knn_scan_range(key, fill, bound, k, xyz, sb, se, qx, qy, qz, lane);
    }
    got = knn_finish(key, fill, k, dk2, lane);
    if (got == k && dk2 <= hl * hl) { exact = true; break; }
  }
  if (!exact) {   // further from the data than the coarsest cell size (or fewer than k points in all): scan everything
    knn_reset(key, fill, bound, lane);
    knn_scan_range(key, fill, bound, k, xyz, 0, n_pts, qx, qy, qz, lane);
    got = knn_finish(key, fill, k, dk2, lane);
  }
  return got;
}

// mean distance to the k nearest reference points, the point itself included (sdf_from_points.cu:158-166)
__global__ void __launch_bounds__(kSdfWarps * 32)
k_knn_mean_distance(const nksr_svh_t svh, const float* __restrict__ xyz, const int32_t* __restrict__ range,
                    const int64_t n_pts, const float ox, const float oy, const float oz,
                    const float* __restrict__ query, const int64_t m, const int k, const int start_level,
                    float* __restrict__ out) {
  __shared__ unsigned long long buf[kSdfWarps][kKnnBuf];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t i = blockIdx.x * (int64_t)kSdfWarps + wid;
  if (i >= m) return;
  const float qx = __ldg(query + 3 * i), qy = __ldg(query + 3 * i + 1), qz = __ldg(query + 3 * i + 2);
  const int got = knn_query(svh, xyz, range, n_pts, ox, oy, oz, start_level, k, qx, qy, qz, buf[wid], lane);
  float s = 0.f;
  for (int t = lane; t < got; t += 32) s += sqrtf(__uint_as_float((unsigned)(buf[wid][t] >> 32)));
  s = warp_sum(s);
  if (lane == 0) out[i] = got > 0 ? s / (float)k : 0.f;
}

template <bool IMLS>
__global__ void __launch_bounds__(kSdfWarps * 32)
k_sdf_from_points(const nksr_svh_t svh, const float* __restrict__ xyz, const float* __restrict__ nrm,
                  const float* __restrict__ ref_std, const int32_t* __restrict__ range, const int64_t n_pts,
                  const float ox, const float oy, const float oz, const float* __restrict__ query, const int64_t m,
                  const int k, const float stdv, const int start_level, float* __restrict__ sdf,
                  float* __restrict__ grad) {
  __shared__ unsigned long long buf[kSdfWarps][kKnnBuf];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t i = blockIdx.x * (int64_t)kSdfWarps + wid;
  if (i >= m) return;
  const float qx = __ldg(query + 3 * i), qy = __ldg(query + 3 * i + 1), qz = __ldg(query + 3 * i + 2);
  const int got = knn_query(svh, xyz, range, n_pts, ox, oy, oz, start_level, k, qx, qy, qz, buf[wid], lane);
  if (got == 0) {
    if (lane == 0) { sdf[i] = 0.f; if (grad) { grad[3 * i] = 0.f; grad[3 * i + 1] = 0.f; grad[3 * i + 2] = 0.f; } }
    return;
  }
  // every lane votes for the neighbours t = lane, lane + 32
  int num_pos = 0;
  float s_dw = 0.f, s_w = 0.f, gx = 0.f, gy = 0.f, gz = 0.f, emin = 3.0e38f;
  float e_t[2] = {0.f, 0.f}, d_t[2] = {0.f, 0.f}, n_t[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int t = lane + 32 * h;
    if (t < got) {
      const int64_t j = (int64_t)(unsigned)(buf[wid][t] & 0xffffffffull);
      const float rx = qx - __ldg(xyz + 3 * j), ry = qy - __ldg(xyz + 3 * j + 1), rz = qz - __ldg(xyz + 3 * j + 2);
      n_t[h][0] = __ldg(nrm + 3 * j); n_t[h][1] = __ldg(nrm + 3 * j + 1); n_t[h][2] = __ldg(nrm + 3 * j + 2);
      d_t[h] = n_t[h][0] * rx + n_t[h][1] * ry + n_t[h][2] * rz;               // d = <n_k, x - p_k>
      if (IMLS) {
        e_t[h] = (rx * rx + ry * ry + rz * rz) / (stdv * stdv);
        emin = fminf(emin, e_t[h]);
      } else if (d_t[h] > 0.f) {
        ++num_pos;
      }
    }
  }
  if (IMLS) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) emin = fminf(emin, __shfl_xor_sync(0xffffffffu, emin, o));
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (lane + 32 * h < got) {
        const float w = expf(-e_t[h] + emin);
        s_w += w;
        s_dw += d_t[h] * w;
        gx += n_t[h][0] * w; gy += n_t[h][1] * w; gz += n_t[h][2] * w;
      }
    }
    s_w = warp_sum(s_w); s_dw = warp_sum(s_dw);
    if (grad) { gx = warp_sum(gx); gy = warp_sum(gy); gz = warp_sum(gz); }
    if (lane == 0) {
      sdf[i] = s_dw / s_w;
      if (grad) { grad[3 * i] = gx / s_w; grad[3 * i + 1] = gy / s_w; grad[3 * i + 2] = gz / s_w; }
    }
    return;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) num_pos += __shfl_xor_sync(0xffffffffu, num_pos, o);
  if (lane == 0) {   // lane 0 holds the nearest neighbour (vote 0)
    const int64_t j = (int64_t)(unsigned)(buf[wid][0] & 0xffffffffull);
    const float rx = qx - __ldg(xyz + 3 * j), ry = qy - __ldg(xyz + 3 * j + 1), rz = qz - __ldg(xyz + 3 * j + 2);
    const float len = sqrtf(rx * rx + ry * ry + rz * rz);
    const float sd = ref_std ? __ldg(ref_std + j) : 1.f;
    float val, ux, uy, uz;
    if (len < stdv * sd) {
      val = fabsf(d_t[0]);
      const float sg = d_t[0] > 0.f ? 1.f : -1.f;
      ux = sg * n_t[0][0]; uy = sg * n_t[0][1]; uz = sg * n_t[0][2];
    } else {
      val = len;
      ux = rx / len; uy = ry / len; uz = rz / len;
    }
    const bool positive = num_pos > got / 2;          // sdf_from_points.cu:136 with num_votes = neighbours found
    sdf[i] = positive ? val : -val;
    if (grad) {
      grad[3 * i] = positive ? ux : -ux; grad[3 * i + 1] = positive ? uy : -uy; grad[3 * i + 2] = positive ? uz : -uz;
    }
  }
}

}  // namespace

extern "C" {

int nksr_knn_mean_distance(const nksr_svh_t* svh, const float* xyz, const int32_t* range, int64_t n_pts,
                           const float* origin3, const float* query, int64_t m, int k, int start_level, float* out,
                           void* stream) {
  if (!svh || !xyz || !range || !origin3 || !query || !out || k < 1 || k > 64 || svh->depth < 1 ||
      svh->depth > NKSR_MAX_DEPTH || start_level < 0 || n_pts < 0)
    return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  k_knn_mean_distance<<<grid_for(m, kSdfWarps), kSdfWarps * 32, 0, as_stream(stream)>>>(
      *svh, xyz, range, n_pts, origin3[0], origin3[1], origin3[2], query, m, k, start_level, out);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_sdf_from_points(const nksr_svh_t* svh, const float* xyz, const float* normal, const float* ref_std,
                         const int32_t* range, int64_t n_pts, const float* origin3, const float* query, int64_t m,
                         int nb_points, float stdv, int imls, int start_level, float* sdf, float* grad, void* stream) {
  if (!svh || !xyz || !normal || !range || !origin3 || !query || !sdf || nb_points < 1 || nb_points > 64 ||
      svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH || start_level < 0 || n_pts < 0)
    return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  const int grid = grid_for(m, kSdfWarps);
  if (imls)
    k_sdf_from_points<true><<<grid, kSdfWarps * 32, 0, as_stream(stream)>>>(
        *svh, xyz, normal, ref_std, range, n_pts, origin3[0], origin3[1], origin3[2], query, m, nb_points, stdv,
        start_level, sdf, grad);
  else
    k_sdf_from_points<false><<<grid, kSdfWarps * 32, 0, as_stream(stream)>>>(
        *svh, xyz, normal, ref_std, range, n_pts, origin3[0], origin3[1], origin3[2], query, m, nb_points, stdv,
        start_level, sdf, grad);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
