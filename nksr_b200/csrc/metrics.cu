// Mesh-quality metrics (the reference's metrics.MeshEvaluator, called from models/nksr_net.py:298-312): area-uniform
// surface sampling of a triangle mesh and exact nearest neighbours with normal agreement.  DESIGN.md SPEC S18.
//
// k_sample_surface: one thread per sample; the triangle comes from a binary search over the caller's per-triangle
// sample bounds, the barycentrics from a counter hash of (seed, sample index), so the samples do not depend on the
// launch configuration.
// k_metric_nearest: the hierarchy search of nearest_common.cuh; the queries it cannot prove (outside the key frame,
// or further than the coarsest cell size from every point) are compacted into a list, and k_metric_far answers them
// by a branch-and-bound over the top-level cells: cells whose point bounding box is further than the best distance so
// far are never scanned.
#include "nearest_common.cuh"

namespace {

constexpr int kSampleThreads = 256;
constexpr int kMetricWarps = 8;

// splitmix64's output mix (SPEC S18: mirrored bit for bit by oracle/metrics.py)
__host__ __device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// uniform in [0, 1) on a 2^-24 grid (exact in fp32) from the hashed seed and the draw counter 2 i + k
__device__ __forceinline__ float hash_uniform(uint64_t hseed, uint64_t counter) {
  return (float)(mix64(hseed + counter) >> 40) * (1.0f / 16777216.0f);
}

__global__ void __launch_bounds__(kSampleThreads)
k_sample_surface(const float* __restrict__ v, const int32_t* __restrict__ f, const int64_t n_tri,
                 const int64_t* __restrict__ start, const int64_t n, const uint64_t hseed, float* __restrict__ out_xyz,
                 float* __restrict__ out_normal, int32_t* __restrict__ out_tri) {
  const int64_t i = blockIdx.x * (int64_t)kSampleThreads + threadIdx.x;
  if (i >= n) return;
  // the last triangle whose first sample is <= i (start[0] = 0, start[n_tri] = n; empty triangles are skipped)
  int64_t lo = 0, hi = n_tri - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (__ldg(start + mid) <= i) lo = mid; else hi = mid - 1;
  }
  const int t = (int)lo;
  const int a = __ldg(f + 3 * (int64_t)t), b = __ldg(f + 3 * (int64_t)t + 1), c = __ldg(f + 3 * (int64_t)t + 2);
  float p0[3], p1[3], p2[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    p0[k] = __ldg(v + 3 * (int64_t)a + k);
    p1[k] = __ldg(v + 3 * (int64_t)b + k);
    p2[k] = __ldg(v + 3 * (int64_t)c + k);
  }
  const float r1 = hash_uniform(hseed, 2 * (uint64_t)i), r2 = hash_uniform(hseed, 2 * (uint64_t)i + 1);
  const float s = sqrtf(r1);
  const float w0 = 1.f - s, w1 = s * (1.f - r2), w2 = s * r2;
#pragma unroll
  for (int k = 0; k < 3; ++k) out_xyz[3 * i + k] = fmaf(w2, p2[k], fmaf(w1, p1[k], w0 * p0[k]));
  // the triangle normal, in fp64 like the areas that gave this triangle its samples
  const double e1x = (double)p1[0] - p0[0], e1y = (double)p1[1] - p0[1], e1z = (double)p1[2] - p0[2];
  const double e2x = (double)p2[0] - p0[0], e2y = (double)p2[1] - p0[1], e2z = (double)p2[2] - p0[2];
  const double nx = e1y * e2z - e1z * e2y, ny = e1z * e2x - e1x * e2z, nz = e1x * e2y - e1y * e2x;
  const double inv = 1.0 / sqrt(nx * nx + ny * ny + nz * nz);
  out_normal[3 * i] = (float)(nx * inv);
  out_normal[3 * i + 1] = (float)(ny * inv);
  out_normal[3 * i + 2] = (float)(nz * inv);
  out_tri[i] = t;
}

// bounding box (lo xyz, hi xyz) of the points of every top-level cell; one warp per cell
__global__ void __launch_bounds__(kMetricWarps * 32)
k_cell_boxes(const float* __restrict__ xyz, const int2* __restrict__ range, const int64_t n_cells,
             float* __restrict__ box) {
  const int lane = threadIdx.x & 31;
  const int64_t c = blockIdx.x * (int64_t)kMetricWarps + (threadIdx.x >> 5);
  if (c >= n_cells) return;
  const int2 r = __ldg(range + c);
  float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f};
  for (int q = r.x + lane; q < r.y; q += 32) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float x = __ldg(xyz + 3 * (int64_t)q + k);
      lo[k] = fminf(lo[k], x);
      hi[k] = fmaxf(hi[k], x);
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[k] = fminf(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
      hi[k] = fmaxf(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
    }
  }
  if (lane < 3) box[6 * c + lane] = lo[lane];
  else if (lane < 6) box[6 * c + lane] = hi[lane - 3];
}

// Lower bound on the squared distance the scan computes for any point of a box: the per-axis gaps are fp32
// differences of the same operands' extremes and the sum is the scan's fma expression, so by monotone rounding the
// bound never exceeds a scanned point's d2.
__device__ __forceinline__ float box_d2(const float* __restrict__ box, const float qx, const float qy,
                                        const float qz) {
  const float gx = fmaxf(fmaxf(__ldg(box) - qx, qx - __ldg(box + 3)), 0.f);
  const float gy = fmaxf(fmaxf(__ldg(box + 1) - qy, qy - __ldg(box + 4)), 0.f);
  const float gz = fmaxf(fmaxf(__ldg(box + 2) - qz, qz - __ldg(box + 5)), 0.f);
  return fmaf(gx, gx, fmaf(gy, gy, gz * gz));
}

// lane 0 of the warp that resolved query i: distance, index and (when both sides have normals) |n_q . n_t| of the
// unit normals; a zero-length normal gives NaN (0/0)
__device__ __forceinline__ void write_result(const int64_t i, const unsigned long long best,
                                             const float* __restrict__ normal, const float* __restrict__ qnormal,
                                             float* __restrict__ out_dist, int32_t* __restrict__ out_idx,
                                             float* __restrict__ out_dot) {
  const int32_t t = (int32_t)(unsigned)(best & 0xffffffffull);
  out_dist[i] = sqrtf(__uint_as_float((unsigned)(best >> 32)));
  out_idx[i] = t;
  if (out_dot && normal && qnormal) {
    float a[3], b[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      a[k] = __ldg(qnormal + 3 * i + k);
      b[k] = __ldg(normal + 3 * (int64_t)t + k);
    }
    const float na = sqrtf(fmaf(a[0], a[0], fmaf(a[1], a[1], a[2] * a[2])));
    const float nb = sqrtf(fmaf(b[0], b[0], fmaf(b[1], b[1], b[2] * b[2])));
    float dot = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) dot = fmaf(__fdiv_rn(a[k], na), __fdiv_rn(b[k], nb), dot);
    out_dot[i] = fabsf(dot);
  }
}

__global__ void __launch_bounds__(kMetricWarps * 32)
k_metric_nearest(const nksr_svh_t svh, const float* __restrict__ xyz, const float* __restrict__ normal,
                 const int32_t* __restrict__ range, const float* __restrict__ query,
                 const float* __restrict__ qnormal, const int64_t m, const float ox, const float oy, const float oz,
                 const int start_level, float* __restrict__ out_dist, int32_t* __restrict__ out_idx,
                 float* __restrict__ out_dot, int32_t* __restrict__ far_list, int32_t* __restrict__ far_count) {
  const int lane = threadIdx.x & 31;
  const int64_t i = blockIdx.x * (int64_t)kMetricWarps + (threadIdx.x >> 5);
  if (i >= m) return;
  const float qx = __ldg(query + 3 * i), qy = __ldg(query + 3 * i + 1), qz = __ldg(query + 3 * i + 2);
  bool exact;
  const unsigned long long best = nearest_on_levels(svh, xyz, range, qx, qy, qz, ox, oy, oz, start_level, lane, exact);
  if (lane != 0) return;
  if (exact) write_result(i, best, normal, qnormal, out_dist, out_idx, out_dot);
  else far_list[atomicAdd(far_count, 1)] = (int32_t)i;
}

// The listed queries, one warp each (grid-stride over the device-side count): the top-level cell with the smallest box
// bound is scanned first, then every other cell whose bound does not exceed the best squared distance so far.
__global__ void __launch_bounds__(kMetricWarps * 32)
k_metric_far(const float* __restrict__ xyz, const float* __restrict__ normal, const int2* __restrict__ range,
             const float* __restrict__ box, const int64_t n_cells, const float* __restrict__ query,
             const float* __restrict__ qnormal, const int32_t* __restrict__ far_list,
             const int32_t* __restrict__ far_count, float* __restrict__ out_dist, int32_t* __restrict__ out_idx,
             float* __restrict__ out_dot) {
  const int lane = threadIdx.x & 31;
  const int count = *far_count;
  for (int w = blockIdx.x * kMetricWarps + (threadIdx.x >> 5); w < count; w += gridDim.x * kMetricWarps) {
    const int64_t i = __ldg(far_list + w);
    const float qx = __ldg(query + 3 * i), qy = __ldg(query + 3 * i + 1), qz = __ldg(query + 3 * i + 2);
    unsigned long long first = kNearNone;       // (bound bits << 32) | cell
    for (int64_t c = lane; c < n_cells; c += 32) {
      const unsigned long long key = near_key(box_d2(box + 6 * c, qx, qy, qz), (unsigned)c);
      first = key < first ? key : first;
    }
    first = warp_min_key(first);
    const int c0 = (int)(unsigned)(first & 0xffffffffull);
    int2 r = __ldg(range + c0);
    unsigned long long best = warp_min_key(near_scan_range(xyz, r.x, r.y, qx, qy, qz, lane, kNearNone));
    for (int64_t cb = 0; cb < n_cells; cb += 32) {
      const int64_t c = cb + lane;
      const float lb = c < n_cells && c != c0 ? box_d2(box + 6 * c, qx, qy, qz) : 3.0e38f;
      unsigned cand = __ballot_sync(0xffffffffu, lb <= __uint_as_float((unsigned)(best >> 32)));
      while (cand) {
        const int s = __ffs(cand) - 1;
        cand &= cand - 1;
        if (__shfl_sync(0xffffffffu, lb, s) > __uint_as_float((unsigned)(best >> 32))) continue;
        r = __ldg(range + cb + s);
        best = warp_min_key(near_scan_range(xyz, r.x, r.y, qx, qy, qz, lane, best));
      }
    }
    if (lane == 0) write_result(i, best, normal, qnormal, out_dist, out_idx, out_dot);
  }
}

}  // namespace

extern "C" {

int nksr_sample_surface(const float* v, const int32_t* f, int64_t n_tri, const int64_t* start, int64_t n, int64_t seed,
                        float* out_xyz, float* out_normal, int32_t* out_tri, void* stream) {
  if (n < 0 || n_tri < 0 || n_tri > INT32_MAX) return NKSR_E_INVALID;
  if (n == 0) return NKSR_OK;
  if (!v || !f || !start || n_tri == 0 || !out_xyz || !out_normal || !out_tri) return NKSR_E_INVALID;
  k_sample_surface<<<grid_for(n, kSampleThreads), kSampleThreads, 0, as_stream(stream)>>>(
      v, f, n_tri, start, n, mix64((uint64_t)seed), out_xyz, out_normal, out_tri);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_metric_nearest(const nksr_svh_t* svh, const float* xyz, const float* normal, const int32_t* range, float* box,
                        int64_t n_pts, const float* query, const float* query_normal, int64_t m, const float* origin3,
                        int start_level, float* out_dist, int32_t* out_idx, float* out_dot, int32_t* far_list,
                        int32_t* far_count, void* stream) {
  if (!svh || !xyz || !range || !box || !origin3 || !far_count || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH ||
      start_level < 0 || n_pts < 1 || n_pts > INT32_MAX || m < 0 || m > INT32_MAX)
    return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  if (!query || !out_dist || !out_idx || !far_list) return NKSR_E_INVALID;
  cudaStream_t st = as_stream(stream);
  const int top = svh->depth - 1;
  const int64_t n_cells = svh->n[top];
  const int2* top_range = reinterpret_cast<const int2*>(range) + svh->offset[top];
  if (cudaMemsetAsync(far_count, 0, sizeof(int32_t), st) != cudaSuccess) return NKSR_E_CUDA;
  k_cell_boxes<<<grid_for(n_cells, kMetricWarps), kMetricWarps * 32, 0, st>>>(xyz, top_range, n_cells, box);
  NKSR_CHECK_LAUNCH();
  k_metric_nearest<<<grid_for(m, kMetricWarps), kMetricWarps * 32, 0, st>>>(
      *svh, xyz, normal, range, query, query_normal, m, origin3[0], origin3[1], origin3[2], start_level, out_dist,
      out_idx, out_dot, far_list, far_count);
  NKSR_CHECK_LAUNCH();
  // the far list's length stays on the device: a fixed grid strides over it
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return NKSR_E_CUDA;
  k_metric_far<<<4 * sms, kMetricWarps * 32, 0, st>>>(xyz, normal, top_range, box, n_cells, query, query_normal,
                                                      far_list, far_count, out_dist, out_idx, out_dot);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
