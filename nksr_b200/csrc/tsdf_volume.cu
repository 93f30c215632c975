// Volume ground truth from sensor rays (the PointTSDFVolume of the reference's groundtruth.bin, consumed by
// dataset/av_gt_geometry.py:141-173 and models/loss.py:221-249).  DESIGN.md SPEC S19.
//
// One thread per ray walks the cells of the dense node grid with a 3D-DDA (Amanatides-Woo), in fp64 and without
// fused multiply-adds (Makefile: --fmad=false), so the traversal and the signed distances are the plain IEEE
// expressions oracle/gt_volume.py evaluates in numpy.
// k_tsdf_init:     key = ~0 (no near observation), volume = NaN (unknown).
// k_tsdf_near:     pass 1, the part of the ray within [r - tau - h, r + tau]: 64-bit atomicMin of
//                  (fp32 bits of |sdf| / tau) << 32 | ray index on the nodes with |sdf| < tau.
// k_tsdf_free:     pass 2, from the ray's start: volume = 1 on nodes with sdf >= tau, up to the first node that holds
//                  a near observation of any ray.
// k_tsdf_finalise: near nodes get sdf / tau of the winning ray, recomputed by the same device function.
// Integer atomics and idempotent stores only: the volume is bitwise repeatable, and its classes do not depend on the
// order of the rays.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kRayThreads = 256;
constexpr int kNodeThreads = 256;
constexpr uint64_t kNoKey = ~0ull;

struct Grid {
  double lo[3];   // volume_min: node 0
  double h;
  int64_t dims[3];
  double tau;
};

struct Ray {
  double s[3], d[3], r;
};

// ray j: s -> p, unit d, length r; false for a non-finite input or a zero length (SPEC S19)
__device__ __forceinline__ bool load_ray(const float* __restrict__ xyz, const float* __restrict__ sensor, int64_t j,
                                         Ray& R) {
  double p[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    R.s[a] = (double)__ldg(sensor + 3 * j + a);
    p[a] = (double)__ldg(xyz + 3 * j + a);
  }
  const double vx = p[0] - R.s[0], vy = p[1] - R.s[1], vz = p[2] - R.s[2];
  R.r = sqrt(vx * vx + vy * vy + vz * vz);
  if (!isfinite(R.r) || !(R.r > 0.0)) return false;
  R.d[0] = vx / R.r;
  R.d[1] = vy / R.r;
  R.d[2] = vz / R.r;
  return true;
}

// sdf = r - <c - s, d> at node (ix, iy, iz), c = lo + i h
__device__ __forceinline__ double node_sdf(const Grid& G, const Ray& R, const int64_t* i) {
  const double cx = G.lo[0] + (double)i[0] * G.h - R.s[0];
  const double cy = G.lo[1] + (double)i[1] * G.h - R.s[1];
  const double cz = G.lo[2] + (double)i[2] * G.h - R.s[2];
  return R.r - (cx * R.d[0] + cy * R.d[1] + cz * R.d[2]);
}

// clip [t_lo, r + tau] to the box (the union of the cells, [lo - h/2, lo + (dims - 1/2) h]) by the slab test
__device__ __forceinline__ bool clip_ray(const Grid& G, const Ray& R, double t_lo, double& t0, double& t1) {
  t0 = t_lo;
  t1 = R.r + G.tau;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double lo = G.lo[a] - 0.5 * G.h, hi = G.lo[a] + ((double)G.dims[a] - 0.5) * G.h;
    if (R.d[a] == 0.0) {
      if (R.s[a] < lo || R.s[a] > hi) return false;
      continue;
    }
    double ta = (lo - R.s[a]) / R.d[a], tb = (hi - R.s[a]) / R.d[a];
    if (ta > tb) { const double t = ta; ta = tb; tb = t; }
    t0 = fmax(t0, ta);
    t1 = fmin(t1, tb);
  }
  return t0 < t1;
}

// Amanatides-Woo walk over the cells the ray passes through on [t0, t1], in order of entry parameter; visit(i, t_entry)
// returns false to stop.  Boundary k of axis a (between cells k - 1 and k) lies at lo + (k - 1/2) h; on equal exit
// parameters the lower axis steps first.
template <typename Visit>
__device__ __forceinline__ void walk(const Grid& G, const Ray& R, double t0, double t1, Visit visit) {
  int64_t i[3], step[3];
  double tmax[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const double x = R.s[a] + t0 * R.d[a];
    int64_t c = (int64_t)floor((x - (G.lo[a] - 0.5 * G.h)) / G.h);
    c = c < 0 ? 0 : (c >= G.dims[a] ? G.dims[a] - 1 : c);
    i[a] = c;
    step[a] = R.d[a] > 0.0 ? 1 : (R.d[a] < 0.0 ? -1 : 0);
    tmax[a] = step[a] == 0 ? INFINITY
                           : (G.lo[a] + ((double)(c + (step[a] > 0 ? 1 : 0)) - 0.5) * G.h - R.s[a]) / R.d[a];
  }
  double te = t0;
  for (;;) {
    if (!visit(i, te)) return;
    // the axis is branched on, not used as an index: the state stays in registers
#define NKSR_DDA_STEP(a)                                                                          \
  {                                                                                               \
    if (!(tmax[a] < t1)) return;                                                                  \
    te = tmax[a];                                                                                 \
    i[a] += step[a];                                                                              \
    if (i[a] < 0 || i[a] >= G.dims[a]) return;                                                    \
    tmax[a] = (G.lo[a] + ((double)(i[a] + (step[a] > 0 ? 1 : 0)) - 0.5) * G.h - R.s[a]) / R.d[a]; \
  }
    if (tmax[0] <= tmax[1] && tmax[0] <= tmax[2]) NKSR_DDA_STEP(0)
    else if (tmax[1] <= tmax[2]) NKSR_DDA_STEP(1)
    else NKSR_DDA_STEP(2)
#undef NKSR_DDA_STEP
  }
}

__device__ __forceinline__ int64_t node_index(const Grid& G, const int64_t* i) {
  return (i[0] * G.dims[1] + i[1]) * G.dims[2] + i[2];
}

__global__ void __launch_bounds__(kNodeThreads)
k_tsdf_init(uint64_t* __restrict__ key, float* __restrict__ volume, int64_t n_nodes) {
  const int64_t v = blockIdx.x * (int64_t)kNodeThreads + threadIdx.x;
  if (v >= n_nodes) return;
  key[v] = kNoKey;
  volume[v] = __int_as_float(0x7fc00000);
}

__global__ void __launch_bounds__(kRayThreads)
k_tsdf_near(const float* __restrict__ xyz, const float* __restrict__ sensor, int64_t n, Grid G,
            unsigned long long* __restrict__ key) {
  const int64_t j = blockIdx.x * (int64_t)kRayThreads + threadIdx.x;
  if (j >= n) return;
  Ray R;
  if (!load_ray(xyz, sensor, j, R)) return;
  // a node within sqrt(3)/2 h of the ray has |t_c - t| < h for every t of its cell, so cells entered before
  // r - tau - h hold no node with sdf < tau
  double t0, t1;
  if (!clip_ray(G, R, fmax(0.0, R.r - G.tau - G.h), t0, t1)) return;
  walk(G, R, t0, t1, [&](const int64_t* i, double) {
    const double sdf = node_sdf(G, R, i);
    const double a = fabs(sdf);
    if (a < G.tau) {
      const float q = (float)(a / G.tau);
      atomicMin(key + node_index(G, i), ((unsigned long long)__float_as_uint(q) << 32) | (unsigned long long)j);
    }
    return true;
  });
}

__global__ void __launch_bounds__(kRayThreads)
k_tsdf_free(const float* __restrict__ xyz, const float* __restrict__ sensor, int64_t n, Grid G,
            const uint64_t* __restrict__ key, float* __restrict__ volume) {
  const int64_t j = blockIdx.x * (int64_t)kRayThreads + threadIdx.x;
  if (j >= n) return;
  Ray R;
  if (!load_ray(xyz, sensor, j, R)) return;
  double t0, t1;
  if (!clip_ray(G, R, 0.0, t0, t1)) return;
  const double t_last = R.r - G.tau + G.h;   // cells entered after this hold no node with sdf >= tau
  walk(G, R, t0, t1, [&](const int64_t* i, double te) {
    if (te > t_last) return false;
    const int64_t v = node_index(G, i);
    if (key[v] != kNoKey) return false;
    if (node_sdf(G, R, i) >= G.tau) volume[v] = 1.0f;
    return true;
  });
}

__global__ void __launch_bounds__(kNodeThreads)
k_tsdf_finalise(const float* __restrict__ xyz, const float* __restrict__ sensor, Grid G,
                const uint64_t* __restrict__ key, float* __restrict__ volume, int64_t n_nodes) {
  const int64_t v = blockIdx.x * (int64_t)kNodeThreads + threadIdx.x;
  if (v >= n_nodes) return;
  const uint64_t k = key[v];
  if (k == kNoKey) return;
  Ray R;
  load_ray(xyz, sensor, (int64_t)(k & 0xffffffffull), R);
  const int64_t i[3] = {v / (G.dims[1] * G.dims[2]), (v / G.dims[2]) % G.dims[1], v % G.dims[2]};
  volume[v] = (float)(node_sdf(G, R, i) / G.tau);
}

bool valid_dims(const int64_t* dims3) {
  if (!dims3) return false;
  int64_t total = 1;
  for (int a = 0; a < 3; ++a) {
    if (dims3[a] < 2 || dims3[a] > INT32_MAX) return false;
    total *= dims3[a];
    if (total > INT32_MAX) return false;
  }
  return true;
}

}  // namespace

extern "C" {

size_t nksr_tsdf_volume_workspace_bytes(const int64_t* dims3) {
  if (!valid_dims(dims3)) return 0;
  return sizeof(uint64_t) * (size_t)(dims3[0] * dims3[1] * dims3[2]);
}

int nksr_tsdf_volume(const float* xyz, const float* sensor, int64_t n, const float* volume_min3, float h,
                     const int64_t* dims3, float tau, float* volume, void* ws, size_t ws_bytes, void* stream) {
  if (!valid_dims(dims3) || !volume_min3 || !volume || n < 0 || n > INT32_MAX) return NKSR_E_INVALID;
  if (!(h > 0.0) || !isfinite(h) || !(tau > 0.0) || !isfinite(tau)) return NKSR_E_INVALID;
  for (int a = 0; a < 3; ++a)
    if (!isfinite(volume_min3[a])) return NKSR_E_INVALID;
  if (n > 0 && (!xyz || !sensor)) return NKSR_E_INVALID;
  const int64_t n_nodes = dims3[0] * dims3[1] * dims3[2];
  if (!ws || ws_bytes < nksr_tsdf_volume_workspace_bytes(dims3)) return NKSR_E_WORKSPACE;
  Grid G;
  for (int a = 0; a < 3; ++a) {
    G.lo[a] = (double)volume_min3[a];
    G.dims[a] = dims3[a];
  }
  G.h = (double)h;
  G.tau = (double)tau;
  uint64_t* key = static_cast<uint64_t*>(ws);
  cudaStream_t st = as_stream(stream);
  k_tsdf_init<<<grid_for(n_nodes, kNodeThreads), kNodeThreads, 0, st>>>(key, volume, n_nodes);
  NKSR_CHECK_LAUNCH();
  if (n == 0) return NKSR_OK;
  k_tsdf_near<<<grid_for(n, kRayThreads), kRayThreads, 0, st>>>(xyz, sensor, n, G,
                                                                  reinterpret_cast<unsigned long long*>(key));
  NKSR_CHECK_LAUNCH();
  k_tsdf_free<<<grid_for(n, kRayThreads), kRayThreads, 0, st>>>(xyz, sensor, n, G, key, volume);
  NKSR_CHECK_LAUNCH();
  k_tsdf_finalise<<<grid_for(n_nodes, kNodeThreads), kNodeThreads, 0, st>>>(xyz, sensor, G, key, volume, n_nodes);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
