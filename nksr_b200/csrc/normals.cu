// Normal estimation by voxel-neighbourhood PCA (SURVEY section 8(f) row 1).
// Replaces nksr.get_estimate_normal_preprocess_fn(knn, max_angle) (examples/recons_waymo.py:36);
// the open CPU twin it follows is examples/recons_waymo_cpu.py:21-41 (kNN-PCA normal, flip to the
// sensor side, drop grazing points).  Neighbourhood = the 27 voxels around the point's voxel of
// a single-level hierarchy sized to hold ~knn points, instead of an exact kNN search.
#include "knn_common.cuh"

namespace {

// moments of the points of each voxel about the voxel centre:
// m[0]=count, m[1..3]=sum d, m[4..9]=sum dxdx,dxdy,dxdz,dydy,dydz,dzdz
__global__ void k_voxel_moments(const int64_t* __restrict__ keys, int64_t n, const int32_t* __restrict__ range,
                                const float* __restrict__ xyz, float w, float* __restrict__ mom) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int ux, uy, uz;
  morton3_decode(__ldg(keys + i), ux, uy, uz);
  const int off = level_offset(0);
  const float cx = ((float)(ux - off) + 0.5f) * w, cy = ((float)(uy - off) + 0.5f) * w,
              cz = ((float)(uz - off) + 0.5f) * w;
  float m[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) m[k] = 0.f;
  const int rb = range[2 * i], re = range[2 * i + 1];
  for (int q = rb; q < re; ++q) {
    const float dx = __ldg(xyz + 3 * (int64_t)q) - cx, dy = __ldg(xyz + 3 * (int64_t)q + 1) - cy,
                dz = __ldg(xyz + 3 * (int64_t)q + 2) - cz;
    m[0] += 1.f; m[1] += dx; m[2] += dy; m[3] += dz;
    m[4] += dx * dx; m[5] += dx * dy; m[6] += dx * dz; m[7] += dy * dy; m[8] += dy * dz; m[9] += dz * dz;
  }
#pragma unroll
  for (int k = 0; k < 10; ++k) mom[i * 10 + k] = m[k];
}

__device__ __forceinline__ void jacobi_rotate(double a[3][3], double v[3][3], int p, int q) {
  if (fabs(a[p][q]) < 1e-300) return;
  double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
  double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
  double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
  for (int k = 0; k < 3; ++k) {
    double akp = a[k][p], akq = a[k][q];
    a[k][p] = c * akp - s * akq;
    a[k][q] = s * akp + c * akq;
  }
  for (int k = 0; k < 3; ++k) {
    double apk = a[p][k], aqk = a[q][k];
    a[p][k] = c * apk - s * aqk;
    a[q][k] = s * apk + c * aqk;
  }
  for (int k = 0; k < 3; ++k) {
    double vkp = v[k][p], vkq = v[k][q];
    v[k][p] = c * vkp - s * vkq;
    v[k][q] = s * vkp + c * vkq;
  }
}

// covariance of the 27-neighbourhood -> eigenvector of the smallest eigenvalue
__global__ void k_voxel_pca(const int32_t* __restrict__ nbr27, const float* __restrict__ mom, int64_t n, float w,
                            float* __restrict__ normal) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  double cnt = 0, s[3] = {0, 0, 0}, m2[6] = {0, 0, 0, 0, 0, 0};
  for (int sl = 0; sl < 27; ++sl) {
    const int nb = __ldg(nbr27 + i * 27 + sl);
    if (nb < 0) continue;
    const float* m = mom + (int64_t)nb * 10;
    const double c = m[0];
    if (c == 0.0) continue;
    int dx, dy, dz;
    slot_to_d(sl, dx, dy, dz);
    const double ox = dx * (double)w, oy = dy * (double)w, oz = dz * (double)w;  // neighbour centre - own centre
    const double sx = m[1], sy = m[2], sz = m[3];
    cnt += c;
    s[0] += sx + c * ox; s[1] += sy + c * oy; s[2] += sz + c * oz;
    m2[0] += m[4] + 2 * sx * ox + c * ox * ox;
    m2[1] += m[5] + sx * oy + sy * ox + c * ox * oy;
    m2[2] += m[6] + sx * oz + sz * ox + c * ox * oz;
    m2[3] += m[7] + 2 * sy * oy + c * oy * oy;
    m2[4] += m[8] + sy * oz + sz * oy + c * oy * oz;
    m2[5] += m[9] + 2 * sz * oz + c * oz * oz;
  }
  float out[3] = {0.f, 0.f, 1.f};
  if (cnt >= 3.0) {
    const double ic = 1.0 / cnt;
    const double mx = s[0] * ic, my = s[1] * ic, mz = s[2] * ic;
    double a[3][3], v[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
    a[0][0] = m2[0] * ic - mx * mx; a[0][1] = a[1][0] = m2[1] * ic - mx * my; a[0][2] = a[2][0] = m2[2] * ic - mx * mz;
    a[1][1] = m2[3] * ic - my * my; a[1][2] = a[2][1] = m2[4] * ic - my * mz; a[2][2] = m2[5] * ic - mz * mz;
    for (int sweep = 0; sweep < 8; ++sweep) {
      jacobi_rotate(a, v, 0, 1);
      jacobi_rotate(a, v, 0, 2);
      jacobi_rotate(a, v, 1, 2);
    }
    int k = 0;
    if (a[1][1] < a[k][k]) k = 1;
    if (a[2][2] < a[k][k]) k = 2;
    double nx = v[0][k], ny = v[1][k], nz = v[2][k];
    double nn = sqrt(nx * nx + ny * ny + nz * nz);
    if (nn > 0) { out[0] = (float)(nx / nn); out[1] = (float)(ny / nn); out[2] = (float)(nz / nn); }
  }
  normal[3 * i] = out[0];
  normal[3 * i + 1] = out[1];
  normal[3 * i + 2] = out[2];
}

// per point: voxel normal, flipped to the sensor side; keep = |cos(view, n)| > cos_min
__global__ void k_orient_normals(const float* __restrict__ xyz, const float* __restrict__ sensor,
                                 const int32_t* __restrict__ base, const float* __restrict__ vox_normal, int64_t m,
                                 float cos_min, float* __restrict__ normal, int32_t* __restrict__ keep) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= m) return;
  const int b = base[i];
  float nx = 0.f, ny = 0.f, nz = 1.f;
  if (b >= 0) { nx = vox_normal[3 * (int64_t)b]; ny = vox_normal[3 * (int64_t)b + 1]; nz = vox_normal[3 * (int64_t)b + 2]; }
  float vx = sensor[3 * i] - xyz[3 * i], vy = sensor[3 * i + 1] - xyz[3 * i + 1], vz = sensor[3 * i + 2] - xyz[3 * i + 2];
  const float vn = sqrtf(vx * vx + vy * vy + vz * vz) + 1e-6f;   // examples/recons_waymo_cpu.py:32-33
  vx /= vn; vy /= vn; vz /= vn;
  const float c = vx * nx + vy * ny + vz * nz;
  if (c < 0.f) { nx = -nx; ny = -ny; nz = -nz; }
  normal[3 * i] = nx; normal[3 * i + 1] = ny; normal[3 * i + 2] = nz;
  keep[i] = (b >= 0 && fabsf(c) > cos_min) ? 1 : 0;
}


// ---------------------------------------------------------------------------------------------------------
// Exact k-nearest-neighbour PCA normals (examples/recons_waymo_cpu.py:26: pcu.estimate_point_cloud_normals_knn
// (xyz, 64)), on a multi-level voxel hash of the Morton-sorted points.  One warp per point:
//   * pick the finest level whose 27-voxel block around the point holds >= 3k points (then the k-th neighbour
//     lies, for surface-like data, within one voxel size of the point);
//   * stream the block's points (contiguous ranges: the points are sorted by Morton key), keep the candidates
//     closer than the current bound in a 128-entry shared-memory buffer, and whenever it fills sort it (bitonic
//     network on packed (distance, index) words) and keep the k best, tightening the bound;
//   * the answer is EXACT when the k-th distance does not exceed the voxel size of the level (everything closer
//     than that lies inside the block); otherwise repeat one level coarser.
// Then the 3 x 3 covariance of the k neighbours (self included) about their mean, its eigenvector of the smallest
// eigenvalue (Jacobi, fp64), orientation to the sensor side and the grazing-angle flag.
constexpr int kKnnWarps = 8;

__global__ void __launch_bounds__(kKnnWarps * 32)
k_knn_normals(const nksr_svh_t svh, const float* __restrict__ xyz, const float* __restrict__ sensor,
              const int32_t* __restrict__ base, const int32_t* __restrict__ range, const int64_t m, const int k,
              const float cos_min, float* __restrict__ normal, int32_t* __restrict__ keep,
              float* __restrict__ eig, int32_t* __restrict__ inexact) {
  __shared__ unsigned long long buf[kKnnWarps][kKnnBuf];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t i = blockIdx.x * (int64_t)kKnnWarps + wid;
  if (i >= m) return;
  unsigned long long* key = buf[wid];
  const float px = __ldg(xyz + 3 * i), py = __ldg(xyz + 3 * i + 1), pz = __ldg(xyz + 3 * i + 2);
  const int L = svh.depth;
  int got = 0;
  bool exact = false;
  for (int l = 0; l < L; ++l) {
    const int b = __ldg(base + (int64_t)l * m + i);
    int rb = 0, re = 0;
    if (b >= 0 && lane < 27) {
      const int v = __ldg(svh.nbr27[l] + (int64_t)b * 27 + lane);
      if (v >= 0) {
        const int2 r = __ldg(reinterpret_cast<const int2*>(range) + svh.offset[l] + v);
        rb = r.x; re = r.y;
      }
    }
    int total = re - rb;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
    if (total < 3 * k && l + 1 < L) continue;
    // ---- scan the block
    int fill;
    float bound;
    const float hl = svh.voxel_size * (float)(1 << l);
    // only neighbours within one cell size can make this level's answer acceptable: prune everything else up front
    // (about two thirds of the block for surface-like data); the coarsest level answers unconditionally
    const float full = l + 1 < L ? hl * hl * 1.0000005f : 3.0e38f;
    // first try a tighter radius: for surface-like data the block's `total` points cover ~9 h^2, so ~1.7 k of them lie
    // within r^2 = 9 h^2 * 1.7 k / (pi * total); then the candidate buffer rarely overflows (one sort per point instead
    // of two or three -- the bitonic network is this kernel's cost).  Too tight (fewer than k found): scan again.
    float first = 9.0f * hl * hl * (1.7f * (float)k) / (3.14159265f * (float)total);
    first = first < full ? first : full;
    float dk2 = 0.f;
    for (int attempt = 0; attempt < 2; ++attempt) {
      const float b0 = attempt == 0 ? first : full;
      knn_reset(key, fill, bound, lane, b0);
      for (int s = 0; s < 27; ++s) {
        const int sb = __shfl_sync(0xffffffffu, rb, s), se = __shfl_sync(0xffffffffu, re, s);
        knn_scan_range(key, fill, bound, k, xyz, sb, se, px, py, pz, lane);
      }
      got = knn_finish(key, fill, k, dk2, lane);
      if (got == k || b0 >= full) break;
    }
    exact = got == k && dk2 <= hl * hl;
    if (exact || l + 1 == L) break;
  }
  // ---- covariance of the neighbours about their mean (coordinates relative to the query point)
  float s[9];
#pragma unroll
  for (int a = 0; a < 9; ++a) s[a] = 0.f;
  for (int t = lane; t < got; t += 32) {
    const int q = (int)(unsigned)(key[t] & 0xffffffffull);
    const float dx = __ldg(xyz + 3 * (int64_t)q) - px, dy = __ldg(xyz + 3 * (int64_t)q + 1) - py,
                dz = __ldg(xyz + 3 * (int64_t)q + 2) - pz;
    s[0] += dx; s[1] += dy; s[2] += dz;
    s[3] = fmaf(dx, dx, s[3]); s[4] = fmaf(dx, dy, s[4]); s[5] = fmaf(dx, dz, s[5]);
    s[6] = fmaf(dy, dy, s[6]); s[7] = fmaf(dy, dz, s[7]); s[8] = fmaf(dz, dz, s[8]);
  }
#pragma unroll
  for (int a = 0; a < 9; ++a) s[a] = warp_sum(s[a]);
  if (lane != 0) return;
  float out[3] = {0.f, 0.f, 1.f};
  double ev[3] = {0.0, 0.0, 0.0};
  if (got >= 3) {
    const double ic = 1.0 / (double)got;
    const double mx = s[0] * ic, my = s[1] * ic, mz = s[2] * ic;
    const double a00 = s[3] * ic - mx * mx, a01 = s[4] * ic - mx * my, a02 = s[5] * ic - mx * mz,
                 a11 = s[6] * ic - my * my, a12 = s[7] * ic - my * mz, a22 = s[8] * ic - mz * mz;
    // closed-form eigenvalues of the symmetric 3 x 3 covariance (trigonometric solution of the characteristic cubic,
    // fp64) and the eigenvector of the smallest one as the largest cross product of two rows of A - lambda I.
    // (The first version ran 8 Jacobi sweeps in fp64 per point: ~1 400 dependent instructions, a quarter of the kernel.)
    const double p1 = a01 * a01 + a02 * a02 + a12 * a12;
    const double q = (a00 + a11 + a22) / 3.0;
    const double b00 = a00 - q, b11 = a11 - q, b22 = a22 - q;
    const double p2 = b00 * b00 + b11 * b11 + b22 * b22 + 2.0 * p1;
    double e_lo = q, e_mid = q, e_hi = q;
    if (p2 > 0.0) {
      const double p = sqrt(p2 / 6.0), ip = 1.0 / p;
      const double c00 = b00 * ip, c11 = b11 * ip, c22 = b22 * ip, c01 = a01 * ip, c02 = a02 * ip, c12 = a12 * ip;
      double r = 0.5 * (c00 * (c11 * c22 - c12 * c12) - c01 * (c01 * c22 - c12 * c02) + c02 * (c01 * c12 - c11 * c02));
      r = r < -1.0 ? -1.0 : (r > 1.0 ? 1.0 : r);
      const double phi = acos(r) / 3.0;
      e_hi = q + 2.0 * p * cos(phi);
      e_lo = q + 2.0 * p * cos(phi + 2.0943951023931953);      // + 2 pi / 3
      e_mid = 3.0 * q - e_hi - e_lo;
    }
    const double m00 = a00 - e_lo, m11 = a11 - e_lo, m22 = a22 - e_lo;
    // rows r0 = (m00, a01, a02), r1 = (a01, m11, a12), r2 = (a02, a12, m22)
    const double x01 = a01 * a12 - a02 * m11, y01 = a02 * a01 - m00 * a12, z01 = m00 * m11 - a01 * a01;   // r0 x r1
    const double x02 = a01 * m22 - a02 * a12, y02 = a02 * a02 - m00 * m22, z02 = m00 * a12 - a01 * a02;   // r0 x r2
    const double x12 = m11 * m22 - a12 * a12, y12 = a12 * a02 - a01 * m22, z12 = a01 * a12 - m11 * a02;   // r1 x r2
    const double n01 = x01 * x01 + y01 * y01 + z01 * z01, n02 = x02 * x02 + y02 * y02 + z02 * z02,
                 n12 = x12 * x12 + y12 * y12 + z12 * z12;
    double nx = x01, ny = y01, nz = z01, nn = n01;
    if (n02 > nn) { nx = x02; ny = y02; nz = z02; nn = n02; }
    if (n12 > nn) { nx = x12; ny = y12; nz = z12; nn = n12; }
    if (nn > 0.0) {
      const double inv = 1.0 / sqrt(nn);
      out[0] = (float)(nx * inv); out[1] = (float)(ny * inv); out[2] = (float)(nz * inv);
    } else if (p2 > 0.0) {     // A - lambda I vanishes: a multiple of the identity shifted by a rank-0 part; keep z
      out[0] = 0.f; out[1] = 0.f; out[2] = 1.f;
    }
    ev[0] = e_lo; ev[1] = e_mid; ev[2] = e_hi;
  }
  float vx = 0.f, vy = 0.f, vz = 0.f, cs = 1.f;
  if (sensor) {
    vx = __ldg(sensor + 3 * i) - px; vy = __ldg(sensor + 3 * i + 1) - py; vz = __ldg(sensor + 3 * i + 2) - pz;
    const float vn = sqrtf(vx * vx + vy * vy + vz * vz) + 1e-6f;   // examples/recons_waymo_cpu.py:32-33
    vx /= vn; vy /= vn; vz /= vn;
    cs = vx * out[0] + vy * out[1] + vz * out[2];
    if (cs < 0.f) { out[0] = -out[0]; out[1] = -out[1]; out[2] = -out[2]; }   // :34-36
  }
  normal[3 * i] = out[0]; normal[3 * i + 1] = out[1]; normal[3 * i + 2] = out[2];
  if (keep) keep[i] = (got >= 3 && fabsf(cs) > cos_min) ? 1 : 0;               // :38-39
  if (eig) {   // ascending eigenvalues (tests skip degenerate neighbourhoods)
    double e0 = ev[0], e1 = ev[1], e2 = ev[2], tsw;
    if (e0 > e1) { tsw = e0; e0 = e1; e1 = tsw; }
    if (e1 > e2) { tsw = e1; e1 = e2; e2 = tsw; }
    if (e0 > e1) { tsw = e0; e0 = e1; e1 = tsw; }
    eig[3 * i] = (float)e0; eig[3 * i + 1] = (float)e1; eig[3 * i + 2] = (float)e2;
  }
  if (inexact && !exact) atomicAdd(inexact, 1);
}

}  // namespace

extern "C" {

int nksr_voxel_moments(const int64_t* keys, int64_t n, const int32_t* range, const float* xyz, float voxel_size,
                       float* mom, void* stream) {
  if (n == 0) return NKSR_OK;
  k_voxel_moments<<<grid_for(n, 128), 128, 0, as_stream(stream)>>>(keys, n, range, xyz, voxel_size, mom);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_voxel_pca_normals(const int32_t* nbr27, const float* mom, int64_t n, float voxel_size, float* normal,
                           void* stream) {
  if (n == 0) return NKSR_OK;
  k_voxel_pca<<<grid_for(n, 128), 128, 0, as_stream(stream)>>>(nbr27, mom, n, voxel_size, normal);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_orient_normals(const float* xyz, const float* sensor, const int32_t* base, const float* vox_normal,
                        int64_t m, float cos_min, float* normal, int32_t* keep, void* stream) {
  if (m == 0) return NKSR_OK;
  k_orient_normals<<<grid_for(m, 256), 256, 0, as_stream(stream)>>>(xyz, sensor, base, vox_normal, m, cos_min,
                                                                     normal, keep);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_knn_normals(const nksr_svh_t* svh, const float* xyz, const float* sensor, const int32_t* base,
                     const int32_t* range, int64_t m, int k, float cos_min, float* normal, int32_t* keep, float* eig,
                     int32_t* inexact, void* stream) {
  if (!svh || !xyz || !base || !range || !normal || k < 3 || k > 64 || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH)
    return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  k_knn_normals<<<grid_for(m, kKnnWarps), kKnnWarps * 32, 0, as_stream(stream)>>>(*svh, xyz, sensor, base, range, m, k,
                                                                                cos_min, normal, keep, eig, inexact);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
