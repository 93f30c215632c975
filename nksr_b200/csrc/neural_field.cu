// The interpolation of the neural field (DESIGN.md SPEC S17, row a6): u(x) = [phi_l(x)] over the given levels, with
// phi_l(x) = sum_s T3_s(tau) F_l[nbr27[b_l(x)][s]] -- the trilinear interpolation of SPEC S4 -- and its VJP
// dF_l[v] = sum_q T3_{slot(v)}(q) g_{q,l}.  The geometry (tau, T3) comes from kernel_eval.cuh, as in the kernel field.
//
// Forward: a group of P lanes (P = the power of two >= C) per query, lane = channel.  On each axis one of the two outer
// tent weights is 0 (tau >= 0: the -1 side, else the +1 side), so only the 8 corners of the trilinear cell are read.
// VJP: deterministic, no floating-point atomics -- the queries are Morton sorted, so the queries whose stencil on
// level l holds voxel v are the contiguous ranges (nksr_row_ranges) of v's 27 neighbours; one warp per voxel, lane =
// channel, gathers them in slot order and range order (the pattern of k_field_bwd_pass2 in field_bwd.cu).
#include "kernel_eval.cuh"

namespace {

constexpr int kWarpsPerBlock = 8;

__device__ __forceinline__ int given_column(unsigned mask, int l) { return __popc(mask & ((1u << l) - 1u)); }

// out[i][g*C + c] = phi_l(x_i)[c] for the g-th given level l; every column of every query is written
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
k_neural_interp(nksr_svh_t svh, nksr_feat_t feat, unsigned mask, const float* __restrict__ xyz, int64_t m, int lanes,
                float* __restrict__ out) {
  const int gsize = lanes;                           // lanes per query (power of two, >= C)
  const int c = (threadIdx.x & 31) & (gsize - 1);
  const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) / gsize;
  if (i >= m) return;
  const int C = feat.channels;
  const int W = C * __popc(mask);
  const float px = __ldg(xyz + 3 * i), py = __ldg(xyz + 3 * i + 1), pz = __ldg(xyz + 3 * i + 2);
  int3 h;
  const bool in_range = half_voxel(px, py, pz, svh.voxel_size * 0.5f, h);
  const int L = svh.depth;
  const double inv0 = 1.0 / (double)svh.voxel_size;
  // containing voxels as k_evaluate / k_locate find them: the coarsest level by search, then child8 down
  int idx = -1;
  if (in_range && svh.n[L - 1] > 0)
    idx = find_key(svh.keys[L - 1], svh.n[L - 1], morton3(h.x >> L, h.y >> L, h.z >> L));
  float* orow = out + i * (int64_t)W;
  for (int l = L - 1; l >= 0; --l) {
    if ((mask >> l) & 1u) {
      float acc = 0.f;
      if (idx >= 0) {
        const int ux = h.x >> (l + 1), uy = h.y >> (l + 1), uz = h.z >> (l + 1);
        const double inv = inv0 * (1.0 / (double)(1 << l));
        const float tx = local_coord(px, inv, voxel_centre(ux, l));
        const float ty = local_coord(py, inv, voxel_centre(uy, l));
        const float tz = local_coord(pz, inv, voxel_centre(uz, l));
        const int sx = tx >= 0.f ? 1 : -1, sy = ty >= 0.f ? 1 : -1, sz = tz >= 0.f ? 1 : -1;
        const int32_t* nrow = svh.nbr27[l] + (int64_t)idx * 27;
        const float* z = feat.z[l];
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const int dx = (k & 4) ? sx : 0, dy = (k & 2) ? sy : 0, dz = (k & 1) ? sz : 0;
          const int nb = __ldg(nrow + (dx + 1) * 9 + (dy + 1) * 3 + (dz + 1));
          if (nb >= 0 && c < C) {
            const float t = stencil_weights(tx, ty, tz, dx, dy, dz).T3();
            acc = fmaf(t, __ldg(z + (int64_t)nb * C + c), acc);
          }
        }
      }
      if (c < C) orow[given_column(mask, l) * C + c] = acc;
    }
    if (l > 0 && idx >= 0) idx = __ldg(svh.child8[l] + (int64_t)idx * 8 + child_octant(h, l));
  }
}

// dF_l[v][c] = sum over v's neighbours u (slot order), over the sorted queries q of u's range (range order) of
// T3_{slot of v in u's stencil}(tau_q) * g[q][col(l)*C + c]; one warp per voxel of level l, lane = channel
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
k_neural_interp_vjp(nksr_svh_t svh, int C, int W, int col, int l, const float* __restrict__ xyz,
                    const int32_t* __restrict__ range, const float* __restrict__ g, float* __restrict__ dfeat) {
  const int lane = threadIdx.x & 31;
  const int64_t v = blockIdx.x * (int64_t)kWarpsPerBlock + (threadIdx.x >> 5);
  if (v >= svh.n[l]) return;
  const double inv = (1.0 / (double)svh.voxel_size) * (1.0 / (double)(1 << l));
  const bool live = lane < C;
  const float* gc = g + col * C + (live ? lane : 0);
  float acc = 0.f;
  for (int s = 0; s < 27; ++s) {
    const int u = __ldg(svh.nbr27[l] + v * 27 + s);
    if (u < 0) continue;
    const int2 r = __ldg(reinterpret_cast<const int2*>(range) + svh.offset[l] + u);
    if (r.x >= r.y) continue;
    int ux, uy, uz;
    morton3_decode(__ldg(svh.keys[l] + u), ux, uy, uz);
    const double cx = voxel_centre(ux, l), cy = voxel_centre(uy, l), cz = voxel_centre(uz, l);
    int dx, dy, dz;
    slot_to_d(26 - s, dx, dy, dz);                   // v sits at offset -d(s) from u
    for (int q = r.x; q < r.y; ++q) {
      const float px = __ldg(xyz + 3 * (int64_t)q), py = __ldg(xyz + 3 * (int64_t)q + 1),
                  pz = __ldg(xyz + 3 * (int64_t)q + 2);
      const float t =
          stencil_weights(local_coord(px, inv, cx), local_coord(py, inv, cy), local_coord(pz, inv, cz), dx, dy, dz)
              .T3();
      if (live) acc = fmaf(t, __ldg(gc + (int64_t)q * W), acc);
    }
  }
  if (live) dfeat[(svh.offset[l] + v) * C + lane] = acc;
}

int check_mask(const nksr_svh_t* svh, int channels, int level_mask) {
  if (!svh || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH) return NKSR_E_INVALID;
  if (channels < 1 || channels > 32) return NKSR_E_INVALID;
  if (level_mask <= 0 || (level_mask >> svh->depth) != 0) return NKSR_E_INVALID;
  return NKSR_OK;
}

}  // namespace

extern "C" {

int nksr_neural_interp(const nksr_svh_t* svh, const nksr_feat_t* feat, int level_mask, const float* xyz, int64_t m,
                       float* out, void* stream) {
  if (!feat) return NKSR_E_INVALID;
  int rc = check_mask(svh, feat->channels, level_mask);
  if (rc != NKSR_OK) return rc;
  if (m < 0 || (m > 0 && (!xyz || !out))) return NKSR_E_INVALID;
  for (int l = 0; l < svh->depth; ++l)
    if (((level_mask >> l) & 1) && svh->n[l] > 0 && !feat->z[l]) return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  int lanes = 1;
  while (lanes < feat->channels) lanes <<= 1;
  const int64_t threads = m * lanes;
  k_neural_interp<<<grid_for(threads, kWarpsPerBlock * 32), kWarpsPerBlock * 32, 0, as_stream(stream)>>>(
      *svh, *feat, (unsigned)level_mask, xyz, m, lanes, out);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_neural_interp_vjp(const nksr_svh_t* svh, int channels, int level_mask, const float* xyz,
                           const int32_t* range, int64_t m, const float* grad, float* dfeat, void* stream) {
  int rc = check_mask(svh, channels, level_mask);
  if (rc != NKSR_OK) return rc;
  if (m < 0 || !dfeat || (m > 0 && (!xyz || !range || !grad))) return NKSR_E_INVALID;
  cudaStream_t s = as_stream(stream);
  const int W = channels * __builtin_popcount((unsigned)level_mask);
  for (int l = 0; l < svh->depth; ++l) {
    if (!((level_mask >> l) & 1) || svh->n[l] == 0) continue;
    if (m == 0) {
      if (cudaMemsetAsync(dfeat + svh->offset[l] * channels, 0, svh->n[l] * channels * sizeof(float), s) != cudaSuccess)
        return NKSR_E_CUDA;
      continue;
    }
    const int col = __builtin_popcount((unsigned)level_mask & ((1u << l) - 1u));
    k_neural_interp_vjp<<<grid_for(svh->n[l], kWarpsPerBlock), kWarpsPerBlock * 32, 0, s>>>(*svh, channels, W, col, l,
                                                                                         xyz, range, grad, dfeat);
  }
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
