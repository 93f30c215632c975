// The interpolation of the neural field (DESIGN.md SPEC S17, row a6): u(x) = [phi_l(x)] over the given levels, with
// phi_l(x) = sum_s T3_s(tau) F_l[nbr27[b_l(x)][s]] -- the trilinear interpolation of SPEC S4 -- and its VJP
// dF_l[v] = sum_q T3_{slot(v)}(q) g_{q,l}; and its position Jacobian J = du/dx (SPEC S17a), J[a] = sum_s dT3_s/dtau_a / W_l
// F_l[nbr27[b_l(x)][s]], with the VJP dF_l[v] = sum_q sum_a dT3_{slot(v),a}(q) / W_l G_{q,a,l}.  The geometry (tau, T3,
// dT3) comes from kernel_eval.cuh, as in the kernel field.  Each kernel is one template: JAC = false is the value
// interpolation, JAC = true the Jacobian, on the same hierarchy walk and the same gather.
//
// Forward: a group of P lanes (P = the power of two >= C) per query, lane = channel.  On each axis one of the two outer
// tent weights is 0 (tau >= 0: the -1 side, else the +1 side), so only the 8 corners of the trilinear cell are read.
// The Jacobian reads them too, and on an axis in the snap zone |tau| < 2^-12 the 4 slots on the far side, whose tent
// derivative (-1/2 or +1/2) is not 0 although their tent value is.
// VJP: deterministic, no floating-point atomics -- the queries are Morton sorted, so the queries whose stencil on
// level l holds voxel v are the contiguous ranges (nksr_row_ranges) of v's 27 neighbours; one warp per voxel, lane =
// channel, gathers them in slot order and range order (the pattern of k_field_bwd_pass2 in field_bwd.cu).
#include "kernel_eval.cuh"

namespace {

constexpr int kWarpsPerBlock = 8;

__device__ __forceinline__ int given_column(unsigned mask, int l) { return __popc(mask & ((1u << l) - 1u)); }

// out[i][g*C + c] = phi_l(x_i)[c] for the g-th given level l; every column of every query is written.  JAC: also
// jac[i][a][g*C + c] = d phi_l(x_i)[c] / dx_a (every entry written), and out may be null
template <bool JAC>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
k_neural_interp(nksr_svh_t svh, nksr_feat_t feat, unsigned mask, const float* __restrict__ xyz, int64_t m, int lanes,
                float* __restrict__ out, float* __restrict__ jac) {
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
  float* orow = (!JAC || out) ? out + i * (int64_t)W : nullptr;
  for (int l = L - 1; l >= 0; --l) {
    if ((mask >> l) & 1u) {
      float acc = 0.f;
      float dj[3] = {0.f, 0.f, 0.f};
      float iw = 0.f;
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
            const StencilWeights w = stencil_weights(tx, ty, tz, dx, dy, dz);
            const float zc = __ldg(z + (int64_t)nb * C + c);
            acc = fmaf(w.T3(), zc, acc);
            if constexpr (JAC) {
#pragma unroll
              for (int a = 0; a < 3; ++a) dj[a] = fmaf(w.dT3(a), zc, dj[a]);
            }
          }
        }
        if constexpr (JAC) {
          // snap zone of axis a: the far-side slots d_a = -s_a (tent value 0, derivative -+1/2), the other two axes
          // on their corners {0, s}; on any other slot off the corners one tent factor of dT3_a is 0
          const float tau[3] = {tx, ty, tz};
          const int sg[3] = {sx, sy, sz};
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            if (!(fabsf(tau[a]) < NKSR_TENT_SNAP)) continue;
            const int b0 = a == 0 ? 1 : 0, b1 = a == 2 ? 1 : 2;
            for (int k = 0; k < 4; ++k) {
              int d[3];
              d[a] = -sg[a];
              d[b0] = (k & 2) ? sg[b0] : 0;
              d[b1] = (k & 1) ? sg[b1] : 0;
              const int nb = __ldg(nrow + (d[0] + 1) * 9 + (d[1] + 1) * 3 + (d[2] + 1));
              if (nb >= 0 && c < C)
                dj[a] = fmaf(stencil_weights(tx, ty, tz, d[0], d[1], d[2]).dT3(a), __ldg(z + (int64_t)nb * C + c),
                             dj[a]);
            }
          }
          iw = (float)inv;
        }
      }
      if (c < C) {
        const int o = given_column(mask, l) * C + c;
        if (!JAC || out) orow[o] = acc;
        if constexpr (JAC) {
          float* jrow = jac + i * (int64_t)(3 * W) + o;
          jrow[0] = dj[0] * iw;
          jrow[W] = dj[1] * iw;
          jrow[2 * W] = dj[2] * iw;
        }
      }
    }
    if (l > 0 && idx >= 0) idx = __ldg(svh.child8[l] + (int64_t)idx * 8 + child_octant(h, l));
  }
}

// dF_l[v][c] = sum over v's neighbours u (slot order), over the sorted queries q of u's range (range order) of
// T3_{slot of v in u's stencil}(tau_q) * g[q][col(l)*C + c]; one warp per voxel of level l, lane = channel.
// JAC: g is (m, 3, W) and the weight of g[q][a][col(l)*C + c] is dT3_a / W_l
template <bool JAC>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
k_neural_interp_vjp(nksr_svh_t svh, int C, int W, int col, int l, const float* __restrict__ xyz,
                    const int32_t* __restrict__ range, const float* __restrict__ g, float* __restrict__ dfeat) {
  const int lane = threadIdx.x & 31;
  const int64_t v = blockIdx.x * (int64_t)kWarpsPerBlock + (threadIdx.x >> 5);
  if (v >= svh.n[l]) return;
  const double inv = (1.0 / (double)svh.voxel_size) * (1.0 / (double)(1 << l));
  const bool live = lane < C;
  const int64_t gstride = JAC ? 3 * (int64_t)W : W;
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
      const StencilWeights w =
          stencil_weights(local_coord(px, inv, cx), local_coord(py, inv, cy), local_coord(pz, inv, cz), dx, dy, dz);
      if (!live) continue;
      const float* gq = gc + (int64_t)q * gstride;
      if constexpr (JAC) {
        acc = fmaf(w.dT3(0), __ldg(gq), acc);
        acc = fmaf(w.dT3(1), __ldg(gq + W), acc);
        acc = fmaf(w.dT3(2), __ldg(gq + 2 * W), acc);
      } else {
        acc = fmaf(w.T3(), __ldg(gq), acc);
      }
    }
  }
  if (live) dfeat[(svh.offset[l] + v) * C + lane] = JAC ? acc * (float)inv : acc;
}

int check_mask(const nksr_svh_t* svh, int channels, int level_mask) {
  if (!svh || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH) return NKSR_E_INVALID;
  if (channels < 1 || channels > 32) return NKSR_E_INVALID;
  if (level_mask <= 0 || (level_mask >> svh->depth) != 0) return NKSR_E_INVALID;
  return NKSR_OK;
}

template <bool JAC>
int launch_interp(const nksr_svh_t* svh, const nksr_feat_t* feat, int level_mask, const float* xyz, int64_t m,
                  float* out, float* jac, void* stream) {
  if (!feat) return NKSR_E_INVALID;
  int rc = check_mask(svh, feat->channels, level_mask);
  if (rc != NKSR_OK) return rc;
  if (m < 0 || (m > 0 && (!xyz || (JAC ? !jac : !out)))) return NKSR_E_INVALID;
  for (int l = 0; l < svh->depth; ++l)
    if (((level_mask >> l) & 1) && svh->n[l] > 0 && !feat->z[l]) return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  int lanes = 1;
  while (lanes < feat->channels) lanes <<= 1;
  const int64_t threads = m * lanes;
  k_neural_interp<JAC><<<grid_for(threads, kWarpsPerBlock * 32), kWarpsPerBlock * 32, 0, as_stream(stream)>>>(
      *svh, *feat, (unsigned)level_mask, xyz, m, lanes, out, jac);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

template <bool JAC>
int launch_vjp(const nksr_svh_t* svh, int channels, int level_mask, const float* xyz, const int32_t* range, int64_t m,
               const float* grad, float* dfeat, void* stream) {
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
    k_neural_interp_vjp<JAC><<<grid_for(svh->n[l], kWarpsPerBlock), kWarpsPerBlock * 32, 0, s>>>(
        *svh, channels, W, col, l, xyz, range, grad, dfeat);
  }
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // namespace

extern "C" {

int nksr_neural_interp(const nksr_svh_t* svh, const nksr_feat_t* feat, int level_mask, const float* xyz, int64_t m,
                       float* out, void* stream) {
  return launch_interp<false>(svh, feat, level_mask, xyz, m, out, nullptr, stream);
}

int nksr_neural_interp_vjp(const nksr_svh_t* svh, int channels, int level_mask, const float* xyz,
                           const int32_t* range, int64_t m, const float* grad, float* dfeat, void* stream) {
  return launch_vjp<false>(svh, channels, level_mask, xyz, range, m, grad, dfeat, stream);
}

int nksr_neural_interp_jacobian(const nksr_svh_t* svh, const nksr_feat_t* feat, int level_mask, const float* xyz,
                                int64_t m, float* out, float* jac, void* stream) {
  return launch_interp<true>(svh, feat, level_mask, xyz, m, out, jac, stream);
}

int nksr_neural_interp_jacobian_vjp(const nksr_svh_t* svh, int channels, int level_mask, const float* xyz,
                                    const int32_t* range, int64_t m, const float* grad, float* dfeat, void* stream) {
  return launch_vjp<true>(svh, channels, level_mask, xyz, range, m, grad, dfeat, stream);
}

}  // extern "C"
