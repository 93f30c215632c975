// Backward of the kernel field (DESIGN.md 4.6): the transpose evaluation dalpha = sum_q c_q E_q, the feature VJP of a
// row functional Q = sum_q sum_s omega_{q,s} E_q[n_s] with respect to z, and the regulariser VJP.
//
// Deterministic by construction, no floating-point atomics: the locations are Morton sorted, so the locations whose
// level-l stencil contains voxel v are the contiguous ranges (nksr_row_ranges) of v's 27 neighbours u.  Pass 1 (one
// warp per location, lane = stencil slot) forms the per-(location, level) vectors phi, dphi_a, psi, psi0, psi_a once;
// pass 2 (one warp per voxel, lane = channel) gathers them over the 27 ranges in slot order and range order, so every
// output is summed in one fixed order.  Both passes take the kernel's geometry from kernel_eval.cuh, as the forward
// does.
#include "kernel_eval.cuh"

namespace {

constexpr int kWarpsPerBlock = 8;

// per-(location, level) record of pass 1, `nq` vectors of C floats:
//   value rows:    phi, [psi]
//   gradient rows: phi, [psi0], and with the full gradient dphi_0..2, [psi_0..2]
// ([..] only when coefficient vectors are given, i.e. for the feature VJP)
__host__ __device__ __forceinline__ int record_vectors(int mode, bool full, bool psi) {
  if (mode == 0) return psi ? 2 : 1;
  const int per = full ? 4 : 1;       // phi (+ dphi_a) ; psi0 (+ psi_a)
  return psi ? 2 * per : per;
}

// pass 1.  coef: per location nvec x (1 or 3) floats (nvec = a1 ? 2 : 1); omega_(a,)s = sum_k coef[k(,a)] a_k[n_s].
template <bool GRAD, bool PSI>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
k_field_bwd_pass1(nksr_svh_t svh, nksr_feat_t feat, const float* __restrict__ xyz, const int32_t* __restrict__ base,
                  int64_t m, bool fullgrad, const float* __restrict__ a0, const float* __restrict__ a1,
                  const float* __restrict__ coef, float* __restrict__ rec) {
  const int lane = threadIdx.x & 31;
  const int64_t i = blockIdx.x * (int64_t)kWarpsPerBlock + (threadIdx.x >> 5);
  if (i >= m) return;
  const int C = feat.channels;
  const int L = svh.depth;
  const bool full = GRAD && fullgrad;
  const int nq = record_vectors(GRAD ? 1 : 0, full, PSI);
  const int nvec = a1 != nullptr ? 2 : 1;
  const int ncf = GRAD ? 3 : 1;
  float cf[2][3] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
  if (PSI) {
    for (int k = 0; k < nvec; ++k)
      for (int a = 0; a < ncf; ++a) cf[k][a] = __ldg(coef + (i * nvec + k) * ncf + a);
  }
  const float px = __ldg(xyz + 3 * i), py = __ldg(xyz + 3 * i + 1), pz = __ldg(xyz + 3 * i + 2);
  // a location outside the range has base -1 on every level (nksr_locate), so its h is never read
  int3 h;
  half_voxel(px, py, pz, svh.voxel_size * 0.5f, h);
  const double inv0 = 1.0 / (double)svh.voxel_size;
  int dx, dy, dz;
  slot_to_d(lane < 27 ? lane : 13, dx, dy, dz);
  for (int l = 0; l < L; ++l) {
    const int b = __ldg(base + (int64_t)l * m + i);
    if (b < 0) continue;                               // pass 2 never reads this record
    const double inv = inv0 * (1.0 / (double)(1 << l));
    const StencilWeights w = stencil_weights(local_coord(px, inv, voxel_centre(h.x >> (l + 1), l)),
                                             local_coord(py, inv, voxel_centre(h.y >> (l + 1), l)),
                                             local_coord(pz, inv, voxel_centre(h.z >> (l + 1), l)), dx, dy, dz);
    const int nb = lane < 27 ? __ldg(svh.nbr27[l] + (int64_t)b * 27 + lane) : -1;
    const bool ok = nb >= 0;
    const float iw = 1.f / (svh.voxel_size * (float)(1 << l));
    const float B3 = w.B3();
    const float T3 = ok ? w.T3() : 0.f;
    float dT3[3] = {0.f, 0.f, 0.f};
    if (full) {
      dT3[0] = ok ? w.dT3(0) : 0.f;
      dT3[1] = ok ? w.dT3(1) : 0.f;
      dT3[2] = ok ? w.dT3(2) : 0.f;
    }
    // psi weights of this slot: value rows omega B; gradient rows (sum_a omega_a dB_a) / W (psi0), omega_a B / W (psi_a)
    float wpsi = 0.f, wpsia[3] = {0.f, 0.f, 0.f};
    if (PSI && ok) {
      const int64_t g = svh.offset[l] + nb;
      const float v0 = __ldg(a0 + g), v1 = a1 != nullptr ? __ldg(a1 + g) : 0.f;
      float om[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) om[a] = a < ncf ? fmaf(cf[1][a], v1, cf[0][a] * v0) : 0.f;
      if (!GRAD) {
        wpsi = om[0] * B3;
      } else {
        wpsi = (om[0] * w.dB(0) + om[1] * w.dB(1) + om[2] * w.dB(2)) * iw;
        if (full) {
#pragma unroll
          for (int a = 0; a < 3; ++a) wpsia[a] = om[a] * B3 * iw;
        }
      }
    }
    const float* zr = feat.z[l] + (int64_t)(ok ? nb : 0) * C;
    float* out = rec + ((int64_t)i * L + l) * nq * C;
    float mine[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) mine[k] = 0.f;
    for (int c = 0; c < C; ++c) {
      const float zc = ok ? __ldg(zr + c) : 0.f;
      float v[8];
      int k = 0;
      v[k++] = warp_sum(T3 * zc);
      if (full)
        for (int a = 0; a < 3; ++a) v[k++] = warp_sum(dT3[a] * zc);
      if (PSI) {
        v[k++] = warp_sum(wpsi * zc);
        if (full)
          for (int a = 0; a < 3; ++a) v[k++] = warp_sum(wpsia[a] * zc);
      }
      if (lane == c)
#pragma unroll
        for (int j = 0; j < 8; ++j) mine[j] = j < k ? v[j] : 0.f;
    }
    if (lane < C)
      for (int k = 0; k < nq; ++k) out[k * C + lane] = mine[k];
  }
}

// pass 2, one warp per voxel v of level l, lane = channel.  Visits the neighbours u of v in slot order; v sits in
// slot 26 - s' of u's stencil (offset -d(s')); every location of u's range in sorted order.
//   VJP (dz_v += ...):  value     omega B phi + T psi
//                       gradient  sum_a omega_a (dB_a phi + B dphi_a) / W + T psi0 + sum_a dT_a psi_a
//   ADJ (dalpha_v = <z_v, Phi>):  value Phi = sum c B phi;  gradient Phi = sum_a c_a (dB_a phi + B dphi_a) / W
template <bool GRAD, bool ADJ>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
k_field_bwd_pass2(nksr_svh_t svh, nksr_feat_t feat, const float* __restrict__ xyz, const int32_t* __restrict__ range,
                  int l, bool fullgrad, const float* __restrict__ a0, const float* __restrict__ a1,
                  const float* __restrict__ coef, const float* __restrict__ rec, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t v = blockIdx.x * (int64_t)kWarpsPerBlock + (threadIdx.x >> 5);
  if (v >= svh.n[l]) return;
  const int C = feat.channels;
  const int L = svh.depth;
  const bool full = GRAD && fullgrad;
  const int nq = record_vectors(GRAD ? 1 : 0, full, !ADJ);
  const int nvec = a1 != nullptr ? 2 : 1;
  const int ncf = GRAD ? 3 : 1;
  const int64_t gv = svh.offset[l] + v;
  float av0 = 0.f, av1 = 0.f;
  if (!ADJ) {
    av0 = __ldg(a0 + gv);
    av1 = a1 != nullptr ? __ldg(a1 + gv) : 0.f;
  }
  const double inv = (1.0 / (double)svh.voxel_size) * (1.0 / (double)(1 << l));
  const float iw = 1.f / (svh.voxel_size * (float)(1 << l));
  const bool live = lane < C;
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
    slot_to_d(26 - s, dx, dy, dz);
    for (int q = r.x; q < r.y; ++q) {
      const float px = __ldg(xyz + 3 * (int64_t)q), py = __ldg(xyz + 3 * (int64_t)q + 1),
                  pz = __ldg(xyz + 3 * (int64_t)q + 2);
      const StencilWeights w =
          stencil_weights(local_coord(px, inv, cx), local_coord(py, inv, cy), local_coord(pz, inv, cz), dx, dy, dz);
      const float B3 = w.B3(), T3 = w.T3();
      const float dB[3] = {w.dB(0), w.dB(1), w.dB(2)}, dT3[3] = {w.dT3(0), w.dT3(1), w.dT3(2)};
      const float* rq = rec + ((int64_t)q * L + l) * nq * C + (live ? lane : 0);
      float om[3];
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        if (a >= ncf) { om[a] = 0.f; continue; }
        const float c0 = __ldg(coef + ((int64_t)q * nvec) * ncf + a);
        if (ADJ) {
          om[a] = c0;
        } else {
          const float c1 = a1 != nullptr ? __ldg(coef + ((int64_t)q * nvec + 1) * ncf + a) : 0.f;
          om[a] = fmaf(c1, av1, c0 * av0);
        }
      }
      if (!live) continue;
      const float phi = __ldg(rq);
      if (!GRAD) {
        acc = fmaf(om[0] * B3, phi, acc);
        if (!ADJ) acc = fmaf(T3, __ldg(rq + C), acc);
      } else {
        float t = (om[0] * dB[0] + om[1] * dB[1] + om[2] * dB[2]) * phi;
        if (full) {
#pragma unroll
          for (int a = 0; a < 3; ++a) t = fmaf(om[a] * B3, __ldg(rq + (1 + a) * C), t);
        }
        acc = fmaf(t, iw, acc);
        if (!ADJ) {
          const int p0 = full ? 4 : 1;                 // psi0, then psi_a
          acc = fmaf(T3, __ldg(rq + p0 * C), acc);
          if (full) {
#pragma unroll
            for (int a = 0; a < 3; ++a) acc = fmaf(dT3[a], __ldg(rq + (p0 + 1 + a) * C), acc);
          }
        }
      }
    }
  }
  if (ADJ) {
    const float zc = live ? __ldg(feat.z[l] + v * C + lane) : 0.f;
    const float d = warp_sum(zc * acc);
    if (lane == 0) out[gv] = d;
  } else if (live) {
    out[gv * C + lane] += acc;
  }
}

// dz_i += w * sum_{i' in N27(i)} B3c(i' - i) (lam_i alpha_i' + alpha_i lam_i') z_i'; one warp per voxel, lane = channel
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
k_regulariser_vjp(nksr_svh_t svh, nksr_feat_t feat, int l, const float* __restrict__ lam,
                  const float* __restrict__ alpha, float w, float* __restrict__ dz) {
  const int lane = threadIdx.x & 31;
  const int64_t v = blockIdx.x * (int64_t)kWarpsPerBlock + (threadIdx.x >> 5);
  if (v >= svh.n[l] || lane >= feat.channels) return;
  const int C = feat.channels;
  const int64_t gv = svh.offset[l] + v;
  const float li = __ldg(lam + gv), ai = __ldg(alpha + gv);
  float acc = 0.f;
  for (int s = 0; s < 27; ++s) {
    const int u = __ldg(svh.nbr27[l] + v * 27 + s);
    if (u < 0) continue;
    int dx, dy, dz;
    slot_to_d(s, dx, dy, dz);
    const float bw = (dx == 0 ? 0.75f : 0.125f) * (dy == 0 ? 0.75f : 0.125f) * (dz == 0 ? 0.75f : 0.125f);
    const int64_t gu = svh.offset[l] + u;
    const float cpl = fmaf(li, __ldg(alpha + gu), ai * __ldg(lam + gu));
    acc = fmaf(bw * cpl, __ldg(feat.z[l] + (int64_t)u * C + lane), acc);
  }
  dz[gv * C + lane] += w * acc;
}

int check_common(const nksr_svh_t* svh, const nksr_feat_t* feat) {
  if (!svh || !feat || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH) return NKSR_E_INVALID;
  if (feat->channels < 1 || feat->channels > 32) return NKSR_E_INVALID;
  return NKSR_OK;
}

int field_bwd(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* xyz, const int32_t* base,
              const int32_t* range, int64_t m, int mode, int approx_kernel_grad, const float* a0, const float* a1,
              const float* coef, float* out, void* ws, size_t ws_bytes, void* stream, bool adjoint) {
  int rc = check_common(svh, feat);
  if (rc != NKSR_OK) return rc;
  if ((mode != 0 && mode != 1) || m < 0 || (m > 0 && (!xyz || !base || !range || !coef)) || !out) return NKSR_E_INVALID;
  if (!adjoint && !a0) return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  if (ws_bytes < nksr_field_bwd_workspace_bytes(svh->depth, m, feat->channels, mode, approx_kernel_grad, !adjoint))
    return NKSR_E_WORKSPACE;
  if (!ws) return NKSR_E_INVALID;
  cudaStream_t s = as_stream(stream);
  float* rec = static_cast<float*>(ws);
  const bool full = mode == 1 && !approx_kernel_grad;
  const int grid1 = grid_for(m, kWarpsPerBlock);
  const nksr_svh_t& sv = *svh;
  const nksr_feat_t& ft = *feat;
#define NKSR_P1(G, P) \
  k_field_bwd_pass1<G, P><<<grid1, kWarpsPerBlock * 32, 0, s>>>(sv, ft, xyz, base, m, full, a0, a1, coef, rec)
  if (mode == 0) { if (adjoint) NKSR_P1(false, false); else NKSR_P1(false, true); }
  else { if (adjoint) NKSR_P1(true, false); else NKSR_P1(true, true); }
#undef NKSR_P1
  NKSR_CHECK_LAUNCH();
  for (int l = 0; l < svh->depth; ++l) {
    if (svh->n[l] == 0) continue;
    const int grid2 = grid_for(svh->n[l], kWarpsPerBlock);
#define NKSR_P2(G, A) \
  k_field_bwd_pass2<G, A><<<grid2, kWarpsPerBlock * 32, 0, s>>>(sv, ft, xyz, range, l, full, a0, a1, coef, rec, out)
    if (mode == 0) { if (adjoint) NKSR_P2(false, true); else NKSR_P2(false, false); }
    else { if (adjoint) NKSR_P2(true, true); else NKSR_P2(true, false); }
#undef NKSR_P2
  }
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // namespace

extern "C" {

size_t nksr_field_bwd_workspace_bytes(int depth, int64_t m, int channels, int mode, int approx_kernel_grad,
                                      int feature_vjp) {
  if (depth < 1 || m < 0 || channels < 1) return 0;
  const int nq = record_vectors(mode, mode == 1 && !approx_kernel_grad, feature_vjp != 0);
  return (size_t)m * (size_t)depth * (size_t)nq * (size_t)channels * sizeof(float);
}

int nksr_evaluate_adjoint(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* xyz, const int32_t* base,
                          const int32_t* range, int64_t m, int mode, int approx_kernel_grad, const float* coef,
                          float* dalpha, void* ws, size_t ws_bytes, void* stream) {
  int rc = check_common(svh, feat);
  if (rc != NKSR_OK || !dalpha) return rc != NKSR_OK ? rc : NKSR_E_INVALID;
  int64_t n = 0;
  for (int l = 0; l < svh->depth; ++l) n += svh->n[l];
  if (m == 0) {
    if (n > 0 && cudaMemsetAsync(dalpha, 0, n * sizeof(float), as_stream(stream)) != cudaSuccess) return NKSR_E_CUDA;
    return NKSR_OK;
  }
  return field_bwd(svh, feat, xyz, base, range, m, mode, approx_kernel_grad, nullptr, nullptr, coef, dalpha, ws,
                   ws_bytes, stream, true);
}

int nksr_feature_vjp(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* xyz, const int32_t* base,
                     const int32_t* range, int64_t m, int mode, int approx_kernel_grad, const float* a0,
                     const float* a1, const float* coef, float* dz, void* ws, size_t ws_bytes, void* stream) {
  return field_bwd(svh, feat, xyz, base, range, m, mode, approx_kernel_grad, a0, a1, coef, dz, ws, ws_bytes, stream,
                   false);
}

int nksr_regulariser_vjp(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* lam, const float* alpha,
                         float w, float* dz, void* stream) {
  int rc = check_common(svh, feat);
  if (rc != NKSR_OK) return rc;
  if (!lam || !alpha || !dz) return NKSR_E_INVALID;
  if (w == 0.f) return NKSR_OK;
  for (int l = 0; l < svh->depth; ++l) {
    if (svh->n[l] == 0) continue;
    k_regulariser_vjp<<<grid_for(svh->n[l], kWarpsPerBlock), kWarpsPerBlock * 32, 0, as_stream(stream)>>>(
        *svh, *feat, l, lam, alpha, w, dz);
  }
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
