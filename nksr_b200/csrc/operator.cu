// Matrix-free application of the inference system A = E^T W E + w_reg R (SPEC S5) straight from the kernel rows, for the
// PCG of KernelField.solve: no count, placement, blocks or fill, and no CSR matrix.  DESIGN 4.2.1.
//
// k_op_gather_scatter: one warp per top-level voxel, lane = stencil slot.  The warp walks the voxel's contiguous range of
// Morton-sorted position locations, then of normal locations.  Per location r it loads the r's lines of every level
// once, forms t_r = w_r E_r x (three values for a gradient location, one per axis) from the x values of the containing
// voxel's 27 neighbours -- fetched once per run of locations with the same containing voxel u_l -- and adds E_l[r][s] t_r
// into a register accumulator per level.  When u_l changes, the accumulator goes to the planar partial sums P[s][u]
// (27 planes of n floats).  A level-l voxel's locations are contiguous and lie inside one top voxel's range, so one warp
// owns every P[.][u] it writes: positions store, normals then add, in a fixed order -- no atomics, and the result is
// bitwise repeatable.  Voxels without locations are never written, and stay zero from the setup's clear.
//
// k_op_apply: one thread per unknown, levels concatenated, grid-stride.  y_i = sum_s P[s][nbr27(i)[26 - s]] (u's slot s
// is i exactly when i's slot 26 - s is u) + w_reg sum_s B3(d_s) <z_i, z_n> x_n over the 27 neighbours n = nbr27(i)[s]:
// the regulariser of gram_row_regulariser, formed on the fly.
//
// Setup (once per solve): the same two kernels with t_r = w_r * target (the right-hand side) and w_r E^2 (the Jacobi
// diagonal) accumulated into a second set of planes.
#include "gram_common.cuh"
#include "operator.cuh"

namespace {

constexpr int kOpWarps = 8;
constexpr int kApplyBlock = 256;

// row forms: value rows (positions), compact gradient lines (approx_kernel_grad), three full gradient rows
enum { kValue = 0, kCompact = 1, kFull = 2 };

template <int KIND, int MAXL, bool SETUP>
__device__ __forceinline__ void op_walk(const nksr_svh_t& svh, const float* __restrict__ e,
                                        const int32_t* __restrict__ base, const float* __restrict__ tgt, int64_t m,
                                        float w, int b, int end, const float* __restrict__ x, float* __restrict__ P,
                                        float* __restrict__ Pd, const int32_t* __restrict__ add_if, int64_t n,
                                        int lane) {
  constexpr int LINES = KIND == kFull ? 3 : 1;   // 128-byte lines per (location, level)
  constexpr int AX = KIND == kValue ? 1 : 3;     // rows per (location, level)
  const int L = svh.depth;
  int cur[MAXL];
  float acc[MAXL], accd[MAXL], xc[MAXL];
#pragma unroll
  for (int l = 0; l < MAXL; ++l) { cur[l] = -1; acc[l] = 0.f; accd[l] = 0.f; xc[l] = 0.f; }
  const int sl = lane < 27 ? lane : 13;
  const CompactSpline spline(c_d27[sl][0], c_d27[sl][1], c_d27[sl][2]);
  const float inv_w0 = 1.f / svh.voxel_size;

  // P[s][u] (+)= acc: lanes < 27; `add_if` (the normal pass): add when the position pass wrote the voxel
  auto flush = [&](int l) {
    const int u = cur[l];
    if (lane < 27) {
      const int64_t g = svh.offset[l] + u;
      const bool add = add_if != nullptr && __ldg(add_if + 2 * g) < __ldg(add_if + 2 * g + 1);
      const int64_t q = (int64_t)lane * n + g;
      P[q] = add ? P[q] + acc[l] : acc[l];
      if (SETUP) Pd[q] = add ? Pd[q] + accd[l] : accd[l];
    }
    acc[l] = 0.f;
    accd[l] = 0.f;
  };

  float nx[MAXL][LINES];   // the next location's lines, requested one location ahead
  auto load_lines = [&](int r, float (&dst)[MAXL][LINES]) {
    const float* p = e + (int64_t)r * L * LINES * NKSR_ROW_STRIDE + lane;
#pragma unroll
    for (int l = 0; l < MAXL; ++l)
#pragma unroll
      for (int a = 0; a < LINES; ++a)
        dst[l][a] = l < L ? __ldcs(p + (l * LINES + a) * NKSR_ROW_STRIDE) : 0.f;
  };
  load_lines(b, nx);
  int bl[MAXL];            // containing voxels of 32 consecutive locations, lane j = location r0 + j
  for (int r = b; r < end; ++r) {
    const int j = (r - b) & 31;
    if (j == 0) {
#pragma unroll
      for (int l = 0; l < MAXL; ++l) bl[l] = (l < L && r + lane < end) ? __ldg(base + (int64_t)l * m + r + lane) : -1;
    }
    float ln[MAXL][LINES];
#pragma unroll
    for (int l = 0; l < MAXL; ++l)
#pragma unroll
      for (int a = 0; a < LINES; ++a) ln[l][a] = nx[l][a];
    if (r + 1 < end) load_lines(r + 1, nx);
#pragma unroll
    for (int l = 0; l < MAXL; ++l) {
      if (l < L) {
        const int u = __shfl_sync(0xffffffffu, bl[l], j);
        if (u != cur[l]) {
          if (cur[l] >= 0) flush(l);
          cur[l] = u;
          if (!SETUP) {
            const int nb = (u >= 0 && lane < 27) ? __ldg(svh.nbr27[l] + (int64_t)u * 27 + lane) : -1;
            xc[l] = nb >= 0 ? __ldg(x + svh.offset[l] + nb) : 0.f;
          }
        }
      }
    }
    // this lane's entries of the location's rows (zero on a level without containing voxel, and in lanes >= 27)
    float ev[MAXL][AX];
#pragma unroll
    for (int l = 0; l < MAXL; ++l) {
      if (KIND == kCompact) {
        float e0 = 0.f, e1 = 0.f, e2 = 0.f;
        if (l < L) spline.grad_rows(ln[l][0], inv_w0 * __int_as_float((127 - l) << 23), lane, e0, e1, e2);
        ev[l][0] = e0;
        ev[l][AX > 1 ? 1 : 0] = e1;
        ev[l][AX > 2 ? 2 : 0] = e2;
      } else {
#pragma unroll
        for (int a = 0; a < AX; ++a) ev[l][a] = ln[l][a];
      }
    }
    float t[AX];
    if (SETUP) {
#pragma unroll
      for (int a = 0; a < AX; ++a) t[a] = KIND == kValue ? 0.f : w * __ldg(tgt + (int64_t)r * 3 + a);
    } else {
#pragma unroll
      for (int a = 0; a < AX; ++a) {
        float s = 0.f;
#pragma unroll
        for (int l = 0; l < MAXL; ++l) s = fmaf(ev[l][a], xc[l], s);
        t[a] = s;
      }
#pragma unroll
      for (int a = 0; a < AX; ++a) t[a] = w * warp_sum(t[a]);
    }
#pragma unroll
    for (int l = 0; l < MAXL; ++l) {
#pragma unroll
      for (int a = 0; a < AX; ++a) {
        acc[l] = fmaf(ev[l][a], t[a], acc[l]);
        if (SETUP) accd[l] = fmaf(w * ev[l][a], ev[l][a], accd[l]);
      }
    }
  }
#pragma unroll
  for (int l = 0; l < MAXL; ++l)
    if (l < L && cur[l] >= 0) flush(l);
}

template <int NKIND, int MAXL, bool SETUP>
__global__ void __launch_bounds__(kOpWarps * 32)
k_op_gather_scatter(nksr_svh_t svh, nksr_constraints_t cs, const int32_t* __restrict__ base_pos,
                    const int32_t* __restrict__ base_nrm, const float* __restrict__ x, float* __restrict__ P,
                    float* __restrict__ Pd, int64_t n, const int* __restrict__ done) {
  if (done && *done) return;
  const int lane = threadIdx.x & 31;
  const int64_t top = blockIdx.x * (int64_t)kOpWarps + (threadIdx.x >> 5);
  const int T = svh.depth - 1;
  if (top >= svh.n[T]) return;
  const int64_t g = svh.offset[T] + top;
  int pb = 0, pe = 0;
  if (cs.n_pos > 0) {
    pb = __ldg(cs.range_pos + 2 * g);
    pe = __ldg(cs.range_pos + 2 * g + 1);
    if (pb < pe)
      op_walk<kValue, MAXL, SETUP>(svh, cs.e_pos, base_pos, nullptr, cs.n_pos, cs.w_pos, pb, pe, x, P, Pd, nullptr, n,
                                   lane);
  }
  if (cs.n_nrm > 0) {
    const int nb = __ldg(cs.range_nrm + 2 * g), ne = __ldg(cs.range_nrm + 2 * g + 1);
    if (nb < ne)
      op_walk<NKIND, MAXL, SETUP>(svh, cs.e_nrm, base_nrm, cs.t_nrm, cs.n_nrm, cs.w_nrm, nb, ne, x, P, Pd,
                                  pb < pe ? cs.range_pos : nullptr, n, lane);
  }
}

// y = sum_s P[s][nbr27(i)[26 - s]] + w_reg R x (SETUP: y = rhs from P, y2 = diag from Pd + w_reg R_ii)
template <bool SETUP>
__global__ void __launch_bounds__(kApplyBlock)
k_op_apply(nksr_svh_t svh, nksr_feat_t feat, float w_reg, const float* __restrict__ P, const float* __restrict__ Pd,
           const float* __restrict__ x, float* __restrict__ y, float* __restrict__ y2, int64_t n,
           double* __restrict__ pap, const int* __restrict__ done) {
  __shared__ double sh[kApplyBlock / 32];
  if (done && *done) return;
  const int C = feat.channels;
  double local = 0.0;
  for (int64_t g = blockIdx.x * (int64_t)kApplyBlock + threadIdx.x; g < n; g += (int64_t)gridDim.x * kApplyBlock) {
    // the level of g: the last one that starts at or before g (an empty level starts where the next one does).
    // Unrolled, so that the level's pointers come from the parameter space, not a local copy of the struct
    int64_t off = 0;
    const int32_t* nbt = svh.nbr27[0];
    const float* zt = feat.z[0];
#pragma unroll
    for (int k = 1; k < NKSR_MAX_DEPTH; ++k)
      if (k < svh.depth && g >= svh.offset[k]) { off = svh.offset[k]; nbt = svh.nbr27[k]; zt = feat.z[k]; }
    const int64_t i = g - off;
    const int32_t* nb = nbt + i * 27;
    const float* zi = zt + i * C;
    float s = 0.f, sd = 0.f, reg = 0.f;
#pragma unroll 3
    for (int k = 0; k < 27; ++k) {
      const int v = __ldg(nb + k);
      if (v < 0) continue;
      const int64_t q = (int64_t)(26 - k) * n + off + v;
      s += __ldg(P + q);
      if (SETUP) sd += __ldg(Pd + q);
      if (w_reg != 0.f && (!SETUP || k == 13)) {
        const float* zn = zt + (int64_t)v * C;
        float d = 0.f;
        for (int c = 0; c < C; ++c) d = fmaf(__ldg(zi + c), __ldg(zn + c), d);
        const int dx = k / 9 - 1, dy = (k / 3) % 3 - 1, dz = k % 3 - 1;
        const float bw = (dx == 0 ? 0.75f : 0.125f) * (dy == 0 ? 0.75f : 0.125f) * (dz == 0 ? 0.75f : 0.125f);
        if (SETUP) sd += w_reg * bw * d;
        else reg = fmaf(w_reg * bw * d, __ldg(x + off + v), reg);
      }
    }
    if (SETUP) {
      y[g] = s;
      y2[g] = sd;
    } else {
      const float yi = s + reg;
      y[g] = yi;
      if (pap) local += (double)yi * (double)__ldg(x + g);
    }
  }
  if (pap) {
    local = warp_sum_d(local);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = local;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < kApplyBlock / 32; ++w) t += sh[w];
      pap[blockIdx.x] = t;
    }
  }
}

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

int64_t op_unknowns(const nksr_svh_t& svh) { return svh.offset[svh.depth - 1] + svh.n[svh.depth - 1]; }

template <bool SETUP>
int gather_scatter_launch(const MfOperator& op, const float* x, const int* done, cudaStream_t s) {
  const int64_t n_top = op.svh.n[op.svh.depth - 1];
  if (n_top == 0) return NKSR_OK;
  const int grid = (int)((n_top + kOpWarps - 1) / kOpWarps);
  const bool compact = op.cs.nrm_compact == 1;
#define NKSR_GS(NK, ML) \
  k_op_gather_scatter<NK, ML, SETUP><<<grid, kOpWarps * 32, 0, s>>>(op.svh, op.cs, op.base_pos, op.base_nrm, x, op.P, \
                                                                     op.Pd, op.n, done)
  if (op.svh.depth <= 4) {
    if (compact) NKSR_GS(kCompact, 4); else NKSR_GS(kFull, 4);
  } else {
    if (compact) NKSR_GS(kCompact, NKSR_MAX_DEPTH); else NKSR_GS(kFull, NKSR_MAX_DEPTH);
  }
#undef NKSR_GS
  return NKSR_OK;
}

bool op_valid(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c, const int32_t* base_pos,
              const int32_t* base_nrm) {
  if (!svh || !feat || !c || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH) return false;
  if (feat->channels < 1 || feat->channels > 32) return false;
  if (c->nrm_compact != 0 && c->nrm_compact != 1) return false;
  if (c->n_pos < 0 || c->n_nrm < 0 || c->n_pos >= INT32_MAX || c->n_nrm >= INT32_MAX) return false;
  if (c->n_pos > 0 && (!c->e_pos || !c->range_pos || !base_pos)) return false;
  if (c->n_nrm > 0 && (!c->e_nrm || !c->range_nrm || !c->t_nrm || !base_nrm)) return false;
  for (int l = 0; l < svh->depth; ++l)
    if (svh->n[l] > 0 && (!svh->nbr27[l] || !feat->z[l])) return false;
  return op_unknowns(*svh) > 0;
}

MfOperator make_op(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                   const int32_t* base_pos, const int32_t* base_nrm, void* ws) {
  MfOperator op;
  op.svh = *svh;
  op.feat = *feat;
  op.cs = *c;
  op.base_pos = base_pos;
  op.base_nrm = base_nrm;
  op.n = op_unknowns(*svh);
  op.P = reinterpret_cast<float*>(ws);
  op.Pd = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(ws) + align256((size_t)27 * op.n * sizeof(float)));
  return op;
}

}  // namespace

int mf_operator_make(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                     const int32_t* base_pos, const int32_t* base_nrm, void* ws, size_t ws_bytes, MfOperator* out) {
  if (!op_valid(svh, feat, c, base_pos, base_nrm) || !ws || !out) return NKSR_E_INVALID;
  if (ws_bytes < nksr_op_workspace_bytes(svh)) return NKSR_E_WORKSPACE;
  *out = make_op(svh, feat, c, base_pos, base_nrm, ws);
  return NKSR_OK;
}

int mf_apply_launch(const MfOperator& op, const float* x, float* y, double* pap, int blocks, const int* done,
                    cudaStream_t s) {
  gather_scatter_launch<false>(op, x, done, s);
  k_op_apply<false><<<blocks, kApplyBlock, 0, s>>>(op.svh, op.feat, op.cs.w_reg, op.P, nullptr, x, y, nullptr, op.n,
                                                   pap, done);
  return NKSR_OK;
}

extern "C" {

size_t nksr_op_workspace_bytes(const nksr_svh_t* svh) {
  if (!svh || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH) return 0;
  return 2 * align256((size_t)27 * op_unknowns(*svh) * sizeof(float)) + 256;
}

int nksr_op_setup(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c, const int32_t* base_pos,
                  const int32_t* base_nrm, float* rhs, float* diag, void* ws, size_t ws_bytes, void* stream) {
  if (!op_valid(svh, feat, c, base_pos, base_nrm) || !rhs || !diag || !ws) return NKSR_E_INVALID;
  if (ws_bytes < nksr_op_workspace_bytes(svh)) return NKSR_E_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const MfOperator op = make_op(svh, feat, c, base_pos, base_nrm, ws);
  // every plane starts at zero: the voxels without locations are never written, here or by nksr_op_apply
  if (cudaMemsetAsync(ws, 0, nksr_op_workspace_bytes(svh), s) != cudaSuccess) return NKSR_E_CUDA;
  gather_scatter_launch<true>(op, nullptr, nullptr, s);
  const int grid = grid_for(op.n, kApplyBlock);
  k_op_apply<true><<<grid, kApplyBlock, 0, s>>>(op.svh, op.feat, op.cs.w_reg, op.P, op.Pd, nullptr, rhs, diag, op.n,
                                                nullptr, nullptr);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_op_apply(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c, const int32_t* base_pos,
                  const int32_t* base_nrm, const float* x, float* y, void* ws, size_t ws_bytes, void* stream) {
  if (!op_valid(svh, feat, c, base_pos, base_nrm) || !x || !y || !ws) return NKSR_E_INVALID;
  if (ws_bytes < nksr_op_workspace_bytes(svh)) return NKSR_E_WORKSPACE;
  const MfOperator op = make_op(svh, feat, c, base_pos, base_nrm, ws);
  mf_apply_launch(op, x, y, nullptr, grid_for(op.n, kApplyBlock), nullptr, as_stream(stream));
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
