// CSR SpMV and Jacobi-preconditioned conjugate gradients (SURVEY section 8 row a4).
// Replaces the solve inside KernelField.solve* (models/nksr_net.py:105-112; tolerance knob
// solver_tol at examples/recons_waymo.py:33; verbose hook models/nksr_net.py:97-98).
//
// All dot products are two-stage and deterministic: every block writes one fp64 partial, the
// consumer kernels re-reduce the (fixed-length) partial array in a fixed order.  The host is not in
// the loop: alpha and beta are formed on the device from the partials, convergence is decided ON THE
// DEVICE (every block of k_pcg_direction reduces the same ||r||^2 partials and block 0 raises a flag
// in device memory that turns every later kernel into a no-op), and the iterations are replayed from a
// CUDA graph of `check_every` iterations -- one host read-back per graph launch, i.e. one per solve for
// the benchmark systems (10-40 iterations) instead of one per iteration.
//
// Second half of the file: the step kernels of the multi-GPU solve (SURVEY section 8e mapping B): a
// Chronopoulos-Gear rearrangement of the same Jacobi-PCG with ONE fused fp64 all-reduce per iteration
// ((r,u), (w,u), (r,r)) and an ownership mask; the collective itself (NCCL) and the halo exchange are
// issued by the host between the kernels (nksr_b200/dist_solve.py).
#include <math.h>

#include "common.cuh"
#include "operator.cuh"
#include "spmv_stream.cuh"

namespace {

constexpr int kBlock = 256;
constexpr int kWarpsPerBlock = kBlock / 32;
constexpr int kGrid = 132 * 8;  // persistent-style grid: 8 blocks per SM (H100 SXM: 132 SMs)

// device-resident solver state (lives at the end of the caller's workspace)
struct PcgCtrl {
  int iters;       // completed iterations (x updates)
  int done;        // 0 running, 1 converged, 2 NaN / breakdown, 3 max_iter reached
  int max_iter;
  int pad;
  double rr;       // ||r||^2 of the current iterate
  double bb;       // ||b||^2
  double target;   // tol^2 * bb
  double gamma_prev, alpha_prev;  // Chronopoulos-Gear recurrences (distributed solve)
};

// sum of val[p] * x[col[p]] over the entries of one row, in every lane of the warp.  The matrix stream: evict-first
// loads (read once per SpMV); x: read-only path, stays in L1/L2.  Four independent 128 B column + value requests per
// lane keep ~1 KB per warp in flight.
__device__ __forceinline__ float row_dot(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                         const float* __restrict__ val, const float* __restrict__ x, int64_t row,
                                         int lane) {
  const int64_t b = __ldg(rowptr + row), e = __ldg(rowptr + row + 1);
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  for (int64_t p = b + lane; p < e; p += 128) {   // predicated tail: absent entries read as (col 0, value 0)
    const bool q1 = p + 32 < e, q2 = p + 64 < e, q3 = p + 96 < e;
    const int c0 = __ldcs(col + p), c1 = q1 ? __ldcs(col + p + 32) : 0, c2 = q2 ? __ldcs(col + p + 64) : 0,
              c3 = q3 ? __ldcs(col + p + 96) : 0;
    const float v0 = __ldcs(val + p), v1 = q1 ? __ldcs(val + p + 32) : 0.f, v2 = q2 ? __ldcs(val + p + 64) : 0.f,
                v3 = q3 ? __ldcs(val + p + 96) : 0.f;
    s0 = fmaf(v0, __ldg(x + c0), s0);
    s1 = fmaf(v1, __ldg(x + c1), s1);
    s2 = fmaf(v2, __ldg(x + c2), s2);
    s3 = fmaf(v3, __ldg(x + c3), s3);
  }
  return warp_sum((s0 + s1) + (s2 + s3));
}

// y = A x, one warp per row, grid-stride over rows.  DOT: also partial[blockIdx] = sum x_i * y_i.
// ctrl (nullable): no-op once the solve is over.
template <bool DOT>
__global__ void __launch_bounds__(kBlock)
k_spmv(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col, const float* __restrict__ val,
       const float* __restrict__ x, float* __restrict__ y, int64_t n, double* __restrict__ partial,
       const PcgCtrl* __restrict__ ctrl) {
  __shared__ double wsum[kWarpsPerBlock];
  if (ctrl && ctrl->done) return;
  const int lane = threadIdx.x & 31;
  const int wid = threadIdx.x >> 5;
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  double local = 0.0;
  for (int64_t row = blockIdx.x * (int64_t)kWarpsPerBlock + wid; row < n; row += nwarps) {
    // (prefetching the next row's pointers was tried and measured slower -- the two loop-carried 64-bit
    // values push the kernel past the 32 registers that keep the persistent 8-blocks-per-SM grid resident)
    const float s = row_dot(rowptr, col, val, x, row, lane);
    if (lane == 0) {
      y[row] = s;
      if (DOT) local += (double)s * (double)__ldg(x + row);
    }
  }
  if (DOT) {
    if (lane == 0) wsum[wid] = local;
    __syncthreads();
    if (threadIdx.x == 0) {
      double t = 0.0;
      for (int w = 0; w < kWarpsPerBlock; ++w) t += wsum[w];
      partial[blockIdx.x] = t;
    }
  }
}

// deterministic block-wide reduction of a fixed-length fp64 array; result broadcast to all threads
__device__ __forceinline__ double reduce_partials(const double* __restrict__ arr, int len, double* sh) {
  double t = 0.0;
  for (int i = threadIdx.x; i < len; i += kBlock) t += arr[i];
  t = warp_sum_d(t);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = t;
  __syncthreads();
  double r = 0.0;
  for (int w = 0; w < kWarpsPerBlock; ++w) r += sh[w];
  __syncthreads();
  return r;
}

__device__ __forceinline__ void block_store_partial(double local, double* sh, double* dst) {
  local = warp_sum_d(local);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int w = 0; w < kWarpsPerBlock; ++w) t += sh[w];
    *dst = t;
  }
  __syncthreads();
}

// x = 0, r = b, z = r/diag, p = z; partials: rz, bb
__global__ void __launch_bounds__(kBlock)
k_pcg_init(const float* __restrict__ b, const float* __restrict__ diag, float* __restrict__ x, float* __restrict__ r,
           float* __restrict__ p, int64_t n, double* __restrict__ part_rz, double* __restrict__ part_bb) {
  __shared__ double sh[kWarpsPerBlock];
  double rz = 0.0, bb = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const float bi = b[i], d = diag[i];
    const float zi = d > 0.f ? bi / d : 0.f;
    x[i] = 0.f;
    r[i] = bi;
    p[i] = zi;
    rz += (double)bi * zi;
    bb += (double)bi * bi;
  }
  block_store_partial(rz, sh, part_rz + blockIdx.x);
  block_store_partial(bb, sh, part_bb + blockIdx.x);
}

// one block: ||b||^2 -> ctrl (target, flags)
__global__ void __launch_bounds__(kBlock)
k_pcg_begin(const double* __restrict__ part_bb, float tol, int max_iter, PcgCtrl* __restrict__ ctrl) {
  __shared__ double sh[kWarpsPerBlock];
  const double bb = reduce_partials(part_bb, kGrid, sh);
  if (threadIdx.x == 0) {
    ctrl->iters = 0;
    ctrl->max_iter = max_iter;
    ctrl->bb = bb;
    ctrl->rr = bb;
    ctrl->target = (double)tol * (double)tol * bb;
    ctrl->gamma_prev = 0.0;
    ctrl->alpha_prev = 0.0;
    ctrl->done = !(bb == bb) ? 2 : (bb > 0.0 ? (max_iter > 0 ? 0 : 3) : 1);
  }
}

// alpha = rz/pAp; x += alpha p; r -= alpha Ap; z = r/diag (kept in ap); partials rz_new, rr
__global__ void __launch_bounds__(kBlock)
k_pcg_update(const float* __restrict__ diag, const float* __restrict__ p, float* __restrict__ ap,
             float* __restrict__ x, float* __restrict__ r, int64_t n, const double* __restrict__ part_rz,
             const double* __restrict__ part_pap, double* __restrict__ part_rz_new, double* __restrict__ part_rr,
             const PcgCtrl* __restrict__ ctrl) {
  __shared__ double sh[kWarpsPerBlock];
  if (ctrl->done) return;
  const double rz = reduce_partials(part_rz, kGrid, sh);
  const double pap = reduce_partials(part_pap, kGrid, sh);
  const float alpha = pap != 0.0 ? (float)(rz / pap) : 0.f;
  double rzn = 0.0, rr = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const float pi = p[i], api = ap[i], d = diag[i];
    x[i] = fmaf(alpha, pi, x[i]);
    const float ri = fmaf(-alpha, api, r[i]);
    r[i] = ri;
    const float zi = d > 0.f ? ri / d : 0.f;
    ap[i] = zi;  // Ap is dead after this point: reuse its storage for z
    rzn += (double)ri * zi;
    rr += (double)ri * ri;
  }
  block_store_partial(rzn, sh, part_rz_new + blockIdx.x);
  block_store_partial(rr, sh, part_rr + blockIdx.x);
}

// convergence test (every block reduces the same ||r||^2 partials, so all blocks agree without talking to
// each other); when the solve goes on: beta = rz_new/rz; p = z + beta p.  Block 0 publishes the verdict for the
// kernels of the NEXT iterations (nothing in this launch reads what it writes).
__global__ void __launch_bounds__(kBlock)
k_pcg_direction(const float* __restrict__ z, float* __restrict__ p, int64_t n, const double* __restrict__ part_rz,
                const double* __restrict__ part_rz_new, const double* __restrict__ part_rr,
                PcgCtrl* __restrict__ ctrl) {
  __shared__ double sh[kWarpsPerBlock];
  if (ctrl->done) return;
  const double rr = reduce_partials(part_rr, kGrid, sh);
  const int it = ctrl->iters + 1;
  int verdict = 0;
  if (!(rr == rr)) verdict = 2;
  else if (rr <= ctrl->target) verdict = 1;
  else if (it >= ctrl->max_iter) verdict = 3;
  if (verdict == 0) {
    const double rz = reduce_partials(part_rz, kGrid, sh);
    const double rzn = reduce_partials(part_rz_new, kGrid, sh);
    const float beta = rz != 0.0 ? (float)(rzn / rz) : 0.f;
    for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock)
      p[i] = fmaf(beta, p[i], z[i]);
  }
  // every block has read ctrl->iters / done before block 0 can get here only if it is the LAST to read; to stay
  // race-free the fields read above (iters, done, target, max_iter) are not written in this kernel: the verdict
  // goes to a separate kernel-boundary-ordered slot
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    ctrl->rr = rr;
    ctrl->pad = verdict | (it << 2);   // consumed by k_pcg_commit
  }
}

// one thread: moves the verdict of k_pcg_direction into the fields the next iteration reads
__global__ void k_pcg_commit(PcgCtrl* __restrict__ ctrl) {
  if (ctrl->done) return;
  ctrl->iters = ctrl->pad >> 2;
  ctrl->done = ctrl->pad & 3;
}

struct PcgWs {
  float *r, *p, *ap;
  double *rz0, *rz1, *pap, *rr, *bb;
  PcgCtrl* ctrl;
};

static size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

static PcgWs carve(void* ws, int64_t n) {
  unsigned char* c = reinterpret_cast<unsigned char*>(ws);
  PcgWs w;
  size_t vec = align256((size_t)n * sizeof(float));
  w.r = reinterpret_cast<float*>(c); c += vec;
  w.p = reinterpret_cast<float*>(c); c += vec;
  w.ap = reinterpret_cast<float*>(c); c += vec;
  size_t part = align256(kGrid * sizeof(double));
  w.rz0 = reinterpret_cast<double*>(c); c += part;
  w.rz1 = reinterpret_cast<double*>(c); c += part;
  w.pap = reinterpret_cast<double*>(c); c += part;
  w.rr = reinterpret_cast<double*>(c); c += part;
  w.bb = reinterpret_cast<double*>(c); c += part;
  w.ctrl = reinterpret_cast<PcgCtrl*>(c);
  return w;
}

// The operator A of a PCG: an assembled CSR matrix (row kernel, or the tile stream when `plan` is set) or, when `mf` is
// set, the matrix-free E^T W E + w_reg R of csrc/operator.cu.  Either way one application writes Ap and the p.Ap
// partials of kGrid blocks; the vector kernels, the graph replay and the verdict do not depend on which.
struct PcgOperator {
  const int64_t* rowptr;
  const int32_t* col;
  const float* val;
  const SpmvPlan* plan;
  const MfOperator* mf;
};

// one PCG iteration on stream s (rz buffers alternate with the iteration parity)
static void launch_iteration(const PcgOperator& A, const float* diag, float* x, int64_t n, const PcgWs& w, int parity,
                             cudaStream_t s, cudaEvent_t e0, cudaEvent_t e1) {
  const int64_t* rowptr = A.rowptr;
  const int32_t* col = A.col;
  const float* val = A.val;
  const SpmvPlan* plan = A.plan;
  double* rz_cur = parity ? w.rz1 : w.rz0;
  double* rz_new = parity ? w.rz0 : w.rz1;
  if (e0) cudaEventRecord(e0, s);
  if (A.mf) {
    mf_apply_launch(*A.mf, w.p, w.ap, w.pap, kGrid, &w.ctrl->done, s);
  } else if (plan) {   // tile stream through the TMA engine + boundary rows, long coarse rows warp per row, then p.Ap
    spmv_stream_launch(rowptr, col, val, w.p, w.ap, *plan, &w.ctrl->done, s);
    if (plan->n_rows < n)
      k_spmv<false><<<kGrid, kBlock, 0, s>>>(rowptr + plan->n_rows, col, val, w.p, w.ap + plan->n_rows,
                                             n - plan->n_rows, nullptr, w.ctrl);
    k_dot_partials<<<kGrid, 256, 0, s>>>(w.p, w.ap, n, w.pap, &w.ctrl->done);
  } else {
    k_spmv<true><<<kGrid, kBlock, 0, s>>>(rowptr, col, val, w.p, w.ap, n, w.pap, w.ctrl);
  }
  if (e1) cudaEventRecord(e1, s);
  k_pcg_update<<<kGrid, kBlock, 0, s>>>(diag, w.p, w.ap, x, w.r, n, rz_cur, w.pap, rz_new, w.rr, w.ctrl);
  k_pcg_direction<<<kGrid, kBlock, 0, s>>>(w.ap, w.p, n, rz_cur, rz_new, w.rr, w.ctrl);
  k_pcg_commit<<<1, 1, 0, s>>>(w.ctrl);
}

static int read_ctrl(const PcgCtrl* dev, PcgCtrl* host, cudaStream_t s) {
  if (cudaMemcpyAsync(host, dev, sizeof(PcgCtrl), cudaMemcpyDeviceToHost, s) != cudaSuccess) return NKSR_E_CUDA;
  if (cudaStreamSynchronize(s) != cudaSuccess) return NKSR_E_CUDA;
  return NKSR_OK;
}

}  // namespace

extern "C" {

int nksr_spmv(const int64_t* rowptr, const int32_t* col, const float* val, const float* x, float* y, int64_t n,
              void* stream) {
  if (n <= 0) return n == 0 ? NKSR_OK : NKSR_E_INVALID;
  int grid = (int)((n + kWarpsPerBlock - 1) / kWarpsPerBlock);
  if (grid > kGrid) grid = kGrid;
  k_spmv<false><<<grid, kBlock, 0, as_stream(stream)>>>(rowptr, col, val, x, y, n, nullptr, nullptr);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

size_t nksr_pcg_workspace_bytes(int64_t n) {
  return 3 * align256((size_t)(n > 0 ? n : 1) * sizeof(float)) + 5 * align256(kGrid * sizeof(double)) +
         align256(sizeof(PcgCtrl)) + 256;
}

}  // extern "C"

static int pcg_solve_impl(const PcgOperator& A, const float* diag, const float* b, float* x, int64_t n, float tol,
                          int max_iter, int check_every, int profile, void* ws, size_t ws_bytes, double* info,
                          void* stream) {
  if (n <= 0 || !info || max_iter < 0) return NKSR_E_INVALID;
  if (ws_bytes < nksr_pcg_workspace_bytes(n)) return NKSR_E_WORKSPACE;
  if (check_every < 1) check_every = 1;
  if (check_every & 1) ++check_every;   // whole pairs of iterations: the rz buffers alternate with the parity
  cudaStream_t s = as_stream(stream);
  PcgWs w = carve(ws, n);
  for (int i = 0; i < 5; ++i) info[i] = 0.0;
  // all partial arrays start at zero (blocks beyond a short grid never write)
  if (cudaMemsetAsync(w.rz0, 0, 5 * align256(kGrid * sizeof(double)) + sizeof(PcgCtrl), s) != cudaSuccess)
    return NKSR_E_CUDA;
  k_pcg_init<<<kGrid, kBlock, 0, s>>>(b, diag, x, w.r, w.p, n, w.rz0, w.bb);
  k_pcg_begin<<<1, kBlock, 0, s>>>(w.bb, tol, max_iter, w.ctrl);
  NKSR_CHECK_LAUNCH();
  PcgCtrl host;
  int rc = NKSR_OK;
  if (profile) {
    // CUDA events around every application of A on this stream (info[2], info[3]); plain launches, checked
    // every `check_every` iterations like the graph path
    const int kMaxEv = 512;
    cudaEvent_t ev[2 * kMaxEv];
    for (int i = 0; i < 2 * kMaxEv; ++i) cudaEventCreate(&ev[i]);
    int n_ev = 0, launched = 0;
    host.done = 0;
    while (rc == NKSR_OK && launched < max_iter) {
      for (int j = 0; j < check_every && launched < max_iter; ++j, ++launched) {
        const bool timed = n_ev < kMaxEv;
        launch_iteration(A, diag, x, n, w, launched & 1, s, timed ? ev[2 * n_ev] : nullptr,
                         timed ? ev[2 * n_ev + 1] : nullptr);
        if (timed) ++n_ev;
      }
      rc = read_ctrl(w.ctrl, &host, s);
      if (host.done) break;
    }
    if (rc == NKSR_OK && launched == 0) rc = read_ctrl(w.ctrl, &host, s);
    if (rc == NKSR_OK) {
      double ms = 0.0;
      const int live = host.iters < n_ev ? host.iters : n_ev;      // launches after convergence are no-ops
      for (int i = 0; i < live; ++i) {
        float t = 0.f;
        cudaEventElapsedTime(&t, ev[2 * i], ev[2 * i + 1]);
        ms += t;
      }
      info[2] = ms;
      info[3] = (double)live;
    }
    for (int i = 0; i < 2 * kMaxEv; ++i) cudaEventDestroy(ev[i]);
  } else {
    // a CUDA graph of `check_every` iterations, captured on a private stream (the caller's stream may be the
    // legacy default stream, which cannot be captured) and replayed on the caller's stream
    cudaStream_t cap = nullptr;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    const int per_graph = check_every < max_iter ? check_every : (max_iter + (max_iter & 1));
    bool ok = max_iter == 0 || cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking) == cudaSuccess;
    if (ok && max_iter > 0) {
      ok = cudaStreamBeginCapture(cap, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
      if (ok) {
        for (int j = 0; j < per_graph; ++j)
          launch_iteration(A, diag, x, n, w, j & 1, cap, nullptr, nullptr);
        ok = cudaStreamEndCapture(cap, &graph) == cudaSuccess && graph != nullptr;
      }
      if (ok) ok = cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess;
    }
    if (!ok) rc = NKSR_E_CUDA;
    host.done = 0;
    int launched = 0;
    while (rc == NKSR_OK && launched < max_iter) {
      if (cudaGraphLaunch(exec, s) != cudaSuccess) { rc = NKSR_E_CUDA; break; }
      launched += per_graph;
      rc = read_ctrl(w.ctrl, &host, s);
      if (host.done) break;
    }
    if (rc == NKSR_OK && launched == 0) rc = read_ctrl(w.ctrl, &host, s);
    if (exec) cudaGraphExecDestroy(exec);
    if (graph) cudaGraphDestroy(graph);
    if (cap) cudaStreamDestroy(cap);
  }
  if (rc != NKSR_OK) return rc;
  if (cudaGetLastError() != cudaSuccess) return NKSR_E_CUDA;
  info[0] = (double)host.iters;
  info[1] = host.bb > 0.0 ? sqrt(host.rr / host.bb) : 0.0;
  info[4] = (double)(host.done == 1 ? 0 : (host.done == 2 ? 2 : 1));   // 0 converged, 1 max_iter, 2 NaN
  return NKSR_OK;
}

extern "C" {

int nksr_pcg_solve(const int64_t* rowptr, const int32_t* col, const float* val, const float* diag, const float* b,
                   float* x, int64_t n, float tol, int max_iter, int check_every, int profile, void* ws,
                   size_t ws_bytes, double* info, void* stream) {
  const PcgOperator A{rowptr, col, val, nullptr, nullptr};
  return pcg_solve_impl(A, diag, b, x, n, tol, max_iter, check_every, profile, ws, ws_bytes, info, stream);
}

int nksr_pcg_solve_matrix_free(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                               const int32_t* base_pos, const int32_t* base_nrm, const float* diag, const float* b,
                               float* x, float tol, int max_iter, int check_every, int profile, void* op_ws,
                               size_t op_ws_bytes, void* ws, size_t ws_bytes, double* info, void* stream) {
  MfOperator mf;
  const int rc = mf_operator_make(svh, feat, c, base_pos, base_nrm, op_ws, op_ws_bytes, &mf);
  if (rc != NKSR_OK) return rc;
  const PcgOperator A{nullptr, nullptr, nullptr, nullptr, &mf};
  return pcg_solve_impl(A, diag, b, x, mf.n, tol, max_iter, check_every, profile, ws, ws_bytes, info, stream);
}

size_t nksr_pcg_stream_workspace_bytes(int64_t n, int64_t nnz) {
  return nksr_pcg_workspace_bytes(n) + spmv_plan_bytes(nnz > 0 ? nnz : 1);
}

int nksr_pcg_solve_stream(const int64_t* rowptr, const int32_t* col, const float* val, const float* diag,
                          const float* b, float* x, int64_t n, int64_t nnz, int64_t split_row, int64_t split_nnz,
                          float tol, int max_iter, int check_every, int profile, void* ws, size_t ws_bytes,
                          double* info, void* stream) {
  if (n <= 0 || nnz <= 0 || split_row < 0 || split_row > n || split_nnz < 0 || split_nnz > nnz) return NKSR_E_INVALID;
  if (ws_bytes < nksr_pcg_stream_workspace_bytes(n, nnz)) return NKSR_E_WORKSPACE;
  const size_t base = nksr_pcg_workspace_bytes(n);
  SpmvPlan plan = spmv_plan_carve(reinterpret_cast<unsigned char*>(ws) + base, split_row, split_nnz);
  if (cudaMemsetAsync(plan.stats, 0, 4 * sizeof(unsigned long long), as_stream(stream)) != cudaSuccess)
    return NKSR_E_CUDA;
  if (split_row == 0 || split_nnz == 0)     // nothing to stream: the plain solver
    return pcg_solve_impl(PcgOperator{rowptr, col, val, nullptr, nullptr}, diag, b, x, n, tol, max_iter, check_every,
                          profile, ws, base, info, stream);
  if (spmv_stream_prepare() != NKSR_OK || spmv_stream_sm_count() <= 0) return NKSR_E_CUDA;
  if (spmv_plan_build(rowptr, plan, as_stream(stream)) != NKSR_OK) return NKSR_E_CUDA;
  return pcg_solve_impl(PcgOperator{rowptr, col, val, &plan, nullptr}, diag, b, x, n, tol, max_iter, check_every,
                        profile, ws, base, info, stream);
}

size_t nksr_spmv_plan_bytes(int64_t nnz) { return spmv_plan_bytes(nnz > 0 ? nnz : 1); }

int nksr_spmv_plan_build(const int64_t* rowptr, int64_t n, int64_t nnz, int64_t split_row, int64_t split_nnz,
                         void* plan_buf, size_t plan_bytes, void* stream) {
  if (n <= 0 || nnz <= 0 || !plan_buf || split_row < 0 || split_row > n || split_nnz < 0 || split_nnz > nnz)
    return NKSR_E_INVALID;
  if (plan_bytes < spmv_plan_bytes(nnz)) return NKSR_E_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  SpmvPlan plan = spmv_plan_carve(plan_buf, split_row, split_nnz);
  if (cudaMemsetAsync(plan.stats, 0, 4 * sizeof(unsigned long long), s) != cudaSuccess) return NKSR_E_CUDA;
  if (split_row == 0 || split_nnz == 0) return NKSR_OK;
  return spmv_plan_build(rowptr, plan, s);
}

int nksr_spmv_plan_stats(const void* plan_buf, int64_t* out, void* stream) {
  if (!plan_buf || !out) return NKSR_E_INVALID;
  cudaStream_t s = as_stream(stream);
  unsigned long long h[4];
  if (cudaMemcpyAsync(h, plan_buf, sizeof(h), cudaMemcpyDeviceToHost, s) != cudaSuccess) return NKSR_E_CUDA;
  if (cudaStreamSynchronize(s) != cudaSuccess) return NKSR_E_CUDA;
  for (int i = 0; i < 4; ++i) out[i] = (int64_t)h[i];
  return NKSR_OK;
}

int nksr_spmv_stream_planned(const int64_t* rowptr, const int32_t* col, const float* val, const float* x, float* y,
                             int64_t n, int64_t nnz, int64_t split_row, int64_t split_nnz, void* plan_buf,
                             void* stream) {
  if (n <= 0 || nnz <= 0 || !plan_buf || split_row < 0 || split_row > n || split_nnz < 0 || split_nnz > nnz)
    return NKSR_E_INVALID;
  cudaStream_t s = as_stream(stream);
  // the streamed part writes every row of [0, split_row), empty ones included; when those rows hold no entry at all,
  // nothing is streamed and they are zeroed here
  if (split_row > 0 && split_nnz == 0 &&
      cudaMemsetAsync(y, 0, (size_t)split_row * sizeof(float), s) != cudaSuccess)
    return NKSR_E_CUDA;
  if (split_row > 0 && split_nnz > 0) {
    const SpmvPlan plan = spmv_plan_carve(plan_buf, split_row, split_nnz);
    if (spmv_stream_prepare() != NKSR_OK) return NKSR_E_CUDA;
    const int rc = spmv_stream_launch(rowptr, col, val, x, y, plan, nullptr, s);
    if (rc != NKSR_OK) return rc;
  }
  // the rows after the streamed ones: the row kernel
  return split_row < n ? nksr_spmv(rowptr + split_row, col, val, x, y + split_row, n - split_row, stream) : NKSR_OK;
}

int nksr_spmv_stream(const int64_t* rowptr, const int32_t* col, const float* val, const float* x, float* y, int64_t n,
                     int64_t nnz, int64_t split_row, int64_t split_nnz, void* plan_buf, size_t plan_bytes,
                     void* stream) {
  const int rc = nksr_spmv_plan_build(rowptr, n, nnz, split_row, split_nnz, plan_buf, plan_bytes, stream);
  if (rc != NKSR_OK) return rc;
  return nksr_spmv_stream_planned(rowptr, col, val, x, y, n, nnz, split_row, split_nnz, plan_buf, stream);
}

}  // extern "C"

// ===================================================================== distributed step kernels
namespace {

// w = A u on the OWNED rows (others: w = 0); partials of (r,u), (w,u), (r,r) over the owned rows
// (8 resident blocks per SM = 32 registers: the persistent 8-blocks-per-SM grid must fit in one wave -- at 40 registers it ran
// in two and took half as long again)
__global__ void __launch_bounds__(kBlock, 8)
k_dcg_spmv(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col, const float* __restrict__ val,
           const uint8_t* __restrict__ owned, const float* __restrict__ r, const float* __restrict__ u,
           float* __restrict__ w, int64_t n, double* __restrict__ part, const PcgCtrl* __restrict__ ctrl) {
  __shared__ double wsum[3][kWarpsPerBlock];
  if (ctrl->done) return;
  const int lane = threadIdx.x & 31;
  const int wid = threadIdx.x >> 5;
  const int64_t nwarps = (int64_t)gridDim.x * kWarpsPerBlock;
  double g = 0.0, d = 0.0, rr = 0.0;
  for (int64_t row = blockIdx.x * (int64_t)kWarpsPerBlock + wid; row < n; row += nwarps) {
    if (!__ldg(owned + row)) {
      if (lane == 0) w[row] = 0.f;
      continue;
    }
    const float s = row_dot(rowptr, col, val, u, row, lane);
    if (lane == 0) {
      w[row] = s;
      const double ri = (double)__ldg(r + row), ui = (double)__ldg(u + row);
      g += ri * ui;
      d += (double)s * ui;
      rr += ri * ri;
    }
  }
  if (lane == 0) { wsum[0][wid] = g; wsum[1][wid] = d; wsum[2][wid] = rr; }
  __syncthreads();
  if (threadIdx.x < 3) {
    double t = 0.0;
    for (int k = 0; k < kWarpsPerBlock; ++k) t += wsum[threadIdx.x][k];
    part[threadIdx.x * kGrid + blockIdx.x] = t;
  }
}

// one block: red[j] = sum of the j-th partial array (fixed order)
__global__ void __launch_bounds__(kBlock)
k_reduce_arrays(const double* __restrict__ part, int arrays, double* __restrict__ red,
                const PcgCtrl* __restrict__ ctrl) {
  __shared__ double sh[kWarpsPerBlock];
  if (ctrl && ctrl->done) return;
  for (int j = 0; j < arrays; ++j) {
    const double t = reduce_partials(part + (size_t)j * kGrid, kGrid, sh);
    if (threadIdx.x == 0) red[j] = t;
  }
}

// x = 0, r = b, u = r/diag on owned rows (0 elsewhere), p = s = 0; partial of (b,b)
__global__ void __launch_bounds__(kBlock)
k_dcg_init(const float* __restrict__ diag, const float* __restrict__ b, const uint8_t* __restrict__ owned,
           float* __restrict__ x, float* __restrict__ r, float* __restrict__ u, float* __restrict__ p,
           float* __restrict__ sv, int64_t n, double* __restrict__ part) {
  __shared__ double sh[kWarpsPerBlock];
  double bb = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const bool own = owned[i] != 0;
    const float bi = own ? b[i] : 0.f, d = diag[i];
    x[i] = 0.f;
    r[i] = bi;
    u[i] = (own && d > 0.f) ? bi / d : 0.f;
    p[i] = 0.f;
    sv[i] = 0.f;
    bb += (double)bi * bi;
  }
  block_store_partial(bb, sh, part + blockIdx.x);
}

__global__ void k_dcg_begin(const double* __restrict__ red, float tol, int max_iter, PcgCtrl* __restrict__ ctrl) {
  const double bb = red[0];
  ctrl->iters = 0;
  ctrl->max_iter = max_iter;
  ctrl->pad = 0;
  ctrl->bb = bb;
  ctrl->rr = bb;
  ctrl->target = (double)tol * (double)tol * bb;
  ctrl->gamma_prev = 0.0;
  ctrl->alpha_prev = 0.0;
  ctrl->done = !(bb == bb) ? 2 : (bb > 0.0 ? (max_iter > 0 ? 0 : 3) : 1);
}

// red = all-reduced {(r,u), (w,u), (r,r)} of the CURRENT iterate.  Converged -> verdict only.  Else
// beta = gamma/gamma_prev, alpha = gamma / (delta - beta*gamma/alpha_prev)  (Chronopoulos & Gear 1989);
// p = u + beta p; s = w + beta s; x += alpha p; r -= alpha s; u = r/diag -- owned rows only.
__global__ void __launch_bounds__(kBlock)
k_dcg_update(const float* __restrict__ diag, const uint8_t* __restrict__ owned, float* __restrict__ x,
             float* __restrict__ r, float* __restrict__ u, const float* __restrict__ w, float* __restrict__ p,
             float* __restrict__ sv, int64_t n, const double* __restrict__ red, PcgCtrl* __restrict__ ctrl) {
  if (ctrl->done) return;
  const double gamma = red[0], delta = red[1], rr = red[2];
  const int it = ctrl->iters;
  int verdict = 0;
  if (!(rr == rr) || !(gamma == gamma)) verdict = 2;
  else if (rr <= ctrl->target) verdict = 1;
  else if (it >= ctrl->max_iter) verdict = 3;
  double alpha = 0.0, beta = 0.0;
  if (verdict == 0) {
    if (it > 0 && ctrl->gamma_prev != 0.0) beta = gamma / ctrl->gamma_prev;
    const double den = (it > 0 && ctrl->alpha_prev != 0.0) ? delta - beta * gamma / ctrl->alpha_prev : delta;
    if (den == 0.0 || !(den == den)) verdict = 2;
    else alpha = gamma / den;
  }
  if (verdict == 0) {
    const float a = (float)alpha, bt = (float)beta;
    for (int64_t i = blockIdx.x * (int64_t)kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
      if (!owned[i]) continue;
      const float pi = fmaf(bt, p[i], u[i]);
      const float si = fmaf(bt, sv[i], w[i]);
      p[i] = pi;
      sv[i] = si;
      x[i] = fmaf(a, pi, x[i]);
      const float ri = fmaf(-a, si, r[i]);
      r[i] = ri;
      const float d = diag[i];
      u[i] = d > 0.f ? ri / d : 0.f;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {   // consumed by k_dcg_commit (kernel-boundary ordered)
    ctrl->rr = rr;
    ctrl->pad = verdict;
    // stash the recurrence scalars where this launch does not read them: the commit kernel moves them
    reinterpret_cast<double*>(ctrl + 1)[0] = gamma;
    reinterpret_cast<double*>(ctrl + 1)[1] = alpha;
  }
}

__global__ void k_dcg_commit(PcgCtrl* __restrict__ ctrl) {
  if (ctrl->done) return;
  ctrl->done = ctrl->pad;
  if (ctrl->pad == 0) {
    ctrl->iters += 1;
    ctrl->gamma_prev = reinterpret_cast<double*>(ctrl + 1)[0];
    ctrl->alpha_prev = reinterpret_cast<double*>(ctrl + 1)[1];
  }
}

__global__ void k_gather_f32(const float* __restrict__ src, const int64_t* __restrict__ idx, int64_t m,
                             float* __restrict__ out) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < m) out[i] = src[idx[i]];
}
__global__ void k_scatter_f32(const float* __restrict__ src, const int64_t* __restrict__ idx, int64_t m,
                              float* __restrict__ dst) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i < m) dst[idx[i]] = src[i];
}

struct DcgWs {
  double* part;   // 3 * kGrid
  PcgCtrl* ctrl;  // followed by 2 stash doubles
};
static DcgWs carve_dcg(void* ws) {
  unsigned char* c = reinterpret_cast<unsigned char*>(ws);
  DcgWs w;
  w.part = reinterpret_cast<double*>(c);
  c += align256(3 * kGrid * sizeof(double));
  w.ctrl = reinterpret_cast<PcgCtrl*>(c);
  return w;
}

}  // namespace

extern "C" {

size_t nksr_dcg_workspace_bytes(void) {
  return align256(3 * kGrid * sizeof(double)) + align256(sizeof(PcgCtrl) + 2 * sizeof(double)) + 256;
}

int nksr_dcg_init(const float* diag, const float* b, const uint8_t* owned, float* x, float* r, float* u, float* p,
                  float* s, int64_t n, void* ws, size_t ws_bytes, double* red, void* stream) {
  if (n <= 0 || !ws || !red) return NKSR_E_INVALID;
  if (ws_bytes < nksr_dcg_workspace_bytes()) return NKSR_E_WORKSPACE;
  cudaStream_t st = as_stream(stream);
  DcgWs w = carve_dcg(ws);
  if (cudaMemsetAsync(ws, 0, nksr_dcg_workspace_bytes(), st) != cudaSuccess) return NKSR_E_CUDA;
  k_dcg_init<<<kGrid, kBlock, 0, st>>>(diag, b, owned, x, r, u, p, s, n, w.part);
  k_reduce_arrays<<<1, kBlock, 0, st>>>(w.part, 3, red, nullptr);   // red[1], red[2] = 0
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_dcg_begin(void* ws, const double* red, float tol, int max_iter, void* stream) {
  if (!ws || !red || max_iter < 0) return NKSR_E_INVALID;
  k_dcg_begin<<<1, 1, 0, as_stream(stream)>>>(red, tol, max_iter, carve_dcg(ws).ctrl);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_dcg_spmv_dots(const int64_t* rowptr, const int32_t* col, const float* val, const uint8_t* owned,
                       const float* r, const float* u, float* w, int64_t n, void* ws, double* red, void* stream) {
  if (n <= 0 || !ws || !red) return NKSR_E_INVALID;
  cudaStream_t st = as_stream(stream);
  DcgWs d = carve_dcg(ws);
  k_dcg_spmv<<<kGrid, kBlock, 0, st>>>(rowptr, col, val, owned, r, u, w, n, d.part, d.ctrl);
  k_reduce_arrays<<<1, kBlock, 0, st>>>(d.part, 3, red, d.ctrl);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_dcg_op_dots(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                     const int32_t* base_pos, const int32_t* base_nrm, void* op_ws, size_t op_ws_bytes,
                     const uint8_t* owned, const float* r, const float* u, float* w, void* ws, double* red,
                     void* stream) {
  if (!ws || !red || !owned || !r || !u || !w) return NKSR_E_INVALID;
  MfOperator mf;
  const int rc = mf_operator_make(svh, feat, c, base_pos, base_nrm, op_ws, op_ws_bytes, &mf);
  if (rc != NKSR_OK) return rc;
  cudaStream_t st = as_stream(stream);
  DcgWs d = carve_dcg(ws);
  // the dots land in the partial arrays of k_dcg_spmv's layout (kGrid blocks of kBlock = 256 threads)
  mf_dcg_launch(mf, owned, r, u, w, d.part, kGrid, &d.ctrl->done, st);
  k_reduce_arrays<<<1, kBlock, 0, st>>>(d.part, 3, red, d.ctrl);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_dcg_update(const float* diag, const uint8_t* owned, float* x, float* r, float* u, const float* w, float* p,
                    float* s, int64_t n, void* ws, const double* red, void* stream) {
  if (n <= 0 || !ws || !red) return NKSR_E_INVALID;
  cudaStream_t st = as_stream(stream);
  DcgWs d = carve_dcg(ws);
  k_dcg_update<<<kGrid, kBlock, 0, st>>>(diag, owned, x, r, u, w, p, s, n, red, d.ctrl);
  k_dcg_commit<<<1, 1, 0, st>>>(d.ctrl);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

/* info (host double[4]): iterations, relative residual, status (0 converged, 1 running/max_iter, 2 NaN), done flag */
int nksr_dcg_status(void* ws, double* info, void* stream) {
  if (!ws || !info) return NKSR_E_INVALID;
  PcgCtrl host;
  const int rc = read_ctrl(carve_dcg(ws).ctrl, &host, as_stream(stream));
  if (rc != NKSR_OK) return rc;
  info[0] = (double)host.iters;
  info[1] = host.bb > 0.0 ? sqrt(host.rr / host.bb) : 0.0;
  info[2] = (double)(host.done == 1 ? 0 : (host.done == 2 ? 2 : 1));
  info[3] = (double)host.done;
  return NKSR_OK;
}

int nksr_gather_f32(const float* src, const int64_t* idx, int64_t m, float* out, void* stream) {
  if (m < 0) return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  k_gather_f32<<<grid_for(m, 256), 256, 0, as_stream(stream)>>>(src, idx, m, out);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_scatter_f32(const float* src, const int64_t* idx, int64_t m, float* dst, void* stream) {
  if (m < 0) return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  k_scatter_f32<<<grid_for(m, 256), 256, 0, as_stream(stream)>>>(src, idx, m, dst);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
