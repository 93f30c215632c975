// Backward of the sparse convolution y = act(bias + res + sum_k x[idx[:, k]] . W[k]) (csrc/sparse_conv.cu), what
// training the U-Net backbone needs (nksr_b200/unet.py, DESIGN 4.3):
//
//   weight gradient   dW[k] = sum_i [idx[i,k] >= 0] x[idx[i,k], :]^T g[i, :]      (c_in x c_out per tap)
//                     db    = sum_i g[i, :]
//   input gradient    dx[j] = sum_k g[idx_t[j,k], :] . W[k]^T  -- nksr_gather_gemm itself over the transposed table
//                     idx_t[j,k] = i  iff  idx[i,k] = j   (nksr_transpose_taps; every U-Net table is injective per tap)
//
// Weight gradient: a reduction over the rows, which must be deterministic and must not lose accuracy with n_out.
//   * The rows are cut into spans by the shapes alone (wgrad_spans below): never by the SM count, so the result is the
//     same bits on every device.  A CTA owns (tap k, TI input channels, TO output channels, span); the tap is the
//     fastest grid dimension, so the CTAs of the K taps that read the same g rows of a span run together and all but
//     one of them find those rows in L2.
//   * Per chunk of 32 rows the CTA gathers x[idx[r, k], ci0 : ci0 + TI] (absent sources as zeros; a chunk without any
//     source for the tap is skipped) and g[r, co0 : co0 + TO] into shared memory (row stride TI + 8 / TO + 8 floats: the
//     transposed fragment reads below hit 32 distinct banks).
//   * fp32 (tf32 = 0): each thread owns (TI / 16) x (TO / 16) entries, one fmaf per row in row order.
//     TF32 (tf32 = 1..3): mma.sync.m16n8k8 with the rows as the MMA's K dimension: A = x chunk^T, B = g chunk, both
//     fragments read transposed out of the row-major tiles and rounded with cvt.rna (as the forward mma.sync kernel).
//     wgmma's TF32 form takes only K-major operands, and here both operands are M- / N-major in memory.
//   * fp32 accumulation over at most kFoldRows = 256 rows, then folded into an fp64 accumulator; each span writes its
//     fp64 partial to the workspace and a second kernel sums the partials in span order.  The fp32 error is that of a
//     256-term sum whatever n_out is.
// No floating-point atomics anywhere; two calls give the same bits.
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kRC = 32;                        // rows per staged chunk
constexpr int kFoldRows = 256;                 // rows summed in fp32 before they are folded into fp64
constexpr int64_t kWsEntries = int64_t(1) << 22;   // fp64 partials the spans may take (32 MB), bounds the span count

// spans of the weight-gradient reduction: a function of the shapes only.  Spans are whole fold blocks; as many as fit
// kWsEntries partials of K * c_in * c_out + c_out values, at most one per fold block.
void wgrad_spans(int64_t n_out, int K, int c_in, int c_out, int64_t* n_spans, int64_t* span_rows) {
  const int64_t folds = (n_out + kFoldRows - 1) / kFoldRows;
  if (folds == 0) { *n_spans = 0; *span_rows = kFoldRows; return; }
  const int64_t per_span = (int64_t)K * c_in * c_out + c_out;
  int64_t s = kWsEntries / per_span;
  if (s < 1) s = 1;
  if (s > folds) s = folds;
  const int64_t per = (folds + s - 1) / s;     // fold blocks per span
  *span_rows = per * kFoldRows;
  *n_spans = (folds + per - 1) / per;
}

__device__ __forceinline__ uint32_t to_tf32(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return r;
}

// D (16x8, fp32) += A (16x8, tf32, row) * B (8x8, tf32, col); fragment layout as in sparse_conv.cu
__device__ __forceinline__ void mma_tf32(float* d, const uint32_t (&a)[4], const uint32_t b0, const uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// Accumulator ownership.  fp32: thread (ty, tx) = (tid / 16, tid % 16) owns ci = ty * MI + i, co = tx * MJ + j.
// TF32: warp w owns ci rows 16 (w % WM) .. + 15 and NT 8-column tiles from co = (w / WM) * NT * 8; lane (g, t) holds
// (ci g, co 2t), (g, 2t+1), (g+8, 2t), (g+8, 2t+1) of each tile, in this order.
template <int TI, int TO, bool TF32>
struct WgradTile {
  static constexpr int MI = TI / 16, MJ = TO / 16;
  static constexpr int WM = TI / 16, WN = 8 / WM, NT = TO / WN / 8;
  static constexpr int N = TF32 ? NT * 4 : MI * MJ;        // accumulators per thread
  __device__ static void coords(const int tid, const int e, int& ci, int& co) {
    if (TF32) {
      const int wid = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
      const int j = e >> 2, q = e & 3;
      ci = (wid % WM) * 16 + g + ((q & 2) ? 8 : 0);
      co = (wid / WM) * NT * 8 + j * 8 + 2 * t + (q & 1);
    } else {
      ci = (tid >> 4) * MI + e / MJ;
      co = (tid & 15) * MJ + e % MJ;
    }
  }
};

template <int TI, int TO, bool TF32>
__global__ void __launch_bounds__(kThreads, 2)
k_wgrad(const float* __restrict__ x, const int32_t* __restrict__ idx, int64_t n_out, int K,
        const float* __restrict__ g, int Cin, int Cout, int64_t span_rows, double* __restrict__ part,
        double* __restrict__ part_db) {
  using T = WgradTile<TI, TO, TF32>;
  constexpr int XS = TI + 8, GS = TO + 8;      // row strides = 8 mod 32
  __shared__ __align__(16) float Xs[kRC * XS];
  __shared__ __align__(16) float Gs[kRC * GS];
  __shared__ int32_t src_s[kRC];
  const int tid = threadIdx.x;
  const int k = blockIdx.x;
  const int n_to = Cout / TO;
  const int ti = blockIdx.y / n_to, to = blockIdx.y % n_to;
  const int ci0 = ti * TI, co0 = to * TO;
  const int64_t span = blockIdx.z;
  const int64_t r_begin = span * span_rows;
  const int64_t r_end = min(n_out, r_begin + span_rows);
  const bool do_db = part_db != nullptr && k == 0 && ti == 0;    // one CTA column also sums g for the bias

  float acc[T::N];
  double accd[T::N];
#pragma unroll
  for (int e = 0; e < T::N; ++e) { acc[e] = 0.f; accd[e] = 0.0; }
  float dbf = 0.f;
  double dbd = 0.0;

  for (int64_t c = 0;; ++c) {
    const int64_t r0 = r_begin + c * kRC;
    if (r0 >= r_end) break;
    int src = -1;
    if (tid < kRC) {
      const int64_t r = r0 + tid;
      if (r < r_end) src = __ldg(idx + r * K + k);
      src_s[tid] = src;
    }
    const bool any = __syncthreads_or(src >= 0);
    if (any || do_db) {
      for (int e = tid; e < kRC * TI / 4; e += kThreads) {
        const int r = e / (TI / 4), q = e % (TI / 4);
        const int s = src_s[r];
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (s >= 0) v = __ldg(reinterpret_cast<const float4*>(x + (int64_t)s * Cin + ci0) + q);
        *reinterpret_cast<float4*>(&Xs[r * XS + q * 4]) = v;
      }
      for (int e = tid; e < kRC * TO / 4; e += kThreads) {
        const int r = e / (TO / 4), q = e % (TO / 4);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r0 + r < r_end) v = __ldg(reinterpret_cast<const float4*>(g + (r0 + r) * Cout + co0) + q);
        *reinterpret_cast<float4*>(&Gs[r * GS + q * 4]) = v;
      }
      __syncthreads();
      if (any) {
        if (TF32) {
          const int wid = tid >> 5, lane = tid & 31, gq = lane >> 2, t = lane & 3;
          const int m0 = (wid % T::WM) * 16, nb = (wid / T::WM) * T::NT * 8;
#pragma unroll
          for (int ks = 0; ks < kRC; ks += 8) {
            uint32_t a[4];
            a[0] = to_tf32(Xs[(ks + t) * XS + m0 + gq]);
            a[1] = to_tf32(Xs[(ks + t) * XS + m0 + gq + 8]);
            a[2] = to_tf32(Xs[(ks + t + 4) * XS + m0 + gq]);
            a[3] = to_tf32(Xs[(ks + t + 4) * XS + m0 + gq + 8]);
#pragma unroll
            for (int j = 0; j < T::NT; ++j) {
              const uint32_t b0 = to_tf32(Gs[(ks + t) * GS + nb + j * 8 + gq]);
              const uint32_t b1 = to_tf32(Gs[(ks + t + 4) * GS + nb + j * 8 + gq]);
              mma_tf32(acc + 4 * j, a, b0, b1);
            }
          }
        } else {
          const int ty = tid >> 4, tx = tid & 15;
#pragma unroll 4
          for (int r = 0; r < kRC; ++r) {
            float av[T::MI], bv[T::MJ];
#pragma unroll
            for (int i = 0; i < T::MI; ++i) av[i] = Xs[r * XS + ty * T::MI + i];
#pragma unroll
            for (int j = 0; j < T::MJ; ++j) bv[j] = Gs[r * GS + tx * T::MJ + j];
#pragma unroll
            for (int i = 0; i < T::MI; ++i)
#pragma unroll
              for (int j = 0; j < T::MJ; ++j) acc[i * T::MJ + j] = fmaf(av[i], bv[j], acc[i * T::MJ + j]);
          }
        }
      }
      if (do_db && tid < TO) {
        for (int r = 0; r < kRC; ++r) dbf += Gs[r * GS + tid];
      }
      __syncthreads();
    }
    if ((c + 1) % (kFoldRows / kRC) == 0) {    // end of a fold block (spans start on fold-block boundaries)
#pragma unroll
      for (int e = 0; e < T::N; ++e) { accd[e] += (double)acc[e]; acc[e] = 0.f; }
      dbd += (double)dbf;
      dbf = 0.f;
    }
  }
#pragma unroll
  for (int e = 0; e < T::N; ++e) accd[e] += (double)acc[e];
  dbd += (double)dbf;

  double* out = part + ((span * K + k) * Cin + ci0) * Cout + co0;
#pragma unroll
  for (int e = 0; e < T::N; ++e) {
    int ci, co;
    T::coords(tid, e, ci, co);
    out[(int64_t)ci * Cout + co] = accd[e];
  }
  if (do_db && tid < TO) part_db[span * Cout + co0 + tid] = dbd;
}

// dW[e] = sum over spans, in span order, of the partials (fp64), then rounded once to fp32; db likewise
__global__ void k_wgrad_reduce(const double* __restrict__ part, const double* __restrict__ part_db, int64_t n_spans,
                               int64_t n_w, int Cout, float* __restrict__ dW, float* __restrict__ db) {
  const int64_t n = n_w + (db ? Cout : 0);
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    double s = 0.0;
    if (e < n_w) {
      for (int64_t p = 0; p < n_spans; ++p) s += part[p * n_w + e];
      dW[e] = (float)s;
    } else {
      const int64_t j = e - n_w;
      for (int64_t p = 0; p < n_spans; ++p) s += part_db[p * Cout + j];
      db[j] = (float)s;
    }
  }
}

template <int TI, int TO, bool TF32>
void launch_wgrad(dim3 grid, cudaStream_t s, const float* x, const int32_t* idx, int64_t n_out, int K, const float* g,
                  int c_in, int c_out, int64_t span_rows, double* part, double* part_db) {
  k_wgrad<TI, TO, TF32><<<grid, kThreads, 0, s>>>(x, idx, n_out, K, g, c_in, c_out, span_rows, part, part_db);
}

template <bool TF32>
void launch_wgrad_tiles(int ti, int to, dim3 grid, cudaStream_t s, const float* x, const int32_t* idx, int64_t n_out,
                        int K, const float* g, int c_in, int c_out, int64_t span_rows, double* part, double* part_db) {
  if (ti == 64 && to == 64) launch_wgrad<64, 64, TF32>(grid, s, x, idx, n_out, K, g, c_in, c_out, span_rows, part, part_db);
  else if (ti == 64) launch_wgrad<64, 32, TF32>(grid, s, x, idx, n_out, K, g, c_in, c_out, span_rows, part, part_db);
  else if (to == 64) launch_wgrad<32, 64, TF32>(grid, s, x, idx, n_out, K, g, c_in, c_out, span_rows, part, part_db);
  else launch_wgrad<32, 32, TF32>(grid, s, x, idx, n_out, K, g, c_in, c_out, span_rows, part, part_db);
}

bool wgrad_shape_ok(int64_t n_out, int K, int c_in, int c_out, int tf32) {
  if (tf32 < 0 || tf32 > 3) return false;
  if (n_out < 0 || K < 1 || c_in < 32 || c_in % 32 != 0 || c_out < 32 || c_out % 32 != 0) return false;
  if (tf32 && K > 32) return false;            // the forward's TF32 limit, kept for the pair
  return true;
}

__global__ void k_fill_i32(int32_t* __restrict__ p, int64_t n, int32_t v) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) p[e] = v;
}

__global__ void k_transpose_scatter(const int32_t* __restrict__ idx, int64_t n, int K, int64_t n_src,
                                    int32_t* __restrict__ idx_t, int32_t* __restrict__ status) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int32_t j = __ldg(idx + e);
    if (j < 0) continue;
    if (j >= n_src) { atomicOr(status, 2); continue; }
    const int64_t i = e / K;
    idx_t[(int64_t)j * K + (e - i * K)] = (int32_t)i;      // plain store: with a collision one writer wins
  }
}

__global__ void k_transpose_verify(const int32_t* __restrict__ idx, int64_t n, int K, int64_t n_src,
                                   const int32_t* __restrict__ idx_t, int32_t* __restrict__ status) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int32_t j = __ldg(idx + e);
    if (j < 0 || j >= n_src) continue;
    const int64_t i = e / K;
    if (idx_t[(int64_t)j * K + (e - i * K)] != (int32_t)i) atomicOr(status, 1);   // the loser of a collision
  }
}

}  // namespace

extern "C" {

size_t nksr_gather_gemm_wgrad_workspace_bytes(int64_t n_out, int K, int c_in, int c_out, int tf32) {
  if (!wgrad_shape_ok(n_out, K, c_in, c_out, tf32)) return 0;
  int64_t n_spans, span_rows;
  wgrad_spans(n_out, K, c_in, c_out, &n_spans, &span_rows);
  return (size_t)n_spans * ((size_t)K * c_in * c_out + c_out) * sizeof(double);
}

int nksr_gather_gemm_wgrad(const float* x, const int32_t* idx, int64_t n_out, int K, const float* g, int c_in,
                           int c_out, float* dW, float* db, void* ws, size_t ws_bytes, int tf32, void* stream) {
  if (!wgrad_shape_ok(n_out, K, c_in, c_out, tf32)) return NKSR_E_INVALID;
  if (!dW) return NKSR_E_INVALID;
  cudaStream_t s = as_stream(stream);
  const int64_t n_w = (int64_t)K * c_in * c_out;
  if (n_out == 0) {                            // empty sum
    if (cudaMemsetAsync(dW, 0, n_w * sizeof(float), s) != cudaSuccess) return NKSR_E_CUDA;
    if (db && cudaMemsetAsync(db, 0, c_out * sizeof(float), s) != cudaSuccess) return NKSR_E_CUDA;
    return NKSR_OK;
  }
  if (!x || !idx || !g) return NKSR_E_INVALID;
  int64_t n_spans, span_rows;
  wgrad_spans(n_out, K, c_in, c_out, &n_spans, &span_rows);
  if (ws_bytes < nksr_gather_gemm_wgrad_workspace_bytes(n_out, K, c_in, c_out, tf32) || !ws) return NKSR_E_WORKSPACE;
  double* part = static_cast<double*>(ws);
  double* part_db = db ? part + n_spans * n_w : nullptr;
  const int ti = c_in % 64 == 0 ? 64 : 32, to = c_out % 64 == 0 ? 64 : 32;
  const dim3 grid((unsigned)K, (unsigned)((c_in / ti) * (c_out / to)), (unsigned)n_spans);
  if (tf32)
    launch_wgrad_tiles<true>(ti, to, grid, s, x, idx, n_out, K, g, c_in, c_out, span_rows, part, part_db);
  else
    launch_wgrad_tiles<false>(ti, to, grid, s, x, idx, n_out, K, g, c_in, c_out, span_rows, part, part_db);
  NKSR_CHECK_LAUNCH();
  const int64_t n_red = n_w + (db ? c_out : 0);
  k_wgrad_reduce<<<(unsigned)std::min<int64_t>((n_red + 255) / 256, 4096), 256, 0, s>>>(part, part_db, n_spans, n_w, c_out,
                                                                                    dW, db);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_transpose_taps(const int32_t* idx, int64_t n_out, int K, int64_t n_src, int32_t* idx_t, int32_t* status,
                        void* stream) {
  if (n_out < 0 || n_src < 0 || K < 1 || n_out > INT32_MAX) return NKSR_E_INVALID;
  if (!status || (n_src > 0 && !idx_t) || (n_out > 0 && !idx)) return NKSR_E_INVALID;
  cudaStream_t s = as_stream(stream);
  const int64_t n_t = n_src * K, n = n_out * K;
  if (n_t > 0) k_fill_i32<<<(unsigned)std::min<int64_t>((n_t + 255) / 256, 8192), 256, 0, s>>>(idx_t, n_t, -1);
  if (n > 0) {
    const unsigned blocks = (unsigned)std::min<int64_t>((n + 255) / 256, 8192);
    k_transpose_scatter<<<blocks, 256, 0, s>>>(idx, n, K, n_src, idx_t, status);
    k_transpose_verify<<<blocks, 256, 0, s>>>(idx, n, K, n_src, idx_t, status);
  }
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
