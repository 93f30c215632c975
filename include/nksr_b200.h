/* nksr_b200 -- C-ABI of the H100-native (sm_90a) NKSR reconstruction hot path.
 *
 * Every entry point is `extern "C"`, takes plain device pointers + sizes + a cudaStream_t
 * (passed as void*), performs NO allocation (the caller owns every buffer, normally torch
 * tensors) and returns 0 or a negative NKSR_E* code.  Variable-size outputs are two-phase:
 * a *_count / capacity call, the caller allocates, a *_fill call.
 *
 * The reference ships this path as the closed `nksr` wheel, so each group below cites the
 * reference CALL SITE whose behaviour it replaces (paths relative to the reference checkout, nv-tlabs/NKSR @ 0d4e369).
 * The reference-side binding is the ctypes shim in nksr_b200/_lib.py (see INTEGRATION.md).
 */
#ifndef NKSR_B200_H
#define NKSR_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define NKSR_API __attribute__((visibility("default")))
#else
#define NKSR_API
#endif

#define NKSR_MAX_DEPTH 8
#define NKSR_ROW_STRIDE 32 /* a kernel-row has 27 stencil slots, padded to one 128 B line */

enum {
  NKSR_OK = 0,
  NKSR_E_INVALID = -1,   /* bad argument                                  */
  NKSR_E_RANGE = -2,     /* coordinate outside the 2^19-voxel key range    */
  NKSR_E_WORKSPACE = -3, /* workspace too small                            */
  NKSR_E_CUDA = -4,      /* a CUDA call failed (cudaGetLastError)          */
  NKSR_E_STRUCTURE = -5  /* hierarchy not parent-closed / table mismatch   */
};

/* Device view of a sparse voxel hierarchy (replaces nksr.SparseFeatureHierarchy internals;
 * contract: models/nksr_net.py:57-62, models/loss.py:33-46). Level l has voxel size
 * voxel_size*2^l; voxels of a level are sorted by 63-bit Morton key. */
typedef struct {
  int32_t depth;
  float voxel_size;
  int64_t n[NKSR_MAX_DEPTH];             /* voxels per level                         */
  int64_t offset[NKSR_MAX_DEPTH];        /* first unknown of the level in alpha      */
  const int64_t* keys[NKSR_MAX_DEPTH];   /* [n] sorted Morton keys                   */
  const int32_t* parent[NKSR_MAX_DEPTH]; /* [n] index at level+1 (NULL at the top)   */
  const int32_t* child8[NKSR_MAX_DEPTH]; /* [n][8] index at level-1, -1 (NULL at 0)  */
  const int32_t* nbr27[NKSR_MAX_DEPTH];  /* [n][27] same-level neighbours, -1        */
  const int32_t* nbr125_top;             /* [n_top][125] 5^3 neighbours of the coarsest level */
} nksr_svh_t;

/* Per-level kernel features z_i (replaces features=feat.basis_features passed to
 * nksr.fields.KernelField, models/nksr_net.py:91-96). */
typedef struct {
  int32_t channels; /* C: 1..32 */
  const float* z[NKSR_MAX_DEPTH]; /* [n_l][C] */
} nksr_feat_t;

NKSR_API const char* nksr_version(void);
NKSR_API const char* nksr_error_string(int code);

/* ---- a1: SparseFeatureHierarchy.build_point_splatting (models/nksr_net.py:57-62) ---- */
/* half-voxel Morton key of every point: morton(floor(x/(W/2)) + 2^20). status[0] |= 1 on range error */
NKSR_API int nksr_point_half_keys(const float* xyz, int64_t n, float voxel_size, int64_t* keys,
                         int32_t* status, void* stream);
NKSR_API size_t nksr_sort_workspace_bytes(int64_t n, int pairs);
NKSR_API int nksr_sort_keys(const int64_t* keys_in, int64_t* keys_out, int64_t n, void* ws,
                   size_t ws_bytes, void* stream);
NKSR_API int nksr_sort_pairs(const int64_t* keys_in, int64_t* keys_out, const int32_t* vals_in,
                    int32_t* vals_out, int64_t n, void* ws, size_t ws_bytes, void* stream);
NKSR_API size_t nksr_unique_workspace_bytes(int64_t n);
/* out = unique(in >> shift) for sorted `in`; *count_out (device int64) = number written */
NKSR_API int nksr_unique_sorted(const int64_t* in, int64_t n, int shift, int64_t* out,
                       int64_t* count_out, void* ws, size_t ws_bytes, void* stream);
/* 8 splat candidates (level-l voxel keys) per unique level-l half key */
NKSR_API int nksr_splat_candidates(const int64_t* half_keys, int64_t n, int64_t* out8, void* stream);
NKSR_API int nksr_parent_index(const int64_t* keys, int64_t n, const int64_t* keys_up, int64_t n_up,
                      int32_t* parent, int32_t* status, void* stream);
NKSR_API int nksr_child_table(const int64_t* keys, const int32_t* parent, int64_t n, int32_t* child8_up,
                     int64_t n_up, void* stream);
NKSR_API int nksr_nbr27_search(const int64_t* keys, int64_t n, int32_t* nbr27, void* stream);
NKSR_API int nksr_nbr125_search(const int64_t* keys, int64_t n, int32_t* nbr125, void* stream);
NKSR_API int nksr_nbr27_from_parent(const int64_t* keys, const int32_t* parent, int64_t n,
                           const int32_t* nbr27_up, const int32_t* child8_up, int32_t* nbr27,
                           void* stream);
/* active_grid_coords() (models/loss.py:36): int32 ijk per voxel */
NKSR_API int nksr_decode_ijk(const int64_t* keys, int64_t n, int level, int32_t* ijk, void* stream);
/* containing voxel per level for M locations: base[l*M + m], -1 if inactive */
NKSR_API int nksr_locate(const nksr_svh_t* svh, const float* xyz, int64_t m, int32_t* base, void* stream);
/* out[i][c] = sum of in[j][c] over the active 27-neighbourhood j of voxel i (feature pooling for
 * the encoder stand-in that feeds models/nksr_net.py:73-78) */
NKSR_API int nksr_pool27(const int32_t* nbr27, const float* in, int64_t n, int channels, float* out,
                void* stream);
/* out[p][c] = sum of in[child][c] over the children of voxel p (n = voxels of the parent level) */
NKSR_API int nksr_pool_children(const int32_t* child8, const float* in, int64_t n, int channels,
                       float* out, void* stream);
/* ---- f2: the sparse convolution of NKSRNetwork's encoder / U-Net (models/nksr_net.py:73-78; unet.f_maps,
 * configs/default/train.yaml:17-18) as a gather-GEMM over the hierarchy's index tables:
 *   y[i,:] = act(bias + res[i,:] + sum_k [idx[i*K+k] >= 0] x[idx[i*K+k],:] . W[k])      W: K x c_in x c_out, row-major
 * idx = nbr27[l] (K = 27): 3x3x3 convolution on level l; idx = child8[l+1] (K = 8): stride-2 convolution l -> l+1.
 * c_in and c_out multiples of 32; bias / res may be NULL; relu: 0/1; tf32: 0 = fp32 FFMA, 1 = mma.sync TF32 (fp32
 * accumulation, operands rounded to TF32 in the kernel, K <= 32), 2 = the same with W already rounded to TF32 by the
 * caller (low 13 mantissa bits zero), 3 = wgmma.mma_async tf32 with the accumulator in registers (K <= 32 x 32-channel
 * steps staged in 128-byte-swizzled shared memory by cp.async; W rounded to TF32 by the caller AND transposed to
 * K x c_out x c_in, the tensor core's K-major operand order) */
NKSR_API int nksr_gather_gemm(const float* x, const int32_t* idx, int64_t n_out, int K, const float* W,
                     const float* bias, const float* res, float* y, int c_in, int c_out, int relu, int tf32,
                     void* stream);
/* Backward of nksr_gather_gemm (csrc/sparse_conv_bwd.cu).  Weight gradient of the same convolution for the output
 * gradient g (n_out x c_out, already multiplied by the activation's derivative):
 *   dW[k] = sum_i [idx[i*K+k] >= 0] x[idx[i*K+k],:]^T g[i,:]   (K x c_in x c_out)    db = sum_i g[i,:] (db may be NULL)
 * Deterministic (no atomics; rows cut into spans fixed by the shapes, fp32 over <= 256 rows, fp64 across them).
 * tf32: 0 = fp32 FFMA; 1..3 = mma.sync TF32 with x and g rounded by cvt.rna.  Shape limits as nksr_gather_gemm;
 * n_out = 0 gives zeros.  ws: nksr_gather_gemm_wgrad_workspace_bytes(...) bytes, else NKSR_E_WORKSPACE. */
NKSR_API size_t nksr_gather_gemm_wgrad_workspace_bytes(int64_t n_out, int K, int c_in, int c_out, int tf32);
NKSR_API int nksr_gather_gemm_wgrad(const float* x, const int32_t* idx, int64_t n_out, int K, const float* g,
                           int c_in, int c_out, float* dW, float* db, void* ws, size_t ws_bytes, int tf32,
                           void* stream);
/* idx_t (n_src x K) = the transpose of a per-tap injective table idx (n_out x K): idx_t[j*K+k] = i iff idx[i*K+k] = j,
 * -1 elsewhere.  The input gradient of the convolution over idx is nksr_gather_gemm over idx_t.  *status (device,
 * zeroed by the caller) |= 1 when two rows share a (source, tap), |= 2 when a source is >= n_src. */
NKSR_API int nksr_transpose_taps(const int32_t* idx, int64_t n_out, int K, int64_t n_src, int32_t* idx_t,
                        int32_t* status, void* stream);
/* first/last+1 sorted location of every level-l voxel: range[2*u], range[2*u+1] */
NKSR_API int nksr_row_ranges(const int32_t* base_l, int64_t m, int32_t* range, int64_t n_l, void* stream);

/* ---- a3: KernelField.solve* Gram assembly (models/nksr_net.py:100-112) ---- */
/* kernel rows, location-major (all lines of one location are contiguous):
 *   mode 0: value rows    e[(m*L + l)*32 + s]             (position constraints)
 *   mode 1: gradient rows e[((m*L + l)*3 + a)*32 + s]     (normal constraints)
 *   mode 2: compact gradient rows e[(m*L + l)*32 + s], s<27: <phi,z_s>, s=27..29: tau
 *           (approx_kernel_grad only; the assembly rebuilds the three rows)
 *   mode | 4 (modes 0 and 1, depth <= 4): interleaved layout, the four levels of a slot are one float4:
 *           value rows e[(m*32 + s)*4 + l], gradient rows e[((m*3 + a)*32 + s)*4 + l]; levels >= depth are zero */
NKSR_API int nksr_build_rows(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* xyz,
                    const int32_t* base, int64_t m, int mode, int approx_kernel_grad, float* e,
                    void* stream);
/* the same rows, bitwise, built one warp per VOXEL: range = nksr_row_ranges of every level (concatenated in level
 * order) of the Morton-SORTED locations xyz; stencil and features are fetched once per voxel.  channels in {4, 8, 16},
 * otherwise NKSR_E_INVALID (callers then use nksr_build_rows) */
NKSR_API int nksr_build_rows_voxel(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* xyz,
                          const int32_t* base, const int32_t* range, int64_t m, int mode, int approx_kernel_grad,
                          float* e, void* stream);
/* structural row lengths of A: cnt[i] (same + coarser levels), cnt_down[i] (finer levels) */
NKSR_API int nksr_gram_count(const nksr_svh_t* svh, int32_t* cnt, int32_t* cnt_down, void* stream);
NKSR_API size_t nksr_scan_workspace_bytes(int64_t n);
/* rowptr[0..n] (int64) = exclusive scan of cnt[i] + cnt_down[i] */
NKSR_API int nksr_gram_rowptr(const int32_t* cnt, const int32_t* cnt_down, int64_t n, int64_t* rowptr,
                     void* ws, size_t ws_bytes, void* stream);
typedef struct {
  const float* e_pos;        /* value rows of the N sorted positions  [N][L][32]      */
  const int32_t* range_pos;  /* per level [n_l][2] (concatenated in level order)      */
  int64_t n_pos;
  float w_pos;
  const float* e_nrm;        /* gradient rows of the K sorted normal locations [K][L][3][32] */
  const int32_t* range_nrm;
  const float* t_nrm;        /* [K][3] targets (sorted order)                          */
  int64_t n_nrm;
  float w_nrm;
  float w_reg;
  int32_t nrm_compact;       /* row-layout code.  0: e_pos [N][L][32], e_nrm [K][L][3][32];  1: e_nrm holds compact rows
                              * [K][L][32] (nksr_build_rows mode 2);  2: both arrays interleaved, e_pos [N][32][4 levels],
                              * e_nrm [K][3][32][4 levels] (nksr_build_rows mode | 4, depth <= 4) */
  /* per-voxel Gram blocks of the coarse levels l >= split_level (nksr_gram_blocks); NULL = none.
   * Block of (level l, voxel u, offset k) starts at (mblock_off[l] + u*(depth-l) + k) * 28*32 floats */
  const float* mblocks;
  int32_t split_level;
  int64_t mblock_off[NKSR_MAX_DEPTH];
} nksr_constraints_t;
/* floats needed for the blocks of levels >= split_level */
NKSR_API int64_t nksr_gram_block_floats(const nksr_svh_t* svh, int split_level);
/* reduce, once per coarse voxel, the 27x27 products of its constraint rows (c->mblock_off and
 * c->split_level must be set; c->mblocks is ignored here) */
NKSR_API int nksr_gram_blocks(const nksr_svh_t* svh, const nksr_constraints_t* c, float* mblocks,
                     void* stream);
/* numeric assembly: fills col/val (CSR, int64 rowptr), rhs b, diag. cursor[n] must be zero. */
NKSR_API int nksr_gram_fill(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                   const int32_t* cnt, const int64_t* rowptr, int32_t* col, float* val,
                   float* rhs, float* diag, int32_t* cursor, void* stream);
/* sort the finer-level (transposed) segment of every row by column: deterministic storage */
NKSR_API int nksr_gram_sort_down(const int32_t* cnt, const int32_t* cnt_down, const int64_t* rowptr,
                        const int32_t* rows, int64_t n_rows, int cap, int32_t* col, float* val,
                        void* stream);

/* -- sort-free placement of the transposed entries (DESIGN.md SPEC S6b): same matrix, no atomics, no sort.
 * Fine voxel j (level l) reaches coarse voxel c (level l+k) through its ancestor a = c - d; its entry sits at
 *   rowptr[c] + cnt[c] + prefix[l][k][c*125 + slot(d)] + rank8[l][k][j*8 + S(d)],  S(d) = axes with |d| = 2. */
typedef struct {
  const int32_t* rank8[NKSR_MAX_DEPTH][NKSR_MAX_DEPTH];   /* [l][k] -> [n_l][8]       */
  const int32_t* prefix[NKSR_MAX_DEPTH][NKSR_MAX_DEPTH];  /* [l][k] -> [n_{l+k}][125] */
} nksr_placement_t;
/* cnt[i] only (same + coarser levels); the transposed lengths come from nksr_gram_place */
NKSR_API int nksr_gram_count_own(const nksr_svh_t* svh, int32_t* cnt, void* stream);
/* tables of one (fine level l, offset k >= 1) pair: rank8 [n_l][8], class_count [n_{l+k}][27] (scratch),
 * prefix [n_{l+k}][125]; advances cnt_down[offset[l+k] + c] by the entries level l adds to row c.
 * cnt_down must start at zero and, for one coarse level, the pairs must be issued in increasing l. */
NKSR_API int nksr_gram_place(const nksr_svh_t* svh, int l, int k, int32_t* rank8, int32_t* class_count,
                    int32_t* prefix, int32_t* cnt_down, void* stream);
/* nksr_gram_fill with the transposed copies written at their final position */
NKSR_API int nksr_gram_fill_placed(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                          const int32_t* cnt, const int64_t* rowptr, const nksr_placement_t* placement,
                          int32_t* col, float* val, float* rhs, float* diag, void* stream);
/* nksr_gram_fill_placed on the rows [row_begin, row_end) only (row_end = -1: to the last row) */
NKSR_API int nksr_gram_fill_placed_rows(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                               const int32_t* cnt, const int64_t* rowptr, const nksr_placement_t* placement,
                               int64_t row_begin, int64_t row_end, int32_t* col, float* val, float* rhs,
                               float* diag, void* stream);
/* the same matrix with the brick fill: the rows of a level below c->split_level that holds at least
 * min_locations_per_voxel constraint locations (positions + normals) per voxel are filled one brick (the level-l voxels
 * under one level-(l+2) key) per block, every constraint line of a source voxel loaded once per brick and multiplied
 * into all its target rows there; every other row runs nksr_gram_fill_placed.  Same CSR pattern and storage order; the
 * 27 per-source partial sums of a bricked row are added in a different (fixed) order.  Compact gradient rows and
 * depth > 4 run nksr_gram_fill_placed on every row. */
NKSR_API int nksr_gram_fill_brick(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                         const int32_t* cnt, const int64_t* rowptr, const nksr_placement_t* placement,
                         int32_t* col, float* val, float* rhs, float* diag, float min_locations_per_voxel,
                         void* stream);

/* the same fill with the sibling-group decomposition (one warp per level-(l+1) voxel = up to eight matrix rows
 * that share their constraint rows, column tables and flush indices): same CSR, same order.  Needs depth <= 4
 * and the virtual level above the coarsest one (svh->parent[depth-1], child8[depth], nbr27[depth]); returns
 * NKSR_E_INVALID otherwise (callers then use nksr_gram_fill_placed). */
NKSR_API int nksr_gram_fill_grouped(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                           const int32_t* cnt, const int64_t* rowptr, const nksr_placement_t* placement,
                           int32_t* col, float* val, float* rhs, float* diag, void* stream);

/* nksr_gram_count_own with one column table per sibling group (same restrictions as nksr_gram_fill_grouped) */
NKSR_API int nksr_gram_count_grouped(const nksr_svh_t* svh, int32_t* cnt, void* stream);

/* ---- a4: PCG (solver_tol, examples/recons_waymo.py:33; verbose, models/nksr_net.py:97) ---- */
NKSR_API int nksr_spmv(const int64_t* rowptr, const int32_t* col, const float* val, const float* x,
              float* y, int64_t n, void* stream);
NKSR_API size_t nksr_pcg_workspace_bytes(int64_t n);
/* Jacobi-PCG from x=0 with the convergence test on the device and the iterations replayed from a CUDA graph
 * of `check_every` iterations (one host read-back per graph launch).  info (host double[5]): [0]=iterations,
 * [1]=relative residual, [4]=status (0 converged, 1 max_iter reached, 2 NaN/breakdown); with profile != 0
 * (plain launches) also [2]=total ms of the live SpMV launches (CUDA events on `stream`, first 512 iterations)
 * and [3]=number of launches timed. */
NKSR_API int nksr_pcg_solve(const int64_t* rowptr, const int32_t* col, const float* val,
                   const float* diag, const float* b, float* x, int64_t n, float tol,
                   int max_iter, int check_every, int profile, void* ws, size_t ws_bytes,
                   double* info, void* stream);

/* -- the same PCG with the SpMV streamed through the TMA engine (csrc/spmv_stream.cuh): the (col, val) arrays are cut
 * into tiles of 4096 entries that one elected thread per CTA moves into a shared-memory ring with bulk async copies
 * (cp.async.bulk + mbarrier); consumer warps form the products in place and reduce the rows from shared memory.  Same
 * result up to the summation order inside a row (fixed, reproducible).  Bulk copies move whole 16-byte units: rowptr
 * must be readable up to index n + 1 (n + 2 entries) and col / val up to the next multiple of 4 entries. */
NKSR_API size_t nksr_pcg_stream_workspace_bytes(int64_t n, int64_t nnz);
/* rows [0, split_row) -- entries [0, split_nnz), split_nnz = rowptr[split_row] -- are streamed; rows >= split_row (the
 * coarse levels, whose transposed segments make rows of tens of thousands of entries) go through the warp-per-row
 * kernel, where a long row streams well and does not stall a tile behind one warp.  split_row = n streams everything. */
NKSR_API int nksr_pcg_solve_stream(const int64_t* rowptr, const int32_t* col, const float* val, const float* diag,
                          const float* b, float* x, int64_t n, int64_t nnz, int64_t split_row, int64_t split_nnz,
                          float tol, int max_iter, int check_every, int profile, void* ws, size_t ws_bytes,
                          double* info, void* stream);
/* y = A x through the same tile stream (plan_buf: nksr_spmv_plan_bytes(nnz) bytes of scratch) */
NKSR_API size_t nksr_spmv_plan_bytes(int64_t nnz);
NKSR_API int nksr_spmv_stream(const int64_t* rowptr, const int32_t* col, const float* val, const float* x, float* y,
                     int64_t n, int64_t nnz, int64_t split_row, int64_t split_nnz, void* plan_buf,
                     size_t plan_bytes, void* stream);

/* ---- e: step kernels of the multi-GPU solve (one global system, SURVEY section 8e mapping B).  A
 * Chronopoulos-Gear arrangement of the same Jacobi-PCG: per iteration ONE halo exchange of u = M^-1 r, one
 * SpMV on the owned rows and ONE fused all-reduce of red[3] = {(r,u), (w,u), (r,r)}; the caller issues the
 * collective (NCCL) on `red` between nksr_dcg_spmv_dots and nksr_dcg_update.  owned[i] != 0: row i belongs to
 * this rank.  All vectors are caller-owned (n floats each); ws: nksr_dcg_workspace_bytes(); red: 3 doubles. */
NKSR_API size_t nksr_dcg_workspace_bytes(void);
/* x=0, r=b, u=r/diag on owned rows; red[0] = local (b,b) -> all-reduce red, then nksr_dcg_begin */
NKSR_API int nksr_dcg_init(const float* diag, const float* b, const uint8_t* owned, float* x, float* r, float* u,
                  float* p, float* s, int64_t n, void* ws, size_t ws_bytes, double* red, void* stream);
NKSR_API int nksr_dcg_begin(void* ws, const double* red, float tol, int max_iter, void* stream);
/* w = A u on owned rows, red = local {(r,u), (w,u), (r,r)}; no-op once the solve is over */
NKSR_API int nksr_dcg_spmv_dots(const int64_t* rowptr, const int32_t* col, const float* val, const uint8_t* owned,
                       const float* r, const float* u, float* w, int64_t n, void* ws, double* red, void* stream);
/* red = all-reduced sums: convergence verdict on the device, else p,s,x,r,u advance one iteration */
NKSR_API int nksr_dcg_update(const float* diag, const uint8_t* owned, float* x, float* r, float* u, const float* w,
                    float* p, float* s, int64_t n, void* ws, const double* red, void* stream);
/* synchronising read-back: info (host double[4]) = iterations, relative residual, status as above, done flag */
NKSR_API int nksr_dcg_status(void* ws, double* info, void* stream);
/* halo packing: out[i] = src[idx[i]] / dst[idx[i]] = src[i] (idx: int64) */
NKSR_API int nksr_gather_f32(const float* src, const int64_t* idx, int64_t m, float* out, void* stream);
NKSR_API int nksr_scatter_f32(const float* src, const int64_t* idx, int64_t m, float* dst, void* stream);

/* ---- a5: field.evaluate_f (models/loss.py:189-198,225) ---- */
NKSR_API int nksr_evaluate(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* alpha,
                  const float* xyz, int64_t m, int want_grad, int approx_kernel_grad,
                  float* f, float* grad, void* stream);

/* ---- a7: field.extract_dual_mesh (models/nksr_net.py:214,284; examples/recons_simple.py:27) ---- */
/* flag[i]=1 if the dual cell with min corner voxel i exists (all 8 voxels active) */
NKSR_API int nksr_mesh_cell_flags(const nksr_svh_t* svh, int32_t* flag, void* stream);
/* min-corner lattice coords (int32 xyz, units W/R) of flagged voxels, in voxel order */
NKSR_API int nksr_mesh_stage0_cells(const nksr_svh_t* svh, const int32_t* flag, const int64_t* scan,
                           int32_t refine, int32_t* cells, void* stream);
/* adaptive hierarchies (models/nksr_net.py:175-179,214): a LEAF of level >= 1 (no children) is meshed as if it were
 * subdivided down to the finest level ("virtual" finest voxels), so all dual cells belong to one lattice.
 * leaf_flags: flag[v] = 1 for childless level-l voxels; virtual_anchors: the 8^l finest-level ijk below every flagged
 * voxel (scan = exclusive scan of flag; anchors [count * 8^l][3]); anchor_flags: flag[i] = 1 if the seven other corner
 * voxels anchor + {0,1}^3 exist, really (level 0) or virtually below a leaf of level < coarse_levels */
NKSR_API int nksr_mesh_leaf_flags(const nksr_svh_t* svh, int level, int32_t* flag, void* stream);
NKSR_API int nksr_mesh_virtual_anchors(const nksr_svh_t* svh, int level, const int32_t* flag, const int64_t* scan,
                              int32_t* anchors, void* stream);
NKSR_API int nksr_mesh_anchor_flags(const nksr_svh_t* svh, const int32_t* anchors, int64_t n, int coarse_levels,
                           int32_t* flag, void* stream);
/* split every cell into g^3 children of size size/g */
NKSR_API int nksr_mesh_split_cells(const int32_t* cells, int64_t n, int32_t size, int32_t g,
                          int32_t* out, void* stream);
/* 8 corner keys per cell: morton(corner - origin) */
NKSR_API int nksr_mesh_corner_keys(const int32_t* cells, int64_t n, int32_t size, int32_t ox, int32_t oy,
                          int32_t oz, int64_t* keys8, void* stream);
/* world positions of lattice keys: W*(0.5 + s/R) */
NKSR_API int nksr_mesh_lattice_pos(const int64_t* keys, int64_t n, int32_t ox, int32_t oy, int32_t oz,
                          float voxel_size, int32_t refine, float* xyz, void* stream);
/* per cell: corner values via binary search of corner keys, case index, crossing flag */
NKSR_API int nksr_mesh_classify(const int64_t* keys8, int64_t n_cells, const int64_t* ukeys,
                       const float* uval, int64_t n_u, float* cval8, int32_t* mc_case,
                       int32_t* crossing, void* stream);
/* gather rows selected by an exclusive scan of flags */
NKSR_API int nksr_compact_rows(const void* in, const int32_t* flag, const int64_t* scan, int64_t n,
                      int32_t row_bytes, void* out, void* stream);
NKSR_API size_t nksr_scan32_workspace_bytes(int64_t n);
NKSR_API int nksr_exclusive_scan32(const int32_t* in, int64_t* out, int64_t n, void* ws, size_t ws_bytes,
                          void* stream); /* out has n+1 entries */
/* per crossing cell: triangle count and 12 edge keys (or -1) */
NKSR_API int nksr_mesh_cell_edges(const int32_t* cells, const int32_t* mc_case, int64_t n, int32_t size,
                         int32_t ox, int32_t oy, int32_t oz, int32_t* ntri, int64_t* ekeys12,
                         void* stream);
/* flag[i] = 1 at the first element of every run of equal non-negative keys (sorted input) */
NKSR_API int nksr_run_heads(const int64_t* keys, int64_t n, int32_t* flag, void* stream);
/* vertices of unique edge keys (src = first cell*12+edge owning it) */
NKSR_API int nksr_mesh_vertices(const int64_t* uekeys, const int32_t* src, int64_t n_v,
                       const int32_t* cells, const float* cval8, int32_t size,
                       float voxel_size, int32_t refine, float* v, void* stream);
NKSR_API int nksr_mesh_triangles(const int32_t* mc_case, const int64_t* ekeys12, const int64_t* tri_scan,
                        int64_t n_cells, const int64_t* uekeys, int64_t n_v, int64_t* tri,
                        void* stream);
/* LayerField mask (models/nksr_net.py:132): 1 if x lies in an active voxel of level < adaptive_depth */
NKSR_API int nksr_layer_mask(const nksr_svh_t* svh, const float* xyz, int64_t m, int adaptive_depth,
                    float* out, void* stream);

/* ---- f1: nksr.get_estimate_normal_preprocess_fn (examples/recons_waymo.py:36; CPU twin
 *      examples/recons_waymo_cpu.py:21-41): voxel-neighbourhood PCA normals ---- */
/* per-voxel moments (count, sum d, sum d d^T; d relative to the voxel centre) of sorted points */
NKSR_API int nksr_voxel_moments(const int64_t* keys, int64_t n, const int32_t* range, const float* xyz,
                       float voxel_size, float* mom10, void* stream);
/* smallest-eigenvalue eigenvector of the covariance over the 27-neighbourhood */
NKSR_API int nksr_voxel_pca_normals(const int32_t* nbr27, const float* mom10, int64_t n, float voxel_size,
                           float* normal, void* stream);
/* per point: its voxel's normal flipped to the sensor side; keep = |cos| > cos_min */
NKSR_API int nksr_orient_normals(const float* xyz, const float* sensor, const int32_t* base,
                        const float* vox_normal, int64_t m, float cos_min, float* normal,
                        int32_t* keep, void* stream);

/* exact k-nearest-neighbour PCA normals (k <= 64, self included) on a multi-level voxel hash of Morton-SORTED points:
 * svh = hierarchy of the points' containing voxels (level l: voxel size voxel_size * 2^l), base[l*m + i] = containing
 * voxel of point i, range = nksr_row_ranges of every level (concatenated in level order).  Per point the finest level
 * whose 27-voxel block holds >= 3k points is searched; the result is exact when the k-th distance <= that voxel size,
 * otherwise the search repeats one level coarser (points still inexact on the coarsest level are counted in *inexact,
 * nullable).  normal: unit eigenvector of the smallest covariance eigenvalue, flipped towards `sensor` (nullable);
 * keep (nullable) = |cos(view, normal)| > cos_min; eig (nullable): [m][3] ascending eigenvalues. */
NKSR_API int nksr_knn_normals(const nksr_svh_t* svh, const float* xyz, const float* sensor, const int32_t* base,
                     const int32_t* range, int64_t m, int k, float cos_min, float* normal, int32_t* keep,
                     float* eig, int32_t* inexact, void* stream);

/* ---- f3: nksr.fields.PCNNField (examples/recons_colored_mesh.py:28-31): nearest data point of m query positions on
 * the same multi-level voxel hash (svh / range as for nksr_knn_normals; xyz = the Morton-sorted cloud; origin3 = HOST
 * float[3], the shift that was applied to the cloud before keying).  out_idx[i] = index (sorted order) of the nearest
 * point (-1 only for an empty cloud); out_d2 (nullable) its squared distance.  A level's answer is accepted when it
 * lies within that level's cell size (then it is exact); a query further than the coarsest cell size from every
 * point (never a mesh vertex) is answered by a scan of all n_pts points. */
NKSR_API int nksr_nearest_point(const nksr_svh_t* svh, const float* xyz, const int32_t* range, int64_t n_pts,
                       const float* query, int64_t m, const float* origin3, int start_level, int32_t* out_idx,
                       float* out_d2, void* stream);

/* ---- f4: the reference's GT-SDF generator ext.sdfgen.sdf_from_points(queries, ref_xyz, ref_normal, nb_points, stdv,
 * compute_grad, imls, adaptive_knn) (ext/sdfgen/sdf_from_points.cu:150-235 + ext/common/kdtree_cuda.cu; call sites
 * dataset/av_gt_geometry.py:63-78, models/loss.py:85).  The reference points live in the same multi-level voxel hash
 * (svh / range / origin3 as for nksr_nearest_point; xyz, normal, ref_std in the Morton-sorted order); search and vote
 * are one kernel.  nksr_knn_mean_distance: out[i] = mean distance from query i to its k nearest reference points
 * (queries = the reference points themselves gives the adaptive ref_std of sdf_from_points.cu:158-166).
 * nksr_sdf_from_points: imls = 0: nearest-neighbour distance / point-to-plane distance with a majority vote for the
 * sign (:92-147), imls = 1: the IMLS average (:33-90); grad nullable; nb_points, k <= 64. */
NKSR_API int nksr_knn_mean_distance(const nksr_svh_t* svh, const float* xyz, const int32_t* range, int64_t n_pts,
                           const float* origin3, const float* query, int64_t m, int k, int start_level,
                           float* out, void* stream);
NKSR_API int nksr_sdf_from_points(const nksr_svh_t* svh, const float* xyz, const float* normal, const float* ref_std,
                         const int32_t* range, int64_t n_pts, const float* origin3, const float* query, int64_t m,
                         int nb_points, float stdv, int imls, int start_level, float* sdf, float* grad,
                         void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NKSR_B200_H */
