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
/* ---- f2b: the structure-grown decoder hierarchy (DESIGN.md SPEC S16; models/nksr_net.py:74-86, dec_tmp_svh).
 * classify: per voxel of level `level`, c = argmax of the 3 logits at logits[i*row_stride] (torch.argmax semantics:
 * first index on a tie, NaN largest), or c = forced[i] when forced != NULL; cls[i] = c, keep[i] = c >= 1,
 * sub[i] = level >= 1 && (c == 2 || (c == 1 && level >= adaptive_depth)). */
NKSR_API int nksr_structure_classify(const float* logits, int64_t row_stride, const int32_t* forced, int64_t n,
                                     int level, int adaptive_depth, int8_t* cls, int32_t* keep, int32_t* sub,
                                     void* stream);
/* children of the subdivided voxels of one level (sub_scan = nksr_exclusive_scan32 of sub, n + 1 entries; the caller
 * sizes the child arrays 8 * sub_scan[n]): child c = 8 sub_scan[i] + o of voxel i has key (keys[i] << 3) | o, parent i
 * and join enc_child8[join[i]*8 + o] (-1 when join[i] < 0 or enc_child8 == NULL); child8 (n x 8) = c, or -1 rows for
 * voxels that are not subdivided.  Deterministic: no atomics, no sort. */
NKSR_API int nksr_structure_grow(const int64_t* keys, const int32_t* sub, const int64_t* sub_scan, int64_t n,
                                 const int32_t* join, const int32_t* enc_child8, int64_t* child_keys,
                                 int32_t* child_parent, int32_t* child_join, int32_t* child8, void* stream);
/* table composition out[i*K+k] = idx[i*K+k] < 0 ? -1 : map[idx[i*K+k]] (n rows of K taps) */
NKSR_API int nksr_compose_taps(const int32_t* idx, int64_t n, int K, const int32_t* map, int32_t* out, void* stream);
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
NKSR_API size_t nksr_scan_workspace_bytes(int64_t n);
/* rowptr[0..n] (int64) = exclusive scan of cnt[i] (same + coarser levels) + cnt_down[i] (finer levels, nksr_gram_place) */
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

/* -- sort-free placement of the transposed entries (DESIGN.md SPEC S6b): no atomics, no sort.
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
/* numeric assembly, one warp per matrix row: fills col/val (CSR, int64 rowptr, row lengths cnt from
 * nksr_gram_count_own / nksr_gram_count_grouped), rhs b and diag; the transposed copies go to their final position */
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
 * must be readable up to index n + 1 (n + 2 entries) and col / val up to the next multiple of 4 entries.  The
 * workspace holds the stream's plan, with room for packed column tiles (nksr_spmv_plan_build): about 2 bytes per
 * nonzero. */
NKSR_API size_t nksr_pcg_stream_workspace_bytes(int64_t n, int64_t nnz);
/* rows [0, split_row) -- entries [0, split_nnz), split_nnz = rowptr[split_row] -- are streamed; rows >= split_row go
 * through the warp-per-row kernel.  split_row = n streams everything (what KernelField does: on the H100 the coarse
 * levels' long rows stream faster as tiles too). */
NKSR_API int nksr_pcg_solve_stream(const int64_t* rowptr, const int32_t* col, const float* val, const float* diag,
                          const float* b, float* x, int64_t n, int64_t nnz, int64_t split_row, int64_t split_nnz,
                          float tol, int max_iter, int check_every, int profile, void* ws, size_t ws_bytes,
                          double* info, void* stream);
/* y = A x through the same tile stream (plan_buf: nksr_spmv_plan_bytes(nnz) bytes of scratch); builds the plan
 * (nksr_spmv_plan_build) and runs it (nksr_spmv_stream_planned) */
NKSR_API size_t nksr_spmv_plan_bytes(int64_t nnz);
NKSR_API int nksr_spmv_stream(const int64_t* rowptr, const int32_t* col, const float* val, const float* x, float* y,
                     int64_t n, int64_t nnz, int64_t split_row, int64_t split_nnz, void* plan_buf,
                     size_t plan_bytes, void* stream);
/* the plan of a tile stream: tile boundaries, and room for packed column tiles.  The first SpMV over the plan packs
 * every tile whose columns lie in at most 8 aligned windows of 8192 columns into window bases plus one uint16 per
 * entry (3-bit window, 13-bit offset); later SpMVs stream 2 bytes per column of such a tile instead of 4.  Valid
 * while rowptr and col are unchanged. */
NKSR_API int nksr_spmv_plan_build(const int64_t* rowptr, int64_t n, int64_t nnz, int64_t split_row, int64_t split_nnz,
                         void* plan_buf, size_t plan_bytes, void* stream);
/* out[4] (host) = packed tiles, entries in packed tiles, streamed tiles, streamed entries of a plan that has run at
 * least one SpMV (the PCG's plan starts nksr_pcg_workspace_bytes(n) bytes into its workspace); synchronises the
 * stream */
NKSR_API int nksr_spmv_plan_stats(const void* plan_buf, int64_t* out, void* stream);
/* y = A x with a plan built by nksr_spmv_plan_build for the same rowptr, col, split_row and split_nnz.  The first
 * launch over a plan writes it (packed slots, headers, counts): a plan belongs to one stream at a time. */
NKSR_API int nksr_spmv_stream_planned(const int64_t* rowptr, const int32_t* col, const float* val, const float* x,
                             float* y, int64_t n, int64_t nnz, int64_t split_row, int64_t split_nnz,
                             void* plan_buf, void* stream);

/* -- the inference system without the matrix (csrc/operator.cu): A x = E^T W E x + w_reg R x applied straight from the
 * kernel rows, which are read once per application.  c: e_pos of the sorted positions, e_nrm / t_nrm of the sorted
 * normal locations, nrm_compact 0 (gradient rows, nksr_build_rows mode 1) or 1 (compact lines, mode 2); range_pos,
 * range_nrm, mblocks and split_level are ignored.  base_pos / base_nrm: [depth][m] containing voxel per level of the
 * same sorted locations (nksr_locate); key_pos / key_nrm: their half-voxel keys (nksr_point_half_keys), ascending.
 * The workspace holds 2 x 27 planes of n floats of per-(stencil slot, voxel) partial sums, the merged location order
 * with its containing voxels (4 (depth + 1) bytes per location), and the work items of at most item_size locations
 * with their edge partials; nksr_op_workspace_bytes gives its size for c->n_pos + c->n_nrm locations. */
NKSR_API size_t nksr_op_workspace_bytes(const nksr_svh_t* svh, const nksr_constraints_t* c, int item_size);
/* once per system: merges the two location orders, cuts the work items (item_size >= 1: at most that many locations,
 * cut only between voxels of levels <= 2, never across a top-level voxel; one such voxel with more locations is an
 * item of its own), then rhs b = E^T W t and the Jacobi diagonal diag(A).  owned (nullable, one byte per unknown,
 * levels concatenated): keep only the locations that have, on some level, an owned unknown among the 27 neighbours of
 * their containing voxel, in the same order.  Rows i with owned[i] != 0 then get the rhs, diagonal and A x of the
 * whole system; the other rows are incomplete.  NULL keeps every location. */
NKSR_API int nksr_op_setup(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                           const int32_t* base_pos, const int32_t* base_nrm, const int64_t* key_pos,
                           const int64_t* key_nrm, const uint8_t* owned, int item_size, float* rhs, float* diag,
                           void* ws, size_t ws_bytes, void* stream);
/* y = A x over a workspace that nksr_op_setup prepared for the same hierarchy, features and constraints.  No atomics:
 * the same x gives bitwise the same y */
NKSR_API int nksr_op_apply(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                           const int32_t* base_pos, const int32_t* base_nrm, const float* x, float* y, void* ws,
                           size_t ws_bytes, void* stream);
/* The constraint values the backward of a matrix-free solve needs (DESIGN 4.6), read from the kernel rows of c (the
 * rows nksr_op_setup used: e_pos, e_nrm with nrm_compact 0 or 1) at the same sorted locations, for two vectors x0, x1
 * (n unknowns each, levels concatenated): out_pos[j][k] = E_j x_k for every sorted position j, out_nrm[j][k][a] = the
 * gradient row a of sorted normal location j times x_k.  No weights are applied.  base_pos / base_nrm as for
 * nksr_op_setup; a location without containing voxel on a level gets nothing from it.  One warp per location, no
 * atomics: bitwise repeatable.  Needs no operator workspace. */
NKSR_API int nksr_op_constraint_values(const nksr_svh_t* svh, const nksr_constraints_t* c, const int32_t* base_pos,
                                       const int32_t* base_nrm, const float* x0, const float* x1, float* out_pos,
                                       float* out_nrm, void* stream);
/* out[5] (host) = byte offsets in a workspace of ws_bytes bytes of the merged location order ([m] int32: r >= 0 position
 * r, ~r normal location r; its first `kept` entries are used), its containing voxels ([depth][m] int32), the item
 * count (int32), the items ([count] int4: begin, end, flags 1 first / 2 last item of its top-level voxel, 0) and the
 * kept location count (int32: m without the owned filter) */
NKSR_API int nksr_op_workspace_layout(const nksr_svh_t* svh, const nksr_constraints_t* c, size_t ws_bytes,
                                      int64_t* out);
/* nksr_pcg_solve with the matrix-free A: op_ws prepared by nksr_op_setup (which gave diag and b), ws of
 * nksr_pcg_workspace_bytes(n) bytes.  profile != 0: info[2] / info[3] time every application of A */
NKSR_API int nksr_pcg_solve_matrix_free(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                                        const int32_t* base_pos, const int32_t* base_nrm, const float* diag,
                                        const float* b, float* x, float tol, int max_iter, int check_every,
                                        int profile, void* op_ws, size_t op_ws_bytes, void* ws, size_t ws_bytes,
                                        double* info, void* stream);

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
/* nksr_dcg_spmv_dots with the matrix-free A of a workspace that nksr_op_setup prepared (with the same owned mask, or
 * NULL): w = A u on owned rows (the arithmetic of nksr_op_apply), w = 0 on the others, red = local {(r,u), (w,u),
 * (r,r)} over the owned rows; n = the hierarchy's unknowns.  No-op once the solve is over */
NKSR_API int nksr_dcg_op_dots(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                              const int32_t* base_pos, const int32_t* base_nrm, void* op_ws, size_t op_ws_bytes,
                              const uint8_t* owned, const float* r, const float* u, float* w, void* ws, double* red,
                              void* stream);
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

/* ---- a5b: backward of the kernel field (training through KernelField.solve / evaluate_f, models/nksr_net.py:91-112,
 * models/loss.py:163-260).  Locations xyz are Morton SORTED, base[l*m + i] = their containing voxels
 * (nksr_locate), range = nksr_row_ranges of every level concatenated in level order (read as int2 pairs: 8-byte
 * aligned).  mode 0: value rows, 1: gradient
 * rows (approx_kernel_grad: without the grad(phi) terms, as the forward).  Deterministic: no atomics, one fixed
 * summation order.  ws: nksr_field_bwd_workspace_bytes(depth, m, C, mode, approx, feature_vjp) bytes (per-location
 * phi / psi vectors), else NKSR_E_WORKSPACE. */
NKSR_API size_t nksr_field_bwd_workspace_bytes(int depth, int64_t m, int channels, int mode, int approx_kernel_grad,
                                               int feature_vjp);
/* dalpha (all unknowns, overwritten) = sum_q coef_q E_q: coef (m) for value rows, (m,3) for gradient rows */
NKSR_API int nksr_evaluate_adjoint(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* xyz,
                          const int32_t* base, const int32_t* range, int64_t m, int mode, int approx_kernel_grad,
                          const float* coef, float* dalpha, void* ws, size_t ws_bytes, void* stream);
/* dz (n_total x C, level blocks at svh->offset, ADDED to) += d/dz sum_q sum_s omega_{q,s} E_q[n_s], with
 * omega_{q,(a,)s} = coef[q,0(,a)] a0[n_s] + coef[q,1(,a)] a1[n_s]; a1 may be NULL (coef then (m) or (m,3)) */
NKSR_API int nksr_feature_vjp(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* xyz, const int32_t* base,
                     const int32_t* range, int64_t m, int mode, int approx_kernel_grad, const float* a0,
                     const float* a1, const float* coef, float* dz, void* ws, size_t ws_bytes, void* stream);
/* dz += w * d/dz (lam^T R alpha), R the regulariser of SPEC S5 without its weight */
NKSR_API int nksr_regulariser_vjp(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* lam,
                         const float* alpha, float w, float* dz, void* stream);

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
/* NeuralField interpolation (models/nksr_net.py:124-130, models/loss.py:120-140; SPEC S17): level_mask = the given
 * levels (bit l, at least one, all < depth; a given level may be empty, its feat->z[l] is then not read).
 * out (m x C*popcount(level_mask), every entry written) = per query the trilinear interpolation of feat->z[l] on each
 * given level in ascending order; 0 where the query has no containing voxel on that level or is non-finite / outside
 * the key range. */
NKSR_API int nksr_neural_interp(const nksr_svh_t* svh, const nksr_feat_t* feat, int level_mask, const float* xyz,
                                int64_t m, float* out, void* stream);
/* its VJP: xyz = Morton SORTED queries (each with a containing voxel on the coarsest level), range = nksr_row_ranges
 * of every level concatenated in level order, grad (m x C*popcount(level_mask)) in the same sorted order.  dfeat
 * (n_total x C, level blocks at svh->offset): the blocks of the given levels are OVERWRITTEN with
 * sum_q T3(q) grad[q]; the others are not touched.  Deterministic: no atomics, one fixed summation order. */
NKSR_API int nksr_neural_interp_vjp(const nksr_svh_t* svh, int channels, int level_mask, const float* xyz,
                                    const int32_t* range, int64_t m, const float* grad, float* dfeat, void* stream);
/* the position Jacobian of nksr_neural_interp (SPEC S17a): jac (m x 3 x C*popcount(level_mask), every entry written)
 * holds jac[i][a][g*C + c] = d out[i][g*C + c] / dx_a, from the tent derivative of SPEC S4 (one-sided in the
 * containing cell, symmetric in the snap zone |tau| < 2^-12) divided by W_l; a row is 0 wherever out is.  out
 * (nullable): when given, written bitwise as nksr_neural_interp writes it. */
NKSR_API int nksr_neural_interp_jacobian(const nksr_svh_t* svh, const nksr_feat_t* feat, int level_mask,
                                         const float* xyz, int64_t m, float* out, float* jac, void* stream);
/* its VJP with respect to the features, under the conventions of nksr_neural_interp_vjp: grad (m x 3 x
 * C*popcount(level_mask)) in the sorted order; the blocks of the given levels of dfeat are OVERWRITTEN with
 * sum_q sum_a dT3_a(q) / W_l grad[q][a]. */
NKSR_API int nksr_neural_interp_jacobian_vjp(const nksr_svh_t* svh, int channels, int level_mask, const float* xyz,
                                             const int32_t* range, int64_t m, const float* grad, float* dfeat,
                                             void* stream);

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

/* ---- metrics.MeshEvaluator (models/nksr_net.py:298-312; DESIGN.md SPEC S17a).
 * nksr_sample_surface: n area-uniform samples of the mesh (v: float[V*3], f: int32[n_tri*3]).  start: int64[n_tri+1],
 * the first sample of every triangle (start[0] = 0, start[n_tri] = n, non-decreasing; the caller forms it from the
 * fp64 area prefix).  Sample i lies on triangle out_tri[i] at the barycentrics of a counter hash of (seed, i);
 * out_normal[i] is that triangle's unit normal.
 * nksr_metric_nearest: for every query, the distance to its nearest point of the Morton-sorted cloud xyz (n_pts >= 1,
 * hashed as for nksr_nearest_point: svh / range / origin3), that point's index in sorted order (ties: the lower
 * index) and, when normal, query_normal and out_dot are all given, |n_q . n_t| of the unit normals.  Exact for
 * every query: those the hierarchy does not resolve are compacted into far_list (int32[m]; *far_count their number,
 * device int32) and answered by a branch-and-bound over the top-level cells, whose point boxes go to box
 * (float[6 * svh->n[depth-1]], workspace). */
NKSR_API int nksr_sample_surface(const float* v, const int32_t* f, int64_t n_tri, const int64_t* start, int64_t n,
                        int64_t seed, float* out_xyz, float* out_normal, int32_t* out_tri, void* stream);
NKSR_API int nksr_metric_nearest(const nksr_svh_t* svh, const float* xyz, const float* normal, const int32_t* range,
                        float* box, int64_t n_pts, const float* query, const float* query_normal, int64_t m,
                        const float* origin3, int start_level, float* out_dist, int32_t* out_idx, float* out_dot,
                        int32_t* far_list, int32_t* far_count, void* stream);

/* ---- PointTSDFVolume ground truth from sensor rays (groundtruth.bin, dataset/av.py:94; consumed by
 * dataset/av_gt_geometry.py:141-173 and models/loss.py:221-249; DESIGN.md SPEC S19).
 * Ray j runs from sensor[j] to xyz[j] (float[n*3] each; rays with a non-finite input or zero length are skipped).
 * Node (i, j, k) sits at volume_min3 + (i, j, k) h (host float[3], evaluated in fp64); dims3 (host int64[3]) >= 2
 * each, product < 2^31; h > 0, tau > 0.  volume (float[dims0*dims1*dims2], [X][Y][Z]) = sdf / tau of the near observation with the
 * smallest |sdf| < tau (ties: the lower ray index), else +1 where a ray passed with sdf >= tau before reaching any
 * near node, else NaN.  Bitwise repeatable; the classes do not depend on the order of the rays.
 * ws: nksr_tsdf_volume_workspace_bytes(dims3) bytes (one 64-bit key per node; 0 for invalid dims), else
 * NKSR_E_WORKSPACE. */
NKSR_API size_t nksr_tsdf_volume_workspace_bytes(const int64_t* dims3);
NKSR_API int nksr_tsdf_volume(const float* xyz, const float* sensor, int64_t n, const float* volume_min3, float h,
                              const int64_t* dims3, float tau, float* volume, void* ws, size_t ws_bytes, void* stream);

/* ---- mesh occupancy by ray parity ('o3d-iou' of metrics.MeshEvaluator, metrics.py:180-188; DESIGN.md SPEC S20).
 * Mesh v: float[V*3], f: int32[n_tri*3] (indices in [0, V), any winding, degenerate and duplicate triangles allowed).
 * Build (an LBVH, one triangle per leaf):
 *   nksr_bvh_keys: scene (device float[8]) = centroid box lo xyz, hi xyz, max |vertex coordinate|, -;
 *     keys (int64[n_tri]) = 63-bit Morton codes of the centroids in that box, idx (int32[n_tri]) = 0..n_tri-1;
 *   the caller sorts (keys, idx) with nksr_sort_pairs;
 *   nksr_bvh_hierarchy: the sorted keys -> nodes (float[16 * (n_tri - 1)]: per internal node the two child boxes and
 *     child codes) and the parent table in ws (ws: nksr_bvh_workspace_bytes(n_tri) bytes, kept for the refit);
 *   nksr_bvh_refit: the sorted idx -> tris (float[12 * n_tri], the triangles in leaf order, the original triangle
 *     index as the int32 bits of each leaf's word 3) and the child boxes.
 * n_tri = 1 needs no nodes (nullable) and no hierarchy call.
 * nksr_mesh_occupancy: inside[i] (uint8[m]) = 1 iff more than k/2 of the k rays from query[i] (float[m*3]) cross the
 * mesh an odd number of times; dirs = device float[k*3] (every component nonzero) or NULL for the first k built-in
 * directions; k odd, 1 <= k <= 9.  Equal bit for bit to testing every triangle (the box test is conservative);
 * n_tri = 0 gives all 0.
 * nksr_mesh_closest (SPEC S21): for every query[i] (float[m*3], finite) the closest triangle of the mesh on the same
 * BVH: dist[i] (float[m]) = sqrt(d2), point[i] (float[m*3]) = the closest point whose d2 that is, tri[i] (int32[m]) =
 * the original triangle index; equal d2 go to the lower index.  Equal bit for bit to testing every triangle (the box
 * bound is conservative); n_tri = 0 gives dist inf, point NaN, tri -1.
 * nksr_mesh_first_hit (SPEC S22): for every ray i from origin[i] along dir[i] (float[m*3] each, finite, dir not all
 * zero, zero components allowed) the first triangle the ray crosses by S20's test at 0 < t <= t_max[i] (float[m],
 * not NaN; t_max NULL: t_max_all for every ray), t = T / det in fp64; equal t go to the lower original index.
 * t[i] (float[m]) = that t rounded to fp32, point[i] (float[m*3]) = origin + t[i] * dir, normal[i] (float[m*3]) =
 * (v1 - v0) x (v2 - v0) / |.| of the original triangle f (int32[n_tri*3]) over v (float[V*3]), the mesh the BVH was
 * built from (NaN for a zero cross product), tri[i] (int32[m]) = the original triangle index.  A miss, and n_tri = 0,
 * give t inf, point and normal NaN, tri -1.  Equal bit for bit to testing every triangle (the slab entry is a
 * conservative bound on t).  Caller-owned buffers, no allocation. */
NKSR_API size_t nksr_bvh_workspace_bytes(int64_t n_tri);
NKSR_API int nksr_bvh_keys(const float* v, const int32_t* f, int64_t n_tri, float* scene, int64_t* keys, int32_t* idx,
                           void* stream);
NKSR_API int nksr_bvh_hierarchy(const int64_t* keys, int64_t n_tri, float* nodes, void* ws, size_t ws_bytes,
                                void* stream);
NKSR_API int nksr_bvh_refit(const float* v, const int32_t* f, const int32_t* idx, int64_t n_tri, float* nodes,
                            float* tris, void* ws, size_t ws_bytes, void* stream);
NKSR_API int nksr_mesh_occupancy(const float* nodes, const float* tris, const float* scene, int64_t n_tri,
                                 const float* query, int64_t m, const float* dirs, int k, uint8_t* inside,
                                 void* stream);
NKSR_API int nksr_mesh_closest(const float* nodes, const float* tris, const float* scene, int64_t n_tri,
                               const float* query, int64_t m, float* dist, float* point, int32_t* tri, void* stream);
NKSR_API int nksr_mesh_first_hit(const float* nodes, const float* tris, const float* scene, int64_t n_tri,
                                 const float* v, const int32_t* f, const float* origin, const float* dir, int64_t m,
                                 const float* t_max, float t_max_all, float* t, float* point, float* normal,
                                 int32_t* tri, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NKSR_B200_H */
