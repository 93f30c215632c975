// The matrix-free inference operator A x = E^T W E x + w_reg R x (csrc/operator.cu), as the PCG driver in solve.cu
// launches it: no Gram matrix is stored, every application reads the kernel rows once.
#pragma once
#include "common.cuh"

struct MfOperator {
  nksr_svh_t svh;
  nksr_feat_t feat;
  nksr_constraints_t cs;     // nrm_compact 0 (full gradient rows) or 1 (compact lines); never interleaved
  const int32_t* base_pos;   // [depth][n_pos] containing voxel of every sorted position, -1 when inactive
  const int32_t* base_nrm;   // [depth][n_nrm] the same for the normal locations
  float* P;                  // [27][n]: per (stencil slot, voxel) partial sums of E^T W E x
  float* Pd;                 // [27][n]: the diagonal's partial sums (setup only)
  int64_t n;
  // the merged walk (nksr_op_setup builds it): positions and normal locations in one half-voxel key order
  int32_t* seq;              // [m] merged location: r >= 0 position r, ~r normal location r
  int32_t* vox;              // [depth][m] containing voxel per level, merged order, -1 when inactive
  int2* top;                 // [n_top] merged range of every top-level voxel
  int32_t* cnt;              // [n_top] items per top voxel, then their exclusive scan in ofs
  int32_t* ofs;
  int32_t* n_items;          // device: number of work items
  void* scan_tmp;
  size_t scan_bytes;
  int64_t* max_items;        // device: the item capacity nksr_op_setup laid the workspace's tail out for
  int4* items;               // [max_items] {begin, end, flags, 0} of the merged sequence, then the edge partials:
                             // [max_items][edge_levels][first | last][27] of runs that span items, and the same for
                             // the diagonal (setup); the kernels find them from *max_items (op_edge_buffers)
  int64_t m;                 // n_pos + n_nrm
  int edge_levels;           // levels above the cut level
  int walk_grid, edge_grid;  // persistent grids (multiples of the SM count)
};

// the operator over a workspace that nksr_op_setup prepared for the same hierarchy and constraints; NKSR_E_INVALID /
// NKSR_E_WORKSPACE as nksr_op_apply
int mf_operator_make(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                     const int32_t* base_pos, const int32_t* base_nrm, void* ws, size_t ws_bytes, MfOperator* out);

// y = A x.  pap != nullptr: also pap[b] = sum of x_i y_i over the rows of block b of a grid of exactly `blocks` blocks
// of 256 threads (the fixed-order partials the PCG reduces).  done != nullptr: every kernel is a no-op once *done.
int mf_apply_launch(const MfOperator& op, const float* x, float* y, double* pap, int blocks, const int* done,
                    cudaStream_t s);

// the distributed solve's step: w = A u on the rows with owned[i] != 0, w = 0 on the others, and dots[j * blocks + b]
// = block b's sums over the owned rows of (r,u), (w,u), (r,r) (j = 0, 1, 2) for a grid of exactly `blocks` blocks of
// 256 threads.  Every kernel is a no-op once *done
int mf_dcg_launch(const MfOperator& op, const uint8_t* owned, const float* r, const float* u, float* w, double* dots,
                  int blocks, const int* done, cudaStream_t s);
