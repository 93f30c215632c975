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
};

// the operator over a workspace that nksr_op_setup prepared for the same hierarchy and constraints; NKSR_E_INVALID /
// NKSR_E_WORKSPACE as nksr_op_apply
int mf_operator_make(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                     const int32_t* base_pos, const int32_t* base_nrm, void* ws, size_t ws_bytes, MfOperator* out);

// y = A x.  pap != nullptr: also pap[b] = sum of x_i y_i over the rows of block b of a grid of exactly `blocks` blocks
// of 256 threads (the fixed-order partials the PCG reduces).  done != nullptr: both kernels are no-ops once *done.
int mf_apply_launch(const MfOperator& op, const float* x, float* y, double* pap, int blocks, const int* done,
                    cudaStream_t s);
