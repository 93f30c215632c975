// Gram-matrix fill, sibling-group decomposition (SURVEY section 8 row a3; replaces the numeric phase of
// KernelField.solve_non_fused / fused_mode, models/nksr_net.py:100-112, examples/recons_waymo.py:33).
//
// Same matrix, same CSR order as the row-per-warp kernel in assemble.cu (SPEC S6 / S6b); what changes is the
// decomposition.  One WARP owns the (up to) eight children of one level-(l+1) voxel P -- eight matrix rows
// of level l that share almost all of their inputs:
//   * the constraint rows they read live in the 4x4x4 level-l voxels around the sibling block (instead of
//     8 x 27 neighbour visits): every 128-byte kernel-row line is loaded ONCE per group and feeds the
//     1..8 siblings it touches from registers (the sibling's own coefficient is a shuffle of the line that is
//     already there, not a second load);
//   * the column voxels of the eight rows all lie in the 6^3 level-l region / the 5^3 neighbourhoods of P's
//     ancestors: one table per group (shared memory) replaces eight times 125 + 64 (L-1-l) parent-table walks;
//   * the slot of a contribution inside a row's accumulation tile is  (uniform base of the source voxel) +
//     (constant of the lane) + (constant of the sibling), so a flush is a load-add-store per level.
// Per-warp shared memory: 8 tiles of 317 structural slots, the column table (216 + 3 x 125), the row ranges of
// the 64 source voxels.  Summation order inside a row: source voxels in x-major order of the 4^3 block, inside
// a voxel positions then normals -- fixed, no atomics, deterministic.
#include "gram_common.cuh"

namespace {

constexpr int kGW = 4;              // sibling groups (warps) per block
constexpr int kTileStride = 320;    // 125 + 3 * 64 = 317 structural slots, padded
constexpr int kTileFloats = 8 * kTileStride;
constexpr int kColTab = 216 + 3 * 125 + 1;
constexpr int kWarpWords = kTileFloats + kColTab + 64 * 4 + 16;   // + row ranges [64][4] + sibling masks [64] bytes

// R[c][:] += a_c * ln[:] for the siblings c of `m8`; a_c = (weighted) coefficient of sibling c in this
// constraint row = slot S + (cx*9 + cy*3 + cz) of the level-l line
template <int NLEV>
__device__ __forceinline__ void accum_row(float (&R)[8][NLEV], const unsigned m8, const int S, const float wl0,
                                          const float (&ln)[NLEV]) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    if (m8 & (1u << c)) {
      const float a = __shfl_sync(0xffffffffu, wl0, S + (c >> 2) * 9 + ((c >> 1) & 1) * 3 + (c & 1));
#pragma unroll
      for (int k2 = 0; k2 + 1 < NLEV; k2 += 2) {
        const float2 r = ffma2_rn(make_float2(a, a), make_float2(ln[k2], ln[k2 + 1]),
                                    make_float2(R[c][k2], R[c][k2 + 1]));
        R[c][k2] = r.x;
        R[c][k2 + 1] = r.y;
      }
      if (NLEV & 1) R[c][NLEV - 1] = fmaf(a, ln[NLEV - 1], R[c][NLEV - 1]);
    }
  }
}

// Column tables of one sibling group (children of the level-(l+1) voxel P): ct[0..215] = the 6^3 level-l voxels
// around the sibling block (through P's 27-stencil `pn`, lane s < 27, and the child tables), then for every
// coarser level l+k the 5^3 neighbourhood of P's ancestor (125 entries each); -1 = inactive.
template <int NLEV>
__device__ __forceinline__ void build_column_tables(const nksr_svh_t& svh, const int l, const int64_t P, const int pn,
                                                    const int Px, const int Py, const int Pz, int* __restrict__ ct,
                                                    const int lane) {
  const int lu = l + 1;
  constexpr int nup = NLEV - 1;
  for (int t0 = 0; t0 < 216; t0 += 32) {
    const int t = t0 + lane;
    const int X = t / 36 - 2, Y = (t / 6) % 6 - 2, Z = t % 6 - 2;
    const int ps = t < 216 ? ((X >> 1) + 1) * 9 + ((Y >> 1) + 1) * 3 + ((Z >> 1) + 1) : 13;
    const int pnv = __shfl_sync(0xffffffffu, pn, ps);
    if (t < 216)
      ct[t] = pnv >= 0 ? __ldg(svh.child8[lu] + (int64_t)pnv * 8 + (((X & 1) << 2) | ((Y & 1) << 1) | (Z & 1))) : -1;
  }
  int a = (int)P;
#pragma unroll
  for (int k = 1; k <= nup; ++k) {
    if (k > 1) a = __ldg(svh.parent[l + k - 1] + a);
    const int ax = Px >> (k - 1), ay = Py >> (k - 1), az = Pz >> (k - 1);
    for (int t = lane; t < 125; t += 32) {
      const int dx = t / 25 - 2, dy = (t / 5) % 5 - 2, dz = t % 5 - 2;
      ct[216 + (k - 1) * 125 + t] = lookup_near(svh, l + k, a, ax, ay, az, ax + dx, ay + dy, az + dz);
    }
  }
}

// column voxel of structural slot t (SPEC S6) of the sibling at (cx,cy,cz) of the block, absolute coordinates
// (gx,gy,gz); k = level offset of the slot, ds / sm = ancestor slot and edge axes of the transposed placement (S6b)
template <int NLEV>
__device__ __forceinline__ int table_column(const int* __restrict__ ct, const int t, const int cx, const int cy,
                                            const int cz, const int gx, const int gy, const int gz, int& k, int& ds,
                                            int& sm) {
  constexpr int nslots = 125 + 64 * (NLEV - 1);
  k = 0; ds = 0; sm = 0;
  if (t < 125) {
    const int dx = t / 25 - 2, dy = (t / 5) % 5 - 2, dz = t % 5 - 2;
    return ct[(cx + dx + 2) * 36 + (cy + dy + 2) * 6 + (cz + dz + 2)];
  }
  if (t >= nslots) return -1;
  int q = t - 125;
  k = 1 + (q >> 6);
  q &= 63;
  const int ccx = (((gx - 1) >> k) - 1) + (q >> 4), ccy = (((gy - 1) >> k) - 1) + ((q >> 2) & 3),
            ccz = (((gz - 1) >> k) - 1) + (q & 3);
  if (ccx > ((gx + 1) >> k) + 1 || ccy > ((gy + 1) >> k) + 1 || ccz > ((gz + 1) >> k) + 1) return -1;
  const int dx = ccx - (gx >> k), dy = ccy - (gy >> k), dz = ccz - (gz >> k);
  ds = (dx + 2) * 25 + (dy + 2) * 5 + (dz + 2);
  sm = ((dx == -2 || dx == 2) ? 4 : 0) | ((dy == -2 || dy == 2) ? 2 : 0) | ((dz == -2 || dz == 2) ? 1 : 0);
  return ct[216 + (k - 1) * 125 + ds];
}

// Structural row lengths (own entries: same level + coarser levels) with the tables of the sibling group:
// replaces one parent-table walk per slot and row by one per table entry and group.
template <int NLEV>
__global__ void __launch_bounds__(256)
k_gram_count_group(const nksr_svh_t svh, const int l, int32_t* __restrict__ cnt) {
  __shared__ int tabs[8][kColTab];
  const int lane = threadIdx.x & 31;
  const int wid = threadIdx.x >> 5;
  const int lu = l + 1;
  const int64_t P = blockIdx.x * (int64_t)8 + wid;
  if (P >= svh.n[lu]) return;
  const int sib = lane < 8 ? __ldg(svh.child8[lu] + P * 8 + lane) : -1;
  const unsigned act = __ballot_sync(0xffffffffu, sib >= 0) & 0xffu;
  if (!act) return;
  const int pn = lane < 27 ? __ldg(svh.nbr27[lu] + P * 27 + lane) : -1;
  int Px, Py, Pz;
  morton3_decode(__ldg(svh.keys[lu] + P), Px, Py, Pz);
  int* ct = tabs[wid];
  build_column_tables<NLEV>(svh, l, P, pn, Px, Py, Pz, ct, lane);
  __syncwarp();
  constexpr int nslots = 125 + 64 * (NLEV - 1);
#pragma unroll 1
  for (int c = 0; c < 8; ++c) {
    if (!(act & (1u << c))) continue;
    const int cx = c >> 2, cy = (c >> 1) & 1, cz = c & 1;
    const int i = __shfl_sync(0xffffffffu, sib, c);
    int n = 0;
    for (int t0 = 0; t0 < nslots; t0 += 32) {
      int k, ds, sm;
      const int cv = table_column<NLEV>(ct, t0 + lane, cx, cy, cz, 2 * Px + cx, 2 * Py + cy, 2 * Pz + cz, k, ds, sm);
      n += __popc(__ballot_sync(0xffffffffu, cv >= 0));
    }
    if (lane == 0) cnt[svh.offset[l] + i] = n;
  }
}

template <int NLEV, bool COMPACT>
__global__ void __launch_bounds__(kGW * 32, 4)
k_gram_fill_group(const nksr_svh_t svh, const nksr_feat_t feat, const nksr_constraints_t cs, const int l,
                  const int32_t* __restrict__ cnt, const int64_t* __restrict__ rowptr,
                  int32_t* __restrict__ col_out, float* __restrict__ val_out, float* __restrict__ rhs,
                  float* __restrict__ diag, const nksr_placement_t place) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31;
  const int wid = threadIdx.x >> 5;
  const int lu = l + 1;
  const int64_t P = blockIdx.x * (int64_t)kGW + wid;
  if (P >= svh.n[lu]) return;
  const int sib = lane < 8 ? __ldg(svh.child8[lu] + P * 8 + lane) : -1;
  const unsigned act = __ballot_sync(0xffffffffu, sib >= 0) & 0xffu;
  if (!act) return;
  const int pn = lane < 27 ? __ldg(svh.nbr27[lu] + P * 27 + lane) : -1;
  int Px, Py, Pz;
  morton3_decode(__ldg(svh.keys[lu] + P), Px, Py, Pz);

  float* tile = smem + wid * kWarpWords;
  int* ct = reinterpret_cast<int*>(tile + kTileFloats);
  int* rng = ct + kColTab;
  unsigned char* m8s = reinterpret_cast<unsigned char*>(rng + 256);
  const int L = svh.depth;
  constexpr int nup = NLEV - 1;
  constexpr int nslots = 125 + 64 * nup;

  for (int t = lane; t < kTileFloats / 4; t += 32) reinterpret_cast<float4*>(tile)[t] = make_float4(0.f, 0.f, 0.f, 0.f);
  build_column_tables<NLEV>(svh, l, P, pn, Px, Py, Pz, ct, lane);
  __syncwarp();
  // ---- the 64 source voxels: constraint-row ranges and the siblings each of them feeds
  const int32_t* rp = cs.range_pos ? cs.range_pos + 2 * svh.offset[l] : nullptr;
  const int32_t* rn = cs.range_nrm ? cs.range_nrm + 2 * svh.offset[l] : nullptr;
  unsigned umask0 = 0u, umask1 = 0u;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int pos = lane + 32 * h;
    const int x = (pos >> 4) - 1, y = ((pos >> 2) & 3) - 1, z = (pos & 3) - 1;
    const int u = ct[(x + 2) * 36 + (y + 2) * 6 + (z + 2)];
    int4 r4 = make_int4(0, 0, 0, 0);
    if (u >= 0) {
      if (rp) { const int2 v = __ldg(reinterpret_cast<const int2*>(rp) + u); r4.x = v.x; r4.y = v.y; }
      if (rn) { const int2 v = __ldg(reinterpret_cast<const int2*>(rn) + u); r4.z = v.x; r4.w = v.y; }
    }
    // sibling c = (cx,cy,cz) is within one voxel of u on an axis unless u sits at -1 (then only cx = 0) or 2 (cx = 1)
    const unsigned mX = x < 0 ? 0x0Fu : (x > 1 ? 0xF0u : 0xFFu);
    const unsigned mY = y < 0 ? 0x33u : (y > 1 ? 0xCCu : 0xFFu);
    const unsigned mZ = z < 0 ? 0x55u : (z > 1 ? 0xAAu : 0xFFu);
    const unsigned m = (r4.x < r4.y || r4.z < r4.w) ? (mX & mY & mZ & act) : 0u;
    reinterpret_cast<int4*>(rng)[pos] = r4;
    m8s[pos] = (unsigned char)m;
    const unsigned bm = __ballot_sync(0xffffffffu, m != 0u);
    if (h == 0) umask0 = bm; else umask1 = bm;
  }
  __syncwarp();

  // lane constants: stencil offset d(s) of this lane's slot, as slot-index increments of the three tile regions
  const int sl = lane < 27 ? lane : 13;
  const int ldx = c_d27[sl][0], ldy = c_d27[sl][1], ldz = c_d27[sl][2];
  const int L0 = ldx * 25 + ldy * 5 + ldz;
  const int Lk = ldx * 16 + ldy * 4 + ldz;
  // per coarser level: A = (2P) >> k (the lower box bound of a sibling with c = 1 is A - 1) and whether the
  // bound of a sibling with c = 0 is one lower (2P a multiple of 2^k), packed 16 / 4 / 1 like the slot index
  int Ak[3][nup > 0 ? nup : 1], Dk[nup > 0 ? nup : 1];
#pragma unroll
  for (int k = 1; k <= nup; ++k) {
    Ak[0][k - 1] = (2 * Px) >> k; Ak[1][k - 1] = (2 * Py) >> k; Ak[2][k - 1] = (2 * Pz) >> k;
    Dk[k - 1] = ((Ak[0][k - 1] - ((2 * Px - 1) >> k)) << 4) | ((Ak[1][k - 1] - ((2 * Py - 1) >> k)) << 2) |
                (Ak[2][k - 1] - ((2 * Pz - 1) >> k));
  }
  const bool use_blocks = cs.mblocks != nullptr && l >= cs.split_level;
  const CompactSpline spline(ldx, ldy, ldz);
  const float inv_wl = 1.f / (svh.voxel_size * (float)(1 << l));

  float R[8][NLEV];
#pragma unroll
  for (int c = 0; c < 8; ++c)
#pragma unroll
    for (int k = 0; k < NLEV; ++k) R[c][k] = 0.f;
  float bsum = 0.f;   // lane c < 8: rhs of sibling c

#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    unsigned um = h == 0 ? umask0 : umask1;
#pragma unroll 1
    while (um) {
      const int pos = 32 * h + __ffs(um) - 1;
      um &= um - 1;
      const int x = (pos >> 4) - 1, y = ((pos >> 2) & 3) - 1, z = (pos & 3) - 1;
      // everything that steers control flow below is derived from ballots / warp reductions, so the compiler
      // knows it is warp-uniform: plain branches, no convergence barriers around the shuffles
      const unsigned m8 = (x < 0 ? 0x0Fu : (x > 1 ? 0xF0u : 0xFFu)) & (y < 0 ? 0x33u : (y > 1 ? 0xCCu : 0xFFu)) &
                          (z < 0 ? 0x55u : (z > 1 ? 0xAAu : 0xFFu)) & act;
      int4 r4 = reinterpret_cast<const int4*>(rng)[pos];
      r4.x = __reduce_max_sync(0xffffffffu, r4.x); r4.y = __reduce_max_sync(0xffffffffu, r4.y);
      r4.z = __reduce_max_sync(0xffffffffu, r4.z); r4.w = __reduce_max_sync(0xffffffffu, r4.w);
      const int S = (1 - x) * 9 + (1 - y) * 3 + (1 - z);
      float B = 0.f;   // lane s: sum over the rows of u of  w * E[row][s] * target
      if (use_blocks) {
        // coarse level: the 27 x 27 products of u's rows were reduced once per voxel (k_gram_blocks); every
        // sibling only picks its line of every block
        const int u = ct[(x + 2) * 36 + (y + 2) * 6 + (z + 2)];
        const float* blk = cs.mblocks + (cs.mblock_off[l] + (int64_t)u * NLEV) * kBlockFloats;
        B = __ldg(blk + 27 * NKSR_ROW_STRIDE + lane);
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          if (m8 & (1u << c)) {
            const int si = S + (c >> 2) * 9 + ((c >> 1) & 1) * 3 + (c & 1);
#pragma unroll
            for (int k = 0; k < NLEV; ++k)
              R[c][k] = __ldg(blk + (int64_t)k * kBlockFloats + si * NKSR_ROW_STRIDE + lane);
          }
        }
      } else {
        for (int q = r4.x; q < r4.y; ++q) {
          const float* p = cs.e_pos + ((int64_t)q * L + l) * NKSR_ROW_STRIDE + lane;
          float ln[NLEV];
#pragma unroll
          for (int k = 0; k < NLEV; ++k) ln[k] = __ldg(p + k * NKSR_ROW_STRIDE);
          accum_row<NLEV>(R, m8, S, cs.w_pos * ln[0], ln);
        }
        if (COMPACT) {
          // one line per (location, level): <phi,z_s> in slots 0..26, tau in 27..29; the three gradient rows
          // dB_a B_b B_c <phi,z_s> / W_level are rebuilt here, once per group instead of once per matrix row
          for (int q = r4.z; q < r4.w; ++q) {
            const float* p = cs.e_nrm + ((int64_t)q * L + l) * NKSR_ROW_STRIDE + lane;
            float e[3][NLEV];
            float iw = inv_wl;
#pragma unroll
            for (int k = 0; k < NLEV; ++k) {
              spline.grad_rows(__ldg(p + k * NKSR_ROW_STRIDE), iw, lane, e[0][k], e[1][k], e[2][k]);
              iw *= 0.5f;
            }
            const float* t = cs.t_nrm + (int64_t)q * 3;
#pragma unroll
            for (int ax = 0; ax < 3; ++ax) {
              const float wl0 = cs.w_nrm * e[ax][0];
              B = fmaf(wl0, __ldg(t + ax), B);
              accum_row<NLEV>(R, m8, S, wl0, e[ax]);
            }
          }
        } else {
          for (int q = r4.z; q < r4.w; ++q) {
            const float* p = cs.e_nrm + ((int64_t)q * L + l) * (3 * NKSR_ROW_STRIDE) + lane;
            const float* t = cs.t_nrm + (int64_t)q * 3;
#pragma unroll
            for (int ax = 0; ax < 3; ++ax) {
              float ln[NLEV];
#pragma unroll
              for (int k = 0; k < NLEV; ++k) ln[k] = __ldg(p + (k * 3 + ax) * NKSR_ROW_STRIDE);
              const float wl0 = cs.w_nrm * ln[0];
              B = fmaf(wl0, __ldg(t + ax), B);
              accum_row<NLEV>(R, m8, S, wl0, ln);
            }
          }
        }
      }
      // ---- flush: slot = base(u) + constant(lane) - constant(sibling)
      const int i0 = (x + 2) * 25 + (y + 2) * 5 + (z + 2) + L0;
      int ik[nup > 0 ? nup : 1];
#pragma unroll
      for (int k = 1; k <= nup; ++k) {
        const int ox = ((2 * Px + x) >> k) - Ak[0][k - 1] + 1, oy = ((2 * Py + y) >> k) - Ak[1][k - 1] + 1,
                  oz = ((2 * Pz + z) >> k) - Ak[2][k - 1] + 1;
        ik[k - 1] = 125 + 64 * (k - 1) + (ox << 4) + (oy << 2) + oz + Lk;
      }
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        if (m8 & (1u << c)) {
          const float bv = __shfl_sync(0xffffffffu, B, S + (c >> 2) * 9 + ((c >> 1) & 1) * 3 + (c & 1));
          if (lane == c) bsum += bv;
          if (lane < 27) {
            float* tc = tile + c * kTileStride;
            tc[i0 - ((c >> 2) * 25 + ((c >> 1) & 1) * 5 + (c & 1))] += R[c][0];
            const int nm = ((c >> 2) ? 0 : 16) | (((c >> 1) & 1) ? 0 : 4) | ((c & 1) ? 0 : 1);
#pragma unroll
            for (int k = 1; k <= nup; ++k) tc[ik[k - 1] + (Dk[k - 1] & nm)] += R[c][k];
          }
#pragma unroll
          for (int k = 0; k < NLEV; ++k) R[c][k] = 0.f;
        }
      }
      __syncwarp();
    }
  }

  // ---- regulariser R_{i,i+d} = w_reg B3(d) <z_i, z_{i+d}>  (SPEC S5), write-out in structural order
  const int C = feat.channels;
  const float bw = (ldx == 0 ? 0.75f : 0.125f) * (ldy == 0 ? 0.75f : 0.125f) * (ldz == 0 ? 0.75f : 0.125f);
#pragma unroll 1
  for (int c = 0; c < 8; ++c) {
    if (!(act & (1u << c))) continue;
    const int cx = c >> 2, cy = (c >> 1) & 1, cz = c & 1;
    const int i = __shfl_sync(0xffffffffu, sib, c);
    float* tc = tile + c * kTileStride;
    if (cs.w_reg != 0.f && lane < 27) {
      const int nb = ct[(cx + ldx + 2) * 36 + (cy + ldy + 2) * 6 + (cz + ldz + 2)];
      if (nb >= 0) {
        const float* zi = feat.z[l] + (int64_t)i * C;
        const float* zn = feat.z[l] + (int64_t)nb * C;
        float d = 0.f;
        for (int ch = 0; ch < C; ++ch) d = fmaf(__ldg(zi + ch), __ldg(zn + ch), d);
        tc[(ldx + 2) * 25 + (ldy + 2) * 5 + (ldz + 2)] += cs.w_reg * bw * d;
      }
    }
    __syncwarp();
    const int64_t row = svh.offset[l] + i;
    const int64_t p0 = rowptr[row];
    const int gx = 2 * Px + cx, gy = 2 * Py + cy, gz = 2 * Pz + cz;
    int written = 0;
#pragma unroll 1
    for (int t0 = 0; t0 < nslots; t0 += 32) {
      const int t = t0 + lane;
      int k, ds, sm;
      const int cv = table_column<NLEV>(ct, t, cx, cy, cz, gx, gy, gz, k, ds, sm);
      const unsigned m = __ballot_sync(0xffffffffu, cv >= 0);
      if (cv >= 0) {
        const int64_t p = p0 + written + __popc(m & ((1u << lane) - 1u));
        const float v = tc[t];
        const int64_t gc = svh.offset[l + k] + cv;
        col_out[p] = (int32_t)gc;
        val_out[p] = v;
        if (k == 0 && cv == i) diag[row] = v;
        if (k > 0) {  // transposed copy, straight to its final slot in the coarse row (SPEC S6b)
          const int64_t q = rowptr[gc] + cnt[gc] + placed_pos(place, l, k, cv, ds, i, sm);
          col_out[q] = (int32_t)row;
          val_out[q] = v;
        }
      }
      written += __popc(m);
    }
    const float bv = __shfl_sync(0xffffffffu, bsum, c);
    if (lane == 0) rhs[row] = bv;
  }
}

}  // namespace

extern "C" {

int nksr_gram_count_grouped(const nksr_svh_t* svh, int32_t* cnt, void* stream) {
  if (!svh || !cnt || svh->depth < 1) return NKSR_E_INVALID;
  if (svh->depth > 4 || svh->depth >= NKSR_MAX_DEPTH || !svh->parent[svh->depth - 1] || !svh->child8[svh->depth] ||
      !svh->nbr27[svh->depth])
    return NKSR_E_INVALID;
  cudaStream_t s = as_stream(stream);
  const int L = svh->depth;
  for (int l = L - 1; l >= 0; --l) {
    const int64_t groups = svh->n[l + 1];
    if (groups == 0 || svh->n[l] == 0) continue;
    const int grid = grid_for(groups, 8);
    switch (L - l) {
      case 1: k_gram_count_group<1><<<grid, 256, 0, s>>>(*svh, l, cnt); break;
      case 2: k_gram_count_group<2><<<grid, 256, 0, s>>>(*svh, l, cnt); break;
      case 3: k_gram_count_group<3><<<grid, 256, 0, s>>>(*svh, l, cnt); break;
      default: k_gram_count_group<4><<<grid, 256, 0, s>>>(*svh, l, cnt); break;
    }
    NKSR_CHECK_LAUNCH();
  }
  return NKSR_OK;
}

int nksr_gram_fill_grouped(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                           const int32_t* cnt, const int64_t* rowptr, const nksr_placement_t* placement,
                           int32_t* col, float* val, float* rhs, float* diag, void* stream) {
  if (!svh || !feat || !c || !placement || svh->depth < 1) return NKSR_E_INVALID;
  if (c->nrm_compact == 2) return NKSR_E_INVALID;     // the interleaved row layout belongs to the row fill
  // needs the virtual level above the coarsest one (parent tables on every level) and at most 4 levels
  if (svh->depth > 4 || svh->depth >= NKSR_MAX_DEPTH || !svh->parent[svh->depth - 1] || !svh->child8[svh->depth] ||
      !svh->nbr27[svh->depth])
    return NKSR_E_INVALID;
  cudaStream_t s = as_stream(stream);
  const size_t smem = (size_t)kGW * kWarpWords * sizeof(float);
  const int L = svh->depth;
  for (int l = L - 1; l >= 0; --l) {
    const int64_t groups = svh->n[l + 1];
    if (groups == 0 || svh->n[l] == 0) continue;
    const int grid = grid_for(groups, kGW);
    const int nlev = L - l;
#define NKSR_GROUP(NLEV, COMPACT)                                                                             \
  do {                                                                                                        \
    if (cudaFuncSetAttribute(k_gram_fill_group<NLEV, COMPACT>, cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                             (int)smem) != cudaSuccess)                                                       \
      return NKSR_E_CUDA;                                                                                     \
    k_gram_fill_group<NLEV, COMPACT><<<grid, kGW * 32, smem, s>>>(*svh, *feat, *c, l, cnt, rowptr, col, val, rhs, \
                                                                  diag, *placement);                          \
  } while (0)
    if (c->nrm_compact) {
      switch (nlev) {
        case 1: NKSR_GROUP(1, true); break;
        case 2: NKSR_GROUP(2, true); break;
        case 3: NKSR_GROUP(3, true); break;
        default: NKSR_GROUP(4, true); break;
      }
    } else {
      switch (nlev) {
        case 1: NKSR_GROUP(1, false); break;
        case 2: NKSR_GROUP(2, false); break;
        case 3: NKSR_GROUP(3, false); break;
        default: NKSR_GROUP(4, false); break;
      }
    }
#undef NKSR_GROUP
    NKSR_CHECK_LAUNCH();
  }
  return NKSR_OK;
}

}  // extern "C"
