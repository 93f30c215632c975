// Device helpers shared by the Gram-assembly kernels (assemble.cu: row-per-warp fill, count, placement,
// blocks; gram_fill_group.cu: sibling-group fill).  Structural slots, column look-ups through the parent
// tables and the sort-free placement argument (DESIGN.md SPEC S6 / S6b).
#pragma once
#include "common.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kMaxSlots = 125 + 64 * (NKSR_MAX_DEPTH - 1);
constexpr int kBlockFloats = 28 * NKSR_ROW_STRIDE;  // one per-voxel Gram block (see k_gram_blocks)

__constant__ signed char c_d27[27][3] = {
    {-1, -1, -1}, {-1, -1, 0}, {-1, -1, 1}, {-1, 0, -1}, {-1, 0, 0}, {-1, 0, 1}, {-1, 1, -1}, {-1, 1, 0}, {-1, 1, 1},
    {0, -1, -1},  {0, -1, 0},  {0, -1, 1},  {0, 0, -1},  {0, 0, 0},  {0, 0, 1},  {0, 1, -1},  {0, 1, 0},  {0, 1, 1},
    {1, -1, -1},  {1, -1, 0},  {1, -1, 1},  {1, 0, -1},  {1, 0, 0},  {1, 0, 1},  {1, 1, -1},  {1, 1, 0},  {1, 1, 1}};

// same-level voxel at offset-space coords (nx,ny,nz) in the 125-neighbourhood of voxel i
// (coords ux,uy,uz): through the parent's 27-stencil and its child table; the top level owns an
// explicit 125-neighbour table.
__device__ __forceinline__ int lookup_near(const nksr_svh_t& svh, int l, int i, int ux, int uy, int uz, int nx,
                                           int ny, int nz) {
  if (svh.parent[l] != nullptr) {  // also true for the top level when the virtual level exists
    const int p = __ldg(svh.parent[l] + i);
    if (p < 0) return -1;
    const int ex = (nx >> 1) - (ux >> 1), ey = (ny >> 1) - (uy >> 1), ez = (nz >> 1) - (uz >> 1);
    const int pn = __ldg(svh.nbr27[l + 1] + (int64_t)p * 27 + (ex + 1) * 9 + (ey + 1) * 3 + (ez + 1));
    if (pn < 0) return -1;
    return __ldg(svh.child8[l + 1] + (int64_t)pn * 8 + (((nx & 1) << 2) | ((ny & 1) << 1) | (nz & 1)));
  }
  return __ldg(svh.nbr125_top + (int64_t)i * 125 + (nx - ux + 2) * 25 + (ny - uy + 2) * 5 + (nz - uz + 2));
}

struct RowGeom {
  int ux, uy, uz;           // offset-space coords of the row voxel
  int anc[NKSR_MAX_DEPTH];  // ancestor index at level l+k (anc[0] = i)
};

__device__ __forceinline__ void row_geom(const nksr_svh_t& svh, int l, int i, RowGeom& g) {
  morton3_decode(__ldg(svh.keys[l] + i), g.ux, g.uy, g.uz);
  g.anc[0] = i;
  int a = i;
#pragma unroll
  for (int k = 1; k < NKSR_MAX_DEPTH; ++k) {
    if (l + k < svh.depth) a = a >= 0 ? __ldg(svh.parent[l + k - 1] + a) : -1;
    g.anc[k] = a;
  }
}

// column voxel (index at its level) of structural slot t of row (l,i); -1 when inactive.
// t < 125: same level; else k = 1 + (t-125)/64 levels up, 4x4x4 candidate box from lo.
__device__ __forceinline__ int slot_column(const nksr_svh_t& svh, int l, const RowGeom& g, int t, int& k_out) {
  if (t < 125) {
    k_out = 0;
    const int dx = t / 25 - 2, dy = (t / 5) % 5 - 2, dz = t % 5 - 2;
    return lookup_near(svh, l, g.anc[0], g.ux, g.uy, g.uz, g.ux + dx, g.uy + dy, g.uz + dz);
  }
  int q = t - 125;
  const int k = 1 + (q >> 6);
  k_out = k;
  q &= 63;
  const int ox = q >> 4, oy = (q >> 2) & 3, oz = q & 3;
  const int cx = (((g.ux - 1) >> k) - 1) + ox, cy = (((g.uy - 1) >> k) - 1) + oy, cz = (((g.uz - 1) >> k) - 1) + oz;
  if (cx > ((g.ux + 1) >> k) + 1 || cy > ((g.uy + 1) >> k) + 1 || cz > ((g.uz + 1) >> k) + 1) return -1;
  int a = g.anc[0];
#pragma unroll
  for (int j = 1; j < NKSR_MAX_DEPTH; ++j)
    if (j == k) a = g.anc[j];
  if (a < 0) return -1;
  return lookup_near(svh, l + k, a, g.ux >> k, g.uy >> k, g.uz >> k, cx, cy, cz);
}

// slot_column plus, for a coarser-level slot, where the transposed copy goes (sort-free placement):
// ds = slot of d = c - a in c's 125-ancestor table (a = ancestor of the row voxel), sm = axes with |d| = 2
__device__ __forceinline__ int slot_column_place(const nksr_svh_t& svh, int l, const RowGeom& g, int t, int& k_out,
                                                 int& ds, int& sm) {
  ds = 0;
  sm = 0;
  const int c = slot_column(svh, l, g, t, k_out);
  if (t >= 125 && c >= 0) {
    const int k = k_out, q = (t - 125) & 63;
    const int dx = (((g.ux - 1) >> k) - 1) + (q >> 4) - (g.ux >> k);
    const int dy = (((g.uy - 1) >> k) - 1) + ((q >> 2) & 3) - (g.uy >> k);
    const int dz = (((g.uz - 1) >> k) - 1) + (q & 3) - (g.uz >> k);
    ds = (dx + 2) * 25 + (dy + 2) * 5 + (dz + 2);
    sm = ((dx == -2 || dx == 2) ? 4 : 0) | ((dy == -2 || dy == 2) ? 2 : 0) | ((dz == -2 || dz == 2) ? 1 : 0);
  }
  return c;
}

// kernel argument of the sort-free placement: empty for the atomic-cursor variant
template <bool PLACED>
struct PlaceArg {
  __device__ __forceinline__ int pos(int, int, int64_t, int, int64_t, int) const { return 0; }
};
template <>
struct PlaceArg<true> {
  nksr_placement_t t;
  __device__ __forceinline__ int pos(int l, int k, int64_t c, int ds, int64_t j, int sm) const {
    return __ldg(t.prefix[l][k] + c * 125 + ds) + __ldg(t.rank8[l][k] + j * 8 + sm);
  }
};

__device__ __forceinline__ void row_of_warp(const nksr_svh_t& svh, int64_t row, int& l, int& i) {
  l = 0;
  while (l + 1 < svh.depth && row >= svh.offset[l + 1]) ++l;
  i = (int)(row - svh.offset[l]);
}

// regulariser R_{i,i+d} = w_reg * B3(d) * <z_i, z_{i+d}> (SPEC S5) added to the row's tile; lane s < 27 owns offset d(s),
// my_u = nbr27[l][i][s] (-1 for the other lanes)
__device__ __forceinline__ void gram_row_regulariser(const nksr_feat_t& feat, const nksr_constraints_t& cs, int l, int i,
                                                     int my_u, int lane, float* __restrict__ acc) {
  if (cs.w_reg == 0.f || my_u < 0) return;
  const int sl = lane < 27 ? lane : 13;
  const int ldx = c_d27[sl][0], ldy = c_d27[sl][1], ldz = c_d27[sl][2];
  const int C = feat.channels;
  const float* zi = feat.z[l] + (int64_t)i * C;
  const float* zn = feat.z[l] + (int64_t)my_u * C;
  float d = 0.f;
  for (int c = 0; c < C; ++c) d = fmaf(__ldg(zi + c), __ldg(zn + c), d);
  const float bw = (ldx == 0 ? 0.75f : 0.125f) * (ldy == 0 ? 0.75f : 0.125f) * (ldz == 0 ? 0.75f : 0.125f);
  acc[(ldx + 2) * 25 + (ldy + 2) * 5 + (ldz + 2)] += cs.w_reg * bw * d;
}

// write-out of row (l,i) from its tile `acc` (indexed by structural slot) in structural order: the 125 same-level slots
// (4 chunks of 32), then the 64 slots of every coarser level (2 chunks each) -- the level offset is uniform inside a chunk,
// so the box bounds, the ancestor and its parent are computed once per level (in the first version a chunk could
// straddle two levels).  Coarser-level entries also go, transposed, to the coarse row's finer-level segment.
template <int MAXL, bool PLACED>
__device__ __forceinline__ void gram_row_writeout(const nksr_svh_t& svh, int l, int i, int64_t row, const RowGeom& g,
                                                  const float* __restrict__ acc, const int32_t* __restrict__ cnt,
                                                  const int64_t* __restrict__ rowptr, int32_t* __restrict__ col_out,
                                                  float* __restrict__ val_out, float* __restrict__ diag,
                                                  int32_t* __restrict__ cursor, const PlaceArg<PLACED>& place, int lane) {
  const int nup = svh.depth - 1 - l;
  const int64_t p0 = rowptr[row];
  int written = 0;
  auto emit = [&](const int c, const int k, const int t, const int ds, const int sm) {
    const unsigned m = __ballot_sync(0xffffffffu, c >= 0);
    if (c >= 0) {
      const int64_t p = p0 + written + __popc(m & ((1u << lane) - 1u));
      const float v = acc[t];
      const int64_t gc = svh.offset[l + k] + c;
      col_out[p] = (int32_t)gc;
      val_out[p] = v;
      if (k == 0 && c == i) diag[row] = v;
      if (k > 0) {  // transposed copy into the coarse row's finer-level segment
        const int64_t q = rowptr[gc] + cnt[gc] +
                          (PLACED ? place.pos(l, k, c, ds, i, sm) : atomicAdd(cursor + gc, 1));
        col_out[q] = (int32_t)row;
        val_out[q] = v;
      }
    }
    written += __popc(m);
  };
  for (int t0 = 0; t0 < 125; t0 += 32) {
    const int t = t0 + lane;
    int k = 0;
    const int c = t < 125 ? slot_column(svh, l, g, t, k) : -1;
    emit(c, 0, t, 0, 0);
  }
#pragma unroll
  for (int k = 1; k < MAXL; ++k) {
    if (k <= nup) {
      const int lox = ((g.ux - 1) >> k) - 1, loy = ((g.uy - 1) >> k) - 1, loz = ((g.uz - 1) >> k) - 1;
      const int hix = ((g.ux + 1) >> k) + 1, hiy = ((g.uy + 1) >> k) + 1, hiz = ((g.uz + 1) >> k) + 1;
      const int ax = g.ux >> k, ay = g.uy >> k, az = g.uz >> k;
      const int a = g.anc[k];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int q = h * 32 + lane;
        const int cx = lox + (q >> 4), cy = loy + ((q >> 2) & 3), cz = loz + (q & 3);
        int c = -1, ds = 0, sm = 0;
        if (a >= 0 && cx <= hix && cy <= hiy && cz <= hiz) {
          c = lookup_near(svh, l + k, a, ax, ay, az, cx, cy, cz);
          const int dx = cx - ax, dy = cy - ay, dz = cz - az;
          ds = (dx + 2) * 25 + (dy + 2) * 5 + (dz + 2);
          sm = ((dx == -2 || dx == 2) ? 4 : 0) | ((dy == -2 || dy == 2) ? 2 : 0) | ((dz == -2 || dz == 2) ? 1 : 0);
        }
        emit(c, k, 125 + 64 * (k - 1) + q, ds, sm);
      }
    }
  }
}

}  // namespace
