// Gram-matrix assembly A = E^T diag(w) E + reg*R into CSR (SURVEY section 8 row a3).
// Replaces the matrix build inside KernelField.solve_non_fused / fused_mode
// (models/nksr_net.py:100-112, examples/recons_waymo.py:33).
//
// Layout (DESIGN.md SPEC S6): unknowns are ordered level-major, Morton inside a level.  Row
// (l,i) stores, in this order, [same-level 125-stencil | coarser level l+1 (<=64) | ... | level
// L-1 | finer-level entries (transposes)].  Only ACTIVE column voxels are stored.  The transposed copies
// go straight to their final slot from two prefix tables (k_place_rank / k_place_prefix, SPEC S6b): no
// atomics and no sort, the same storage order on every run.
//
// Numeric phase: one warp per row.  For each of the 27 voxels u around i, the constraint rows
// whose containing voxel is u form one contiguous range (locations are Morton sorted); every
// such row r contributes  w * E[r,i] * E[r, :]  and all rows of u share the same 27-stencils on
// level l and on every coarser level, so lane s accumulates stencil slot s in a register and
// the warp flushes once per u into a per-warp shared-memory tile indexed by structural slot --
// no atomics, deterministic summation order.  Profiles of the first version showed the
// kernel to be instruction-issue / L2-latency bound, hence: neighbour indices and row ranges are
// fetched lane-parallel once per row; constraint rows are stored location-major so every line is a
// compile-time offset from one pointer; two levels are accumulated per float2 pair of FMAs; 64 registers keep
// 32 warps per SM resident; and on the coarse levels (a voxel owns hundreds of constraint rows) the
// 27 x 27 products are reduced once per voxel by k_gram_blocks and the rows only gather block lines.
// Optional compact gradient rows (approx_kernel_grad: one line <phi,z_s> + tau per location and level,
// the three rows rebuilt with nine FMAs) trade 2/3 of the row memory for ALU work.
#include <stdlib.h>

#include <cub/cub.cuh>

#include "gram_common.cuh"

namespace {

// own entries only (the transposed segments are sized by k_place_prefix)
__global__ void __launch_bounds__(kWarps * 32)
k_gram_count(nksr_svh_t svh, int64_t n_total, int32_t* __restrict__ cnt) {
  const int lane = threadIdx.x & 31;
  const int64_t row = blockIdx.x * (int64_t)kWarps + (threadIdx.x >> 5);
  if (row >= n_total) return;
  int l, i;
  row_of_warp(svh, row, l, i);
  RowGeom g;
  row_geom(svh, l, i, g);
  const int nslots = 125 + 64 * (svh.depth - 1 - l);
  int c = 0;
  for (int t0 = 0; t0 < nslots; t0 += 32) {
    int t = t0 + lane, k = 0;
    int col = t < nslots ? slot_column(svh, l, g, t, k) : -1;
    c += __popc(__ballot_sync(0xffffffffu, col >= 0));
  }
  if (lane == 0) cnt[row] = c;
}

struct AddPair {
  const int32_t* a;
  const int32_t* b;
  __host__ __device__ __forceinline__ int64_t operator()(const int64_t& i) const { return (int64_t)a[i] + b[i]; }
};

__global__ void k_set_last(const int32_t* cnt, const int32_t* cnt_down, int64_t n, int64_t* rowptr) {
  if (threadIdx.x == 0 && blockIdx.x == 0) rowptr[n] = rowptr[n - 1] + cnt[n - 1] + cnt_down[n - 1];
}

// ---------------------------------------------------------------- sort-free transposed placement
// (SPEC S6b; formula checked on the CPU by oracle/placement_proto.py + tests/test_cpu_placement.py)
// Fine voxel j (level l, coords u) stores an entry for the coarse voxel c (level l+k) iff c lies in
// [((u-1)>>k)-1, ((u+1)>>k)+1] per axis.  With a = u>>k the ancestor of j:  c-a in {-1,0,1} always
// qualifies, c-a = -2 needs u on the LOW edge of the ancestor block (u mod 2^k == 0) and c-a = +2 on
// the HIGH edge.  So the fine voxels reaching c are, for each of the 125 ancestors a = c-d, the
// descendants of a in an edge class that depends on d only, and the descendants of one ancestor are
// contiguous in Morton order.  Ordering c's transposed segment by (level l, slot of d, Morton index j):
//     position(j -> c) = prefix[c][slot(d)] + rank of j among the class(d) descendants of a
// -- two small tables from prefix sums; no atomics, no sort, deterministic by construction.
//
// edge type per axis: 0 = interior, 1 = low edge, 2 = high edge (never both: 2^k >= 2)
__device__ __forceinline__ int edge_type(int u, int m) { return (u & m) == 0 ? 1 : ((u & m) == m ? 2 : 0); }

// One warp per ancestor a (level l+k): rank8[j*8 + S] = rank of descendant j among the descendants
// that share j's edge types on the axes in S (S = 4*x + 2*y + z; only defined when j is on an edge
// for every axis of S; S = 0: index of j inside the block); class_count[a*27 + cls] = members of the
// class cls = 9*rx + 3*ry + rz, r in {0 any, 1 low, 2 high}.
__global__ void __launch_bounds__(kWarps * 32)
k_place_rank(nksr_svh_t svh, int l, int k, int32_t* __restrict__ rank8, int32_t* __restrict__ class_count) {
  const int lane = threadIdx.x & 31;
  const int lu = l + k;
  const int64_t a = blockIdx.x * (int64_t)kWarps + (threadIdx.x >> 5);
  if (a >= svh.n[lu]) return;
  int64_t first, end;
  if (k == 1 && svh.child8[lu] != nullptr) {
    // children are contiguous in Morton order: one 32-byte row of the child table instead of two binary searches
    // over the level's keys (the searches were most of the rank kernels' time)
    const int c = lane < 8 ? __ldg(svh.child8[lu] + a * 8 + lane) : -1;
    int lo = c >= 0 ? c : 0x7fffffff, hi = c;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o));
      hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o));
    }
    lo = __shfl_sync(0xffffffffu, lo, 0);
    hi = __shfl_sync(0xffffffffu, hi, 0);
    first = hi >= 0 ? lo : 0;
    end = hi >= 0 ? hi + 1 : 0;
  } else {
    const int64_t ka = __ldg(svh.keys[lu] + a);
    const int64_t nl = svh.n[l];
    first = lower_bound_key(svh.keys[l], nl, ka << (3 * k));
    end = lower_bound_key(svh.keys[l], nl, (ka + 1) << (3 * k));
  }
  const int m = (1 << k) - 1;
  const unsigned lt = (1u << lane) - 1u;
  int run[27];
#pragma unroll
  for (int c = 0; c < 27; ++c) run[c] = 0;
  for (int64_t j0 = first; j0 < end; j0 += 32) {
    const int64_t j = j0 + lane;
    const bool in = j < end;
    int ex = 0, ey = 0, ez = 0;
    if (in) {
      int x, y, z;
      morton3_decode(__ldg(svh.keys[l] + j), x, y, z);
      ex = edge_type(x, m); ey = edge_type(y, m); ez = edge_type(z, m);
    }
#pragma unroll
    for (int c = 0; c < 27; ++c) {
      const int rx = c / 9, ry = (c / 3) % 3, rz = c % 3;
      const bool mem = in && (rx == 0 || ex == rx) && (ry == 0 || ey == ry) && (rz == 0 || ez == rz);
      const unsigned b = __ballot_sync(0xffffffffu, mem);
      if (mem) rank8[j * 8 + ((rx ? 4 : 0) | (ry ? 2 : 0) | (rz ? 1 : 0))] = run[c] + __popc(b & lt);
      run[c] += __popc(b);
    }
  }
#pragma unroll
  for (int c = 0; c < 27; ++c)
    if (lane == c) class_count[a * 27 + c] = run[c];
}

// One warp per coarse voxel c (level l+k): exclusive prefix over the 125 ancestors a = c - d (slot
// t = (dx+2)*25 + (dy+2)*5 + (dz+2), d = c - a) of the class counts, starting at the current length of
// c's transposed segment (the finer levels handled before); the segment length is advanced.
__global__ void __launch_bounds__(kWarps * 32)
k_place_prefix(nksr_svh_t svh, int l, int k, const int32_t* __restrict__ class_count,
               int32_t* __restrict__ prefix, int32_t* __restrict__ cnt_down) {
  const int lane = threadIdx.x & 31;
  const int lu = l + k;
  const int64_t c = blockIdx.x * (int64_t)kWarps + (threadIdx.x >> 5);
  if (c >= svh.n[lu]) return;
  int cx, cy, cz;
  morton3_decode(__ldg(svh.keys[lu] + c), cx, cy, cz);
  int32_t* len = cnt_down + svh.offset[lu] + c;
  int carry = *len;
  __syncwarp();
  for (int t0 = 0; t0 < 125; t0 += 32) {
    const int t = t0 + lane;
    int v = 0;
    if (t < 125) {
      const int dx = t / 25 - 2, dy = (t / 5) % 5 - 2, dz = t % 5 - 2;
      const int a = lookup_near(svh, lu, (int)c, cx, cy, cz, cx - dx, cy - dy, cz - dz);
      const int cls = (dx == -2 ? 9 : (dx == 2 ? 18 : 0)) + (dy == -2 ? 3 : (dy == 2 ? 6 : 0)) +
                      (dz == -2 ? 1 : (dz == 2 ? 2 : 0));
      if (a >= 0) v = __ldg(class_count + (int64_t)a * 27 + cls);
    }
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int up = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += up;
    }
    if (t < 125) prefix[c * 125 + t] = carry + inc - v;
    carry += __shfl_sync(0xffffffffu, inc, 31);
  }
  if (lane == 0) *len = carry;
}

// Per-voxel Gram blocks for the COARSE levels (l >= split_level), where a voxel owns hundreds to
// thousands of constraint rows: one warp per (voxel u, level offset k) reduces
//   M[si][s] = sum_rows w * E_l[row][si] * E_{l+k}[row][s]      (27 x 27, lane s keeps column s)
// ONCE, instead of each of the 27 matrix rows around u streaming all of u's constraint rows again.
// Block layout: 28 lines of 32 floats -- lines 0..26 = M[si][:], line 27 = rhs share per si (k = 0).
// m[s] += el[s] * ek for the 27 stencil slots s (lane = column of the block, m[s] = row s): the weighted level-l line
// `el` of the constraint row is staged in shared memory and read back as seven broadcast 128-bit loads feeding 14
// float2 FMA pairs -- the first version fetched the 28 values with 28 shuffles per row, two thirds of its instructions
__device__ __forceinline__ void gram_block_update(float (&m)[28], const float* __restrict__ el_line, float ek) {
  const float2 ek2 = make_float2(ek, ek);
  const float4* l4 = reinterpret_cast<const float4*>(el_line);
#pragma unroll
  for (int j = 0; j < 7; ++j) {
    const float4 a = l4[j];                                    // slot 27 is padding (zero)
    const float2 r0 = ffma2_rn(make_float2(a.x, a.y), ek2, make_float2(m[4 * j], m[4 * j + 1]));
    const float2 r1 = ffma2_rn(make_float2(a.z, a.w), ek2, make_float2(m[4 * j + 2], m[4 * j + 3]));
    m[4 * j] = r0.x; m[4 * j + 1] = r0.y; m[4 * j + 2] = r1.x; m[4 * j + 3] = r1.y;
  }
}

// level c (uniform) of an interleaved row element (four levels per float4)
__device__ __forceinline__ float level_of(const float4& v, const int c) {
  return c == 0 ? v.x : (c == 1 ? v.y : (c == 2 ? v.z : v.w));
}

// ILV: rows in the interleaved layout [location][rows][32][4 levels] (nksr_build_rows mode | 4, depth <= 4): one 128-bit
// load per (location, axis) brings both lines of the block
template <int MAXL, bool ILV>
__global__ void __launch_bounds__(kWarps * 32)
k_gram_blocks(nksr_svh_t svh, nksr_constraints_t cs, float* __restrict__ mblocks) {
  __shared__ __align__(16) float stage[kWarps][3][32];
  const int lane = threadIdx.x & 31;
  const int wid = threadIdx.x >> 5;
  int64_t w = blockIdx.x * (int64_t)kWarps + wid;
  int l = cs.split_level;
  while (l < svh.depth && w >= svh.n[l] * (svh.depth - l)) { w -= svh.n[l] * (svh.depth - l); ++l; }
  if (l >= svh.depth) return;
  const int L = svh.depth;
  const int nlev = L - l;
  const int u = (int)(w / nlev), k = (int)(w - (int64_t)u * nlev);
  float m[28];
#pragma unroll
  for (int s = 0; s < 28; ++s) m[s] = 0.f;
  float bvec = 0.f;
  if (cs.range_pos) {
    const int32_t* rp = cs.range_pos + 2 * (svh.offset[l] + u);
    const int pb = __ldg(rp), pe = __ldg(rp + 1);
    for (int q = pb; q < pe; ++q) {
      float e0, ek;
      if (ILV) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(cs.e_pos) + (int64_t)q * NKSR_ROW_STRIDE + lane);
        e0 = level_of(v, l);
        ek = level_of(v, l + k);
      } else {
        const float* p0 = cs.e_pos + ((int64_t)q * L + l) * NKSR_ROW_STRIDE + lane;
        e0 = __ldg(p0);
        ek = k == 0 ? e0 : __ldg(p0 + k * NKSR_ROW_STRIDE);
      }
      stage[wid][0][lane] = cs.w_pos * e0;
      __syncwarp();
      gram_block_update(m, stage[wid][0], ek);
      __syncwarp();
    }
  }
  if (cs.range_nrm) {
    const int32_t* rn = cs.range_nrm + 2 * (svh.offset[l] + u);
    const int nb = __ldg(rn), ne = __ldg(rn + 1);
    // (requesting the lines of location q + 1 before location q is multiplied in was tried: slower)
    for (int q = nb; q < ne; ++q) {
      const float* p0 = cs.e_nrm + ((int64_t)q * L + l) * (3 * NKSR_ROW_STRIDE) + lane;
      float ek[3];
#pragma unroll
      for (int ax = 0; ax < 3; ++ax) {
        float e0;
        if (ILV) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(cs.e_nrm) + ((int64_t)q * 3 + ax) * NKSR_ROW_STRIDE + lane);
          e0 = level_of(v, l);
          ek[ax] = level_of(v, l + k);
        } else {
          e0 = __ldg(p0 + ax * NKSR_ROW_STRIDE);
          ek[ax] = k == 0 ? e0 : __ldg(p0 + (k * 3 + ax) * NKSR_ROW_STRIDE);
        }
        const float el = cs.w_nrm * e0;
        if (k == 0) bvec = fmaf(el, __ldg(cs.t_nrm + (int64_t)q * 3 + ax), bvec);
        stage[wid][ax][lane] = el;
      }
      __syncwarp();
#pragma unroll
      for (int ax = 0; ax < 3; ++ax) gram_block_update(m, stage[wid][ax], ek[ax]);
      __syncwarp();
    }
  }
  float* blk = mblocks + (cs.mblock_off[l] + (int64_t)u * nlev + k) * kBlockFloats;
#pragma unroll
  for (int s = 0; s < 27; ++s) blk[s * NKSR_ROW_STRIDE + lane] = m[s];
  blk[27 * NKSR_ROW_STRIDE + lane] = bvec;
}

// ILV (MAXL == 4): rows in the interleaved layout -- one 128-bit load per lane brings the four levels of a location
// (value rows) or of one axis of it (gradient rows): 1 + 3 wide loads per visited location instead of 4 + 12 narrow ones
// (with narrow loads the LSU was the busiest unit of the kernel).  Same products in the same order: the matrix is
// bitwise the one of the plain layout.
template <bool COMPACT, int MAXL, int MINB, bool ILV>
__global__ void __launch_bounds__(kWarps * 32, MINB)
k_gram_fill(nksr_svh_t svh, nksr_feat_t feat, nksr_constraints_t cs, int64_t row_begin, int64_t row_end,
            const int32_t* __restrict__ cnt, const int64_t* __restrict__ rowptr, int32_t* __restrict__ col_out,
            float* __restrict__ val_out, float* __restrict__ rhs, float* __restrict__ diag,
            const nksr_placement_t place) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31;
  const int wid = threadIdx.x >> 5;
  // coarse rows own thousands of constraint rows, fine rows a few dozen: schedule the heavy
  // (coarse, high index) rows first so that the tail of the grid is made of light rows
  const int64_t row = row_end - 1 - (blockIdx.x * (int64_t)kWarps + wid);
  if (row < row_begin) return;
  int l, i;
  row_of_warp(svh, row, l, i);
  const int L = svh.depth;
  const int nup = L - 1 - l;
  const int nslots = 125 + 64 * nup;
  float* acc = smem + wid * kMaxSlots;
  for (int t = lane; t < nslots; t += 32) acc[t] = 0.f;
  RowGeom g;
  row_geom(svh, l, i, g);
  const int64_t N = cs.n_pos, K = cs.n_nrm;
  const int32_t* rp = cs.range_pos ? cs.range_pos + 2 * svh.offset[l] : nullptr;
  const int32_t* rn = cs.range_nrm ? cs.range_nrm + 2 * svh.offset[l] : nullptr;
  float bsum = 0.f;
  const int sl = lane < 27 ? lane : 13;
  const int ldx = c_d27[sl][0], ldy = c_d27[sl][1], ldz = c_d27[sl][2];
  // flush bases: lane us < 27 is also the source voxel u = i + d(us); base of u in the tile on every level without
  // the lane's own stencil offset, packed two per word:  same level: (d+2) in the 5^3 box;  level l+k: position of
  // (u >> k) in the 4^3 box that starts at ((i-1) >> k) - 1
  const int lane_l0 = ldx * 25 + ldy * 5 + ldz, lane_lk = ldx * 16 + ldy * 4 + ldz;
  unsigned flush_a, flush_b;
  {
    int b[4];
    b[0] = 62 + lane_l0;
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      const int ox = ((g.ux + ldx) >> k) - (((g.ux - 1) >> k) - 1), oy = ((g.uy + ldy) >> k) - (((g.uy - 1) >> k) - 1),
                oz = ((g.uz + ldz) >> k) - (((g.uz - 1) >> k) - 1);
      b[k] = 125 + 64 * (k - 1) + (ox << 4) + (oy << 2) + oz;
    }
    flush_a = (unsigned)b[0] | ((unsigned)b[1] << 16);
    flush_b = (unsigned)b[2] | ((unsigned)b[3] << 16);
  }
  // lane-parallel prefetch of the 27 neighbour voxels and their constraint-row ranges
  const int my_u = lane < 27 ? __ldg(svh.nbr27[l] + (int64_t)i * 27 + lane) : -1;
  int my_pb = 0, my_pe = 0, my_nb = 0, my_ne = 0;
  if (my_u >= 0) {
    if (rp) { my_pb = __ldg(rp + 2 * (int64_t)my_u); my_pe = __ldg(rp + 2 * (int64_t)my_u + 1); }
    if (rn) { my_nb = __ldg(rn + 2 * (int64_t)my_u); my_ne = __ldg(rn + 2 * (int64_t)my_u + 1); }
  }
  const CompactSpline spline(ldx, ldy, ldz);
  const float inv_wl = 1.f / (svh.voxel_size * (float)(1 << l));
  // rows are stored location-major ([q][L][rows][32]): level stride is a compile-time constant
  constexpr int pos_level = NKSR_ROW_STRIDE;
  constexpr int nrm_level = NKSR_ROW_STRIDE * (COMPACT ? 1 : 3);
  (void)N; (void)K;
  const bool use_blocks = cs.mblocks != nullptr && l >= cs.split_level;
  __syncwarp();

  for (int us = 0; us < 27; ++us) {
    const int u = __shfl_sync(0xffffffffu, my_u, us);
    if (u < 0) continue;
    const int pb = __shfl_sync(0xffffffffu, my_pb, us), pe = __shfl_sync(0xffffffffu, my_pe, us);
    const int nb = __shfl_sync(0xffffffffu, my_nb, us), ne = __shfl_sync(0xffffffffu, my_ne, us);
    if (pb == pe && nb == ne) continue;
    const int si = 26 - us;  // slot of i inside u's stencil
    float r[MAXL];
#pragma unroll
    for (int k = 0; k < MAXL; ++k) r[k] = 0.f;
    if (use_blocks) {
      // coarse level: the 27 x 27 products of u's constraint rows were reduced once per voxel by
      // k_gram_blocks; this row only picks its line of every block (and its share of the rhs)
      const float* blk = cs.mblocks + (cs.mblock_off[l] + (int64_t)u * (nup + 1)) * kBlockFloats;
      bsum += __ldg(blk + 27 * NKSR_ROW_STRIDE + si);
#pragma unroll
      for (int k = 0; k < MAXL; ++k)
        if (k <= nup) r[k] = __ldg(blk + (int64_t)k * kBlockFloats + si * NKSR_ROW_STRIDE + lane);
    } else {
    if (ILV) {
      float2 a01 = make_float2(0.f, 0.f), a23 = make_float2(0.f, 0.f);     // ABSOLUTE levels 0,1 | 2,3
      const float4* ep = reinterpret_cast<const float4*>(cs.e_pos) + lane;
      for (int q = pb; q < pe; ++q) {
        const float4 v = __ldg(ep + (int64_t)q * NKSR_ROW_STRIDE);
        const float a = cs.w_pos * __shfl_sync(0xffffffffu, level_of(v, l), si);
        a01 = ffma2_rn(make_float2(a, a), make_float2(v.x, v.y), a01);
        a23 = ffma2_rn(make_float2(a, a), make_float2(v.z, v.w), a23);
      }
      const float4* en = reinterpret_cast<const float4*>(cs.e_nrm) + lane;
      for (int q = nb; q < ne; ++q) {
        const float4* p = en + (int64_t)q * (3 * NKSR_ROW_STRIDE);
        // own coefficients: broadcast loads of level l of slot si (see the note in the plain loop below)
        const float* ps = cs.e_nrm + ((int64_t)q * (3 * NKSR_ROW_STRIDE) + si) * 4 + l;
        const float* t = cs.t_nrm + (int64_t)q * 3;
#pragma unroll
        for (int ax = 0; ax < 3; ++ax) {
          const float a = cs.w_nrm * __ldg(ps + ax * (4 * NKSR_ROW_STRIDE));
          bsum = fmaf(a, __ldg(t + ax), bsum);
          const float4 v = __ldg(p + ax * NKSR_ROW_STRIDE);
          a01 = ffma2_rn(make_float2(a, a), make_float2(v.x, v.y), a01);
          a23 = ffma2_rn(make_float2(a, a), make_float2(v.z, v.w), a23);
        }
      }
      // absolute -> relative levels (l is uniform in the warp)
      if (l == 0) { r[0] = a01.x; r[1] = a01.y; r[2] = a23.x; r[3] = a23.y; }
      else if (l == 1) { r[0] = a01.y; r[1] = a23.x; r[2] = a23.y; }
      else if (l == 2) { r[0] = a23.x; r[1] = a23.y; }
      else { r[0] = a23.y; }
    } else {
    // fp32 FMAs on float2 pairs: two levels per step, same IEEE result per lane
    float2 r2[MAXL / 2];
#pragma unroll
    for (int k2 = 0; k2 < MAXL / 2; ++k2) r2[k2] = make_float2(0.f, 0.f);
    for (int q = pb; q < pe; ++q) {
      const float* pk = cs.e_pos + ((int64_t)q * L + l) * NKSR_ROW_STRIDE + lane;
      float ln[MAXL];
#pragma unroll
      for (int k = 0; k < MAXL; ++k) ln[k] = k <= nup ? __ldg(pk + k * pos_level) : 0.f;
      const float a = cs.w_pos * __shfl_sync(0xffffffffu, ln[0], si);
#pragma unroll
      for (int k2 = 0; k2 < MAXL / 2; ++k2)
        r2[k2] = ffma2_rn(make_float2(a, a), make_float2(ln[2 * k2], ln[2 * k2 + 1]), r2[k2]);
    }
    if (COMPACT) {
      // one line per (location, level): <phi,z_s> in slots 0..26, tau in 27..29;
      // E_a[s] = dB_a B_b B_c <phi,z_s> / W_level
      for (int q = nb; q < ne; ++q) {
        const float* pk = cs.e_nrm + ((int64_t)q * L + l) * NKSR_ROW_STRIDE + lane;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, iw = inv_wl;
#pragma unroll
        for (int k = 0; k < MAXL; ++k) {
          if (k <= nup) {
            const float line = __ldg(pk);
            pk += nrm_level;
            float e0, e1, e2;
            spline.grad_rows(line, iw, lane, e0, e1, e2);
            if (k == 0) {
              a0 = cs.w_nrm * __shfl_sync(0xffffffffu, e0, si);
              a1 = cs.w_nrm * __shfl_sync(0xffffffffu, e1, si);
              a2 = cs.w_nrm * __shfl_sync(0xffffffffu, e2, si);
              const float* t = cs.t_nrm + (int64_t)q * 3;
              bsum = fmaf(a0, __ldg(t), fmaf(a1, __ldg(t + 1), fmaf(a2, __ldg(t + 2), bsum)));
            }
            r[k] = fmaf(a0, e0, fmaf(a1, e1, fmaf(a2, e2, r[k])));
            iw *= 0.5f;
          }
        }
      }
    } else {
      // (a "wide" variant -- 80 registers, three blocks per SM, two normal locations = 30 line loads in flight per warp
      // -- was measured slower and removed)
      for (int q = nb; q < ne; ++q) {
        const float* p0 = cs.e_nrm + ((int64_t)q * L + l) * (3 * NKSR_ROW_STRIDE);
        const float* t = cs.t_nrm + (int64_t)q * 3;
        // (the own coefficient stays a broadcast LOAD here: fetching it by shuffle from the level-l line -- as the position
        // loop does -- ties the three axes' loads to the shuffles' completion and was measured slower)
#pragma unroll
        for (int ax = 0; ax < 3; ++ax) {
          const float a = cs.w_nrm * __ldg(p0 + ax * NKSR_ROW_STRIDE + si);
          bsum = fmaf(a, __ldg(t + ax), bsum);
          const float* pk = p0 + ax * NKSR_ROW_STRIDE + lane;
#pragma unroll
          for (int k2 = 0; k2 < MAXL / 2; ++k2) {
            const float l0 = 2 * k2 <= nup ? __ldg(pk + (2 * k2) * nrm_level) : 0.f;
            const float l1 = 2 * k2 + 1 <= nup ? __ldg(pk + (2 * k2 + 1) * nrm_level) : 0.f;
            r2[k2] = ffma2_rn(make_float2(a, a), make_float2(l0, l1), r2[k2]);
          }
        }
      }
    }
#pragma unroll
    for (int k2 = 0; k2 < MAXL / 2; ++k2) { r[2 * k2] += r2[k2].x; r[2 * k2 + 1] += r2[k2].y; }
    }  // !ILV
    }  // !use_blocks
    // flush: every lane < 27 owns a distinct structural slot per level; slot = base of the source voxel (computed once
    // per row by lane `us`, see flush_base above) + constant of the lane.  (The per-lane index arithmetic
    // of the first version was a fifth of the kernel's instructions.)
    {
      const unsigned wa = __shfl_sync(0xffffffffu, flush_a, us), wb = __shfl_sync(0xffffffffu, flush_b, us);
      if (lane < 27) {
        acc[(int)(wa & 0xffffu) + lane_l0] += r[0];
        if (MAXL > 1 && 1 <= nup) acc[(int)(wa >> 16) + lane_lk] += r[1];
        if (MAXL > 2 && 2 <= nup) acc[(int)(wb & 0xffffu) + lane_lk] += r[2];
        if (MAXL > 3 && 3 <= nup) acc[(int)(wb >> 16) + lane_lk] += r[3];
#pragma unroll
        for (int k = 4; k < MAXL; ++k) {      // hierarchies deeper than 4 levels: the general formula
          if (k <= nup) {
            const int vx = g.ux + c_d27[us][0], vy = g.uy + c_d27[us][1], vz = g.uz + c_d27[us][2];
            const int ox = ((vx >> k) + ldx) - (((g.ux - 1) >> k) - 1);
            const int oy = ((vy >> k) + ldy) - (((g.uy - 1) >> k) - 1);
            const int oz = ((vz >> k) + ldz) - (((g.uz - 1) >> k) - 1);
            acc[125 + 64 * (k - 1) + (ox << 4) + (oy << 2) + oz] += r[k];
          }
        }
      }
    }
    __syncwarp();
  }
  gram_row_regulariser(feat, cs, l, i, my_u, lane, acc);
  __syncwarp();
  gram_row_writeout<MAXL>(svh, l, i, row, g, acc, cnt, rowptr, col_out, val_out, diag, place, lane);
  if (lane == 0) rhs[row] = bsum;
}

static int64_t total_unknowns(const nksr_svh_t* svh) {
  return svh->offset[svh->depth - 1] + svh->n[svh->depth - 1];
}

}  // namespace

extern "C" {

int nksr_gram_count_own(const nksr_svh_t* svh, int32_t* cnt, void* stream) {
  if (!svh || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH) return NKSR_E_INVALID;
  if (!svh->nbr125_top && !svh->parent[svh->depth - 1]) return NKSR_E_INVALID;
  const int64_t n = total_unknowns(svh);
  if (n == 0) return NKSR_OK;
  k_gram_count<<<grid_for(n, kWarps), kWarps * 32, 0, as_stream(stream)>>>(*svh, n, cnt);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_gram_place(const nksr_svh_t* svh, int l, int k, int32_t* rank8, int32_t* class_count, int32_t* prefix,
                    int32_t* cnt_down, void* stream) {
  if (!svh || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH || l < 0 || k < 1 || l + k >= svh->depth)
    return NKSR_E_INVALID;
  if (!svh->nbr125_top && !svh->parent[svh->depth - 1]) return NKSR_E_INVALID;
  if (!rank8 || !class_count || !prefix || !cnt_down) return NKSR_E_INVALID;
  const int64_t n_up = svh->n[l + k];
  if (n_up == 0 || svh->n[l] == 0) return NKSR_OK;
  const int grid = grid_for(n_up, kWarps);
  k_place_rank<<<grid, kWarps * 32, 0, as_stream(stream)>>>(*svh, l, k, rank8, class_count);
  NKSR_CHECK_LAUNCH();
  k_place_prefix<<<grid, kWarps * 32, 0, as_stream(stream)>>>(*svh, l, k, class_count, prefix, cnt_down);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

size_t nksr_scan_workspace_bytes(int64_t n) {
  size_t bytes = 0;
  cub::CountingInputIterator<int64_t> cnt_it(0);
  cub::TransformInputIterator<int64_t, AddPair, cub::CountingInputIterator<int64_t>> it(cnt_it,
                                                                                        AddPair{nullptr, nullptr});
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, it, (int64_t*)nullptr, n);
  return bytes + 256;
}

int nksr_gram_rowptr(const int32_t* cnt, const int32_t* cnt_down, int64_t n, int64_t* rowptr, void* ws,
                     size_t ws_bytes, void* stream) {
  if (n <= 0) return NKSR_E_INVALID;
  cub::CountingInputIterator<int64_t> cnt_it(0);
  cub::TransformInputIterator<int64_t, AddPair, cub::CountingInputIterator<int64_t>> it(cnt_it,
                                                                                        AddPair{cnt, cnt_down});
  size_t need = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, need, it, rowptr, n);
  if (need > ws_bytes) return NKSR_E_WORKSPACE;
  if (cub::DeviceScan::ExclusiveSum(ws, need, it, rowptr, n, as_stream(stream)) != cudaSuccess) return NKSR_E_CUDA;
  k_set_last<<<1, 32, 0, as_stream(stream)>>>(cnt, cnt_down, n, rowptr);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int64_t nksr_gram_block_floats(const nksr_svh_t* svh, int split_level) {
  if (!svh || split_level < 0) return 0;
  int64_t blocks = 0;
  for (int l = split_level; l < svh->depth; ++l) blocks += svh->n[l] * (svh->depth - l);
  return blocks * kBlockFloats;
}

int nksr_gram_blocks(const nksr_svh_t* svh, const nksr_constraints_t* c, float* mblocks, void* stream) {
  if (!svh || !c || !mblocks || c->nrm_compact == 1 || c->split_level < 0 || c->split_level > svh->depth)
    return NKSR_E_INVALID;
  const bool ilv = c->nrm_compact == 2;               // interleaved rows (both arrays), depth <= 4
  if (ilv && svh->depth > 4) return NKSR_E_INVALID;
  int64_t warps = 0;
  for (int l = c->split_level; l < svh->depth; ++l) warps += svh->n[l] * (svh->depth - l);
  if (warps == 0) return NKSR_OK;
  const int grid = grid_for(warps, kWarps);
  if (ilv)
    k_gram_blocks<4, true><<<grid, kWarps * 32, 0, as_stream(stream)>>>(*svh, *c, mblocks);
  else if (svh->depth <= 4)
    k_gram_blocks<4, false><<<grid, kWarps * 32, 0, as_stream(stream)>>>(*svh, *c, mblocks);
  else
    k_gram_blocks<NKSR_MAX_DEPTH, false><<<grid, kWarps * 32, 0, as_stream(stream)>>>(*svh, *c, mblocks);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_gram_fill_placed(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                          const int32_t* cnt, const int64_t* rowptr, const nksr_placement_t* placement,
                          int32_t* col, float* val, float* rhs, float* diag, void* stream) {
  return nksr_gram_fill_placed_rows(svh, feat, c, cnt, rowptr, placement, 0, -1, col, val, rhs, diag, stream);
}

int nksr_gram_fill_placed_rows(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                               const int32_t* cnt, const int64_t* rowptr, const nksr_placement_t* placement,
                               int64_t row_begin, int64_t row_end, int32_t* col, float* val, float* rhs, float* diag,
                               void* stream) {
  if (!svh || !feat || !c || !placement || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH) return NKSR_E_INVALID;
  if (!svh->nbr125_top && !svh->parent[svh->depth - 1]) return NKSR_E_INVALID;
  const int64_t n = total_unknowns(svh);
  if (row_end < 0) row_end = n;
  if (row_begin < 0 || row_begin > row_end || row_end > n) return NKSR_E_INVALID;
  if (row_begin == row_end) return NKSR_OK;
  cudaStream_t s = as_stream(stream);
  const size_t smem = (size_t)kWarps * kMaxSlots * sizeof(float);
  const int grid = grid_for(row_end - row_begin, kWarps);
#define NKSR_FILL(COMPACT, MAXL, MINB, ILV)                                                                  \
  k_gram_fill<COMPACT, MAXL, MINB, ILV><<<grid, kWarps * 32, smem, s>>>(                                     \
      *svh, *feat, *c, row_begin, row_end, cnt, rowptr, col, val, rhs, diag, *placement)
  // 4 resident blocks per SM (64 registers) for depth <= 4; 5 blocks (48 registers) was measured
  // 1.7x slower (register starvation cuts the loads in flight per warp)
  if (c->nrm_compact == 2) {                          // interleaved rows
    if (svh->depth > 4) return NKSR_E_INVALID;
    NKSR_FILL(false, 4, 4, true);
  } else if (svh->depth <= 4) {
    if (c->nrm_compact) NKSR_FILL(true, 4, 4, false); else NKSR_FILL(false, 4, 4, false);
  } else {
    if (c->nrm_compact) NKSR_FILL(true, NKSR_MAX_DEPTH, 2, false); else NKSR_FILL(false, NKSR_MAX_DEPTH, 2, false);
  }
#undef NKSR_FILL
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
