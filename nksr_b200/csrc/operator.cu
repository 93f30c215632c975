// Matrix-free application of the inference system A = E^T W E + w_reg R (SPEC S5) straight from the kernel rows, for the
// PCG of KernelField.solve: no count, placement, blocks or fill, and no CSR matrix.  DESIGN 4.2.1.
//
// Setup (nksr_op_setup, once per solve) merges the Morton-sorted positions and normal locations into one sequence by
// their half-voxel keys (positions first on equal keys), so that every voxel's locations of both kinds are one
// contiguous run at every level.  It cuts each top-level voxel's run into work items of at most S locations, cut only
// where no voxel of a level <= kCutLevel continues (a single such voxel longer than S is an item of its own).
//
// k_op_walk: a persistent grid of warps steps over the items, lane = stencil slot.  Per location r the warp loads r's
// lines of every level once (two locations ahead), forms t_r = w_r E_r x (three values for a gradient location, one
// per axis) from the x values of the containing voxel's 27 neighbours -- fetched once per run of locations with the
// same containing voxel u_l, one run ahead, their nbr27 rows two runs ahead -- and adds E_l[r][s] t_r into a register
// accumulator per level.  The run bookkeeping is done per window of 32 locations, lane-parallel: one ballot per level
// marks the run starts, and inside the window every branch is warp-uniform.  When u_l changes, the accumulator is
// stored once to the planar partial sums P[s][u] (27 planes of n floats).  A voxel of a level <= kCutLevel lies inside
// one item; a coarser voxel's run may span items, and then every item stores its piece to an edge buffer, which
// k_op_edges sums in item order and stores to P once (whether a piece goes there is decided once per item).  The
// stores to P go through a per-warp buffer in shared memory, 32 voxels at a time, one plane after the other.  No
// atomics: each P[.][u] has one writer, and the result is bitwise repeatable and independent of the grid.  Voxels
// without locations are never written, and stay zero from the setup's clear.
//
// k_op_apply: one thread per unknown, levels concatenated, grid-stride.  y_i = sum_s P[s][nbr27(i)[26 - s]] (u's slot s
// is i exactly when i's slot 26 - s is u) + w_reg sum_s B3(d_s) <z_i, z_n> x_n over the 27 neighbours n = nbr27(i)[s]:
// the regulariser of gram_row_regulariser, formed on the fly.
//
// Setup also runs the walk with t_r = w_r * target (the right-hand side) and w_r E^2 (the Jacobi diagonal) accumulated
// into a second set of planes.
#include <cub/cub.cuh>

#include "gram_common.cuh"
#include "operator.cuh"

namespace {

constexpr int kOpWarps = 4;          // warps per block of the walk
constexpr int kApplyBlock = 256;
constexpr int kEdgeBlock = 256;
// items are cut at boundaries of the voxels of levels <= kCutLevel.  The macro exists to measure the alternatives
// (DESIGN 4.2.1); the default is what the measurements chose.
#ifndef NKSR_OP_CUT_LEVEL
#define NKSR_OP_CUT_LEVEL 2
#endif
constexpr int kCutLevel = NKSR_OP_CUT_LEVEL;
constexpr int kItemFirst = 1, kItemLast = 2;   // item flags: first / last item of its top voxel

// row forms: value rows (positions), compact gradient lines (approx_kernel_grad), three full gradient rows
enum { kValue = 0, kCompact = 1, kFull = 2 };

__device__ __forceinline__ int op_cut_level(int depth) { return depth - 1 < kCutLevel ? depth - 1 : kCutLevel; }

// the edge partials of the rhs / application (e) and of the diagonal (d), after the items, each 256-byte aligned; laid
// out for the capacity nksr_op_setup recorded, whatever workspace size a later application is given
struct EdgeBuffers { float* e; float* d; };
__device__ __forceinline__ EdgeBuffers op_edge_buffers(const MfOperator& op) {
  const uint64_t mi = (uint64_t)*op.max_items;
  const uint64_t a = (reinterpret_cast<uint64_t>(op.items) + mi * sizeof(int4) + 255) & ~(uint64_t)255;
  const uint64_t b = (a + mi * op.edge_levels * 2 * 27 * sizeof(float) + 255) & ~(uint64_t)255;
  return {reinterpret_cast<float*>(a), reinterpret_cast<float*>(b)};
}

// ------------------------------------------------------------------------------------------------- setup: the items
// owned-location filter: keep[i] = 1 when location i (positions, then normal locations) has, on some level l, an owned
// unknown among the 27 neighbours of its containing voxel -- the only rows it contributes to.  One warp per location,
// lane = stencil slot
__global__ void k_op_keep(nksr_svh_t svh, const int32_t* __restrict__ bp, int64_t np, const int32_t* __restrict__ bn,
                          int64_t nn, const uint8_t* __restrict__ owned, int32_t* __restrict__ keep) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (i >= np + nn) return;
  const bool pos = i < np;
  const int32_t* b = pos ? bp + i : bn + (i - np);
  const int64_t nb = pos ? np : nn;
  bool any = false;
  for (int l = 0; l < svh.depth && !any; ++l) {
    const int v = __ldg(b + l * nb);
    if (v < 0) continue;
    const int u = lane < 27 ? __ldg(svh.nbr27[l] + (int64_t)v * 27 + lane) : -1;
    any = __any_sync(0xffffffffu, u >= 0 && __ldg(owned + svh.offset[l] + u) != 0);
  }
  if (lane == 0) keep[i] = any ? 1 : 0;
}

// merged position of every location: positions first on equal keys (a stable merge of the two sorted key lists).
// keep != nullptr: the exclusive scan of the filter's flags over m + 1 entries; only the kept locations are merged, to
// the first keep[m] slots, in the same relative order
__global__ void k_op_merge(const int64_t* __restrict__ kp, int64_t np, const int64_t* __restrict__ kn, int64_t nn,
                           const int32_t* __restrict__ bp, const int32_t* __restrict__ bn, int L,
                           const int32_t* __restrict__ keep, int32_t* __restrict__ seq, int32_t* __restrict__ vox) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const int64_t m = np + nn;
  if (i >= m) return;
  if (keep && keep[i + 1] == keep[i]) return;
  const bool pos = i < np;
  const int64_t r = pos ? i : i - np;
  const int64_t key = pos ? kp[r] : kn[r];
  const int64_t* other = pos ? kn : kp;
  int64_t lo = 0, hi = pos ? nn : np;   // positions: #normals with key < k; normals: #positions with key <= k
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    const int64_t v = __ldg(other + mid);
    if (pos ? v < key : v <= key) lo = mid + 1; else hi = mid;
  }
  // the same count over the kept locations only: kept ones of my kind before me plus kept ones of the other before me
  const int64_t rank = !keep ? r + lo
                     : pos ? keep[i] + (keep[np + lo] - keep[np]) : (keep[i] - keep[np]) + keep[lo];
  seq[rank] = pos ? (int32_t)r : ~(int32_t)r;
  const int32_t* b = pos ? bp : bn;
  const int64_t nb = pos ? np : nn;
  for (int l = 0; l < L; ++l) vox[l * m + rank] = __ldg(b + l * nb + r);
}

// merged range of every top-level voxel (zero-length for voxels without locations: the workspace starts cleared)
__global__ void k_op_top_ranges(const int32_t* __restrict__ vt, int64_t m, int2* __restrict__ top) {
  const int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (k >= m) return;
  const int t = vt[k];
  if (t < 0) return;
  if (k == 0 || vt[k - 1] != t) top[t].x = (int)k;
  if (k == m - 1 || vt[k + 1] != t) top[t].y = (int)(k + 1);
}

// one warp per top voxel: greedy items of at most S locations, cut only before a location k where no voxel of a level
// <= cut continues from k - 1; when there is no such k within S locations, the item runs to the next one.
// !WRITE: cnt[g] = items of voxel g.  WRITE: items at ofs[g], and the last voxel's warp stores the item count.
template <bool WRITE>
__global__ void k_op_cut(const int32_t* __restrict__ vox, int64_t m, const int2* __restrict__ top, int64_t n_top,
                         int cut, int S, int32_t* __restrict__ cnt, const int32_t* __restrict__ ofs,
                         int4* __restrict__ items, int32_t* __restrict__ n_items) {
  const int lane = threadIdx.x & 31;
  const int64_t g = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  if (g >= n_top) return;
  const int2 rg = top[g];
  const int s = rg.x, e = rg.y;
  auto legal = [&](int k) {
    for (int l = 0; l <= cut; ++l) {
      const int p = __ldg(vox + l * m + k - 1);
      if (p >= 0 && p == __ldg(vox + l * m + k)) return false;
    }
    return true;
  };
  const int o = WRITE ? ofs[g] : 0;
  int a = s, c = 0;
  while (a < e) {
    const int64_t lim = (int64_t)a + S < e ? (int64_t)a + S : e;
    int b = -1;
    if (lim == e) {
      b = e;
    } else {
      for (int hi = (int)lim; hi > a && b < 0; hi -= 32) {   // the largest legal cut in (a, lim]
        const int k = hi - lane;
        const unsigned bal = __ballot_sync(0xffffffffu, k > a && legal(k));
        if (bal) b = hi - (__ffs(bal) - 1);
      }
      for (int lo = (int)lim + 1; b < 0; lo += 32) {          // none: the first one after lim (e at the latest)
        const int k = lo + lane;
        const unsigned bal = __ballot_sync(0xffffffffu, k >= e || legal(k));
        if (bal) b = lo + __ffs(bal) - 1;
      }
    }
    if (WRITE && lane == 0) items[o + c] = make_int4(a, b, (a == s ? kItemFirst : 0) | (b == e ? kItemLast : 0), 0);
    ++c;
    a = b;
  }
  if (!WRITE && lane == 0) cnt[g] = c;
  if (WRITE && lane == 0 && g == n_top - 1) *n_items = o + c;
}

// ------------------------------------------------------------------------------------------- the walk of one item
// The warp steps over the item in windows of 32 merged locations.  Each window is read lane-parallel (lane j =
// location k0 + j: sequence entry and containing voxel per level), and one ballot per level marks where a run of
// locations with the same containing voxel starts.  Inside the window every branch is warp-uniform: a run start is a
// bit test, its voxel one shuffle.  The next window is held as well, so that a run start can find the next two runs
// of its level in the run-start masks and request their x values and nbr27 rows one and two runs ahead.
// A warp's finished partial sums on their way to P: up to 32 voxels, one row of 27 slots each (stride 33, so that both
// the row-wise writes and the column-wise reads are free of bank conflicts), and the voxels' unknown indices.  A full
// buffer is drained plane by plane: the buffered voxels are nearly consecutive, so each plane's store touches a few
// sectors, where a voxel's own store would touch 27
constexpr int kStage = 33;
struct PStage {
  float* v;     // [32][kStage] acc
  float* d;     // [32][kStage] accd (setup)
  int64_t* g;   // [32] offset[l] + u
  int n;        // voxels held, warp-uniform
};

template <bool SETUP>
__device__ __forceinline__ void op_stage_drain(const MfOperator& op, PStage& ps, int lane) {
  __syncwarp();
  if (lane < ps.n) {
    const int64_t g = ps.g[lane];
    float* p = op.P + g;
    float* pd = SETUP ? op.Pd + g : nullptr;
#pragma unroll 9
    for (int s = 0; s < 27; ++s) {
      p[(int64_t)s * op.n] = ps.v[lane * kStage + s];
      if (SETUP) pd[(int64_t)s * op.n] = ps.d[lane * kStage + s];
    }
  }
  __syncwarp();
  ps.n = 0;
}

template <int NKIND, int MAXL, bool SETUP>
__device__ __forceinline__ void op_walk_item(const MfOperator& op, const float* __restrict__ x, int it, int4 item,
                                             EdgeBuffers eb, PStage& ps, int lane) {
  constexpr unsigned kAll = 0xffffffffu;
  constexpr int LINES = NKIND == kFull ? 3 : 1;     // 128-byte lines per (location, level) of the widest row
  const nksr_svh_t& svh = op.svh;
  const int L = svh.depth;
  const int cut = op_cut_level(L);
  const int64_t m = op.m;
  const int32_t* __restrict__ vox = op.vox;
  const int b = item.x, e = item.y;
  const int sl = lane < 27 ? lane : 13;
  const CompactSpline spline(c_d27[sl][0], c_d27[sl][1], c_d27[sl][2]);
  const float inv_w0 = 1.f / svh.voxel_size;

  // bit l (16 + l): the item's first (last) run on level l > cut continues from the previous (into the next) item
  bool cont = false;
  if (lane < L && !(item.z & kItemFirst)) {
    const int p = __ldg(vox + lane * m + b - 1);
    cont = p >= 0 && p == __ldg(vox + lane * m + b);
  } else if (lane >= 16 && lane - 16 < L && !(item.z & kItemLast)) {
    const int p = __ldg(vox + (lane - 16) * m + e);
    cont = p >= 0 && p == __ldg(vox + (lane - 16) * m + e - 1);
  }
  const unsigned above = (0xffffu << (cut + 1)) & 0xffffu;
  const unsigned edge = __ballot_sync(kAll, cont) & (above | above << 16);

  // windows A (locations k0 + j) and B (k0 + 32 + j): sequence entry q, containing voxels v, and per level the run
  // starts s (bit j: location j's voxel differs from the one before it; -1 before the item)
  int qa, qb, va[MAXL], vb[MAXL];
  unsigned sa[MAXL], sb[MAXL];
  auto load_win = [&](int k0, int& q, int (&v)[MAXL]) {
    const int k = k0 + lane;
    const bool in = k < e;
    q = in ? __ldg(op.seq + k) : 0;
#pragma unroll
    for (int l = 0; l < MAXL; ++l) v[l] = (in && l < L) ? __ldg(vox + l * m + k) : -1;
  };
  auto starts_b = [&]() {   // B's run starts; B's lane 0 follows A's lane 31
#pragma unroll
    for (int l = 0; l < MAXL; ++l)
      sb[l] = __ballot_sync(kAll, vb[l] != __shfl_sync(kAll, lane == 31 ? va[l] : vb[l], (lane + 31) & 31));
  };
  load_win(b, qa, va);
  load_win(b + 32, qb, vb);
#pragma unroll
  for (int l = 0; l < MAXL; ++l) {
    const int p = __shfl_up_sync(kAll, va[l], 1);
    sa[l] = __ballot_sync(kAll, va[l] != (lane == 0 ? -1 : p));
  }
  starts_b();

  // the lines of the next locations, requested AHEAD locations before they are visited: sequence entry, the lines
  // of every level and (setup) the target values.  The three-line rows take one location, to stay in the registers
  constexpr int AHEAD = NKIND == kFull ? 1 : 2;
  constexpr int TN = SETUP ? 3 : 1;
  struct Stage {
    int q;
    float ln[MAXL][LINES];
    float tn[TN];
  };
  auto load_stage = [&](int q, Stage& s) {
    s.q = q;
    if (q >= 0) {
      const float* p = op.cs.e_pos + (int64_t)q * L * NKSR_ROW_STRIDE + lane;
#pragma unroll
      for (int l = 0; l < MAXL; ++l)
#pragma unroll
        for (int a = 0; a < LINES; ++a) s.ln[l][a] = (a == 0 && l < L) ? __ldcs(p + l * NKSR_ROW_STRIDE) : 0.f;
#pragma unroll
      for (int a = 0; a < TN; ++a) s.tn[a] = 0.f;
    } else {
      const float* p = op.cs.e_nrm + (int64_t)~q * L * LINES * NKSR_ROW_STRIDE + lane;
#pragma unroll
      for (int l = 0; l < MAXL; ++l)
#pragma unroll
        for (int a = 0; a < LINES; ++a) s.ln[l][a] = l < L ? __ldcs(p + (l * LINES + a) * NKSR_ROW_STRIDE) : 0.f;
#pragma unroll
      for (int a = 0; a < TN; ++a) s.tn[a] = SETUP ? __ldg(op.cs.t_nrm + (int64_t)~q * 3 + a) : 0.f;
    }
  };
  Stage st[AHEAD];
#pragma unroll
  for (int s = 0; s < AHEAD; ++s) {
    const int q = __shfl_sync(kAll, qa, s);
    if (b + s < e) load_stage(q, st[s]);
  }

  // per level: the current run's voxel, accumulators and x values, the x values of the next run (xn) and the nbr27
  // entry of the run after it (nn).  Bit l / 16 + l of req: they were requested (the run's start lay in the windows)
  int cur[MAXL], nn[MAXL];
  float acc[MAXL], accd[MAXL], xc[MAXL], xn[MAXL];
#pragma unroll
  for (int l = 0; l < MAXL; ++l) {
    cur[l] = -1; nn[l] = -1;
    acc[l] = 0.f; accd[l] = 0.f; xc[l] = 0.f; xn[l] = 0.f;
  }
  unsigned req = 0;
  unsigned first = 0xffffffffu;   // bit l: the current level-l run started at the item's first location
  auto nbr_of = [&](int l, int v) { return (v >= 0 && lane < 27) ? __ldg(svh.nbr27[l] + (int64_t)v * 27 + lane) : -1; };
  auto x_of = [&](int l, int nb) { return nb >= 0 ? __ldg(x + svh.offset[l] + nb) : 0.f; };

  // P[s][u] = acc through the warp's staging buffer, or the item's edge slot when u's run continues into the
  // previous or the next item
  auto flush = [&](int l, bool last) {
    const bool f = (first >> l) & 1u;
    const bool to_edge = (f && ((edge >> l) & 1u)) || (last && ((edge >> (16 + l)) & 1u));
    if (to_edge) {
      if (lane < 27) {
        const int64_t q = (((int64_t)it * op.edge_levels + (l - cut - 1)) * 2 + (f ? 0 : 1)) * 27 + lane;
        eb.e[q] = acc[l];
        if (SETUP) eb.d[q] = accd[l];
      }
    } else {
      if (lane < 27) {
        ps.v[ps.n * kStage + lane] = acc[l];
        if (SETUP) ps.d[ps.n * kStage + lane] = accd[l];
      }
      if (lane == 0) ps.g[ps.n] = svh.offset[l] + cur[l];
      if (++ps.n == 32) op_stage_drain<SETUP>(op, ps, lane);
    }
  };

  for (int k0 = b; k0 < e; k0 += 32) {
    const int nj = e - k0 < 32 ? e - k0 : 32;
    for (int j = 0; j < nj; ++j) {
      const int k = k0 + j;
      Stage nx;
      {
        const int ja = j + AHEAD;
        const int q = __shfl_sync(kAll, ja < 32 ? qa : qb, ja & 31);
        if (k + AHEAD < e) load_stage(q, nx);
      }

      // runs starting at this location: the finished run goes out, the new one's x values come in, and the next
      // two runs' x values and nbr27 rows are requested
#pragma unroll
      for (int l = 0; l < MAXL; ++l) {
        if (l < L && ((sa[l] >> j) & 1u)) {
          const int v = __shfl_sync(kAll, va[l], j);
          if (cur[l] >= 0) flush(l, false);
          if (k > b) first &= ~(1u << l);
          cur[l] = v;
          acc[l] = 0.f;
          accd[l] = 0.f;
          if (!SETUP) {
            xc[l] = v < 0 ? 0.f : ((req >> l) & 1u) ? xn[l] : x_of(l, nbr_of(l, v));
            uint64_t rest = ((uint64_t)sb[l] << 32 | sa[l]) & (~0ull << (j + 1));
            const int j1 = __ffsll((long long)rest) - 1;
            rest &= rest - 1;
            const int j2 = __ffsll((long long)rest) - 1;
            const int v1 = __shfl_sync(kAll, j1 < 32 ? va[l] : vb[l], j1 & 31);
            const int v2 = __shfl_sync(kAll, j2 < 32 ? va[l] : vb[l], j2 & 31);
            // the next run is the one whose nbr27 entry the previous run start requested, when it found it
            xn[l] = j1 < 0 ? 0.f : x_of(l, ((req >> (16 + l)) & 1u) ? nn[l] : nbr_of(l, v1));
            nn[l] = j2 < 0 ? -1 : nbr_of(l, v2);
            req = (req & ~(0x10001u << l)) | (j1 >= 0 ? 1u << l : 0u) | (j2 >= 0 ? 0x10000u << l : 0u);
          }
        }
      }

      // this location's rows: t = w E x, then acc += E t
      const Stage& cs = st[0];
      auto visit = [&](auto kind_tag) {
        constexpr int KIND = decltype(kind_tag)::value;
        constexpr int AX = KIND == kValue ? 1 : 3;
        const float w = KIND == kValue ? op.cs.w_pos : op.cs.w_nrm;
        float ev[MAXL][AX];   // zero on a level without containing voxel, and in lanes >= 27
#pragma unroll
        for (int l = 0; l < MAXL; ++l) {
          if (KIND == kCompact) {
            float e0 = 0.f, e1 = 0.f, e2 = 0.f;
            if (l < L) spline.grad_rows(cs.ln[l][0], inv_w0 * __int_as_float((127 - l) << 23), lane, e0, e1, e2);
            ev[l][0] = e0;
            ev[l][AX > 1 ? 1 : 0] = e1;
            ev[l][AX > 2 ? 2 : 0] = e2;
          } else {
#pragma unroll
            for (int a = 0; a < AX; ++a) ev[l][a] = cs.ln[l][a];
          }
        }
        float t[AX];
        if (SETUP) {
#pragma unroll
          for (int a = 0; a < AX; ++a) t[a] = KIND == kValue ? 0.f : w * cs.tn[a < TN ? a : 0];
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
      };
      if (cs.q >= 0) visit(std::integral_constant<int, kValue>());
      else visit(std::integral_constant<int, NKIND>());

#pragma unroll
      for (int s = 0; s + 1 < AHEAD; ++s) st[s] = st[s + 1];
      st[AHEAD - 1] = nx;
    }
    if (k0 + 32 < e) {   // slide the windows
      qa = qb;
#pragma unroll
      for (int l = 0; l < MAXL; ++l) { va[l] = vb[l]; sa[l] = sb[l]; }
      load_win(k0 + 64, qb, vb);
      starts_b();
    }
  }
#pragma unroll
  for (int l = 0; l < MAXL; ++l)
    if (l < L && cur[l] >= 0) flush(l, true);
}

template <int NKIND, int MAXL, bool SETUP>
// depth <= 4: at most 102 registers for the application (5 blocks per SM), 128 for the setup walk, which holds the
// diagonal's accumulators and buffer as well (4 blocks per SM)
__global__ void __launch_bounds__(kOpWarps * 32, MAXL <= 4 ? (SETUP ? 4 : 5) : 1)
k_op_walk(MfOperator op, const float* __restrict__ x, const int* __restrict__ done) {
  __shared__ float s_v[kOpWarps][SETUP ? 2 : 1][32 * kStage];
  __shared__ int64_t s_g[kOpWarps][32];
  if (done && *done) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  PStage ps{s_v[warp][0], SETUP ? s_v[warp][SETUP ? 1 : 0] : nullptr, s_g[warp], 0};
  // the warp's item index and bounds through redux.sync: warp-uniform values, and the compiler sees them as such
  const int n_items = (int)__reduce_max_sync(0xffffffffu, (unsigned)*op.n_items);
  const EdgeBuffers eb = op_edge_buffers(op);
  for (int it = (int)__reduce_max_sync(0xffffffffu, blockIdx.x * kOpWarps + warp); it < n_items;
       it += gridDim.x * kOpWarps) {
    const int4 item = op.items[it];
    op_walk_item<NKIND, MAXL, SETUP>(op, x, it,
                                     make_int4((int)__reduce_max_sync(0xffffffffu, (unsigned)item.x),
                                               (int)__reduce_max_sync(0xffffffffu, (unsigned)item.y),
                                               (int)__reduce_max_sync(0xffffffffu, (unsigned)item.z), 0),
                                     eb, ps, lane);
  }
  if (ps.n > 0) op_stage_drain<SETUP>(op, ps, lane);
}

// one warp per (item, level above the cut): a run that starts in the item and continues into the next ones is summed
// over its pieces in item order and stored to P once
template <bool SETUP>
__global__ void __launch_bounds__(kEdgeBlock) k_op_edges(MfOperator op, const int* __restrict__ done) {
  if (done && *done) return;
  const int NL = op.edge_levels;
  const int lane = threadIdx.x & 31;
  const int cut = op_cut_level(op.svh.depth);
  const int64_t units = (int64_t)*op.n_items * NL;
  const EdgeBuffers eb = op_edge_buffers(op);
  const int64_t stride = (int64_t)gridDim.x * (kEdgeBlock / 32);
  for (int64_t w = (blockIdx.x * (int64_t)kEdgeBlock + threadIdx.x) >> 5; w < units; w += stride) {
    const int it = (int)(w / NL), j = (int)(w % NL), l = cut + 1 + j;
    const int4 item = op.items[it];
    if (item.z & kItemLast) continue;
    const int32_t* v = op.vox + l * op.m;
    const int u = __ldg(v + item.y - 1);
    if (u < 0 || __ldg(v + item.y) != u) continue;                            // the item's last run ends in it
    const bool in_first = __ldg(v + item.x) == u;
    if (in_first && !(item.z & kItemFirst) && __ldg(v + item.x - 1) == u) continue;   // summed where it starts
    int64_t q = (((int64_t)it * NL + j) * 2 + (in_first ? 0 : 1)) * 27 + lane;
    float s = 0.f, sd = 0.f;
    if (lane < 27) {
      s = eb.e[q];
      if (SETUP) sd = eb.d[q];
    }
    for (int i = it + 1;; ++i) {
      const int4 nxt = op.items[i];
      q = (((int64_t)i * NL + j) * 2) * 27 + lane;
      if (lane < 27) {
        s += eb.e[q];
        if (SETUP) sd += eb.d[q];
      }
      if ((nxt.z & kItemLast) || __ldg(v + nxt.y) != u) break;
    }
    if (lane < 27) {
      const int64_t p = (int64_t)lane * op.n + op.svh.offset[l] + u;
      op.P[p] = s;
      if (SETUP) op.Pd[p] = sd;
    }
  }
}

// row g of y = sum_s P[s][nbr27(i)[26 - s]] + w_reg R x (SETUP: y = rhs from P, y2 = diag from Pd + w_reg R_ii)
template <bool SETUP>
__device__ __forceinline__ void op_apply_row(const nksr_svh_t& svh, const nksr_feat_t& feat, float w_reg,
                                             const float* __restrict__ P, const float* __restrict__ Pd,
                                             const float* __restrict__ x, int64_t n, int64_t g, float& y, float& y2) {
  const int C = feat.channels;
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
    y = s;
    y2 = sd;
  } else {
    y = s + reg;
  }
}

// one thread per unknown, grid-stride: y (and y2) of op_apply_row; pap != nullptr: pap[b] = block b's sum of x_i y_i
template <bool SETUP>
__global__ void __launch_bounds__(kApplyBlock)
k_op_apply(nksr_svh_t svh, nksr_feat_t feat, float w_reg, const float* __restrict__ P, const float* __restrict__ Pd,
           const float* __restrict__ x, float* __restrict__ y, float* __restrict__ y2, int64_t n,
           double* __restrict__ pap, const int* __restrict__ done) {
  __shared__ double sh[kApplyBlock / 32];
  if (done && *done) return;
  double local = 0.0;
  for (int64_t g = blockIdx.x * (int64_t)kApplyBlock + threadIdx.x; g < n; g += (int64_t)gridDim.x * kApplyBlock) {
    float yi, y2i;
    op_apply_row<SETUP>(svh, feat, w_reg, P, Pd, x, n, g, yi, y2i);
    y[g] = yi;
    if (SETUP) y2[g] = y2i;
    else if (pap) local += (double)yi * (double)__ldg(x + g);
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

// the distributed solve's step (x = u): w = A u on the rows with owned[g] != 0 (op_apply_row, the arithmetic of
// k_op_apply) and 0 on the others; dots[j * gridDim.x + block] = the block's sums over the owned rows of (r,u), (w,u),
// (r,r) for j = 0, 1, 2.  (4 blocks per SM caps it at 64 registers: without the cap ptxas held it at 40 and spilled
// the three accumulators)
__global__ void __launch_bounds__(kApplyBlock, 4)
k_op_apply_dcg(nksr_svh_t svh, nksr_feat_t feat, float w_reg, const float* __restrict__ P,
               const uint8_t* __restrict__ owned, const float* __restrict__ r, const float* __restrict__ u,
               float* __restrict__ w, int64_t n, double* __restrict__ dots, const int* __restrict__ done) {
  __shared__ double sh[3][kApplyBlock / 32];
  if (*done) return;
  double ru = 0.0, wu = 0.0, rr = 0.0;
  for (int64_t g = blockIdx.x * (int64_t)kApplyBlock + threadIdx.x; g < n; g += (int64_t)gridDim.x * kApplyBlock) {
    if (!__ldg(owned + g)) {
      w[g] = 0.f;
      continue;
    }
    float wi, unused;
    op_apply_row<false>(svh, feat, w_reg, P, nullptr, u, n, g, wi, unused);
    w[g] = wi;
    const double ri = (double)__ldg(r + g), ui = (double)__ldg(u + g);
    ru += ri * ui;
    wu += (double)wi * ui;
    rr += ri * ri;
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  ru = warp_sum_d(ru);
  wu = warp_sum_d(wu);
  rr = warp_sum_d(rr);
  if (lane == 0) { sh[0][wid] = ru; sh[1][wid] = wu; sh[2][wid] = rr; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double t0 = 0.0, t1 = 0.0, t2 = 0.0;
    for (int k = 0; k < kApplyBlock / 32; ++k) { t0 += sh[0][k]; t1 += sh[1][k]; t2 += sh[2][k]; }
    dots[blockIdx.x] = t0;
    dots[gridDim.x + blockIdx.x] = t1;
    dots[2 * gridDim.x + blockIdx.x] = t2;
  }
}

// ------------------------------------------------------------------------------- constraint values for the backward
// E_j x0 and E_j x1 at location j (KIND kValue: one value row; kCompact / kFull: the three gradient rows), read from the
// resident rows: one warp, lane = stencil slot.  Per level the containing voxel, then its nbr27 entry and the lines,
// then the x values of both vectors are requested for every level before any is used; each line is read once and
// serves both vectors.  A level without containing voxel contributes nothing.  The per-lane sums run over the levels in
// ascending order and are then reduced over the warp, the order of the walk's t_r: E_j x here is bitwise the walk's.
// out (2 x AX floats at j): the AX values of x0, then those of x1
template <int KIND, int MAXL>
__device__ __forceinline__ void op_location_values(const nksr_svh_t& svh, const float* __restrict__ rows,
                                                   const int32_t* __restrict__ base, int64_t nb, int64_t j,
                                                   const float* __restrict__ x0, const float* __restrict__ x1,
                                                   float* __restrict__ out, int lane) {
  constexpr int AX = KIND == kValue ? 1 : 3;
  constexpr int LINES = KIND == kFull ? 3 : 1;
  const int L = svh.depth;
  int v[MAXL];
#pragma unroll
  for (int l = 0; l < MAXL; ++l) v[l] = l < L ? __ldg(base + l * nb + j) : -1;
  const float* p = rows + j * L * LINES * NKSR_ROW_STRIDE + lane;
  int nbr[MAXL];
  float ln[MAXL][LINES];
#pragma unroll
  for (int l = 0; l < MAXL; ++l) {
    nbr[l] = (v[l] >= 0 && lane < 27) ? __ldg(svh.nbr27[l] + (int64_t)v[l] * 27 + lane) : -1;
#pragma unroll
    for (int a = 0; a < LINES; ++a) ln[l][a] = v[l] >= 0 ? __ldcs(p + (l * LINES + a) * NKSR_ROW_STRIDE) : 0.f;
  }
  float xa[MAXL], xb[MAXL];
#pragma unroll
  for (int l = 0; l < MAXL; ++l) {
    const int64_t g = nbr[l] >= 0 ? svh.offset[l] + nbr[l] : -1;
    xa[l] = g >= 0 ? __ldg(x0 + g) : 0.f;
    xb[l] = g >= 0 ? __ldg(x1 + g) : 0.f;
  }
  const int sl = lane < 27 ? lane : 13;
  const CompactSpline spline(c_d27[sl][0], c_d27[sl][1], c_d27[sl][2]);
  const float inv_w0 = 1.f / svh.voxel_size;
  float sa[AX], sb[AX];
#pragma unroll
  for (int a = 0; a < AX; ++a) sa[a] = sb[a] = 0.f;
#pragma unroll
  for (int l = 0; l < MAXL; ++l) {
    float ev[AX];
    if (KIND == kCompact) {
      float e0 = 0.f, e1 = 0.f, e2 = 0.f;
      if (l < L) spline.grad_rows(ln[l][0], inv_w0 * __int_as_float((127 - l) << 23), lane, e0, e1, e2);
      ev[0] = e0;
      ev[AX > 1 ? 1 : 0] = e1;
      ev[AX > 2 ? 2 : 0] = e2;
    } else {
#pragma unroll
      for (int a = 0; a < AX; ++a) ev[a] = ln[l][a < LINES ? a : 0];
    }
#pragma unroll
    for (int a = 0; a < AX; ++a) {
      sa[a] = fmaf(ev[a], xa[l], sa[a]);
      sb[a] = fmaf(ev[a], xb[l], sb[a]);
    }
  }
#pragma unroll
  for (int a = 0; a < AX; ++a) {
    sa[a] = warp_sum(sa[a]);
    sb[a] = warp_sum(sb[a]);
  }
  if (lane == 0) {
#pragma unroll
    for (int a = 0; a < AX; ++a) {
      out[a] = sa[a];
      out[AX + a] = sb[a];
    }
  }
}

// one warp per location: the sorted positions, then the sorted normal locations
template <int NKIND, int MAXL>
__global__ void __launch_bounds__(kApplyBlock)
k_op_constraint_values(nksr_svh_t svh, nksr_constraints_t cs, const int32_t* __restrict__ base_pos,
                       const int32_t* __restrict__ base_nrm, const float* __restrict__ x0,
                       const float* __restrict__ x1, float* __restrict__ out_pos, float* __restrict__ out_nrm) {
  const int lane = threadIdx.x & 31;
  const int64_t i = (blockIdx.x * (int64_t)kApplyBlock + threadIdx.x) >> 5;
  if (i < cs.n_pos) {
    op_location_values<kValue, MAXL>(svh, cs.e_pos, base_pos, cs.n_pos, i, x0, x1, out_pos + 2 * i, lane);
  } else if (i < cs.n_pos + cs.n_nrm) {
    const int64_t j = i - cs.n_pos;
    op_location_values<NKIND, MAXL>(svh, cs.e_nrm, base_nrm, cs.n_nrm, j, x0, x1, out_nrm + 6 * j, lane);
  }
}

// -------------------------------------------------------------------------------------------------------- host side
size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

int64_t op_unknowns(const nksr_svh_t& svh) { return svh.offset[svh.depth - 1] + svh.n[svh.depth - 1]; }

int edge_levels(const nksr_svh_t& svh) {
  const int cut = svh.depth - 1 < kCutLevel ? svh.depth - 1 : kCutLevel;
  return svh.depth - 1 - cut;
}

// workspace: P, Pd, the merged sequence and its voxels, top ranges, item counts and offsets, the item count, the
// owned-location filter's flags and the kept count, the scans' scratch (the fixed part), then as many items with their
// edge slots as the rest holds
struct OpLayout {
  size_t P, Pd, seq, vox, top, cnt, ofs, n_items, max_items, keep, n_kept, scan, scan_bytes, fixed;
  size_t per_item;   // item record + its edge slots (rhs and diagonal)
};

OpLayout op_layout(const nksr_svh_t& svh, int64_t m) {
  OpLayout o;
  const int64_t n = op_unknowns(svh), n_top = svh.n[svh.depth - 1];
  size_t top_scan = 0, keep_scan = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, top_scan, (const int32_t*)nullptr, (int32_t*)nullptr,
                                (int)(n_top > 0 ? n_top : 1));
  cub::DeviceScan::ExclusiveSum(nullptr, keep_scan, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(m + 1));
  o.scan_bytes = top_scan > keep_scan ? top_scan : keep_scan;
  size_t at = 0;
  auto take = [&](size_t bytes) { const size_t p = at; at += align256(bytes); return p; };
  o.P = take((size_t)27 * n * sizeof(float));
  o.Pd = take((size_t)27 * n * sizeof(float));
  o.seq = take((size_t)m * sizeof(int32_t));
  o.vox = take((size_t)svh.depth * m * sizeof(int32_t));
  o.top = take((size_t)n_top * sizeof(int2));
  o.cnt = take((size_t)n_top * sizeof(int32_t));
  o.ofs = take((size_t)n_top * sizeof(int32_t));
  o.n_items = take(sizeof(int32_t));
  o.max_items = take(sizeof(int64_t));
  o.keep = take((size_t)(m + 1) * sizeof(int32_t));
  o.n_kept = take(sizeof(int32_t));
  o.scan = take(o.scan_bytes);
  o.fixed = at;
  o.per_item = sizeof(int4) + 2 * (size_t)edge_levels(svh) * 2 * 27 * sizeof(float);
  return o;
}

// greedy items: two consecutive items of one top voxel hold more than S locations together
int64_t op_max_items(const nksr_svh_t& svh, int64_t m, int S) {
  return 2 * ((m + S - 1) / S) + svh.n[svh.depth - 1];
}

int sm_count() {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return 132;
  return sms > 0 ? sms : 132;
}

// resident blocks per SM of the walk kernel this operator launches
template <bool SETUP>
int walk_blocks_per_sm(const MfOperator& op) {
  const bool compact = op.cs.nrm_compact == 1, deep = op.svh.depth > 4;
  const void* f = deep ? (compact ? (const void*)k_op_walk<kCompact, NKSR_MAX_DEPTH, SETUP>
                                  : (const void*)k_op_walk<kFull, NKSR_MAX_DEPTH, SETUP>)
                       : (compact ? (const void*)k_op_walk<kCompact, 4, SETUP> : (const void*)k_op_walk<kFull, 4, SETUP>);
  int blocks = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, f, kOpWarps * 32, 0) != cudaSuccess || blocks < 1)
    blocks = 1;
  return blocks;
}

template <bool SETUP>
void walk_launch(const MfOperator& op, const float* x, const int* done, cudaStream_t s) {
  const bool compact = op.cs.nrm_compact == 1;
  // the setup walk, once per solve, has its own occupancy (see k_op_walk)
  const int grid = SETUP ? sm_count() * walk_blocks_per_sm<true>(op) : op.walk_grid;
#define NKSR_WALK(NK, ML) k_op_walk<NK, ML, SETUP><<<grid, kOpWarps * 32, 0, s>>>(op, x, done)
  if (op.svh.depth <= 4) {
    if (compact) NKSR_WALK(kCompact, 4); else NKSR_WALK(kFull, 4);
  } else {
    if (compact) NKSR_WALK(kCompact, NKSR_MAX_DEPTH); else NKSR_WALK(kFull, NKSR_MAX_DEPTH);
  }
#undef NKSR_WALK
  if (op.edge_levels > 0) k_op_edges<SETUP><<<op.edge_grid, kEdgeBlock, 0, s>>>(op, done);
}

bool op_valid(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c, const int32_t* base_pos,
              const int32_t* base_nrm) {
  if (!svh || !feat || !c || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH) return false;
  if (feat->channels < 1 || feat->channels > 32) return false;
  if (c->nrm_compact != 0 && c->nrm_compact != 1) return false;
  if (c->n_pos < 0 || c->n_nrm < 0 || c->n_pos + c->n_nrm >= INT32_MAX) return false;
  if (c->n_pos > 0 && (!c->e_pos || !base_pos)) return false;
  if (c->n_nrm > 0 && (!c->e_nrm || !c->t_nrm || !base_nrm)) return false;
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
  op.m = c->n_pos + c->n_nrm;
  const OpLayout o = op_layout(*svh, op.m);
  unsigned char* w = reinterpret_cast<unsigned char*>(ws);
  op.P = reinterpret_cast<float*>(w + o.P);
  op.Pd = reinterpret_cast<float*>(w + o.Pd);
  op.seq = reinterpret_cast<int32_t*>(w + o.seq);
  op.vox = reinterpret_cast<int32_t*>(w + o.vox);
  op.top = reinterpret_cast<int2*>(w + o.top);
  op.cnt = reinterpret_cast<int32_t*>(w + o.cnt);
  op.ofs = reinterpret_cast<int32_t*>(w + o.ofs);
  op.n_items = reinterpret_cast<int32_t*>(w + o.n_items);
  op.scan_tmp = w + o.scan;
  op.scan_bytes = o.scan_bytes;
  op.edge_levels = edge_levels(*svh);
  op.max_items = reinterpret_cast<int64_t*>(w + o.max_items);
  op.items = reinterpret_cast<int4*>(w + o.fixed);
  const int sms = sm_count();
  op.walk_grid = sms * walk_blocks_per_sm<false>(op);
  op.edge_grid = sms * 8;
  return op;
}

size_t workspace_bytes(const nksr_svh_t& svh, int64_t m, int item_size) {
  const OpLayout o = op_layout(svh, m);
  return o.fixed + (size_t)op_max_items(svh, m, item_size) * o.per_item + 768;
}

}  // namespace

int mf_operator_make(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                     const int32_t* base_pos, const int32_t* base_nrm, void* ws, size_t ws_bytes, MfOperator* out) {
  if (!op_valid(svh, feat, c, base_pos, base_nrm) || !ws || !out) return NKSR_E_INVALID;
  if (ws_bytes < op_layout(*svh, c->n_pos + c->n_nrm).fixed + 768) return NKSR_E_WORKSPACE;
  *out = make_op(svh, feat, c, base_pos, base_nrm, ws);
  return NKSR_OK;
}

int mf_apply_launch(const MfOperator& op, const float* x, float* y, double* pap, int blocks, const int* done,
                    cudaStream_t s) {
  walk_launch<false>(op, x, done, s);
  k_op_apply<false><<<blocks, kApplyBlock, 0, s>>>(op.svh, op.feat, op.cs.w_reg, op.P, nullptr, x, y, nullptr, op.n,
                                                   pap, done);
  return NKSR_OK;
}

int mf_dcg_launch(const MfOperator& op, const uint8_t* owned, const float* r, const float* u, float* w, double* dots,
                  int blocks, const int* done, cudaStream_t s) {
  walk_launch<false>(op, u, done, s);
  k_op_apply_dcg<<<blocks, kApplyBlock, 0, s>>>(op.svh, op.feat, op.cs.w_reg, op.P, owned, r, u, w, op.n, dots, done);
  return NKSR_OK;
}

extern "C" {

size_t nksr_op_workspace_bytes(const nksr_svh_t* svh, const nksr_constraints_t* c, int item_size) {
  if (!svh || !c || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH || item_size < 1) return 0;
  if (c->n_pos < 0 || c->n_nrm < 0) return 0;
  return workspace_bytes(*svh, c->n_pos + c->n_nrm, item_size);
}

int nksr_op_setup(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c, const int32_t* base_pos,
                  const int32_t* base_nrm, const int64_t* key_pos, const int64_t* key_nrm, const uint8_t* owned,
                  int item_size, float* rhs, float* diag, void* ws, size_t ws_bytes, void* stream) {
  if (!op_valid(svh, feat, c, base_pos, base_nrm) || !rhs || !diag || !ws || item_size < 1) return NKSR_E_INVALID;
  if ((c->n_pos > 0 && !key_pos) || (c->n_nrm > 0 && !key_nrm)) return NKSR_E_INVALID;
  const int64_t m = c->n_pos + c->n_nrm;
  if (ws_bytes < workspace_bytes(*svh, m, item_size)) return NKSR_E_WORKSPACE;
  cudaStream_t s = as_stream(stream);
  const MfOperator op = make_op(svh, feat, c, base_pos, base_nrm, ws);
  // every plane starts at zero (the voxels without locations are never written, here or by nksr_op_apply), and so do
  // the top ranges and the item count.  The tail holds as many items as fit; the kernels lay it out from the
  // capacity recorded here, so later applications need not be given the same workspace size
  const OpLayout o = op_layout(*svh, m);
  const int64_t max_items = (int64_t)((ws_bytes - o.fixed - 768) / o.per_item);
  if (cudaMemsetAsync(ws, 0, o.fixed, s) != cudaSuccess) return NKSR_E_CUDA;
  if (cudaMemcpyAsync(op.max_items, &max_items, sizeof(int64_t), cudaMemcpyHostToDevice, s) != cudaSuccess)
    return NKSR_E_CUDA;
  unsigned char* w = reinterpret_cast<unsigned char*>(ws);
  int32_t* keep = reinterpret_cast<int32_t*>(w + o.keep);
  int32_t* n_kept = reinterpret_cast<int32_t*>(w + o.n_kept);
  const int32_t m32 = (int32_t)m;
  if (!owned && cudaMemcpyAsync(n_kept, &m32, sizeof(int32_t), cudaMemcpyHostToDevice, s) != cudaSuccess)
    return NKSR_E_CUDA;
  const int64_t n_top = svh->n[svh->depth - 1];
  if (m > 0 && n_top > 0) {
    if (owned) {
      // the filter: flags, their exclusive scan in place over m + 1 entries (keep[m] = 0 from the clear, so keep[m]
      // becomes the kept count), and the vox entries past the kept ones read as "no voxel"
      k_op_keep<<<grid_for(m * 32, 256), 256, 0, s>>>(*svh, base_pos, c->n_pos, base_nrm, c->n_nrm, owned, keep);
      size_t kb = op.scan_bytes;
      if (cub::DeviceScan::ExclusiveSum(op.scan_tmp, kb, keep, keep, (int)(m + 1), s) != cudaSuccess)
        return NKSR_E_CUDA;
      if (cudaMemcpyAsync(n_kept, keep + m, sizeof(int32_t), cudaMemcpyDeviceToDevice, s) != cudaSuccess ||
          cudaMemsetAsync(op.vox, 0xff, (size_t)svh->depth * m * sizeof(int32_t), s) != cudaSuccess)
        return NKSR_E_CUDA;
    }
    k_op_merge<<<grid_for(m, 256), 256, 0, s>>>(key_pos, c->n_pos, key_nrm, c->n_nrm, base_pos, base_nrm, svh->depth,
                                               owned ? keep : nullptr, op.seq, op.vox);
    k_op_top_ranges<<<grid_for(m, 256), 256, 0, s>>>(op.vox + (int64_t)(svh->depth - 1) * m, m, op.top);
    const int cut = svh->depth - 1 < kCutLevel ? svh->depth - 1 : kCutLevel;
    const int grid = grid_for(n_top * 32, 256);
    k_op_cut<false><<<grid, 256, 0, s>>>(op.vox, m, op.top, n_top, cut, item_size, op.cnt, nullptr, nullptr, nullptr);
    size_t tb = op.scan_bytes;
    if (cub::DeviceScan::ExclusiveSum(op.scan_tmp, tb, op.cnt, op.ofs, (int)n_top, s) != cudaSuccess)
      return NKSR_E_CUDA;
    k_op_cut<true><<<grid, 256, 0, s>>>(op.vox, m, op.top, n_top, cut, item_size, nullptr, op.ofs, op.items,
                                        op.n_items);
    walk_launch<true>(op, nullptr, nullptr, s);
  }
  const int grid = grid_for(op.n, kApplyBlock);
  k_op_apply<true><<<grid, kApplyBlock, 0, s>>>(op.svh, op.feat, op.cs.w_reg, op.P, op.Pd, nullptr, rhs, diag, op.n,
                                                nullptr, nullptr);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_op_apply(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c, const int32_t* base_pos,
                  const int32_t* base_nrm, const float* x, float* y, void* ws, size_t ws_bytes, void* stream) {
  if (!op_valid(svh, feat, c, base_pos, base_nrm) || !x || !y || !ws) return NKSR_E_INVALID;
  MfOperator op;
  const int rc = mf_operator_make(svh, feat, c, base_pos, base_nrm, ws, ws_bytes, &op);
  if (rc != NKSR_OK) return rc;
  mf_apply_launch(op, x, y, nullptr, grid_for(op.n, kApplyBlock), nullptr, as_stream(stream));
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_op_constraint_values(const nksr_svh_t* svh, const nksr_constraints_t* c, const int32_t* base_pos,
                              const int32_t* base_nrm, const float* x0, const float* x1, float* out_pos,
                              float* out_nrm, void* stream) {
  if (!svh || !c || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH || !x0 || !x1) return NKSR_E_INVALID;
  if (c->nrm_compact != 0 && c->nrm_compact != 1) return NKSR_E_INVALID;
  if (c->n_pos < 0 || c->n_nrm < 0) return NKSR_E_INVALID;
  if (c->n_pos > 0 && (!c->e_pos || !base_pos || !out_pos)) return NKSR_E_INVALID;
  if (c->n_nrm > 0 && (!c->e_nrm || !base_nrm || !out_nrm)) return NKSR_E_INVALID;
  for (int l = 0; l < svh->depth; ++l)
    if (svh->n[l] > 0 && !svh->nbr27[l]) return NKSR_E_INVALID;
  const int64_t m = c->n_pos + c->n_nrm;
  if (m == 0) return NKSR_OK;
  const int grid = grid_for(m * 32, kApplyBlock);
  cudaStream_t s = as_stream(stream);
#define NKSR_VALUES(NK, ML) \
  k_op_constraint_values<NK, ML><<<grid, kApplyBlock, 0, s>>>(*svh, *c, base_pos, base_nrm, x0, x1, out_pos, out_nrm)
  if (svh->depth <= 4) {
    if (c->nrm_compact == 1) NKSR_VALUES(kCompact, 4); else NKSR_VALUES(kFull, 4);
  } else {
    if (c->nrm_compact == 1) NKSR_VALUES(kCompact, NKSR_MAX_DEPTH); else NKSR_VALUES(kFull, NKSR_MAX_DEPTH);
  }
#undef NKSR_VALUES
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_op_workspace_layout(const nksr_svh_t* svh, const nksr_constraints_t* c, size_t ws_bytes, int64_t* out) {
  if (!svh || !c || !out || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH || c->n_pos < 0 || c->n_nrm < 0)
    return NKSR_E_INVALID;
  const OpLayout o = op_layout(*svh, c->n_pos + c->n_nrm);
  if (ws_bytes < o.fixed + 768) return NKSR_E_WORKSPACE;
  out[0] = (int64_t)o.seq;
  out[1] = (int64_t)o.vox;
  out[2] = (int64_t)o.n_items;
  out[3] = (int64_t)o.fixed;
  out[4] = (int64_t)o.n_kept;
  return NKSR_OK;
}

}  // extern "C"
