// Gram-matrix fill, brick decomposition of the fine levels (the rows of the levels below the block split level).
//
// Same matrix, same CSR order as the row-per-warp kernel in assemble.cu (SPEC S6 / S6b).  What changes is the loop
// nest.  The row kernel streams, for every matrix row i, the constraint lines of each of the 27 voxels u around i, so
// every line is loaded once per active neighbour row (27 times in a dense region).  Here one block owns a BRICK of
// rows -- the level-l voxels that share key >> 3*LB, contiguous in Morton order -- with one accumulation tile per row
// in shared memory, indexed by structural slot exactly like the row kernel's tile.  The source voxels of the brick
// are the union of its rows' 27-neighbourhoods ((2^LB + 2)^3 positions); each source u is visited once per level
// offset k: its lines are loaded once and multiplied into every target row si of u inside the brick,
//     M_u[si][s] = sum over u's constraint rows (positions, then normals by axis) of  w E_l[si] * E_{l+k}[s]
// (lane = column s, the weighted level-l value staged in shared memory and read back as broadcasts, as in
// k_gram_blocks), only for the targets that are active rows of the brick -- so the FMA count is the row kernel's, and
// only the lines of the brick's halo are loaded by more than one block.
//
// Each M_u[si] is the per-(row, source) partial sum of the row kernel, the same operations in the same order.  The
// partials are flushed into the row tiles in 27 colour phases (local source coordinates mod 3 per axis) with a
// block barrier between phases: two sources of one colour never share a target row, so the flushes are plain
// shared-memory adds, without atomics.  A row therefore adds its 27 partials in phase order instead of the row
// kernel's neighbour order, and its rhs chain runs in the same phase order (carried in shared memory): the values
// differ from the row kernel's by the reassociation of those 27 terms, and are reproducible run to run.  The
// regulariser and the write-out (gram_common.cuh) are the row kernel's.
//
// Blocks are assigned fixed windows of 8^LB voxel indices and process the bricks that START in their window (a
// brick holds at most 8^LB voxels), so no brick list is stored and the schedule does not depend on the GPU.  The
// bricks of a window are consecutive runs of rows, and a block packs them greedily, in order, into batches of at most
// 8^LB rows (the tile), kBatchBricks bricks and a bound on their source voxels that fits the source list; setup, the
// 27 phases and the write-out run once per batch.  Each brick keeps its own local frame and colours: a source voxel
// in the halo of two bricks of a batch is two entries, each flushing only into its own brick's rows, so every row
// still adds its partials in the same phase order and the system is bitwise the one-brick-at-a-time schedule's.
//
// Inside an item (one source, one level offset) a warp streams the source's constraint lines through a ring of
// kLineRing locations in shared memory with cp.async: location q is multiplied in while the lines of the next three
// are on their way, without holding them in registers (one location ahead in registers was what the item loop could
// afford, and the items are chains of dependent line loads).  The values and their order are unchanged.
//
// Measured per level on the benchmark system (H100 SXM at 700 W, DESIGN.md 4.1): the brick fill wins where a voxel
// owns many constraint locations (level 2: 18 per voxel, 44 ms against 90 ms for the row kernel) and loses where it
// owns few (level 1, 4.9 per voxel: 112 against 83 ms; level 0, 1.7 per voxel, where tiles and rings leave room for
// one block per SM: 454 against 105 ms).  So a level is bricked only when it holds at least `min_locations_per_voxel`
// constraint locations per voxel, the row kernel fills the others.
#include "gram_common.cuh"

namespace {

constexpr int kBrickWarps = 8;
// brick = the level-l descendants of one level-(l+2) key: 4^3 rows (bricks of 2^3 rows were measured 2.1x slower)
constexpr int kBrickLog2 = 2;
// bricks in one batch, at most (the brick index of a source entry takes 4 bits)
constexpr int kBatchBricks = 16;
// locations whose lines a warp has in flight: each location's lines are copied into a per-warp ring of shared memory
// (cp.async, no registers held) kLineRing - 1 locations ahead of the one being multiplied in
constexpr int kLineRing = 4;
// one ring slot: level l and level l + k of the three lines of a location (one for a position) per lane, and the
// location's three normal targets
constexpr int kSlotWords = 6 * 32 + 4;
// dynamic shared memory per block that leaves room for two blocks per SM (228 KB per SM, 1 KB reserved per block, a
// few static words), and for one
constexpr size_t kTwoBlockSmemBytes = (size_t)113 * 1024 - 64;
constexpr size_t kOneBlockSmemBytes = (size_t)227 * 1024 - 64;

template <int LB>
struct Brick {
  static constexpr int S = 1 << LB;               // rows per axis
  static constexpr int NB = S * S * S;            // rows per brick, and per batch, at most
  static constexpr int R = S + 2;                 // source voxels per axis
  static constexpr int NS = R * R * R;
  static_assert(NB <= 64 && NS <= 256, "the start mask holds 64 rows, a row map entry a signed char, a source "
                                       "position 8 bits");
  // one source entry: ranges int4 | target mask | brick and position u16 | its place in the phase order u16
  static constexpr size_t kSourceBytes = sizeof(int4) + sizeof(unsigned) + 2 * sizeof(unsigned short);
  // shared-memory words beside the source list: tiles [NB][ts] | rhs [NB] | row maps [kBatchBricks][NB] bytes |
  // brick origins int4 [kBatchBricks] | phase counts, offsets, cursors [3][32] | per warp: 3 staged lines + target
  // list [4][32] + line ring [kLineRing][kSlotWords]
  static constexpr int kWarpWords = 128 + kLineRing * kSlotWords;
  static constexpr size_t fixed_words(int ts) {
    return (size_t)NB * ts + NB + kBatchBricks * NB / 4 + 4 * kBatchBricks + 3 * 32 + kBrickWarps * kWarpWords;
  }
  static constexpr size_t words(int ts, int cap) { return fixed_words(ts) + (size_t)cap * kSourceBytes / 4; }
};

// m[j] += st[j] * ek for the nt compacted targets j (four per broadcast 128-bit load)
__device__ __forceinline__ void brick_fma(float (&m)[28], const float* __restrict__ st, const float ek, const int nt) {
  const float4* s4 = reinterpret_cast<const float4*>(st);
#pragma unroll
  for (int j = 0; j < 7; ++j) {
    if (4 * j < nt) {
      const float4 a = s4[j];
      m[4 * j] = fmaf(a.x, ek, m[4 * j]);
      m[4 * j + 1] = fmaf(a.y, ek, m[4 * j + 1]);
      m[4 * j + 2] = fmaf(a.z, ek, m[4 * j + 2]);
      m[4 * j + 3] = fmaf(a.w, ek, m[4 * j + 3]);
    }
  }
}

__device__ __forceinline__ void cp_async4(float* dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// request into ring slot `slot` this lane's level-l value (word lane) and, for k > 0, level-(l + k) value (word
// 32 + lane) of the position row of location q
template <bool ILV>
__device__ __forceinline__ void brick_issue_pos(const nksr_constraints_t& cs, int q, int L, int l, int k, int lane,
                                                float* slot) {
  const float* p0 = ILV ? cs.e_pos + ((int64_t)q * NKSR_ROW_STRIDE + lane) * 4 + l
                        : cs.e_pos + ((int64_t)q * L + l) * NKSR_ROW_STRIDE + lane;
  cp_async4(slot + lane, p0);
  if (k) cp_async4(slot + 32 + lane, p0 + (ILV ? k : k * NKSR_ROW_STRIDE));
}

// the same for the three gradient rows of normal location q (level l at word ax * 32 + lane, level l + k at
// (3 + ax) * 32 + lane), and, for k = 0, its three targets (words 192..194, one lane each)
template <bool ILV>
__device__ __forceinline__ void brick_issue_nrm(const nksr_constraints_t& cs, int q, int L, int l, int k, int lane,
                                                float* slot) {
#pragma unroll
  for (int ax = 0; ax < 3; ++ax) {
    const float* p0 = ILV ? cs.e_nrm + (((int64_t)q * 3 + ax) * NKSR_ROW_STRIDE + lane) * 4 + l
                          : cs.e_nrm + (((int64_t)q * L + l) * 3 + ax) * NKSR_ROW_STRIDE + lane;
    cp_async4(slot + ax * 32 + lane, p0);
    if (k) cp_async4(slot + (3 + ax) * 32 + lane, p0 + (ILV ? k : k * 3 * NKSR_ROW_STRIDE));
  }
  if (k == 0 && lane < 3) cp_async4(slot + 192 + lane, cs.t_nrm + (int64_t)q * 3 + lane);
}

// ILV: rows in the interleaved layout (four levels of a slot per float4); else one line per (location, level, axis)
template <int LB, bool ILV>
__global__ void __launch_bounds__(kBrickWarps * 32, 2)
k_gram_fill_brick(const nksr_svh_t svh, const nksr_feat_t feat, const nksr_constraints_t cs, const int l,
                  const int cap, const int32_t* __restrict__ cnt, const int64_t* __restrict__ rowptr,
                  int32_t* __restrict__ col_out, float* __restrict__ val_out, float* __restrict__ rhs,
                  float* __restrict__ diag, const nksr_placement_t place) {
  using B = Brick<LB>;
  extern __shared__ __align__(16) float smem[];
  __shared__ unsigned s_starts[2];
  __shared__ int s_nsrc;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int L = svh.depth, nup = L - 1 - l, nlev = nup + 1;
  const int ts = (125 + 64 * nup + 3) & ~3;
  int4* rng = reinterpret_cast<int4*>(smem);
  float* tile = reinterpret_cast<float*>(rng + cap);
  float* brhs = tile + B::NB * ts;
  unsigned* smask = reinterpret_cast<unsigned*>(brhs + B::NB);
  unsigned short* smeta = reinterpret_cast<unsigned short*>(smask + cap);
  unsigned short* order = smeta + cap;
  signed char* posmap = reinterpret_cast<signed char*>(order + cap);
  int4* borig = reinterpret_cast<int4*>(posmap + kBatchBricks * B::NB);
  int* pcnt = reinterpret_cast<int*>(borig + kBatchBricks);
  int* poff = pcnt + 32;
  int* pcur = poff + 32;
  float* stage = reinterpret_cast<float*>(pcur + 32) + wid * B::kWarpWords;
  int* tlist = reinterpret_cast<int*>(stage + 96);
  float* ring = stage + 128;

  const int64_t nl = svh.n[l];
  const int64_t* keys = svh.keys[l];
  const int64_t w0 = (int64_t)blockIdx.x * B::NB;
  if (wid < 2) {
    const int64_t i = w0 + tid;
    const bool st = tid < B::NB && i < nl &&
                    (i == 0 || (__ldg(keys + i) >> (3 * LB)) != (__ldg(keys + i - 1) >> (3 * LB)));
    const unsigned bal = __ballot_sync(0xffffffffu, st);
    if (lane == 0) s_starts[wid] = bal;
  }
  __syncthreads();
  uint64_t starts = s_starts[0] | ((uint64_t)s_starts[1] << 32);
  if (!starts) return;
  // rows of the window's last brick, which may run past the window (the others end where the next one starts)
  const int last = 63 - __clzll((long long)starts);
  int nlast;
  {
    const int64_t lkey = __ldg(keys + w0 + last) >> (3 * LB);
    int in = 0;
    if (tid < B::NB) {
      const int64_t i = w0 + last + tid;
      in = i < nl && (__ldg(keys + i) >> (3 * LB)) == lkey;
    }
    nlast = __syncthreads_count(in);
  }
  const int32_t* rp = cs.range_pos ? cs.range_pos + 2 * svh.offset[l] : nullptr;
  const int32_t* rn = cs.range_nrm ? cs.range_nrm + 2 * svh.offset[l] : nullptr;
  // this lane's stencil offset as slot increments of the same-level box and of a coarser level's 4^3 box
  const int sl = lane < 27 ? lane : 13;
  const int lane_l0 = c_d27[sl][0] * 25 + c_d27[sl][1] * 5 + c_d27[sl][2];
  const int lane_lk = c_d27[sl][0] * 16 + c_d27[sl][1] * 4 + c_d27[sl][2];

  while (starts) {
    // ---- the batch: consecutive bricks, taken greedily while their rows fit the tiles and the bound on their
    // sources (a brick of n rows has at most min(6^3, 27 n)) fits the source list.  Its rows are one run of voxel
    // indices [b0, b0 + nrows); this thread's batch row tid belongs to brick my_brick, which starts at row my_first.
    const int64_t b0 = w0 + (__ffsll((long long)starts) - 1);
    int nb = 0, nrows = 0, nsrc = 0, my_brick = -1, my_first = 0;
    while (starts && nb < kBatchBricks) {
      const int s0 = __ffsll((long long)starts) - 1;
      const uint64_t rest = starts & (starts - 1);
      const int n = rest ? (__ffsll((long long)rest) - 1) - s0 : nlast;
      const int ns = min(B::NS, 27 * n);
      if (nrows + n > B::NB || nsrc + ns > cap) break;
      if (tid >= nrows && tid < nrows + n) { my_brick = nb; my_first = nrows; }
      nrows += n;
      nsrc += ns;
      ++nb;
      starts = rest;
    }

    // ---- reset the tiles, map the batch's rows and collect its source voxels
    for (int t = tid; t < nb * B::NB / 4; t += blockDim.x) reinterpret_cast<int*>(posmap)[t] = -1;
    for (int t = tid; t < nrows * ts / 4; t += blockDim.x)
      reinterpret_cast<float4*>(tile)[t] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int t = tid; t < nrows; t += blockDim.x) brhs[t] = 0.f;
    if (tid < 32) pcnt[tid] = 0;
    if (tid == 0) s_nsrc = 0;
    __syncthreads();
    if (tid < nrows) {
      int x, y, z;
      morton3_decode(__ldg(keys + b0 + tid), x, y, z);
      const int bx = (x >> LB) << LB, by = (y >> LB) << LB, bz = (z >> LB) << LB;
      posmap[my_brick * B::NB + (((x - bx) * B::S) + (y - by)) * B::S + (z - bz)] = (signed char)tid;
      if (tid == my_first) borig[my_brick] = make_int4(bx, by, bz, 0);
    }
    __syncthreads();
    // per halo position of every brick: the mask of its target slots si that are rows of that brick; the source
    // voxel (a neighbour of any of those rows), its constraint-row ranges, and an entry when it has constraint rows
    for (int t = tid; t < nb * B::NS; t += blockDim.x) {
      const int j = t / B::NS, pos = t - j * B::NS;
      const signed char* pm = posmap + j * B::NB;
      const int lx = pos / (B::R * B::R) - 1, ly = (pos / B::R) % B::R - 1, lz = pos % B::R - 1;
      unsigned m = 0u;
      int row = -1, srow = 0;
      for (int s = 0; s < 27; ++s) {
        const int rx = lx + c_d27[s][0], ry = ly + c_d27[s][1], rz = lz + c_d27[s][2];
        if (rx >= 0 && rx < B::S && ry >= 0 && ry < B::S && rz >= 0 && rz < B::S) {
          const int r = pm[(rx * B::S + ry) * B::S + rz];
          if (r >= 0) {
            m |= 1u << s;
            if (row < 0) { row = r; srow = s; }
          }
        }
      }
      if (!m) continue;
      const int v = __ldg(svh.nbr27[l] + (b0 + row) * 27 + (26 - srow));    // offset -d(srow) from that row
      if (v < 0) continue;
      int4 r4 = make_int4(0, 0, 0, 0);
      if (rp) { const int2 a = __ldg(reinterpret_cast<const int2*>(rp) + v); r4.x = a.x; r4.y = a.y; }
      if (rn) { const int2 a = __ldg(reinterpret_cast<const int2*>(rn) + v); r4.z = a.x; r4.w = a.y; }
      if (!(r4.x < r4.y || r4.z < r4.w)) continue;
      const int e = atomicAdd(&s_nsrc, 1);        // < cap: the batch was cut by the bound on its sources
      rng[e] = r4;
      smask[e] = m;
      smeta[e] = (unsigned short)(j << 8 | pos);
      atomicAdd(&pcnt[((lx + 1) % 3) * 9 + ((ly + 1) % 3) * 3 + (lz + 1) % 3], 1);
    }
    __syncthreads();
    // colour phases: the sources whose brick-local coordinates are (cx,cy,cz) mod 3.  Two sources of one colour
    // never share a target row, so the order of a phase's items changes no value.
    if (wid == 0) {
      const int c = lane < 27 ? pcnt[lane] : 0;
      int incl = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      poff[lane] = incl - c;
      pcur[lane] = incl - c;
    }
    __syncthreads();
    for (int e = tid; e < s_nsrc; e += blockDim.x) {
      const int pos = smeta[e] & 255;
      const int p = ((pos / (B::R * B::R)) % 3) * 9 + (((pos / B::R) % B::R) % 3) * 3 + (pos % B::R) % 3;
      order[atomicAdd(&pcur[p], 1)] = (unsigned short)e;
    }
    __syncthreads();

    for (int p = 0; p < 27; ++p) {
      const int nitems = pcnt[p] * nlev;
      if (!nitems) continue;                      // (uniform: nothing to order)
      const int o0 = poff[p];
      for (int it = wid; it < nitems; it += kBrickWarps) {
        // ---- one (source u, level offset k): lane s < 27 is target slot s of u when bit s of the mask is set
        const int e = order[o0 + it / nlev], k = it % nlev;
        const unsigned tm = smask[e];
        const int nt = __popc(tm);
        const int4 r4 = rng[e];
        const int meta = smeta[e], pos = meta & 255;
        const signed char* pm = posmap + (meta >> 8) * B::NB;
        const int4 bo = borig[meta >> 8];
        const int lx = pos / (B::R * B::R) - 1, ly = (pos / B::R) % B::R - 1, lz = pos % B::R - 1;  // brick-local
        const bool mine = lane < 27 && ((tm >> lane) & 1u);
        const int rank = __popc(tm & ((1u << lane) - 1u));
        int trow = 0;
        float b = 0.f;
        __syncwarp();
        if (mine) {
          tlist[rank] = lane;
          trow = pm[((lx + c_d27[lane][0]) * B::S + ly + c_d27[lane][1]) * B::S + lz + c_d27[lane][2]];
          if (k == 0) b = brhs[trow];
        }
        float m[28];
#pragma unroll
        for (int j = 0; j < 28; ++j) m[j] = 0.f;
        // (location q is multiplied in while the lines of the next kLineRing - 1 locations are on their way; one
        // commit group per location, empty past the end, so that wait_group counts locations)
        const int npos = r4.y - r4.x;
#pragma unroll
        for (int d = 0; d < kLineRing - 1; ++d) {
          if (d < npos) brick_issue_pos<ILV>(cs, r4.x + d, L, l, k, lane, ring + d * kSlotWords);
          cp_async_commit();
        }
        for (int i = 0; i < npos; ++i) {
          if (i + kLineRing - 1 < npos)
            brick_issue_pos<ILV>(cs, r4.x + i + kLineRing - 1, L, l, k, lane,
                                 ring + ((i + kLineRing - 1) % kLineRing) * kSlotWords);
          cp_async_commit();
          cp_async_wait<kLineRing - 1>();
          const float* sl = ring + (i % kLineRing) * kSlotWords;
          const float e0 = sl[lane], ek = k == 0 ? e0 : sl[32 + lane];
          __syncwarp();
          if (mine) stage[rank] = cs.w_pos * e0;
          __syncwarp();
          brick_fma(m, stage, ek, nt);
        }
        const int nnrm = r4.w - r4.z;
#pragma unroll
        for (int d = 0; d < kLineRing - 1; ++d) {
          if (d < nnrm) brick_issue_nrm<ILV>(cs, r4.z + d, L, l, k, lane, ring + d * kSlotWords);
          cp_async_commit();
        }
        for (int i = 0; i < nnrm; ++i) {
          if (i + kLineRing - 1 < nnrm)
            brick_issue_nrm<ILV>(cs, r4.z + i + kLineRing - 1, L, l, k, lane,
                                 ring + ((i + kLineRing - 1) % kLineRing) * kSlotWords);
          cp_async_commit();
          cp_async_wait<kLineRing - 1>();
          const float* sl = ring + (i % kLineRing) * kSlotWords;
          __syncwarp();                              // (the targets were copied by lanes 0..2)
#pragma unroll
          for (int ax = 0; ax < 3; ++ax) {
            const float el = cs.w_nrm * sl[ax * 32 + lane];
            if (mine) {
              if (k == 0) b = fmaf(el, sl[192 + ax], b);
              stage[ax * 32 + rank] = el;
            }
          }
          __syncwarp();
#pragma unroll
          for (int ax = 0; ax < 3; ++ax) brick_fma(m, stage + ax * 32, k == 0 ? sl[ax * 32 + lane] : sl[(3 + ax) * 32 + lane], nt);
        }
        if (mine && k == 0) brhs[trow] = b;
        __syncwarp();
        // ---- flush into the target rows' tiles: the slot of column u + d(lane) in row i = u + d(si) is the row
        // kernel's base of the source (d(u - i) = -d(si)) plus the lane constant
        const int ux = bo.x + lx, uy = bo.y + ly, uz = bo.z + lz;       // source voxel, absolute
#pragma unroll
        for (int j = 0; j < 27; ++j) {
          if (j < nt) {
            const int si = tlist[j];
            const int dx = c_d27[si][0], dy = c_d27[si][1], dz = c_d27[si][2];
            const int r = pm[((lx + dx) * B::S + ly + dy) * B::S + lz + dz];
            int base;
            if (k == 0) {
              base = 62 - (dx * 25 + dy * 5 + dz) + lane_l0;
            } else {
              const int gx = ux + dx, gy = uy + dy, gz = uz + dz;   // row voxel, absolute
              const int ox = (ux >> k) - (((gx - 1) >> k) - 1), oy = (uy >> k) - (((gy - 1) >> k) - 1),
                        oz = (uz >> k) - (((gz - 1) >> k) - 1);
              base = 125 + 64 * (k - 1) + (ox << 4) + (oy << 2) + oz + lane_lk;
            }
            if (lane < 27) tile[r * ts + base] += m[j];
          }
        }
      }
      __syncthreads();
    }

    // ---- regulariser and write-out, one warp per row
    for (int r = wid; r < nrows; r += kBrickWarps) {
      const int i = (int)(b0 + r);
      const int64_t row = svh.offset[l] + i;
      RowGeom g;
      row_geom(svh, l, i, g);
      const int my_u = lane < 27 ? __ldg(svh.nbr27[l] + (int64_t)i * 27 + lane) : -1;
      float* acc = tile + r * ts;
      gram_row_regulariser(feat, cs, l, i, my_u, lane, acc);
      __syncwarp();
      gram_row_writeout<4>(svh, l, i, row, g, acc, cnt, rowptr, col_out, val_out, diag, place, lane);
      if (lane == 0) rhs[row] = brhs[r];
    }
    __syncthreads();
  }
}

template <int LB, bool ILV>
int launch_brick_level(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c, int l,
                       const int32_t* cnt, const int64_t* rowptr, const nksr_placement_t& place, int32_t* col, float* val,
                       float* rhs, float* diag, cudaStream_t s) {
  using B = Brick<LB>;
  const int ts = (125 + 64 * (svh->depth - 1 - l) + 3) & ~3;
  // the source list takes what two blocks per SM leave beside the tiles (one block on level 0 of a depth-4
  // hierarchy, whose tiles and line rings leave too little), up to the most a batch can need
  const size_t fixed = B::fixed_words(ts) * sizeof(float);
  const size_t budget = fixed + B::NS * B::kSourceBytes <= kTwoBlockSmemBytes ? kTwoBlockSmemBytes : kOneBlockSmemBytes;
  const size_t room = (budget - fixed) / B::kSourceBytes;
  const int cap = (int)(room < (size_t)27 * B::NB ? room : (size_t)27 * B::NB) & ~3;
  if (cap < B::NS) return NKSR_E_INVALID;
  const size_t smem = B::words(ts, cap) * sizeof(float);
  if (cudaFuncSetAttribute(k_gram_fill_brick<LB, ILV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
      cudaSuccess)
    return NKSR_E_CUDA;
  k_gram_fill_brick<LB, ILV><<<grid_for(svh->n[l], B::NB), kBrickWarps * 32, smem, s>>>(
      *svh, *feat, *c, l, cap, cnt, rowptr, col, val, rhs, diag, place);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // namespace

extern "C" {

int nksr_gram_fill_brick(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c,
                         const int32_t* cnt, const int64_t* rowptr, const nksr_placement_t* placement, int32_t* col,
                         float* val, float* rhs, float* diag, float min_locations_per_voxel, void* stream) {
  if (!svh || !feat || !c || !placement || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH) return NKSR_E_INVALID;
  if (!(min_locations_per_voxel >= 0.f)) return NKSR_E_INVALID;
  // compact gradient rows and hierarchies deeper than 4 levels: the row fill on every row
  const int nb = (c->nrm_compact == 1 || svh->depth > 4) ? 0 : (c->split_level < svh->depth ? c->split_level : svh->depth);
  if (nb < 0) return NKSR_E_INVALID;
  cudaStream_t s = as_stream(stream);
  const double locations = (double)c->n_pos + (double)c->n_nrm;
  for (int l = 0; l < nb; ++l) {
    if (svh->n[l] == 0) continue;
    if (locations < (double)min_locations_per_voxel * (double)svh->n[l]) {   // sparse level: the row fill
      const int rc = nksr_gram_fill_placed_rows(svh, feat, c, cnt, rowptr, placement, svh->offset[l],
                                                svh->offset[l] + svh->n[l], col, val, rhs, diag, stream);
      if (rc != NKSR_OK) return rc;
      continue;
    }
    const int rc =
        c->nrm_compact == 2
            ? launch_brick_level<kBrickLog2, true>(svh, feat, c, l, cnt, rowptr, *placement, col, val, rhs, diag, s)
            : launch_brick_level<kBrickLog2, false>(svh, feat, c, l, cnt, rowptr, *placement, col, val, rhs, diag, s);
    if (rc != NKSR_OK) return rc;
  }
  const int64_t n = svh->offset[svh->depth - 1] + svh->n[svh->depth - 1];
  const int64_t rest = nb < svh->depth ? svh->offset[nb] : n;
  return nksr_gram_fill_placed_rows(svh, feat, c, cnt, rowptr, placement, rest, n, col, val, rhs, diag, stream);
}

}  // extern "C"
