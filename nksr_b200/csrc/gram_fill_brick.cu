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
// brick holds at most 8^LB voxels), so no brick list is stored and the schedule does not depend on the GPU.
//
// Measured per level on the benchmark system (H100 SXM at a 400 W power limit, DESIGN.md 4.1): the brick fill wins
// where a voxel owns many constraint locations (level 2: 18 per voxel, 75 ms against 99 ms for the row kernel) and loses
// where it owns one or two (level 0: 302 against 125 ms; level 1, about 5 per voxel: 148 against 98 ms).  Its 27 phases
// run one after another, each a chain of dependent loads, and a sparse level gives them too little work to hide that:
// so a level is bricked only when it holds at least `min_locations_per_voxel` constraint locations per voxel, the row
// kernel fills the others.
#include "gram_common.cuh"

namespace {

constexpr int kBrickWarps = 8;
// brick = the level-l descendants of one level-(l+2) key: 4^3 rows (bricks of 2^3 rows were measured 2.1x slower)
constexpr int kBrickLog2 = 2;

template <int LB>
struct Brick {
  static constexpr int S = 1 << LB;               // rows per axis
  static constexpr int NB = S * S * S;            // rows per brick, at most
  static constexpr int R = S + 2;                 // source voxels per axis
  static constexpr int NS = R * R * R;
  static constexpr int NC = (R + 2) / 3;          // sources of one colour per axis, at most
  static_assert(NC * NC * NC <= 8 && NB <= 64, "phase lists hold 8 sources, the start mask 64 rows");
  // shared-memory words: ranges int4[NS] | tiles [NB][ts] | rhs [NB] | posmap [NB] | row coords [NB] | sources [NS] |
  // target masks [NS] | phase lists [27][8] + counts [32] | per warp: 3 staged lines + target list [4][32]
  static constexpr size_t words(int ts) {
    return (size_t)4 * NS + (size_t)NB * ts + 3 * NB + 2 * NS + 27 * 8 + 32 + kBrickWarps * 128;
  }
};

__device__ __forceinline__ float level_of(const float4& v, const int c) {
  return c == 0 ? v.x : (c == 1 ? v.y : (c == 2 ? v.z : v.w));
}

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

// level l (e0) and level l + k (ek) of this lane's slot in the position row of location q
template <bool ILV>
__device__ __forceinline__ void brick_load_pos(const nksr_constraints_t& cs, int q, int L, int l, int k, int lane,
                                               float& e0, float& ek) {
  if (ILV) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(cs.e_pos) + (int64_t)q * NKSR_ROW_STRIDE + lane);
    e0 = level_of(v, l);
    ek = level_of(v, l + k);
  } else {
    const float* p0 = cs.e_pos + ((int64_t)q * L + l) * NKSR_ROW_STRIDE + lane;
    e0 = __ldg(p0);
    ek = k == 0 ? e0 : __ldg(p0 + k * NKSR_ROW_STRIDE);
  }
}

// the same for the three gradient rows of normal location q
template <bool ILV>
__device__ __forceinline__ void brick_load_nrm(const nksr_constraints_t& cs, int q, int L, int l, int k, int lane,
                                               float (&e0)[3], float (&ek)[3]) {
#pragma unroll
  for (int ax = 0; ax < 3; ++ax) {
    if (ILV) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(cs.e_nrm) + ((int64_t)q * 3 + ax) * NKSR_ROW_STRIDE + lane);
      e0[ax] = level_of(v, l);
      ek[ax] = level_of(v, l + k);
    } else {
      const float* p0 = cs.e_nrm + (((int64_t)q * L + l) * 3 + ax) * NKSR_ROW_STRIDE + lane;
      e0[ax] = __ldg(p0);
      ek[ax] = k == 0 ? e0[ax] : __ldg(p0 + k * 3 * NKSR_ROW_STRIDE);
    }
  }
}

// ILV: rows in the interleaved layout (four levels of a slot per float4); else one line per (location, level, axis)
template <int LB, bool ILV>
__global__ void __launch_bounds__(kBrickWarps * 32)
k_gram_fill_brick(const nksr_svh_t svh, const nksr_feat_t feat, const nksr_constraints_t cs, const int l,
                  const int32_t* __restrict__ cnt, const int64_t* __restrict__ rowptr, int32_t* __restrict__ col_out,
                  float* __restrict__ val_out, float* __restrict__ rhs, float* __restrict__ diag,
                  const PlaceArg<true> place) {
  using B = Brick<LB>;
  extern __shared__ __align__(16) float smem[];
  __shared__ unsigned s_starts[2];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int L = svh.depth, nup = L - 1 - l, nlev = nup + 1;
  const int ts = (125 + 64 * nup + 3) & ~3;
  int4* rng = reinterpret_cast<int4*>(smem);
  float* tile = reinterpret_cast<float*>(rng + B::NS);
  float* brhs = tile + B::NB * ts;
  int* posmap = reinterpret_cast<int*>(brhs + B::NB);
  int* rloc = posmap + B::NB;
  int* src = rloc + B::NB;
  unsigned* tmask = reinterpret_cast<unsigned*>(src + B::NS);
  int* plist = reinterpret_cast<int*>(tmask + B::NS);
  int* pcnt = plist + 27 * 8;
  float* stage = reinterpret_cast<float*>(pcnt + 32) + wid * 128;
  int* tlist = reinterpret_cast<int*>(stage + 96);

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
  const int32_t* rp = cs.range_pos ? cs.range_pos + 2 * svh.offset[l] : nullptr;
  const int32_t* rn = cs.range_nrm ? cs.range_nrm + 2 * svh.offset[l] : nullptr;
  // this lane's stencil offset as slot increments of the same-level box and of a coarser level's 4^3 box
  const int sl = lane < 27 ? lane : 13;
  const int lane_l0 = c_d27[sl][0] * 25 + c_d27[sl][1] * 5 + c_d27[sl][2];
  const int lane_lk = c_d27[sl][0] * 16 + c_d27[sl][1] * 4 + c_d27[sl][2];

  while (starts) {
    const int64_t first = w0 + (__ffsll((long long)starts) - 1);
    starts &= starts - 1;
    const int64_t bkey = __ldg(keys + first) >> (3 * LB);
    int in = 0;
    if (tid < B::NB) {
      const int64_t i = first + tid;
      in = i < nl && (__ldg(keys + i) >> (3 * LB)) == bkey;
    }
    const int nrows = __syncthreads_count(in);
    int bx, by, bz;
    morton3_decode(bkey, bx, by, bz);
    bx <<= LB; by <<= LB; bz <<= LB;

    // ---- reset the tiles, map the brick's rows and collect its source voxels
    for (int t = tid; t < B::NB; t += blockDim.x) posmap[t] = -1;
    for (int t = tid; t < B::NS; t += blockDim.x) src[t] = -1;
    for (int t = tid; t < nrows * ts / 4; t += blockDim.x)
      reinterpret_cast<float4*>(tile)[t] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int t = tid; t < nrows; t += blockDim.x) brhs[t] = 0.f;
    __syncthreads();
    if (tid < nrows) {
      int x, y, z;
      morton3_decode(__ldg(keys + first + tid), x, y, z);
      const int r = (((x - bx) * B::S) + (y - by)) * B::S + (z - bz);
      posmap[r] = tid;
      rloc[tid] = r;
    }
    __syncthreads();
    for (int t = tid; t < nrows * 27; t += blockDim.x) {     // (several rows may name one source: same value)
      const int r = t / 27, s = t - 27 * r;
      const int v = __ldg(svh.nbr27[l] + (first + r) * 27 + s);
      if (v >= 0) {
        const int q = rloc[r];
        const int lx = q / (B::S * B::S) + c_d27[s][0] + 1, ly = (q / B::S) % B::S + c_d27[s][1] + 1,
                  lz = q % B::S + c_d27[s][2] + 1;
        src[(lx * B::R + ly) * B::R + lz] = v;
      }
    }
    __syncthreads();
    // per source: constraint-row ranges and the mask of its target slots si that are rows of this brick
    for (int t = tid; t < B::NS; t += blockDim.x) {
      const int v = src[t];
      int4 r4 = make_int4(0, 0, 0, 0);
      unsigned m = 0u;
      if (v >= 0) {
        if (rp) { const int2 a = __ldg(reinterpret_cast<const int2*>(rp) + v); r4.x = a.x; r4.y = a.y; }
        if (rn) { const int2 a = __ldg(reinterpret_cast<const int2*>(rn) + v); r4.z = a.x; r4.w = a.y; }
        if (r4.x < r4.y || r4.z < r4.w) {
          const int lx = t / (B::R * B::R) - 1, ly = (t / B::R) % B::R - 1, lz = t % B::R - 1;
          for (int s = 0; s < 27; ++s) {
            const int rx = lx + c_d27[s][0], ry = ly + c_d27[s][1], rz = lz + c_d27[s][2];
            if (rx >= 0 && rx < B::S && ry >= 0 && ry < B::S && rz >= 0 && rz < B::S &&
                posmap[(rx * B::S + ry) * B::S + rz] >= 0)
              m |= 1u << s;
          }
        }
      }
      rng[t] = r4;
      tmask[t] = m;
    }
    __syncthreads();
    // colour phases: the sources whose local coordinates are (cx,cy,cz) mod 3 and that feed at least one row
    for (int p = wid; p < 27; p += kBrickWarps) {
      int t = -1;
      if (lane < B::NC * B::NC * B::NC) {
        const int lx = p / 9 + 3 * (lane / (B::NC * B::NC)), ly = (p / 3) % 3 + 3 * ((lane / B::NC) % B::NC),
                  lz = p % 3 + 3 * (lane % B::NC);
        if (lx < B::R && ly < B::R && lz < B::R) {
          t = (lx * B::R + ly) * B::R + lz;
          if (!tmask[t]) t = -1;
        }
      }
      const unsigned bal = __ballot_sync(0xffffffffu, t >= 0);
      if (t >= 0) plist[p * 8 + __popc(bal & ((1u << lane) - 1u))] = t;
      if (lane == 0) pcnt[p] = __popc(bal);
    }
    __syncthreads();

    for (int p = 0; p < 27; ++p) {
      const int nitems = pcnt[p] * nlev;
      for (int it = wid; it < nitems; it += kBrickWarps) {
        // ---- one (source u, level offset k): lane s < 27 is target slot s of u when bit s of the mask is set
        const int t = plist[p * 8 + it / nlev], k = it % nlev;
        const unsigned tm = tmask[t];
        const int nt = __popc(tm);
        const int4 r4 = rng[t];
        const int lx = t / (B::R * B::R) - 1, ly = (t / B::R) % B::R - 1, lz = t % B::R - 1;  // row-local coords
        const bool mine = lane < 27 && ((tm >> lane) & 1u);
        const int rank = __popc(tm & ((1u << lane) - 1u));
        int trow = 0;
        float b = 0.f;
        __syncwarp();
        if (mine) {
          tlist[rank] = lane;
          trow = posmap[((lx + c_d27[lane][0]) * B::S + ly + c_d27[lane][1]) * B::S + lz + c_d27[lane][2]];
          if (k == 0) b = brhs[trow];
        }
        float m[28];
#pragma unroll
        for (int j = 0; j < 28; ++j) m[j] = 0.f;
        // (the lines of location q + 1 are requested before location q is multiplied in: one location's loads per
        // iteration otherwise leave the warp waiting on L2 once per location)
        float e0 = 0.f, ek = 0.f;
        if (r4.x < r4.y) brick_load_pos<ILV>(cs, r4.x, L, l, k, lane, e0, ek);
        for (int q = r4.x; q < r4.y; ++q) {
          float e0n = 0.f, ekn = 0.f;
          if (q + 1 < r4.y) brick_load_pos<ILV>(cs, q + 1, L, l, k, lane, e0n, ekn);
          __syncwarp();
          if (mine) stage[rank] = cs.w_pos * e0;
          __syncwarp();
          brick_fma(m, stage, ek, nt);
          e0 = e0n;
          ek = ekn;
        }
        float n0[3] = {0.f, 0.f, 0.f}, nk[3] = {0.f, 0.f, 0.f};
        if (r4.z < r4.w) brick_load_nrm<ILV>(cs, r4.z, L, l, k, lane, n0, nk);
        for (int q = r4.z; q < r4.w; ++q) {
          float n0n[3] = {0.f, 0.f, 0.f}, nkn[3] = {0.f, 0.f, 0.f};
          if (q + 1 < r4.w) brick_load_nrm<ILV>(cs, q + 1, L, l, k, lane, n0n, nkn);
          __syncwarp();
#pragma unroll
          for (int ax = 0; ax < 3; ++ax) {
            const float el = cs.w_nrm * n0[ax];
            if (mine) {
              if (k == 0) b = fmaf(el, __ldg(cs.t_nrm + (int64_t)q * 3 + ax), b);
              stage[ax * 32 + rank] = el;
            }
          }
          __syncwarp();
#pragma unroll
          for (int ax = 0; ax < 3; ++ax) brick_fma(m, stage + ax * 32, nk[ax], nt);
#pragma unroll
          for (int ax = 0; ax < 3; ++ax) { n0[ax] = n0n[ax]; nk[ax] = nkn[ax]; }
        }
        if (mine && k == 0) brhs[trow] = b;
        __syncwarp();
        // ---- flush into the target rows' tiles: the slot of column u + d(lane) in row i = u + d(si) is the row
        // kernel's base of the source (d(u - i) = -d(si)) plus the lane constant
        const int ux = bx + lx, uy = by + ly, uz = bz + lz;       // source voxel, absolute
#pragma unroll
        for (int j = 0; j < 27; ++j) {
          if (j < nt) {
            const int si = tlist[j];
            const int dx = c_d27[si][0], dy = c_d27[si][1], dz = c_d27[si][2];
            const int r = posmap[((lx + dx) * B::S + ly + dy) * B::S + lz + dz];
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
      const int i = (int)(first + r);
      const int64_t row = svh.offset[l] + i;
      RowGeom g;
      row_geom(svh, l, i, g);
      const int my_u = lane < 27 ? __ldg(svh.nbr27[l] + (int64_t)i * 27 + lane) : -1;
      float* acc = tile + r * ts;
      gram_row_regulariser(feat, cs, l, i, my_u, lane, acc);
      __syncwarp();
      gram_row_writeout<4, true>(svh, l, i, row, g, acc, cnt, rowptr, col_out, val_out, diag, nullptr, place, lane);
      if (lane == 0) rhs[row] = brhs[r];
    }
    __syncthreads();
  }
}

template <int LB, bool ILV>
int launch_brick_level(const nksr_svh_t* svh, const nksr_feat_t* feat, const nksr_constraints_t* c, int l,
                       const int32_t* cnt, const int64_t* rowptr, const PlaceArg<true>& place, int32_t* col, float* val,
                       float* rhs, float* diag, cudaStream_t s) {
  const int ts = (125 + 64 * (svh->depth - 1 - l) + 3) & ~3;
  const size_t smem = Brick<LB>::words(ts) * sizeof(float);
  if (cudaFuncSetAttribute(k_gram_fill_brick<LB, ILV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
      cudaSuccess)
    return NKSR_E_CUDA;
  k_gram_fill_brick<LB, ILV><<<grid_for(svh->n[l], Brick<LB>::NB), kBrickWarps * 32, smem, s>>>(
      *svh, *feat, *c, l, cnt, rowptr, col, val, rhs, diag, place);
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
  PlaceArg<true> place;
  place.t = *placement;
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
            ? launch_brick_level<kBrickLog2, true>(svh, feat, c, l, cnt, rowptr, place, col, val, rhs, diag, s)
            : launch_brick_level<kBrickLog2, false>(svh, feat, c, l, cnt, rowptr, place, col, val, rhs, diag, s);
    if (rc != NKSR_OK) return rc;
  }
  const int64_t n = svh->offset[svh->depth - 1] + svh->n[svh->depth - 1];
  const int64_t rest = nb < svh->depth ? svh->offset[nb] : n;
  return nksr_gram_fill_placed_rows(svh, feat, c, cnt, rowptr, placement, rest, n, col, val, rhs, diag, stream);
}

}  // extern "C"
