// Streaming CSR SpMV for sm_90a: the matrix never goes through the L1 / register path.
// (SURVEY section 8 row a4; the CG SpMV is the kernel BASELINE.json names for the HBM roofline.)
//
// The (col, val) stream is cut into fixed tiles of kTile entries.  One elected producer thread per CTA moves whole
// tiles (column indices, values and the slice of row pointers that covers them) from HBM into a ring of
// shared-memory stages with 1-D bulk async copies (cp.async.bulk.shared::cluster.global, the TMA engine; SASS
// UBLKCP) that signal an mbarrier with their byte count; the consumer warps never issue a load for the matrix:
//   phase 1  every thread turns its share of the tile into products  val * x[col]  in place (the x gathers are
//            the only global loads of the kernel, perfectly balanced, 8 independent gathers per thread);
//   phase 2  one warp per row sums the row's products from shared memory in a fixed order and writes y.
// (A one-phase consumer -- warp per row straight from shared memory, no CTA barrier, 24 warps -- was measured slower
// on the short rows.)
// A row cut by a tile boundary is owned by the tile it starts in; the tiles it continues into leave their part in
// head[tile] and k_spmv_heads adds the parts in tile order -- no atomics, bitwise reproducible.
// The memory pipeline (kStages x 36 KB per CTA, 2 CTAs per SM) is independent of what the warps are waiting for,
// which is what the warp-per-row kernel lacked (profiled: most warps stalled on the scoreboard, DRAM well below its peak).
//
// Packed column tiles.  At 0.79 of the data-sheet bandwidth the stream is bound by the bytes it moves, and the int32
// columns are a third of them.  A tile covers a few dozen consecutive Morton rows, so its columns fall in a few narrow
// index windows (one or two per level).  Once per plan, every tile is examined: when its columns lie in at most
// kPackWindows aligned windows of 2^kPackBits columns, the window bases go to the tile's header and one
// uint16 per entry (3-bit window selector, 13-bit offset) to the tile's 8 KB slot; the producer then moves 8 KB of
// offsets instead of 16 KB of columns.  Other tiles stay raw and are read from `col`.  Phase 1 decodes the same column
// indices, so the products, their order and y are bitwise those of the raw stream.
// The first SpMV over a plan packs the tiles as it streams them (the plan marks every tile unexamined): its consumers
// hold the raw columns anyway, so packing costs that launch the 2-byte writes and not another pass over col (a
// separate pack kernel took longer than the packed tiles saved over a 10-iteration solve).
#pragma once
#include "common.cuh"

namespace {

constexpr int kTile = 4096;             // entries per tile: 16 KB of columns + 16 KB of values
constexpr int kTileRows = 512;          // row pointers staged per tile (int64): 4 KB
constexpr int kStages = 3;
constexpr int kStreamWarps = 16;        // consumer warps per CTA (8 warps left the x gathers latency bound)
constexpr int kStreamThreads = (kStreamWarps + 1) * 32;   // + the producer warp
constexpr int kStreamCtasPerSm = 2;
constexpr int kPackWindows = 8;         // window selector: 3 bits
constexpr int kPackBits = 13;           // offset inside a window: 13 bits, windows of 8192 columns

struct __align__(16) TileHdr {
  int32_t base[kPackWindows];           // first column of each window (packed tiles)
  int32_t packed;                       // 1: the tile's columns are in its packed slot, 0: read them from col
  int32_t pad[3];
};
struct __align__(16) SpmvStage {
  int32_t col[kTile];                   // raw columns, or kTile uint16 (selector, offset) pairs in the first half
  float val[kTile];
  int64_t rp[kTileRows];
  TileHdr hdr;
};
struct SpmvSmem {
  SpmvStage st[kStages];
  unsigned long long full[kStages];
  unsigned long long empty[kStages];
  unsigned set[2][kPackWindows + 1];    // packing: a tile's windows (empty: ~0) + overflow flag, by tile parity
};

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "NKSR_WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra NKSR_DONE_%=;\n"
      "bra NKSR_WAIT_%=;\n"
      "NKSR_DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// 1-D bulk copy global -> shared, completion counted in bytes on `bar` (src, dst and bytes multiples of 16)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// first_row[t] = row that contains entry t * kTile (last row whose start is <= that entry); first_row[0] = 0, so that
// tile 0 also writes the empty rows the matrix may start with; first_row[ntiles] = n
__global__ void k_spmv_plan(const int64_t* __restrict__ rowptr, int64_t n, int64_t ntiles,
                            int32_t* __restrict__ first_row) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t > ntiles) return;
  if (t == ntiles) { first_row[t] = (int32_t)n; return; }
  if (t == 0) { first_row[0] = 0; return; }
  const int64_t e = t * kTile;
  int64_t lo = 0, hi = n;   // first row with rowptr[row] > e
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (__ldg(rowptr + mid) <= e) lo = mid + 1; else hi = mid;
  }
  first_row[t] = (int32_t)(lo - 1);
}

// the consumers of an unexamined tile, holding its columns c[j] (entry tid + j * 512): collect the tile's windows
// (col >> kPackBits) in a set of kPackWindows slots (set[it & 1]: one warp leader per distinct window of a warp claims
// the first slot that is free or holds it, by compare-and-swap, so a window has one slot); with no overflow, write the
// tile's packed slot, selector = the window's slot.  The slot order depends on timing, the decoded columns do not.
// Writes the header either way.  stats[0] += packed tiles, stats[1] += their entries (integer atomics).  The caller
// clears the set after the CTA barrier that follows.
template <int kPer>
__device__ __forceinline__ void pack_tile(unsigned* set, const int (&c)[kPer], int cnt, int64_t t,
                                          TileHdr* __restrict__ hdr, uint16_t* __restrict__ pk,
                                          unsigned long long* __restrict__ stats) {
  const int tid = threadIdx.x, lane = tid & 31;
  unsigned sels = 0;          // 4 bits per entry: the window's slot
#pragma unroll
  for (int j = 0; j < kPer; ++j) {
    const bool live = tid + j * (kStreamWarps * 32) < cnt;
    const unsigned w = live ? (unsigned)c[j] >> kPackBits : 0xffffffffu;
    const unsigned same = __match_any_sync(0xffffffffu, w);
    const int leader = __ffs(same) - 1;
    unsigned slot = 0;
    if (live && lane == leader) {
      for (slot = 0; slot < kPackWindows; ++slot) {
        const unsigned old = atomicCAS(set + slot, 0xffffffffu, w);
        if (old == 0xffffffffu || old == w) break;
      }
      if (slot == kPackWindows) set[kPackWindows] = 1u;   // a ninth window: the tile stays raw
    }
    sels |= (__shfl_sync(0xffffffffu, slot, leader) & 7u) << (4 * j);
  }
  asm volatile("bar.sync 1, %0;" ::"n"(kStreamWarps * 32) : "memory");
  if (set[kPackWindows] != 0u) {
    if (tid == 0) hdr[t].packed = 0;
    return;
  }
  const int64_t e0 = t * kTile;
#pragma unroll
  for (int j = 0; j < kPer; ++j) {
    const int e = tid + j * (kStreamWarps * 32);
    const unsigned v = e < cnt ? (((sels >> (4 * j)) & 7u) << kPackBits) | ((unsigned)c[j] & ((1u << kPackBits) - 1))
                               : 0u;
    pk[e0 + e] = (uint16_t)v;
  }
  if (tid == 0) {
#pragma unroll
    for (int k = 0; k < kPackWindows; ++k) hdr[t].base[k] = set[k] != 0xffffffffu ? (int32_t)(set[k] << kPackBits) : 0;
    hdr[t].packed = 1;
    atomicAdd(stats, 1ull);
    atomicAdd(stats + 1, (unsigned long long)cnt);
  }
}

// y = A x for the rows that START inside each tile; head[t] = the part of tile t that belongs to a row started
// earlier.  rowptr must be readable up to index n + 1 and col / val up to the next multiple of 4 entries (the bulk
// copies move whole 16-byte units); `done` (nullable): the solve is over, do nothing.
__global__ void __launch_bounds__(kStreamThreads, kStreamCtasPerSm)
k_spmv_stream(const int64_t* __restrict__ rowptr, const int32_t* __restrict__ col, const float* __restrict__ val,
              const float* __restrict__ x, float* __restrict__ y, int64_t n, int64_t nnz, int64_t ntiles,
              const int32_t* __restrict__ first_row, float* __restrict__ head, TileHdr* __restrict__ hdr,
              uint16_t* __restrict__ pk, unsigned long long* __restrict__ stats, const int* __restrict__ done) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  SpmvSmem& sm = *reinterpret_cast<SpmvSmem*>(smem_raw);
  if (done && *done) return;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (blockIdx.x == 0 && tid == 0) {
    stats[2] = (unsigned long long)ntiles;
    stats[3] = (unsigned long long)nnz;
  }
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], kStreamWarps); }
    for (int i = 0; i < 2 * (kPackWindows + 1); ++i) (&sm.set[0][0])[i] = (i % (kPackWindows + 1)) < kPackWindows ? ~0u : 0u;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (wid == kStreamWarps) {
    // ---------------- producer: one thread feeds the ring
    if (lane == 0) {
      int it = 0;
      for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
        const int s = it % kStages;
        const unsigned use = (unsigned)(it / kStages);
        if (use > 0) mbar_wait(&sm.empty[s], (use - 1) & 1);
        const int64_t e0 = t * kTile;
        const int64_t cnt = (nnz - e0 < kTile) ? (nnz - e0) : kTile;
        const unsigned ebytes = (unsigned)(((cnt + 3) & ~(int64_t)3) * 4);
        const bool packed = hdr[t].packed == 1;
        const unsigned cbytes = packed ? (unsigned)(((cnt + 7) & ~(int64_t)7) * 2) : ebytes;
        const int64_t ra = first_row[t] & ~1;                       // 16-byte aligned start of the row-pointer slice
        int64_t rcount = (int64_t)first_row[t + 1] + 2 - ra;        // ... up to rowptr[first_row[t+1] + 1]
        if (ra + rcount > n + 1) rcount = n + 1 - ra;
        rcount = (rcount + 1) & ~(int64_t)1;
        const bool staged = rcount <= kTileRows;
        const unsigned rbytes = staged ? (unsigned)(rcount * 8) : 0u;
        mbar_expect_tx(&sm.full[s], (unsigned)sizeof(TileHdr) + cbytes + ebytes + rbytes);
        bulk_g2s(&sm.st[s].hdr, hdr + t, (unsigned)sizeof(TileHdr), &sm.full[s]);
        if (packed) bulk_g2s(sm.st[s].col, pk + e0, cbytes, &sm.full[s]);
        else bulk_g2s(sm.st[s].col, col + e0, ebytes, &sm.full[s]);
        bulk_g2s(sm.st[s].val, val + e0, ebytes, &sm.full[s]);
        if (staged) bulk_g2s(sm.st[s].rp, rowptr + ra, rbytes, &sm.full[s]);
      }
    }
    return;
  }

  // ---------------- consumers
  int it = 0;
  for (int64_t t = blockIdx.x; t < ntiles; t += gridDim.x, ++it) {
    const int s = it % kStages;
    const unsigned use = (unsigned)(it / kStages);
    SpmvStage& st = sm.st[s];
    mbar_wait(&sm.full[s], use & 1);
    const int64_t e0 = t * kTile;
    const int cnt = (int)((nnz - e0 < kTile) ? (nnz - e0) : kTile);
    // phase 1: products in place.  All 16 column indices of the thread first, then 16 independent x gathers in flight,
    // then the multiplies (a loop of  val[e] *= x[col[e]]  serialises on the shared-memory store)
    {
      constexpr int kPer = kTile / (kStreamWarps * 32);
      int c[kPer];
      float xv[kPer];
      if (st.hdr.packed == 1) {
        const uint16_t* off = reinterpret_cast<const uint16_t*>(st.col);
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
          const int e = tid + j * (kStreamWarps * 32);
          const unsigned v = off[e];
          c[j] = e < cnt ? st.hdr.base[v >> kPackBits] + (int)(v & ((1u << kPackBits) - 1)) : 0;
        }
      } else {
#pragma unroll
        for (int j = 0; j < kPer; ++j) {
          const int e = tid + j * (kStreamWarps * 32);
          c[j] = e < cnt ? st.col[e] : 0;
        }
      }
#pragma unroll
      for (int j = 0; j < kPer; ++j) xv[j] = __ldg(x + c[j]);
      // an unexamined tile is packed while its gathers are in flight
      if (st.hdr.packed < 0) pack_tile<kPer>(sm.set[it & 1], c, cnt, t, hdr, pk, stats);
#pragma unroll
      for (int j = 0; j < kPer; ++j) {
        const int e = tid + j * (kStreamWarps * 32);
        st.val[e] *= xv[j];
      }
    }
    asm volatile("bar.sync 1, %0;" ::"n"(kStreamWarps * 32) : "memory");
    // (set[it & 1] is next used by tile it + 2, after the barrier above of tile it + 1)
    if (tid < kPackWindows + 1) sm.set[it & 1][tid] = tid < kPackWindows ? ~0u : 0u;
    // phase 2: one warp per row of the tile
    const int r0 = first_row[t];
    const int64_t ra = r0 & ~1;
    int64_t rcount = (int64_t)first_row[t + 1] + 2 - ra;
    if (ra + rcount > n + 1) rcount = n + 1 - ra;
    const bool staged = ((rcount + 1) & ~(int64_t)1) <= kTileRows;
    const int64_t* rp = staged ? st.rp : rowptr + ra;               // rp[i] = rowptr[ra + i]
    const int64_t e1 = e0 + cnt;
    const int64_t rlast = first_row[t + 1] < n ? first_row[t + 1] : n - 1;   // last row the slice describes
    for (int64_t row = r0 + wid; row <= rlast; row += kStreamWarps) {
      const int64_t b = rp[row - ra];
      const int64_t e = rp[row - ra + 1];
      // an empty row that starts exactly at the tile's end belongs to no later tile (first_row[t + 1] is the last
      // row starting there): this tile writes its zero.  With first_row[0] = 0 for the rows before entry 0, every
      // row of [0, n) is written
      if (b > e1 || (b == e1 && e > b)) break;
      const int lo = (int)((b > e0 ? b : e0) - e0), hi = (int)((e < e1 ? e : e1) - e0);
      float acc = 0.f;
      for (int p = lo + lane; p < hi; p += 32) acc += st.val[p];
      acc = warp_sum(acc);
      if (lane == 0) {
        if (b >= e0) y[row] = acc; else head[t] = acc;
      }
    }
    // the stage was written through the generic proxy (products in place); order those writes before the bulk
    // copy (async proxy) that refills it
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.empty[s]);
  }
}

// rows cut by tile boundaries: the owner (the tile the row starts in) holds the first part in y[row]; add the
// parts left by the following tiles, in tile order.  One thread per tile.
__global__ void k_spmv_heads(const int64_t* __restrict__ rowptr, float* __restrict__ y, int64_t n, int64_t nnz,
                             int64_t ntiles, const int32_t* __restrict__ first_row, const float* __restrict__ head,
                             const int* __restrict__ done) {
  if (done && *done) return;
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= ntiles) return;
  const int64_t e0 = t * kTile;
  const int64_t e1 = (nnz - e0 < kTile) ? nnz : e0 + kTile;
  if (e1 >= nnz) return;                                 // nothing continues past the last tile
  const int64_t row = first_row[t + 1];                  // row holding the first entry of the next tile
  const int64_t b = __ldg(rowptr + row);
  if (b >= e1 || b < e0) return;                         // starts exactly at the boundary / owned by an earlier tile
  const int64_t e = __ldg(rowptr + row + 1);
  float s = y[row];
  for (int64_t tt = t + 1; tt < ntiles && tt * kTile < e; ++tt) s += head[tt];
  y[row] = s;
}

// partial[blockIdx] = sum a_i * b_i (fp64), fixed order
__global__ void __launch_bounds__(256)
k_dot_partials(const float* __restrict__ a, const float* __restrict__ b, int64_t n, double* __restrict__ partial,
               const int* __restrict__ done) {
  __shared__ double sh[8];
  if (done && *done) return;
  double t = 0.0;
  for (int64_t i = blockIdx.x * (int64_t)256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256)
    t += (double)a[i] * (double)b[i];
  t = warp_sum_d(t);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double r = 0.0;
    for (int w = 0; w < 8; ++w) r += sh[w];
    partial[blockIdx.x] = r;
  }
}

struct SpmvPlan {
  int64_t n_rows;       // rows [0, n_rows) are streamed (entries [0, nnz)); the caller handles the remaining rows
  int64_t nnz, ntiles;
  unsigned long long* stats;   // [4]: packed tiles, entries in packed tiles, streamed tiles, streamed entries (after
                               // the first SpMV)
  int32_t* first_row;   // [ntiles + 1]
  float* head;          // [ntiles]
  TileHdr* hdr;         // [ntiles]
  uint16_t* pk;         // [ntiles * kTile]: the packed slots
};

// plan buffer: stats | first_row | head | hdr | packed slots; stats first, so that a built plan is queried without
// knowing how many entries it streams
static size_t spmv_align256(size_t v) { return (v + 255) & ~(size_t)255; }
static int64_t spmv_tiles(int64_t nnz) { return (nnz + kTile - 1) / kTile; }
static size_t spmv_plan_bytes(int64_t nnz) {
  const int64_t nt = spmv_tiles(nnz);
  return 256 + spmv_align256((size_t)(nt + 1) * 4) + spmv_align256((size_t)nt * 4) +
         spmv_align256((size_t)nt * sizeof(TileHdr)) + (size_t)nt * kTile * sizeof(uint16_t) + 256;
}
static SpmvPlan spmv_plan_carve(void* buf, int64_t n_rows, int64_t nnz) {
  SpmvPlan p;
  p.n_rows = n_rows;
  p.nnz = nnz;
  p.ntiles = spmv_tiles(nnz);
  unsigned char* c = reinterpret_cast<unsigned char*>(buf);
  p.stats = reinterpret_cast<unsigned long long*>(c);
  c += 256;
  p.first_row = reinterpret_cast<int32_t*>(c);
  c += spmv_align256((size_t)(p.ntiles + 1) * 4);
  p.head = reinterpret_cast<float*>(c);
  c += spmv_align256((size_t)p.ntiles * 4);
  p.hdr = reinterpret_cast<TileHdr*>(c);
  c += spmv_align256((size_t)p.ntiles * sizeof(TileHdr));
  p.pk = reinterpret_cast<uint16_t*>(c);
  return p;
}
// tile boundaries; every tile marked unexamined (packed = -1), so that the first SpMV packs it.  p.stats must be zero
static int spmv_plan_build(const int64_t* rowptr, const SpmvPlan& p, cudaStream_t s) {
  const int64_t work = p.ntiles + 1;
  k_spmv_plan<<<grid_for(work, 256), 256, 0, s>>>(rowptr, p.n_rows, p.ntiles, p.first_row);
  if (cudaMemsetAsync(p.hdr, 0xff, (size_t)p.ntiles * sizeof(TileHdr), s) != cudaSuccess) return NKSR_E_CUDA;
  return cudaGetLastError() == cudaSuccess ? NKSR_OK : NKSR_E_CUDA;
}
// once per call site, outside any stream capture: opt in to the shared-memory ring on the current device
static int spmv_stream_prepare() {
  return cudaFuncSetAttribute(k_spmv_stream, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SpmvSmem)) ==
                 cudaSuccess
             ? NKSR_OK
             : NKSR_E_CUDA;
}
static int spmv_stream_sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}
// y = A x through the tile stream (+ the boundary rows)
static int spmv_stream_launch(const int64_t* rowptr, const int32_t* col, const float* val, const float* x, float* y,
                              const SpmvPlan& p, const int* done, cudaStream_t s) {
  const int64_t n = p.n_rows;
  int64_t grid = (int64_t)spmv_stream_sm_count() * kStreamCtasPerSm;
  if (grid > p.ntiles) grid = p.ntiles;
  if (grid < 1) return NKSR_OK;
  k_spmv_stream<<<(int)grid, kStreamThreads, sizeof(SpmvSmem), s>>>(rowptr, col, val, x, y, n, p.nnz, p.ntiles,
                                                                    p.first_row, p.head, p.hdr, p.pk, p.stats, done);
  k_spmv_heads<<<grid_for(p.ntiles, 256), 256, 0, s>>>(rowptr, y, n, p.nnz, p.ntiles, p.first_row, p.head, done);
  return cudaGetLastError() == cudaSuccess ? NKSR_OK : NKSR_E_CUDA;
}

}  // namespace
