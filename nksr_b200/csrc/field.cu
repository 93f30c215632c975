// Kernel-row construction for the Gram assembly (row a3) and field evaluation (row a5).
// Call sites replaced: KernelField.solve_non_fused (models/nksr_net.py:100-112) and
// field.evaluate_f (models/loss.py:189-198,225).
#include "kernel_eval.cuh"

namespace {

constexpr int kWarpsPerBlock = 8;

// one warp per (location, level): writes a 128-byte value row (MODE 0), three gradient rows
// (MODE 1) or one compact gradient row (MODE 2, approx_kernel_grad only): slots 0..26 hold
// <phi(x), z_s>, slots 27..29 the local coordinate tau -- the three gradient rows
// dB_a B_b B_c <phi,z_s> / W_l are rebuilt from it inside the assembly kernel.
// One warp per LOCATION, all levels in one (unrolled) loop: the point is read once, the per-level
// dependent chains (base -> key -> neighbours -> features) of the levels overlap, and the grid
// has L times fewer blocks than a warp per (location, level).
// ILV (depth <= 4): "levels in the lane" layout -- the four levels of one (location, axis, slot) are one float4,
// [m][rows][32 slots][4 levels]: the assembly reads all levels of a location with ONE 128-bit load per lane (512
// contiguous bytes per warp) instead of one 32-bit load per level, and this kernel writes them with one 128-bit store.
template <int MODE, int MAXL, bool ILV>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
k_build_rows(nksr_svh_t svh, nksr_feat_t feat, const float* __restrict__ xyz, const int32_t* __restrict__ base,
             int64_t m, bool fullgrad, float* __restrict__ e) {
  const int lane = threadIdx.x & 31;
  const int64_t i = blockIdx.x * (int64_t)kWarpsPerBlock + (threadIdx.x >> 5);
  if (i >= m) return;
  constexpr bool GRAD = MODE == 1;
  constexpr int ROWS = GRAD ? 3 : 1;
  const float px = __ldg(xyz + 3 * i), py = __ldg(xyz + 3 * i + 1), pz = __ldg(xyz + 3 * i + 2);
  // half-voxel coordinates of the point: the containing voxel on level l is h >> (l+1), so no key has to be loaded
  // and decoded per level.  A point outside the range has base -1 on every level (nksr_locate), so h is never read.
  int3 h;
  half_voxel(px, py, pz, svh.voxel_size * 0.5f, h);
  const double inv0 = 1.0 / (double)svh.voxel_size;
  // location-major layout [m][L][rows][32]: all lines of one location are contiguous, so the
  // assembly kernel reaches them with compile-time offsets from one base pointer
  float* out0 = e + (int64_t)i * svh.depth * ROWS * NKSR_ROW_STRIDE;
  float kv[MAXL][ROWS];            // ILV only: the levels of this lane's slot (dead code otherwise)
#pragma unroll
  for (int l = 0; l < MAXL; ++l)
#pragma unroll
    for (int a = 0; a < ROWS; ++a) kv[l][a] = 0.f;
#pragma unroll
  for (int l = 0; l < MAXL; ++l) {
    if (l < svh.depth) {
      float* out = out0 + l * ROWS * NKSR_ROW_STRIDE;
      const int b = __ldg(base + (int64_t)l * m + i);
      if (b < 0) {
        if (!ILV) {
          out[lane] = 0.f;
          if (GRAD) { out[32 + lane] = 0.f; out[64 + lane] = 0.f; }
        }
      } else {
        const float wl = svh.voxel_size * (float)(1 << l);
        LaneKernel r = eval_level_lane<GRAD>(svh.nbr27[l], feat.z[l], feat.channels, l, wl, inv0, px, py, pz, b,
                                             h.x >> (l + 1), h.y >> (l + 1), h.z >> (l + 1), fullgrad, lane);
        if (ILV) {
#pragma unroll
          for (int a = 0; a < ROWS; ++a) kv[l][a] = GRAD ? r.dk[a] : r.k;
        } else if (GRAD) {
          out[lane] = r.dk[0];
          out[32 + lane] = r.dk[1];
          out[64 + lane] = r.dk[2];
        } else if (MODE == 2) {
          out[lane] = lane < 27 ? r.dot : (lane < 30 ? r.tau[lane - 27] : 0.f);
        } else {
          out[lane] = r.k;
        }
      }
    }
  }
  if (ILV) {
    float4* o4 = reinterpret_cast<float4*>(e) + ((int64_t)i * ROWS) * NKSR_ROW_STRIDE + lane;
#pragma unroll
    for (int a = 0; a < ROWS; ++a)
      o4[a * NKSR_ROW_STRIDE] = make_float4(kv[0][a], kv[1 % MAXL][a], kv[2 % MAXL][a], kv[3 % MAXL][a]);
  }
}

// ---- kernel rows, one warp per VOXEL (the default): all locations whose containing voxel on level l is u share u's
// 27-stencil and its features, and they are contiguous (locations are Morton sorted).  The warp-per-location kernel
// above re-gathers 27 feature rows per location and level -- 27 L1 wavefronts per channel load, the measured limit of
// that kernel; here the stencil and the features (C <= 16, as float4
// registers) are fetched ONCE per voxel and the loop over the voxel's locations is ALU + shuffles + the row stores.
// Same geometry (kernel_eval.cuh) and the channel loop in the same order: bitwise the rows of k_build_rows.
template <int MODE, int NC4>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
k_build_rows_voxel(nksr_svh_t svh, nksr_feat_t feat, const float* __restrict__ xyz, const int32_t* __restrict__ range,
                   int l, bool fullgrad, float* __restrict__ e) {
  const int lane = threadIdx.x & 31;
  const int64_t u = blockIdx.x * (int64_t)kWarpsPerBlock + (threadIdx.x >> 5);
  if (u >= svh.n[l]) return;
  const int2 r = __ldg(reinterpret_cast<const int2*>(range) + svh.offset[l] + u);
  if (r.x >= r.y) return;
  constexpr bool GRAD = MODE == 1;
  constexpr int ROWS = GRAD ? 3 : 1;
  int ux, uy, uz;
  morton3_decode(__ldg(svh.keys[l] + u), ux, uy, uz);
  const int nb = lane < 27 ? __ldg(svh.nbr27[l] + u * 27 + lane) : -1;
  const bool ok = nb >= 0;
  float zc[NC4 * 4];
#pragma unroll
  for (int q = 0; q < NC4; ++q) {
    const float4 v = ok ? __ldg(reinterpret_cast<const float4*>(feat.z[l] + (int64_t)nb * (NC4 * 4)) + q)
                        : make_float4(0.f, 0.f, 0.f, 0.f);
    zc[4 * q] = v.x; zc[4 * q + 1] = v.y; zc[4 * q + 2] = v.z; zc[4 * q + 3] = v.w;
  }
  int dx, dy, dz;
  slot_to_d(lane < 27 ? lane : 13, dx, dy, dz);
  const double cx = voxel_centre(ux, l), cy = voxel_centre(uy, l), cz = voxel_centre(uz, l);
  const double inv = (1.0 / (double)svh.voxel_size) * (1.0 / (double)(1 << l));
  const float iw = 1.f / (svh.voxel_size * (float)(1 << l));
  const int L = svh.depth;
  for (int q = r.x; q < r.y; ++q) {
    const float px = __ldg(xyz + 3 * (int64_t)q), py = __ldg(xyz + 3 * (int64_t)q + 1), pz = __ldg(xyz + 3 * (int64_t)q + 2);
    const float tx = local_coord(px, inv, cx), ty = local_coord(py, inv, cy), tz = local_coord(pz, inv, cz);
    const StencilWeights w = stencil_weights(tx, ty, tz, dx, dy, dz);
    const float B3 = w.B3();
    const float T3 = ok ? w.T3() : 0.f;
    float dT3[3] = {0.f, 0.f, 0.f};
    if (GRAD) {
      dT3[0] = ok ? w.dT3(0) : 0.f;
      dT3[1] = ok ? w.dT3(1) : 0.f;
      dT3[2] = ok ? w.dT3(2) : 0.f;
    }
    float dot = 0.f, ddot[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int c = 0; c < NC4 * 4; ++c) {
      const float phi = warp_sum(T3 * zc[c]);
      dot = fmaf(phi, zc[c], dot);
      if (GRAD && fullgrad) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          const float dphi = warp_sum(dT3[a] * zc[c]);
          ddot[a] = fmaf(dphi, zc[c], ddot[a]);
        }
      }
    }
    float* out = e + ((int64_t)q * L + l) * ROWS * NKSR_ROW_STRIDE;
    if (GRAD) {
      out[lane] = ok ? (w.dB(0) * dot + B3 * ddot[0]) * iw : 0.f;
      out[32 + lane] = ok ? (w.dB(1) * dot + B3 * ddot[1]) * iw : 0.f;
      out[64 + lane] = ok ? (w.dB(2) * dot + B3 * ddot[2]) * iw : 0.f;
    } else if (MODE == 2) {
      const float tau = lane == 27 ? tx : (lane == 28 ? ty : tz);
      out[lane] = lane < 27 ? (ok ? dot : 0.f) : (lane < 30 ? tau : 0.f);
    } else {
      out[lane] = ok ? B3 * dot : 0.f;
    }
  }
}

// locations whose containing voxel on some level is inactive (e.g. the centre of a childless voxel on the level
// below): their lines of that level are zero
template <int ROWS>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
k_zero_inactive_rows(int depth, const int32_t* __restrict__ base, int64_t m, float* __restrict__ e) {
  const int lane = threadIdx.x & 31;
  const int64_t i = blockIdx.x * (int64_t)kWarpsPerBlock + (threadIdx.x >> 5);
  if (i >= m) return;
  for (int l = 0; l < depth; ++l) {
    if (__ldg(base + (int64_t)l * m + i) >= 0) continue;
    float* out = e + ((int64_t)i * depth + l) * ROWS * NKSR_ROW_STRIDE;
#pragma unroll
    for (int r = 0; r < ROWS; ++r) out[r * 32 + lane] = 0.f;
  }
}

// one warp per query: f(x) = sum_l sum_s alpha * K ; containing voxels found by top search + descent
template <bool GRAD>
__global__ void __launch_bounds__(kWarpsPerBlock * 32)
k_evaluate(nksr_svh_t svh, nksr_feat_t feat, const float* __restrict__ alpha, const float* __restrict__ xyz,
           int64_t m, bool fullgrad, float* __restrict__ f, float* __restrict__ g) {
  const int lane = threadIdx.x & 31;
  const int64_t i = blockIdx.x * (int64_t)kWarpsPerBlock + (threadIdx.x >> 5);
  if (i >= m) return;
  const float px = __ldg(xyz + 3 * i), py = __ldg(xyz + 3 * i + 1), pz = __ldg(xyz + 3 * i + 2);
  int3 h;
  const bool in_range = half_voxel(px, py, pz, svh.voxel_size * 0.5f, h);
  const int L = svh.depth;
  const double inv0 = 1.0 / (double)svh.voxel_size;
  int idx = -1;
  if (in_range && svh.n[L - 1] > 0)
    idx = find_key(svh.keys[L - 1], svh.n[L - 1], morton3(h.x >> L, h.y >> L, h.z >> L));
  float accf = 0.f, accg[3] = {0.f, 0.f, 0.f};
  for (int l = L - 1; l >= 0; --l) {
    if (idx < 0) break;  // parent closure: nothing active below
    const float wl = svh.voxel_size * (float)(1 << l);
    LaneKernel r = eval_level_lane<GRAD>(svh.nbr27[l], feat.z[l], feat.channels, l, wl, inv0, px, py, pz, idx,
                                         h.x >> (l + 1), h.y >> (l + 1), h.z >> (l + 1), fullgrad, lane);
    float a = r.nb >= 0 ? __ldg(alpha + svh.offset[l] + r.nb) : 0.f;
    accf = fmaf(a, r.k, accf);
    if (GRAD) {
      accg[0] = fmaf(a, r.dk[0], accg[0]);
      accg[1] = fmaf(a, r.dk[1], accg[1]);
      accg[2] = fmaf(a, r.dk[2], accg[2]);
    }
    if (l > 0) idx = __ldg(svh.child8[l] + (int64_t)idx * 8 + child_octant(h, l));
  }
  accf = warp_sum(accf);
  if (GRAD) {
    accg[0] = warp_sum(accg[0]);
    accg[1] = warp_sum(accg[1]);
    accg[2] = warp_sum(accg[2]);
  }
  if (lane == 0) {
    f[i] = accf;
    if (GRAD) { g[3 * i] = accg[0]; g[3 * i + 1] = accg[1]; g[3 * i + 2] = accg[2]; }
  }
}

// f(x) for RUNS of consecutive queries (C == 4, value only): the mesher evaluates lattice points in Morton order, so
// consecutive queries share their containing voxel on the coarse levels almost always and on the finest level about
// half of the time.  One warp walks kEvalRun consecutive queries and keeps, per level, the containing voxel with its
// 27 neighbours, their features (one float4) and coefficients in registers; a level is re-fetched only when the
// query leaves the voxel.  k_evaluate re-gathers all of it per query and level (three 27-wavefront gathers each).  Same geometry
// (kernel_eval.cuh) and the channel loop in the same order: bitwise the values of k_evaluate<false>.
constexpr int kEvalRun = 8;
constexpr int kEvalMaxL = 4;

__global__ void __launch_bounds__(kWarpsPerBlock * 32)
k_evaluate_runs(nksr_svh_t svh, nksr_feat_t feat, const float* __restrict__ alpha, const float* __restrict__ xyz,
                int64_t m, float* __restrict__ f) {
  const int lane = threadIdx.x & 31;
  const int64_t q0 = (blockIdx.x * (int64_t)kWarpsPerBlock + (threadIdx.x >> 5)) * kEvalRun;
  if (q0 >= m) return;
  const int L = svh.depth;
  const float half_w = svh.voxel_size * 0.5f;
  const double inv0 = 1.0 / (double)svh.voxel_size;
  int dx, dy, dz;
  slot_to_d(lane < 27 ? lane : 13, dx, dy, dz);
  // cached state per level: voxel coordinates, index, this lane's neighbour, its features and coefficient
  int cux[kEvalMaxL], cuy[kEvalMaxL], cuz[kEvalMaxL], cidx[kEvalMaxL], cnb[kEvalMaxL];
  float4 cz[kEvalMaxL];
  float ca[kEvalMaxL];
#pragma unroll
  for (int ll = 0; ll < kEvalMaxL; ++ll) {      // indexed by position in the coarse-to-fine walk: static after unrolling
    cux[ll] = cuy[ll] = cuz[ll] = -1; cidx[ll] = -1; cnb[ll] = -1; ca[ll] = 0.f;
    cz[ll] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const int64_t q1 = q0 + kEvalRun < m ? q0 + kEvalRun : m;
  for (int64_t i = q0; i < q1; ++i) {
    const float px = __ldg(xyz + 3 * i), py = __ldg(xyz + 3 * i + 1), pz = __ldg(xyz + 3 * i + 2);
    int3 h;
    const bool in_range = half_voxel(px, py, pz, half_w, h);
    float accf = 0.f;
    int idx = -1;
    bool alive = in_range && svh.n[L - 1] > 0;
#pragma unroll
    for (int ll = 0; ll < kEvalMaxL; ++ll) {
      const int l = L - 1 - ll;                    // coarse to fine
      if (l < 0 || !alive) continue;
      const int vx = h.x >> (l + 1), vy = h.y >> (l + 1), vz = h.z >> (l + 1);
      if (vx != cux[ll] || vy != cuy[ll] || vz != cuz[ll]) {   // left the voxel on this level: re-fetch it
        int nidx;
        if (l == L - 1) {
          nidx = find_key(svh.keys[l], svh.n[l], morton3(vx, vy, vz));
        } else {
          nidx = idx >= 0 ? __ldg(svh.child8[l + 1] + (int64_t)idx * 8 + child_octant(h, l + 1)) : -1;
        }
        cux[ll] = vx; cuy[ll] = vy; cuz[ll] = vz; cidx[ll] = nidx;
        cnb[ll] = -1; ca[ll] = 0.f; cz[ll] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (nidx >= 0 && lane < 27) {
          const int nb = __ldg(svh.nbr27[l] + (int64_t)nidx * 27 + lane);
          cnb[ll] = nb;
          if (nb >= 0) {
            cz[ll] = __ldg(reinterpret_cast<const float4*>(feat.z[l] + (int64_t)nb * 4));
            ca[ll] = __ldg(alpha + svh.offset[l] + nb);
          }
        }
      }
      idx = cidx[ll];
      if (idx < 0) { alive = false; continue; }   // parent closure: nothing active below
      const double inv = inv0 * (1.0 / (double)(1 << l));
      const StencilWeights w =
          stencil_weights(local_coord(px, inv, voxel_centre(vx, l)), local_coord(py, inv, voxel_centre(vy, l)),
                          local_coord(pz, inv, voxel_centre(vz, l)), dx, dy, dz);
      const bool ok = cnb[ll] >= 0;
      const float B3 = w.B3();
      const float T3 = ok ? w.T3() : 0.f;
      float dot = 0.f;
      const float zc[4] = {cz[ll].x, cz[ll].y, cz[ll].z, cz[ll].w};
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float phi = warp_sum(T3 * zc[c]);
        dot = fmaf(phi, zc[c], dot);
      }
      const float kval = ok ? B3 * dot : 0.f;
      accf = fmaf(ok ? ca[ll] : 0.f, kval, accf);
    }
    accf = warp_sum(accf);
    if (lane == 0) f[i] = accf;
  }
}

// LayerField mask: 1 when the containing voxel of some level < adaptive_depth is active
__global__ void k_layer_mask(nksr_svh_t svh, const float* __restrict__ xyz, int64_t m, int adaptive_depth,
                             float* __restrict__ out) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= m) return;
  int3 h;
  float r = 0.f;
  if (half_voxel(__ldg(xyz + 3 * i), __ldg(xyz + 3 * i + 1), __ldg(xyz + 3 * i + 2), svh.voxel_size * 0.5f, h)) {
    int top = adaptive_depth < svh.depth ? adaptive_depth : svh.depth;
    for (int l = 0; l < top; ++l) {
      if (svh.n[l] == 0) continue;
      int sh = l + 1;
      if (find_key(svh.keys[l], svh.n[l], morton3(h.x >> sh, h.y >> sh, h.z >> sh)) >= 0) { r = 1.f; break; }
    }
  }
  out[i] = r;
}

}  // namespace

extern "C" {

int nksr_build_rows(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* xyz, const int32_t* base,
                    int64_t m, int mode, int approx_kernel_grad, float* e, void* stream) {
  if (!svh || !feat || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH || feat->channels < 1) return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  const int grid = grid_for(m, kWarpsPerBlock);
  cudaStream_t s = as_stream(stream);
  // mode | 4: the interleaved layout [m][rows][32][4 levels] (value and gradient rows, depth <= 4)
  const bool ilv = (mode & 4) != 0;
  mode &= ~4;
  if (mode < 0 || mode > 2 || (mode == 2 && !approx_kernel_grad)) return NKSR_E_INVALID;
  if (ilv && (mode == 2 || svh->depth > 4)) return NKSR_E_INVALID;
  const bool full = mode == 1 && !approx_kernel_grad;
#define NKSR_ROWS(MODE, MAXL) \
  k_build_rows<MODE, MAXL, false><<<grid, kWarpsPerBlock * 32, 0, s>>>(*svh, *feat, xyz, base, m, full, e)
  if (ilv) {
    if (mode == 0) k_build_rows<0, 4, true><<<grid, kWarpsPerBlock * 32, 0, s>>>(*svh, *feat, xyz, base, m, full, e);
    else k_build_rows<1, 4, true><<<grid, kWarpsPerBlock * 32, 0, s>>>(*svh, *feat, xyz, base, m, full, e);
  } else if (svh->depth <= 4) {
    if (mode == 0) NKSR_ROWS(0, 4); else if (mode == 1) NKSR_ROWS(1, 4); else NKSR_ROWS(2, 4);
  } else {
    if (mode == 0) NKSR_ROWS(0, NKSR_MAX_DEPTH); else if (mode == 1) NKSR_ROWS(1, NKSR_MAX_DEPTH);
    else NKSR_ROWS(2, NKSR_MAX_DEPTH);
  }
#undef NKSR_ROWS
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_build_rows_voxel(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* xyz, const int32_t* base,
                          const int32_t* range, int64_t m, int mode, int approx_kernel_grad, float* e, void* stream) {
  if (!svh || !feat || !range || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH) return NKSR_E_INVALID;
  if (mode < 0 || mode > 2 || (mode == 2 && !approx_kernel_grad)) return NKSR_E_INVALID;
  const int C = feat->channels;
  if (C != 4 && C != 8 && C != 16) return NKSR_E_INVALID;     // features are held as float4 registers
  if (m == 0) return NKSR_OK;
  cudaStream_t s = as_stream(stream);
  const bool full = mode == 1 && !approx_kernel_grad;
  const int zgrid = grid_for(m, kWarpsPerBlock);
  if (mode == 1) k_zero_inactive_rows<3><<<zgrid, kWarpsPerBlock * 32, 0, s>>>(svh->depth, base, m, e);
  else k_zero_inactive_rows<1><<<zgrid, kWarpsPerBlock * 32, 0, s>>>(svh->depth, base, m, e);
  for (int l = 0; l < svh->depth; ++l) {
    if (svh->n[l] == 0) continue;
    const int grid = grid_for(svh->n[l], kWarpsPerBlock);
#define NKSR_VROWS(MODE, NC4) \
  k_build_rows_voxel<MODE, NC4><<<grid, kWarpsPerBlock * 32, 0, s>>>(*svh, *feat, xyz, range, l, full, e)
#define NKSR_VROWS_C(MODE)                                                     \
  do {                                                                         \
    if (C == 4) NKSR_VROWS(MODE, 1); else if (C == 8) NKSR_VROWS(MODE, 2); else NKSR_VROWS(MODE, 4); \
  } while (0)
    if (mode == 0) NKSR_VROWS_C(0); else if (mode == 1) NKSR_VROWS_C(1); else NKSR_VROWS_C(2);
#undef NKSR_VROWS_C
#undef NKSR_VROWS
  }
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_evaluate(const nksr_svh_t* svh, const nksr_feat_t* feat, const float* alpha, const float* xyz, int64_t m,
                  int want_grad, int approx_kernel_grad, float* f, float* grad, void* stream) {
  if (!svh || !feat || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH || feat->channels < 1) return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  int grid = grid_for(m, kWarpsPerBlock);
  if (want_grad)
    k_evaluate<true><<<grid, kWarpsPerBlock * 32, 0, as_stream(stream)>>>(*svh, *feat, alpha, xyz, m,
                                                                          !approx_kernel_grad, f, grad);
  else if (feat->channels == 4 && svh->depth <= kEvalMaxL)
    k_evaluate_runs<<<grid_for((m + kEvalRun - 1) / kEvalRun, kWarpsPerBlock), kWarpsPerBlock * 32, 0,
                      as_stream(stream)>>>(*svh, *feat, alpha, xyz, m, f);
  else
    k_evaluate<false><<<grid, kWarpsPerBlock * 32, 0, as_stream(stream)>>>(*svh, *feat, alpha, xyz, m, false, f,
                                                                           grad);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_layer_mask(const nksr_svh_t* svh, const float* xyz, int64_t m, int adaptive_depth, float* out,
                    void* stream) {
  if (!svh || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH) return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  k_layer_mask<<<grid_for(m, 256), 256, 0, as_stream(stream)>>>(*svh, xyz, m, adaptive_depth, out);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
