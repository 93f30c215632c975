// Dual marching cubes with MISE refinement (SURVEY section 8 row a7).
// Replaces field.extract_dual_mesh(grid_upsample, mise_iter, max_points)
// (models/nksr_net.py:214,284; examples/recons_simple.py:27; examples/recons_colored_mesh.py:30).
//
// DESIGN.md SPEC S8-S10: lattice point s (int3, units W/R, R = grid_upsample * 2^mise_iter) sits
// at world position W*(0.5 + s/R), so voxel centres are lattice points s = R*ijk.  A cell is
// (min corner s, size).  Stage-0 cells = cubes spanned by 2x2x2 active finest voxels (the dual
// of the primal grid).  The host drives: corner keys -> sort/unique -> evaluate -> classify ->
// compact crossing cells -> split, and finally edges -> weld -> vertices + triangles.
#include <cub/cub.cuh>

#include "common.cuh"
#include "mc_tables.inc"

namespace {

__global__ void k_cell_flags(nksr_svh_t svh, int32_t* __restrict__ flag) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= svh.n[0]) return;
  const int32_t* nb = svh.nbr27[0] + i * 27;
  int ok = 1;
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    int s = (((c >> 2) & 1) + 1) * 9 + (((c >> 1) & 1) + 1) * 3 + ((c & 1) + 1);
    ok &= (__ldg(nb + s) >= 0);
  }
  flag[i] = ok;
}

__global__ void k_stage0_cells(nksr_svh_t svh, const int32_t* __restrict__ flag, const int64_t* __restrict__ scan,
                               int32_t refine, int32_t* __restrict__ cells) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= svh.n[0] || !flag[i]) return;
  int ux, uy, uz;
  morton3_decode(__ldg(svh.keys[0] + i), ux, uy, uz);
  const int off = level_offset(0);
  int64_t o = scan[i] * 3;
  cells[o] = (ux - off) * refine;
  cells[o + 1] = (uy - off) * refine;
  cells[o + 2] = (uz - off) * refine;
}

__global__ void k_split_cells(const int32_t* __restrict__ cells, int64_t n, int32_t sub, int32_t g,
                              int32_t* __restrict__ out) {
  const int g3 = g * g * g;
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n * g3) return;
  int64_t i = t / g3;
  int c = (int)(t - i * g3);
  int cx = c / (g * g), cy = (c / g) % g, cz = c % g;
  out[3 * t] = cells[3 * i] + cx * sub;
  out[3 * t + 1] = cells[3 * i + 1] + cy * sub;
  out[3 * t + 2] = cells[3 * i + 2] + cz * sub;
}

__global__ void k_corner_keys(const int32_t* __restrict__ cells, int64_t n, int32_t size, int ox, int oy, int oz,
                              int64_t* __restrict__ keys8) {
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n * 8) return;
  int64_t i = t >> 3;
  int c = (int)(t & 7);
  int x = cells[3 * i] - ox + ((c >> 2) & 1) * size;
  int y = cells[3 * i + 1] - oy + ((c >> 1) & 1) * size;
  int z = cells[3 * i + 2] - oz + (c & 1) * size;
  keys8[t] = morton3(x, y, z);
}

__global__ void k_lattice_pos(const int64_t* __restrict__ keys, int64_t n, int ox, int oy, int oz, float w,
                              float refine, float* __restrict__ xyz) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int x, y, z;
  morton3_decode(keys[i], x, y, z);
  // fp32, same op order as the oracle: W * (0.5 + s / R)
  xyz[3 * i] = __fmul_rn(w, __fadd_rn(0.5f, __fdiv_rn((float)(x + ox), refine)));
  xyz[3 * i + 1] = __fmul_rn(w, __fadd_rn(0.5f, __fdiv_rn((float)(y + oy), refine)));
  xyz[3 * i + 2] = __fmul_rn(w, __fadd_rn(0.5f, __fdiv_rn((float)(z + oz), refine)));
}

__global__ void k_classify(const int64_t* __restrict__ keys8, int64_t n_cells, const int64_t* __restrict__ ukeys,
                           const float* __restrict__ uval, int64_t n_u, float* __restrict__ cval8,
                           int32_t* __restrict__ mc_case, int32_t* __restrict__ crossing) {
  // one thread per corner; 8 consecutive lanes form a cell
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  const bool live = t < n_cells * 8;
  float v = 0.f;
  if (live) {
    int j = find_key(ukeys, n_u, keys8[t]);
    v = j >= 0 ? uval[j] : 0.f;
    cval8[t] = v;
  }
  unsigned bits = __ballot_sync(0xffffffffu, live && v > 0.f);
  if (live && (t & 7) == 0) {
    int lane = threadIdx.x & 31;
    int cs = (int)((bits >> lane) & 0xffu);
    mc_case[t >> 3] = cs;
    crossing[t >> 3] = (cs != 0 && cs != 255) ? 1 : 0;
  }
}

__global__ void k_compact_rows(const uint32_t* __restrict__ in, const int32_t* __restrict__ flag,
                               const int64_t* __restrict__ scan, int64_t n, int32_t words,
                               uint32_t* __restrict__ out) {
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n * words) return;
  int64_t i = t / words;
  int wq = (int)(t - i * words);
  if (flag[i]) out[scan[i] * words + wq] = in[t];
}

struct ToI64 {
  __host__ __device__ __forceinline__ int64_t operator()(const int32_t& v) const { return (int64_t)v; }
};

__global__ void k_scan_last(const int32_t* in, int64_t* out, int64_t n) {
  if (threadIdx.x == 0 && blockIdx.x == 0) out[n] = out[n - 1] + in[n - 1];
}

__global__ void k_cell_edges(const int32_t* __restrict__ cells, const int32_t* __restrict__ mc_case, int64_t n,
                             int32_t size, int ox, int oy, int oz, int32_t* __restrict__ ntri,
                             int64_t* __restrict__ ekeys) {
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n * 12) return;
  int64_t i = t / 12;
  int e = (int)(t - i * 12);
  const int cs = mc_case[i];
  const int a = c_mc_edges[e][0], b = c_mc_edges[e][1], ax = c_mc_edges[e][2];
  int64_t k = -1;
  if (((cs >> a) & 1) != ((cs >> b) & 1)) {
    int x = cells[3 * i] - ox + ((a >> 2) & 1) * size;
    int y = cells[3 * i + 1] - oy + ((a >> 1) & 1) * size;
    int z = cells[3 * i + 2] - oz + (a & 1) * size;
    k = (morton3(x, y, z) << 2) | ax;
  }
  ekeys[t] = k;
  if (e == 0) ntri[i] = c_mc_count[cs];
}

__global__ void k_run_heads(const int64_t* __restrict__ keys, int64_t n, int32_t* __restrict__ flag) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int64_t k = keys[i];
  flag[i] = (k >= 0 && (i == 0 || keys[i - 1] != k)) ? 1 : 0;
}

__global__ void k_vertices(const int64_t* __restrict__ uekeys, const int32_t* __restrict__ src, int64_t n_v,
                           const int32_t* __restrict__ cells, const float* __restrict__ cval8, int32_t size, float w,
                           float refine, float* __restrict__ v) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n_v) return;
  const int s = src[i];
  const int64_t cell = s / 12;
  const int e = s - (int)cell * 12;
  const int a = c_mc_edges[e][0], b = c_mc_edges[e][1], ax = c_mc_edges[e][2];
  const float fa = cval8[cell * 8 + a], fb = cval8[cell * 8 + b];
  int lx = cells[3 * cell] + ((a >> 2) & 1) * size;
  int ly = cells[3 * cell + 1] + ((a >> 1) & 1) * size;
  int lz = cells[3 * cell + 2] + (a & 1) * size;
  float p[3];
  p[0] = __fmul_rn(w, __fadd_rn(0.5f, __fdiv_rn((float)lx, refine)));
  p[1] = __fmul_rn(w, __fadd_rn(0.5f, __fdiv_rn((float)ly, refine)));
  p[2] = __fmul_rn(w, __fadd_rn(0.5f, __fdiv_rn((float)lz, refine)));
  const double tpar = (double)fa / ((double)fa - (double)fb);
  const double step = (double)__fdiv_rn(__fmul_rn(w, (float)size), refine);
  p[ax] = (float)((double)p[ax] + tpar * step);
  v[3 * i] = p[0];
  v[3 * i + 1] = p[1];
  v[3 * i + 2] = p[2];
}

__global__ void k_triangles(const int32_t* __restrict__ mc_case, const int64_t* __restrict__ ekeys,
                            const int64_t* __restrict__ tri_scan, int64_t n_cells,
                            const int64_t* __restrict__ uekeys, int64_t n_v, int64_t* __restrict__ tri) {
  // one thread per (cell, triangle slot 0..4)
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n_cells * 5) return;
  int64_t i = t / 5;
  int q = (int)(t - i * 5);
  const int cs = mc_case[i];
  if (q >= c_mc_count[cs]) return;
  int64_t o = (tri_scan[i] + q) * 3;
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    int e = c_mc_tri[cs][3 * q + j];
    tri[o + j] = find_key(uekeys, n_v, ekeys[i * 12 + e]);
  }
}


// ---- adaptive hierarchies (models/nksr_net.py:175-179,214): where a voxel of level l >= 1 is a LEAF (its children were
// pruned) the field is still defined, so the mesher treats the leaf as if it were subdivided down to the finest level:
// "virtual" finest voxels.  Dual cells are then cubes between the centres of 2x2x2 finest voxels, real or virtual --
// one family of cells on one lattice, hence no cracks and no duplicates across level transitions.
__global__ void k_leaf_flags(nksr_svh_t svh, int l, int32_t* __restrict__ flag) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= svh.n[l]) return;
  const int32_t* ch = svh.child8[l] + i * 8;
  int any = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) any |= (__ldg(ch + k) >= 0);
  flag[i] = !any;
}

// 8^l finest-level coordinates (ijk, not offset) below every flagged level-l voxel, x-major inside a leaf
__global__ void k_virtual_anchors(nksr_svh_t svh, int l, const int32_t* __restrict__ flag,
                                  const int64_t* __restrict__ scan, int32_t* __restrict__ out) {
  const int per = 1 << (3 * l);
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= svh.n[l] * (int64_t)per) return;
  const int64_t i = t >> (3 * l);
  if (!flag[i]) return;
  const int d = (int)(t & (per - 1));
  const int m = (1 << l) - 1;
  const int dx = d >> (2 * l), dy = (d >> l) & m, dz = d & m;
  int ux, uy, uz;
  morton3_decode(__ldg(svh.keys[l] + i), ux, uy, uz);
  const int off = level_offset(l);
  const int64_t o = (scan[i] * per + d) * 3;
  out[o] = ((ux - off) << l) + dx;
  out[o + 1] = ((uy - off) << l) + dy;
  out[o + 2] = ((uz - off) << l) + dz;
}

// finest voxel (x,y,z) exists: really, or virtually below a leaf of one of the levels 1 .. coarse-1
__device__ __forceinline__ bool voxel_exists(const nksr_svh_t& svh, int coarse, int x, int y, int z) {
  const int o0 = level_offset(0);
  if (find_key(svh.keys[0], svh.n[0], morton3(x + o0, y + o0, z + o0)) >= 0) return true;
  for (int l = 1; l < coarse; ++l) {
    const int o = level_offset(l);
    const int v = find_key(svh.keys[l], svh.n[l], morton3((x >> l) + o, (y >> l) + o, (z >> l) + o));
    if (v < 0) continue;
    const int32_t* ch = svh.child8[l] + (int64_t)v * 8;
    int any = 0;
#pragma unroll
    for (int k = 0; k < 8; ++k) any |= (__ldg(ch + k) >= 0);
    if (!any) return true;
  }
  return false;
}

__global__ void k_anchor_flags(nksr_svh_t svh, const int32_t* __restrict__ anchors, int64_t n, int coarse,
                               int32_t* __restrict__ flag) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int x = anchors[3 * i], y = anchors[3 * i + 1], z = anchors[3 * i + 2];
  int ok = 1;
  for (int c = 1; c < 8 && ok; ++c) ok &= voxel_exists(svh, coarse, x + ((c >> 2) & 1), y + ((c >> 1) & 1), z + (c & 1));
  flag[i] = ok;
}

}  // namespace

extern "C" {

int nksr_mesh_leaf_flags(const nksr_svh_t* svh, int level, int32_t* flag, void* stream) {
  if (!svh || level < 1 || level >= svh->depth || !svh->child8[level]) return NKSR_E_INVALID;
  if (svh->n[level] == 0) return NKSR_OK;
  k_leaf_flags<<<grid_for(svh->n[level], 256), 256, 0, as_stream(stream)>>>(*svh, level, flag);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

// (levels above 6 are refused: 8^7 anchors per leaf; meshing.py MAX_VIRTUAL_LEVEL states the same limit)
int nksr_mesh_virtual_anchors(const nksr_svh_t* svh, int level, const int32_t* flag, const int64_t* scan,
                              int32_t* anchors, void* stream) {
  if (!svh || level < 1 || level >= svh->depth || level > 6) return NKSR_E_INVALID;
  if (svh->n[level] == 0) return NKSR_OK;
  const int64_t work = svh->n[level] << (3 * level);
  k_virtual_anchors<<<grid_for(work, 256), 256, 0, as_stream(stream)>>>(*svh, level, flag, scan, anchors);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_anchor_flags(const nksr_svh_t* svh, const int32_t* anchors, int64_t n, int coarse_levels, int32_t* flag,
                           void* stream) {
  if (!svh || coarse_levels < 1 || coarse_levels > svh->depth) return NKSR_E_INVALID;
  for (int l = 1; l < coarse_levels; ++l)
    if (!svh->child8[l]) return NKSR_E_INVALID;
  if (n == 0) return NKSR_OK;
  k_anchor_flags<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(*svh, anchors, n, coarse_levels, flag);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_cell_flags(const nksr_svh_t* svh, int32_t* flag, void* stream) {
  if (!svh || svh->depth < 1) return NKSR_E_INVALID;
  if (svh->n[0] == 0) return NKSR_OK;
  k_cell_flags<<<grid_for(svh->n[0], 256), 256, 0, as_stream(stream)>>>(*svh, flag);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_stage0_cells(const nksr_svh_t* svh, const int32_t* flag, const int64_t* scan, int32_t refine,
                           int32_t* cells, void* stream) {
  if (!svh || svh->depth < 1 || refine < 1) return NKSR_E_INVALID;
  if (svh->n[0] == 0) return NKSR_OK;
  k_stage0_cells<<<grid_for(svh->n[0], 256), 256, 0, as_stream(stream)>>>(*svh, flag, scan, refine, cells);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_split_cells(const int32_t* cells, int64_t n, int32_t size, int32_t g, int32_t* out, void* stream) {
  if (g < 1 || size % g) return NKSR_E_INVALID;
  if (n == 0) return NKSR_OK;
  k_split_cells<<<grid_for(n * g * g * g, 256), 256, 0, as_stream(stream)>>>(cells, n, size / g, g, out);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_corner_keys(const int32_t* cells, int64_t n, int32_t size, int32_t ox, int32_t oy, int32_t oz,
                          int64_t* keys8, void* stream) {
  if (n == 0) return NKSR_OK;
  k_corner_keys<<<grid_for(n * 8, 256), 256, 0, as_stream(stream)>>>(cells, n, size, ox, oy, oz, keys8);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_lattice_pos(const int64_t* keys, int64_t n, int32_t ox, int32_t oy, int32_t oz, float voxel_size,
                          int32_t refine, float* xyz, void* stream) {
  if (n == 0) return NKSR_OK;
  k_lattice_pos<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(keys, n, ox, oy, oz, voxel_size, (float)refine,
                                                                  xyz);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_classify(const int64_t* keys8, int64_t n_cells, const int64_t* ukeys, const float* uval, int64_t n_u,
                       float* cval8, int32_t* mc_case, int32_t* crossing, void* stream) {
  if (n_cells == 0) return NKSR_OK;
  k_classify<<<grid_for(n_cells * 8, 256), 256, 0, as_stream(stream)>>>(keys8, n_cells, ukeys, uval, n_u, cval8,
                                                                         mc_case, crossing);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_compact_rows(const void* in, const int32_t* flag, const int64_t* scan, int64_t n, int32_t row_bytes,
                      void* out, void* stream) {
  if (row_bytes <= 0 || (row_bytes & 3)) return NKSR_E_INVALID;
  if (n == 0) return NKSR_OK;
  const int words = row_bytes / 4;
  k_compact_rows<<<grid_for(n * words, 256), 256, 0, as_stream(stream)>>>(
      reinterpret_cast<const uint32_t*>(in), flag, scan, n, words, reinterpret_cast<uint32_t*>(out));
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

size_t nksr_scan32_workspace_bytes(int64_t n) {
  size_t bytes = 0;
  cub::TransformInputIterator<int64_t, ToI64, const int32_t*> it((const int32_t*)nullptr, ToI64());
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, it, (int64_t*)nullptr, n);
  return bytes + 256;
}

int nksr_exclusive_scan32(const int32_t* in, int64_t* out, int64_t n, void* ws, size_t ws_bytes, void* stream) {
  if (n < 0) return NKSR_E_INVALID;
  if (n == 0) {
    cudaMemsetAsync(out, 0, sizeof(int64_t), as_stream(stream));
    return NKSR_OK;
  }
  cub::TransformInputIterator<int64_t, ToI64, const int32_t*> it(in, ToI64());
  size_t need = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, need, it, out, n);
  if (need > ws_bytes) return NKSR_E_WORKSPACE;
  if (cub::DeviceScan::ExclusiveSum(ws, need, it, out, n, as_stream(stream)) != cudaSuccess) return NKSR_E_CUDA;
  k_scan_last<<<1, 32, 0, as_stream(stream)>>>(in, out, n);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_cell_edges(const int32_t* cells, const int32_t* mc_case, int64_t n, int32_t size, int32_t ox,
                         int32_t oy, int32_t oz, int32_t* ntri, int64_t* ekeys12, void* stream) {
  if (n == 0) return NKSR_OK;
  k_cell_edges<<<grid_for(n * 12, 256), 256, 0, as_stream(stream)>>>(cells, mc_case, n, size, ox, oy, oz, ntri,
                                                                      ekeys12);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_run_heads(const int64_t* keys, int64_t n, int32_t* flag, void* stream) {
  if (n == 0) return NKSR_OK;
  k_run_heads<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(keys, n, flag);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_vertices(const int64_t* uekeys, const int32_t* src, int64_t n_v, const int32_t* cells,
                       const float* cval8, int32_t size, float voxel_size, int32_t refine, float* v, void* stream) {
  if (n_v == 0) return NKSR_OK;
  k_vertices<<<grid_for(n_v, 256), 256, 0, as_stream(stream)>>>(uekeys, src, n_v, cells, cval8, size, voxel_size,
                                                                 (float)refine, v);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_triangles(const int32_t* mc_case, const int64_t* ekeys12, const int64_t* tri_scan, int64_t n_cells,
                        const int64_t* uekeys, int64_t n_v, int64_t* tri, void* stream) {
  if (n_cells == 0) return NKSR_OK;
  k_triangles<<<grid_for(n_cells * 5, 256), 256, 0, as_stream(stream)>>>(mc_case, ekeys12, tri_scan, n_cells, uekeys,
                                                                         n_v, tri);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
