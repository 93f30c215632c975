// Sparse voxel hierarchy construction (SURVEY section 8 row a1).
// Replaces nksr.SparseFeatureHierarchy.build_point_splatting (models/nksr_net.py:57-62) and the
// grid accessors used at models/loss.py:33-46.  Integer work only: results are bit-exact
// against oracle/nksr_oracle.py (OracleSVH).
#include <cub/cub.cuh>

#include "common.cuh"

namespace {

__global__ void k_point_half_keys(const float* __restrict__ xyz, int64_t n, float half_w,
                                  int64_t* __restrict__ keys, int32_t* __restrict__ status) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int3 h;
  if (!half_voxel(__ldg(xyz + 3 * i), __ldg(xyz + 3 * i + 1), __ldg(xyz + 3 * i + 2), half_w, h)) atomicOr(status, 1);
  keys[i] = morton3(h.x, h.y, h.z);
}

struct ShiftOp {
  int shift;
  __host__ __device__ __forceinline__ int64_t operator()(const int64_t& k) const { return k >> shift; }
};

__global__ void k_splat_candidates(const int64_t* __restrict__ hk, int64_t n, int64_t* __restrict__ out) {
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n * 8) return;
  int64_t i = t >> 3;
  int a = (int)(t & 7);
  int hx, hy, hz;
  morton3_decode(__ldg(hk + i), hx, hy, hz);
  // base = (h-1)>>1 in offset space (offset 2^(20-l) is even), then the 8 nearest centres
  int bx = ((hx - 1) >> 1) + ((a >> 2) & 1);
  int by = ((hy - 1) >> 1) + ((a >> 1) & 1);
  int bz = ((hz - 1) >> 1) + (a & 1);
  out[t] = morton3(bx, by, bz);
}

__global__ void k_parent_index(const int64_t* __restrict__ keys, int64_t n, const int64_t* __restrict__ keys_up,
                               int64_t n_up, int32_t* __restrict__ parent, int32_t* __restrict__ status) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int p = find_key(keys_up, n_up, __ldg(keys + i) >> 3);
  if (p < 0) atomicOr(status, 2);
  parent[i] = p;
}

__global__ void k_child_table(const int64_t* __restrict__ keys, const int32_t* __restrict__ parent, int64_t n,
                              int32_t* __restrict__ child8_up) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int p = parent[i];
  if (p >= 0) child8_up[(int64_t)p * 8 + (int)(keys[i] & 7)] = (int32_t)i;
}

__global__ void k_nbr27_search(const int64_t* __restrict__ keys, int64_t n, int32_t* __restrict__ nbr) {
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n * 27) return;
  int64_t i = t / 27;
  int s = (int)(t - i * 27);
  int ux, uy, uz, dx, dy, dz;
  morton3_decode(__ldg(keys + i), ux, uy, uz);
  slot_to_d(s, dx, dy, dz);
  ux += dx; uy += dy; uz += dz;
  int r = -1;
  if (ux >= 0 && uy >= 0 && uz >= 0 && ux < NKSR_KEY_LIMIT && uy < NKSR_KEY_LIMIT && uz < NKSR_KEY_LIMIT)
    r = find_key(keys, n, morton3(ux, uy, uz));
  nbr[t] = r;
}

__global__ void k_nbr125_search(const int64_t* __restrict__ keys, int64_t n, int32_t* __restrict__ nbr) {
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n * 125) return;
  int64_t i = t / 125;
  int s = (int)(t - i * 125);
  int ux, uy, uz;
  morton3_decode(__ldg(keys + i), ux, uy, uz);
  ux += s / 25 - 2; uy += (s / 5) % 5 - 2; uz += s % 5 - 2;
  int r = -1;
  if (ux >= 0 && uy >= 0 && uz >= 0 && ux < NKSR_KEY_LIMIT && uy < NKSR_KEY_LIMIT && uz < NKSR_KEY_LIMIT)
    r = find_key(keys, n, morton3(ux, uy, uz));
  nbr[t] = r;
}

__global__ void k_nbr27_from_parent(const int64_t* __restrict__ keys, const int32_t* __restrict__ parent, int64_t n,
                                    const int32_t* __restrict__ nbr_up, const int32_t* __restrict__ child8_up,
                                    int32_t* __restrict__ nbr) {
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n * 27) return;
  int64_t i = t / 27;
  int s = (int)(t - i * 27);
  int ux, uy, uz, dx, dy, dz;
  morton3_decode(__ldg(keys + i), ux, uy, uz);
  slot_to_d(s, dx, dy, dz);
  int nx = ux + dx, ny = uy + dy, nz = uz + dz;
  int ex = (nx >> 1) - (ux >> 1), ey = (ny >> 1) - (uy >> 1), ez = (nz >> 1) - (uz >> 1);
  int p = __ldg(parent + i);
  int r = -1;
  if (p >= 0) {
    int pn = __ldg(nbr_up + (int64_t)p * 27 + (ex + 1) * 9 + (ey + 1) * 3 + (ez + 1));
    if (pn >= 0) r = __ldg(child8_up + (int64_t)pn * 8 + (((nx & 1) << 2) | ((ny & 1) << 1) | (nz & 1)));
  }
  nbr[t] = r;
}

__global__ void k_decode_ijk(const int64_t* __restrict__ keys, int64_t n, int off, int32_t* __restrict__ ijk) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int ux, uy, uz;
  morton3_decode(keys[i], ux, uy, uz);
  ijk[3 * i + 0] = ux - off;
  ijk[3 * i + 1] = uy - off;
  ijk[3 * i + 2] = uz - off;
}

// containing voxel on every level: search the coarsest level, then walk child8 down
__global__ void k_locate(nksr_svh_t svh, const float* __restrict__ xyz, int64_t m, float half_w,
                         int32_t* __restrict__ base) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= m) return;
  int3 h;
  const bool ok = half_voxel(__ldg(xyz + 3 * i), __ldg(xyz + 3 * i + 1), __ldg(xyz + 3 * i + 2), half_w, h);
  const int L = svh.depth;
  int idx = -1;
  if (ok && svh.n[L - 1] > 0) idx = find_key(svh.keys[L - 1], svh.n[L - 1], morton3(h.x >> L, h.y >> L, h.z >> L));
  base[(int64_t)(L - 1) * m + i] = idx;
  for (int l = L - 2; l >= 0; --l) {
    if (idx >= 0) idx = __ldg(svh.child8[l + 1] + (int64_t)idx * 8 + child_octant(h, l + 1));
    base[(int64_t)l * m + i] = idx;
  }
}

// out[i][c] = sum over the active 27-neighbourhood of in[nb][c]; one warp per voxel, lane = slot
__global__ void k_pool27(const int32_t* __restrict__ nbr27, const float* __restrict__ in, int64_t n, int channels,
                         float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t i = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= n) return;
  const int nb = lane < 27 ? __ldg(nbr27 + i * 27 + lane) : -1;
  for (int c = 0; c < channels; ++c) {
    float v = nb >= 0 ? __ldg(in + (int64_t)nb * channels + c) : 0.f;
    v = warp_sum(v);
    if (lane == 0) out[i * channels + c] = v;
  }
}

// out[p][c] = sum over the (<= 8) children of voxel p of in[child][c]
__global__ void k_pool_children(const int32_t* __restrict__ child8, const float* __restrict__ in, int64_t n,
                                int channels, float* __restrict__ out) {
  int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n * channels) return;
  const int64_t p = t / channels;
  const int c = (int)(t - p * channels);
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int ch = __ldg(child8 + p * 8 + j);
    if (ch >= 0) s += __ldg(in + (int64_t)ch * channels + c);
  }
  out[t] = s;
}

__global__ void k_row_ranges(const int32_t* __restrict__ base, int64_t m, int32_t* __restrict__ range) {
  int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= m) return;
  int b = base[i];
  if (b < 0) return;
  if (i == 0 || base[i - 1] != b) range[2 * (int64_t)b] = (int32_t)i;
  if (i == m - 1 || base[i + 1] != b) range[2 * (int64_t)b + 1] = (int32_t)(i + 1);
}

}  // namespace

extern "C" {

const char* nksr_version(void) { return "nksr_b200 0.1 (sm_90a)"; }

const char* nksr_error_string(int code) {
  switch (code) {
    case NKSR_OK: return "ok";
    case NKSR_E_INVALID: return "invalid argument";
    case NKSR_E_RANGE: return "coordinate outside the supported voxel range";
    case NKSR_E_WORKSPACE: return "workspace too small";
    case NKSR_E_CUDA: return "CUDA error";
    case NKSR_E_STRUCTURE: return "hierarchy structure error";
    default: return "unknown error";
  }
}

int nksr_point_half_keys(const float* xyz, int64_t n, float voxel_size, int64_t* keys, int32_t* status,
                         void* stream) {
  if (n < 0 || !(voxel_size > 0.f)) return NKSR_E_INVALID;
  if (n == 0) return NKSR_OK;
  float half_w = voxel_size * 0.5f;
  k_point_half_keys<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(xyz, n, half_w, keys, status);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

size_t nksr_sort_workspace_bytes(int64_t n, int pairs) {
  size_t bytes = 0;
  if (pairs)
    cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const int64_t*)nullptr, (int64_t*)nullptr,
                                    (const int32_t*)nullptr, (int32_t*)nullptr, n);
  else
    cub::DeviceRadixSort::SortKeys(nullptr, bytes, (const int64_t*)nullptr, (int64_t*)nullptr, n);
  return bytes + 256;
}

int nksr_sort_keys(const int64_t* keys_in, int64_t* keys_out, int64_t n, void* ws, size_t ws_bytes, void* stream) {
  if (n == 0) return NKSR_OK;
  size_t need = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, need, keys_in, keys_out, n);
  if (need > ws_bytes) return NKSR_E_WORKSPACE;
  // keys are non-negative 63-bit Morton codes: sort bits [0,63)
  if (cub::DeviceRadixSort::SortKeys(ws, need, keys_in, keys_out, n, 0, 63, as_stream(stream)) != cudaSuccess)
    return NKSR_E_CUDA;
  return NKSR_OK;
}

int nksr_sort_pairs(const int64_t* keys_in, int64_t* keys_out, const int32_t* vals_in, int32_t* vals_out, int64_t n,
                    void* ws, size_t ws_bytes, void* stream) {
  if (n == 0) return NKSR_OK;
  size_t need = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, need, keys_in, keys_out, vals_in, vals_out, n);
  if (need > ws_bytes) return NKSR_E_WORKSPACE;
  if (cub::DeviceRadixSort::SortPairs(ws, need, keys_in, keys_out, vals_in, vals_out, n, 0, 63,
                                      as_stream(stream)) != cudaSuccess)
    return NKSR_E_CUDA;
  return NKSR_OK;
}

size_t nksr_unique_workspace_bytes(int64_t n) {
  size_t bytes = 0;
  cub::TransformInputIterator<int64_t, ShiftOp, const int64_t*> it((const int64_t*)nullptr, ShiftOp{0});
  cub::DeviceSelect::Unique(nullptr, bytes, it, (int64_t*)nullptr, (int64_t*)nullptr, n);
  return bytes + 256;
}

int nksr_unique_sorted(const int64_t* in, int64_t n, int shift, int64_t* out, int64_t* count_out, void* ws,
                       size_t ws_bytes, void* stream) {
  if (n < 0 || shift < 0 || shift > 62) return NKSR_E_INVALID;
  if (n == 0) {
    cudaMemsetAsync(count_out, 0, sizeof(int64_t), as_stream(stream));
    return NKSR_OK;
  }
  cub::TransformInputIterator<int64_t, ShiftOp, const int64_t*> it(in, ShiftOp{shift});
  size_t need = 0;
  cub::DeviceSelect::Unique(nullptr, need, it, out, count_out, n);
  if (need > ws_bytes) return NKSR_E_WORKSPACE;
  if (cub::DeviceSelect::Unique(ws, need, it, out, count_out, n, as_stream(stream)) != cudaSuccess)
    return NKSR_E_CUDA;
  return NKSR_OK;
}

int nksr_splat_candidates(const int64_t* half_keys, int64_t n, int64_t* out8, void* stream) {
  if (n == 0) return NKSR_OK;
  k_splat_candidates<<<grid_for(n * 8, 256), 256, 0, as_stream(stream)>>>(half_keys, n, out8);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_parent_index(const int64_t* keys, int64_t n, const int64_t* keys_up, int64_t n_up, int32_t* parent,
                      int32_t* status, void* stream) {
  if (n == 0) return NKSR_OK;
  k_parent_index<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(keys, n, keys_up, n_up, parent, status);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_child_table(const int64_t* keys, const int32_t* parent, int64_t n, int32_t* child8_up, int64_t n_up,
                     void* stream) {
  if (cudaMemsetAsync(child8_up, 0xFF, (size_t)n_up * 8 * sizeof(int32_t), as_stream(stream)) != cudaSuccess)
    return NKSR_E_CUDA;
  if (n == 0) return NKSR_OK;
  k_child_table<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(keys, parent, n, child8_up);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_nbr27_search(const int64_t* keys, int64_t n, int32_t* nbr27, void* stream) {
  if (n == 0) return NKSR_OK;
  k_nbr27_search<<<grid_for(n * 27, 256), 256, 0, as_stream(stream)>>>(keys, n, nbr27);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_nbr125_search(const int64_t* keys, int64_t n, int32_t* nbr125, void* stream) {
  if (n == 0) return NKSR_OK;
  k_nbr125_search<<<grid_for(n * 125, 256), 256, 0, as_stream(stream)>>>(keys, n, nbr125);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_nbr27_from_parent(const int64_t* keys, const int32_t* parent, int64_t n, const int32_t* nbr27_up,
                           const int32_t* child8_up, int32_t* nbr27, void* stream) {
  if (n == 0) return NKSR_OK;
  k_nbr27_from_parent<<<grid_for(n * 27, 256), 256, 0, as_stream(stream)>>>(keys, parent, n, nbr27_up, child8_up,
                                                                              nbr27);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_decode_ijk(const int64_t* keys, int64_t n, int level, int32_t* ijk, void* stream) {
  if (level < 0 || level >= NKSR_MAX_DEPTH) return NKSR_E_INVALID;
  if (n == 0) return NKSR_OK;
  k_decode_ijk<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(keys, n, level_offset(level), ijk);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_locate(const nksr_svh_t* svh, const float* xyz, int64_t m, int32_t* base, void* stream) {
  if (!svh || svh->depth < 1 || svh->depth > NKSR_MAX_DEPTH) return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  k_locate<<<grid_for(m, 256), 256, 0, as_stream(stream)>>>(*svh, xyz, m, svh->voxel_size * 0.5f, base);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_pool27(const int32_t* nbr27, const float* in, int64_t n, int channels, float* out, void* stream) {
  if (channels < 1) return NKSR_E_INVALID;
  if (n == 0) return NKSR_OK;
  k_pool27<<<grid_for(n, 8), 256, 0, as_stream(stream)>>>(nbr27, in, n, channels, out);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_pool_children(const int32_t* child8, const float* in, int64_t n, int channels, float* out, void* stream) {
  if (channels < 1) return NKSR_E_INVALID;
  if (n == 0) return NKSR_OK;
  k_pool_children<<<grid_for(n * channels, 256), 256, 0, as_stream(stream)>>>(child8, in, n, channels, out);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_row_ranges(const int32_t* base_l, int64_t m, int32_t* range, int64_t n_l, void* stream) {
  if (cudaMemsetAsync(range, 0, (size_t)n_l * 2 * sizeof(int32_t), as_stream(stream)) != cudaSuccess)
    return NKSR_E_CUDA;
  if (m == 0) return NKSR_OK;
  k_row_ranges<<<grid_for(m, 256), 256, 0, as_stream(stream)>>>(base_l, m, range);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
