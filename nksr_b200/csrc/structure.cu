// The structure-grown decoder hierarchy (DESIGN.md SPEC S16): classify the voxels of one level from the structure
// head's logits (or forced classes), then emit the children of the subdivided voxels with their tables.  The
// reference's decoder grows dec_tmp_svh the same way (models/nksr_net.py:74-86).  Integer work only: no atomics and no
// sort; children come out in (parent, octant) order, which is already Morton-sorted and unique.
#include "common.cuh"

namespace {

// argmax with torch.argmax semantics: the first index wins a tie, a NaN counts as larger than every number (the
// first NaN wins among NaNs)
__device__ __forceinline__ int argmax3(float a, float b, float c) {
  int best = 0;
  float bv = a;
  if (!isnan(bv) && (isnan(b) || b > bv)) { best = 1; bv = b; }
  if (!isnan(bv) && (isnan(c) || c > bv)) { best = 2; }
  return best;
}

__global__ void k_structure_classify(const float* __restrict__ logits, int64_t row_stride,
                                     const int32_t* __restrict__ forced, int64_t n, int level, int adaptive_depth,
                                     int8_t* __restrict__ cls, int32_t* __restrict__ keep, int32_t* __restrict__ sub) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int c;
  if (forced) {
    c = __ldg(forced + i);
  } else {
    const float* r = logits + i * row_stride;
    c = argmax3(__ldg(r), __ldg(r + 1), __ldg(r + 2));
  }
  cls[i] = (int8_t)c;
  keep[i] = c >= 1;
  sub[i] = level >= 1 && (c == 2 || (c == 1 && level >= adaptive_depth));
}

// one thread per (voxel of level l, octant o): child c = 8 scan[i] + o of a subdivided voxel i gets key (key << 3) | o,
// parent i and join E.child8[l][join[i]][o]; child8[i][o] = c, or -1 for a voxel that is not subdivided
__global__ void k_structure_grow(const int64_t* __restrict__ keys, const int32_t* __restrict__ sub,
                                 const int64_t* __restrict__ sub_scan, int64_t n, const int32_t* __restrict__ join,
                                 const int32_t* __restrict__ enc_child8, int64_t* __restrict__ child_keys,
                                 int32_t* __restrict__ child_parent, int32_t* __restrict__ child_join,
                                 int32_t* __restrict__ child8) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= n * 8) return;
  const int64_t i = t >> 3;
  const int o = (int)(t & 7);
  if (!__ldg(sub + i)) {
    child8[t] = -1;
    return;
  }
  const int64_t c = __ldg(sub_scan + i) * 8 + o;
  child8[t] = (int32_t)c;
  child_keys[c] = (__ldg(keys + i) << 3) | o;
  child_parent[c] = (int32_t)i;
  const int j = __ldg(join + i);
  child_join[c] = (j >= 0 && enc_child8) ? __ldg(enc_child8 + (int64_t)j * 8 + o) : -1;
}

__global__ void k_compose_taps(const int32_t* __restrict__ idx, int64_t total, const int32_t* __restrict__ map,
                               int32_t* __restrict__ out) {
  const int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int v = __ldg(idx + t);
  out[t] = v < 0 ? -1 : __ldg(map + v);
}

}  // namespace

extern "C" {

int nksr_structure_classify(const float* logits, int64_t row_stride, const int32_t* forced, int64_t n, int level,
                            int adaptive_depth, int8_t* cls, int32_t* keep, int32_t* sub, void* stream) {
  if (n < 0 || level < 0 || level >= NKSR_MAX_DEPTH) return NKSR_E_INVALID;
  if (n == 0) return NKSR_OK;
  if (!forced && (!logits || row_stride < 3)) return NKSR_E_INVALID;
  k_structure_classify<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(logits, row_stride, forced, n, level,
                                                                          adaptive_depth, cls, keep, sub);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_structure_grow(const int64_t* keys, const int32_t* sub, const int64_t* sub_scan, int64_t n,
                        const int32_t* join, const int32_t* enc_child8, int64_t* child_keys, int32_t* child_parent,
                        int32_t* child_join, int32_t* child8, void* stream) {
  if (n < 0) return NKSR_E_INVALID;
  if (n == 0) return NKSR_OK;
  k_structure_grow<<<grid_for(n * 8, 256), 256, 0, as_stream(stream)>>>(keys, sub, sub_scan, n, join, enc_child8,
                                                                         child_keys, child_parent, child_join, child8);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_compose_taps(const int32_t* idx, int64_t n, int K, const int32_t* map, int32_t* out, void* stream) {
  if (n < 0 || K < 1) return NKSR_E_INVALID;
  if (n == 0) return NKSR_OK;
  k_compose_taps<<<grid_for(n * K, 256), 256, 0, as_stream(stream)>>>(idx, n * K, map, out);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
