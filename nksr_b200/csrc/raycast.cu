// Mesh occupancy by ray parity (the evaluator's 'o3d-iou'; DESIGN.md SPEC S20): an LBVH over the triangles and one
// traversal kernel that counts the crossings of K rays per query.
//
// Build: k_bvh_bounds (centroid box and the largest |vertex coordinate|) -> k_bvh_keys (63-bit Morton keys of the
// centroids) -> nksr_sort_pairs (the caller) -> k_bvh_hierarchy (Karras, HPG 2012: one thread per internal node, ties
// between equal keys broken by index) -> k_bvh_refit (one thread per leaf, bottom-up with per-node arrival flags; min /
// max does not depend on the arrival order, so the boxes are deterministic).  One triangle per leaf; every internal
// node stores its two child boxes and child codes (64 B), and the triangles are copied in leaf order (48 B each), their vertices in lexicographic order.
//
// Query: k_mesh_occupancy, one thread per query, the K directions in turn, every crossing counted (no early exit, so
// the traversal order does not matter).  The box test is conservative with respect to the exact triangle test: boxes
// are padded by delta(q) = 2^-19 (M + |q|_inf), which bounds every rounding of the sheared frame, and the slab test
// inflates its far distance as in Ize, "Robust BVH Ray Traversal" (JCGT 2013).  So the count, and the occupancy, is
// the brute-force rule's bit for bit.
//
// Distance: k_mesh_closest, one thread per query, best-first over the same LBVH (nearer child first, the farther one
// pushed with its bound).  SPEC S21's point-triangle routine gives each triangle's closest point; a child box is
// skipped only when its padded lower bound is strictly above the best squared distance so far, and the bound never
// exceeds the routine's d2 of any triangle inside, so the answer, ties to the lower original index included, is the
// brute force's bit for bit.
//
// First hit: k_mesh_first_hit, one thread per ray (its own origin, direction and t_max), nearest-entry-first over the
// same LBVH.  SPEC S22's candidates are S20's crossings, each at t = T / det; a child box is skipped only when its
// padded slab entry is strictly above the best t so far or t_max, and that entry never exceeds the t of a candidate
// inside, so the hit, ties to the lower original index included, is the brute force's bit for bit.
//
// Built with --fmad=false: the rules round every fp32 and fp64 product and sum on their own (SPEC S20, S21).
#include "common.cuh"

namespace {

constexpr int kBvhThreads = 256;
constexpr int kOccThreads = 128;
// Karras depth bound: a child's range shares strictly more leading bits of the (63-bit key, 31-bit index) pair than
// its parent's, so a root-to-leaf path has at most 95 internal nodes and the stack (one entry per level) at most 95
constexpr int kStack = 96;
constexpr int kMaxRays = 9;

// The default ray directions of SPEC S20 (the first K are used): no zero component, no two components of equal
// magnitude, no component below 0.15 in magnitude.  oracle/metrics.py states the same list.
__constant__ float kDefaultDirs[kMaxRays][3] = {
    {-0x1.8815a2p-3f, 0x1.480a34p-1f, 0x1.7cb0ecp-1f},
    {0x1.c613e2p-2f, 0x1.286306p-1f, -0x1.5e5c32p-1f},
    {-0x1.3433a6p-2f, -0x1.42e6aap-3f, -0x1.e18a22p-1f},
    {0x1.2ed1f8p-1f, -0x1.69843ep-1f, -0x1.8ebf20p-2f},
    {-0x1.9f3f84p-1f, 0x1.c1902cp-3f, 0x1.15a29ep-1f},
    {0x1.ac4238p-2f, -0x1.62a6b6p-1f, -0x1.2cdb7cp-1f},
    {-0x1.b7da02p-1f, 0x1.3c78c4p-3f, 0x1.f3a8dap-2f},
    {0x1.3037d2p-2f, -0x1.35be2ep-1f, 0x1.7a3dacp-1f},
    {-0x1.1448b4p-1f, -0x1.78b382p-1f, -0x1.a314ecp-2f},
};

// order-preserving float <-> uint for atomic min / max
__device__ __forceinline__ unsigned f2o(float x) {
  const unsigned u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float o2f(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__device__ __forceinline__ void load_tri(const float* __restrict__ v, const int32_t* __restrict__ f, int64_t t,
                                         float p[3][3]) {
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const int64_t i = __ldg(f + 3 * t + c);
#pragma unroll
    for (int k = 0; k < 3; ++k) p[c][k] = __ldg(v + 3 * i + k);
  }
}

__device__ __forceinline__ float centroid(const float p[3][3], int k) { return (p[0][k] + p[1][k] + p[2][k]) * (1.f / 3.f); }

// scene[0..5] (centroid lo xyz, hi xyz) and scene[6] (max |vertex coordinate|) as ordered uints, pre-set by k_bvh_scene_init
__global__ void __launch_bounds__(kBvhThreads)
k_bvh_bounds(const float* __restrict__ v, const int32_t* __restrict__ f, const int64_t n_tri,
             unsigned* __restrict__ scene) {
  float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f}, mx = 0.f;
  for (int64_t t = blockIdx.x * (int64_t)kBvhThreads + threadIdx.x; t < n_tri; t += (int64_t)gridDim.x * kBvhThreads) {
    float p[3][3];
    load_tri(v, f, t, p);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const float c = centroid(p, k);
      lo[k] = fminf(lo[k], c);
      hi[k] = fmaxf(hi[k], c);
      mx = fmaxf(mx, fmaxf(fabsf(p[0][k]), fmaxf(fabsf(p[1][k]), fabsf(p[2][k]))));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      lo[k] = fminf(lo[k], __shfl_xor_sync(0xffffffffu, lo[k], o));
      hi[k] = fmaxf(hi[k], __shfl_xor_sync(0xffffffffu, hi[k], o));
    }
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      atomicMin(scene + k, f2o(lo[k]));
      atomicMax(scene + 3 + k, f2o(hi[k]));
    }
    atomicMax(scene + 6, f2o(mx));
  }
}

__device__ __forceinline__ uint64_t spread21(uint64_t x) {
  x &= 0x1fffffull;
  x = (x | x << 32) & 0x1f00000000ffffull;
  x = (x | x << 16) & 0x1f0000ff0000ffull;
  x = (x | x << 8) & 0x100f00f00f00f00full;
  x = (x | x << 4) & 0x10c30c30c30c30c3ull;
  x = (x | x << 2) & 0x1249249249249249ull;
  return x;
}

// keys[t] = 63-bit Morton code of triangle t's centroid in the centroid box (21 bits per axis), idx[t] = t;
// k_bvh_scene_floats then turns scene back into floats for the queries
__global__ void __launch_bounds__(kBvhThreads)
k_bvh_keys(const float* __restrict__ v, const int32_t* __restrict__ f, const int64_t n_tri,
           const unsigned* __restrict__ scene, int64_t* __restrict__ keys, int32_t* __restrict__ idx) {
  const int64_t t = blockIdx.x * (int64_t)kBvhThreads + threadIdx.x;
  if (t >= n_tri) return;
  float p[3][3];
  load_tri(v, f, t, p);
  uint64_t key = 0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float lo = o2f(__ldg(scene + k)), ext = o2f(__ldg(scene + 3 + k)) - lo;
    const float s = ext > 0.f ? (centroid(p, k) - lo) / ext : 0.f;
    const float q = fminf(fmaxf(s, 0.f), 1.f) * 2097151.f;
    key |= spread21((uint64_t)q) << (2 - k);
  }
  keys[t] = (int64_t)key;
  idx[t] = (int32_t)t;
}

__global__ void k_bvh_scene_init(unsigned* __restrict__ scene) {
  const int k = threadIdx.x;
  if (k < 8) scene[k] = k < 3 ? 0xffffffffu : 0u;
}

__global__ void k_bvh_scene_floats(unsigned* __restrict__ scene) {
  const int k = threadIdx.x;
  if (k < 7) scene[k] = __float_as_uint(o2f(scene[k]));
}

// common prefix length of the (key, index) pairs i and j; -1 outside [0, n)
__device__ __forceinline__ int delta(const int64_t* __restrict__ keys, const int64_t n, const int64_t i,
                                     const int64_t j) {
  if (j < 0 || j >= n) return -1;
  const uint64_t a = (uint64_t)__ldg(keys + i), b = (uint64_t)__ldg(keys + j);
  if (a != b) return __clzll((long long)(a ^ b));
  return 64 + __clz((int)((uint32_t)i ^ (uint32_t)j));
}

// node layout (16 floats): [lo0 xyz, child0] [hi0 xyz, child1] [lo1 xyz, 0] [hi1 xyz, 0]; child >= 0: internal node,
// child < 0: leaf ~child (the triangle at that position of the leaf order).  parent: int32[2 n - 1], internal nodes
// first, then the leaves; the root (node 0) has -1.
__global__ void __launch_bounds__(kBvhThreads)
k_bvh_hierarchy(const int64_t* __restrict__ keys, const int64_t n, float* __restrict__ nodes,
                int32_t* __restrict__ parent) {
  const int64_t i = blockIdx.x * (int64_t)kBvhThreads + threadIdx.x;
  if (i >= n - 1) return;
  const int d = delta(keys, n, i, i + 1) - delta(keys, n, i, i - 1) > 0 ? 1 : -1;
  const int dmin = delta(keys, n, i, i - d);
  int64_t lmax = 2;
  while (delta(keys, n, i, i + lmax * d) > dmin) lmax <<= 1;
  int64_t l = 0;
  for (int64_t s = lmax >> 1; s > 0; s >>= 1)
    if (delta(keys, n, i, i + (l + s) * d) > dmin) l += s;
  const int64_t j = i + l * d;
  const int dnode = delta(keys, n, i, j);
  int64_t s = 0;
  for (int64_t step = l;;) {
    step = (step + 1) >> 1;
    if (delta(keys, n, i, i + (s + step) * d) > dnode) s += step;
    if (step <= 1) break;
  }
  const int64_t g = i + s * d + (d < 0 ? -1 : 0);
  const int64_t first = i < j ? i : j, last = i < j ? j : i;
  const int32_t left = first == g ? ~(int32_t)g : (int32_t)g;
  const int32_t right = last == g + 1 ? ~(int32_t)(g + 1) : (int32_t)(g + 1);
  nodes[16 * i + 3] = __int_as_float(left);
  nodes[16 * i + 7] = __int_as_float(right);
  nodes[16 * i + 11] = 0.f;
  nodes[16 * i + 15] = 0.f;
  parent[left >= 0 ? left : n - 1 + ~left] = (int32_t)i;
  parent[right >= 0 ? right : n - 1 + ~right] = (int32_t)i;
  if (i == 0) parent[0] = -1;
}

__device__ __forceinline__ bool lex_less(const float a[3], const float b[3]) {
  return a[0] < b[0] || (a[0] == b[0] && (a[1] < b[1] || (a[1] == b[1] && a[2] < b[2])));
}

__device__ __forceinline__ void swap3(float a[3], float b[3]) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float t = a[k];
    a[k] = b[k];
    b[k] = t;
  }
}

// one thread per leaf: copy the triangle in leaf order, write its box into the parent's slot, and climb while this
// thread is the second to arrive at a node
__global__ void __launch_bounds__(kBvhThreads)
k_bvh_refit(const float* __restrict__ v, const int32_t* __restrict__ f, const int32_t* __restrict__ idx,
            const int64_t n, const int32_t* __restrict__ parent, int32_t* __restrict__ flags,
            float* __restrict__ nodes, float4* __restrict__ tris) {
  const int64_t j = blockIdx.x * (int64_t)kBvhThreads + threadIdx.x;
  if (j >= n) return;
  float p[3][3];
  const int32_t orig = __ldg(idx + j);
  load_tri(v, f, orig, p);
  // SPEC S20 tests the vertices in lexicographic (x, y, z) order, so neither the winding nor the rotation of a
  // triangle changes how its sums are rounded
  if (lex_less(p[1], p[0])) swap3(p[0], p[1]);
  if (lex_less(p[2], p[1])) swap3(p[1], p[2]);
  if (lex_less(p[1], p[0])) swap3(p[0], p[1]);
  // the first vertex's .w carries the original triangle index, which the distance query reports and breaks ties on
  tris[3 * j] = make_float4(p[0][0], p[0][1], p[0][2], __int_as_float(orig));
  tris[3 * j + 1] = make_float4(p[1][0], p[1][1], p[1][2], 0.f);
  tris[3 * j + 2] = make_float4(p[2][0], p[2][1], p[2][2], 0.f);
  if (n == 1) return;
  float lo[3], hi[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    lo[k] = fminf(p[0][k], fminf(p[1][k], p[2][k]));
    hi[k] = fmaxf(p[0][k], fmaxf(p[1][k], p[2][k]));
  }
  int32_t code = ~(int32_t)j;
  int32_t node = __ldg(parent + n - 1 + j);
  while (node >= 0) {
    float* nd = nodes + 16 * (int64_t)node;
    const int slot = __float_as_int(__ldcg(nd + 3)) == code ? 0 : 1;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      __stcg(nd + 8 * slot + k, lo[k]);
      __stcg(nd + 8 * slot + 4 + k, hi[k]);
    }
    __threadfence();
    if (atomicAdd(flags + node, 1) == 0) return;
    __threadfence();
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      lo[k] = fminf(lo[k], __ldcg(nd + 8 * (1 - slot) + k));
      hi[k] = fmaxf(hi[k], __ldcg(nd + 8 * (1 - slot) + 4 + k));
    }
    code = node;
    node = __ldcg(parent + node);
  }
}

// Ize's slab test on the box padded by pad: origin o, reciprocal direction r; the far distance is inflated by
// 1 + 2^-20 (> 1 + 2 gamma_3), and only t >= 0 counts.  tn is the entry distance (in units of the direction), which
// the first-hit traversal orders and bounds by (DESIGN.md section 4.7)
__device__ __forceinline__ bool slab_entry(const float4 lo, const float4 hi, const float pad, const float o[3],
                                           const float r[3], float& tn) {
  const float t0x = (lo.x - pad - o[0]) * r[0], t1x = (hi.x + pad - o[0]) * r[0];
  const float t0y = (lo.y - pad - o[1]) * r[1], t1y = (hi.y + pad - o[1]) * r[1];
  const float t0z = (lo.z - pad - o[2]) * r[2], t1z = (hi.z + pad - o[2]) * r[2];
  tn = fmaxf(fmaxf(fminf(t0x, t1x), fminf(t0y, t1y)), fminf(t0z, t1z));
  const float tf = fminf(fminf(fmaxf(t0x, t1x), fmaxf(t0y, t1y)), fmaxf(t0z, t1z)) * (1.f + 0x1p-20f);
  return tf >= 0.f && tn <= tf;
}

__device__ __forceinline__ bool slab_hit(const float4 lo, const float4 hi, const float pad, const float o[3],
                                         const float r[3]) {
  float tn;
  return slab_entry(lo, hi, pad, o, r, tn);
}

// the ray's frame (SPEC S20): kz = argmax |d| (first on ties), kx, ky the next two cyclically, swapped when d[kz] < 0
struct RayFrame {
  int kx, ky, kz;
  float sx, sy, sz;
};

__device__ __forceinline__ RayFrame ray_frame(const float d[3]) {
  int kz = 0;
  if (fabsf(d[1]) > fabsf(d[kz])) kz = 1;
  if (fabsf(d[2]) > fabsf(d[kz])) kz = 2;
  int kx = kz == 2 ? 0 : kz + 1, ky = kx == 2 ? 0 : kx + 1;
  if (d[kz] < 0.f) {
    const int s = kx;
    kx = ky;
    ky = s;
  }
  return {kx, ky, kz, __fdiv_rn(d[kx], d[kz]), __fdiv_rn(d[ky], d[kz]), __fdiv_rn(1.f, d[kz])};
}

__device__ __forceinline__ float pick(const float a[3], int k) { return k == 0 ? a[0] : (k == 1 ? a[1] : a[2]); }

// does edge (P, Q) own the origin when its edge function is 0: the inward normal s (Qy - Py, Px - Qx) has a positive
// x, or a zero x and a positive y (s = sign of det)
__device__ __forceinline__ bool owns(const float px, const float py, const float qx, const float qy, const bool pos) {
  return pos ? (qy > py || (qy == py && px > qx)) : (qy < py || (qy == py && px < qx));
}

// SPEC S20's crossing test of the ray from the query (o) along the frame's direction with triangle t; on a crossing
// the ray parameter of SPEC S22 is T / det
__device__ __forceinline__ bool crossing(const float4* __restrict__ tris, const int64_t t, const float o[3],
                                         const RayFrame& fr, double& T, double& det) {
  float sx[3], sy[3], sz[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float4 w = __ldg(tris + 3 * t + c);
    const float a[3] = {w.x - o[0], w.y - o[1], w.z - o[2]};
    const float az = pick(a, fr.kz);
    sx[c] = pick(a, fr.kx) - fr.sx * az;
    sy[c] = pick(a, fr.ky) - fr.sy * az;
    sz[c] = fr.sz * az;
  }
  double U = (double)sx[2] * sy[1] - (double)sy[2] * sx[1];
  double V = (double)sx[0] * sy[2] - (double)sy[0] * sx[2];
  double W = (double)sx[1] * sy[0] - (double)sy[1] * sx[0];
  if ((U < 0.0 || V < 0.0 || W < 0.0) && (U > 0.0 || V > 0.0 || W > 0.0)) return false;
  det = U + V + W;
  if (det == 0.0) return false;
  const bool pos = det > 0.0;
  if (U == 0.0 && !owns(sx[1], sy[1], sx[2], sy[2], pos)) return false;
  if (V == 0.0 && !owns(sx[2], sy[2], sx[0], sy[0], pos)) return false;
  if (W == 0.0 && !owns(sx[0], sy[0], sx[1], sy[1], pos)) return false;
  T = U * (double)sz[0] + V * (double)sz[1] + W * (double)sz[2];
  return pos ? T > 0.0 : T < 0.0;
}

__device__ __forceinline__ bool crosses(const float4* __restrict__ tris, const int64_t t, const float o[3],
                                        const RayFrame& fr) {
  double T, det;
  return crossing(tris, t, o, fr, T, det);
}

__global__ void __launch_bounds__(kOccThreads)
k_mesh_occupancy(const float4* __restrict__ nodes, const float4* __restrict__ tris, const float* __restrict__ scene,
                 const int64_t n_tri, const float* __restrict__ query, const int64_t m, const float* __restrict__ dirs,
                 const int k_rays, uint8_t* __restrict__ inside) {
  __shared__ RayFrame frames[kMaxRays];
  __shared__ float recip[kMaxRays][3];
  if (threadIdx.x < k_rays) {
    const int r = threadIdx.x;
    const float d[3] = {dirs ? dirs[3 * r] : kDefaultDirs[r][0], dirs ? dirs[3 * r + 1] : kDefaultDirs[r][1],
                        dirs ? dirs[3 * r + 2] : kDefaultDirs[r][2]};
    frames[r] = ray_frame(d);
#pragma unroll
    for (int k = 0; k < 3; ++k) recip[r][k] = __fdiv_rn(1.f, d[k]);
  }
  __syncthreads();
  const int64_t i = blockIdx.x * (int64_t)kOccThreads + threadIdx.x;
  if (i >= m) return;
  const float o[3] = {__ldg(query + 3 * i), __ldg(query + 3 * i + 1), __ldg(query + 3 * i + 2)};
  // every rounding of the sheared frame moves a crossing by less than 2^-19 (M + |q|_inf) (SPEC S20)
  const float pad = (__ldg(scene + 6) + fmaxf(fabsf(o[0]), fmaxf(fabsf(o[1]), fabsf(o[2])))) * 0x1p-19f;
  int votes = 0;
  int32_t stack[kStack];
  for (int r = 0; r < k_rays; ++r) {
    const RayFrame fr = frames[r];
    const float rc[3] = {recip[r][0], recip[r][1], recip[r][2]};
    int parity = 0;
    if (n_tri == 1) {
      parity = crosses(tris, 0, o, fr);
    } else {
      int sp = 0;
      int32_t node = 0;
      for (;;) {
        const float4* nd = nodes + 4 * (int64_t)node;
        const float4 a = __ldg(nd), b = __ldg(nd + 1), c = __ldg(nd + 2), e = __ldg(nd + 3);
        const int32_t c0 = __float_as_int(a.w), c1 = __float_as_int(b.w);
        const bool h0 = slab_hit(a, b, pad, o, rc), h1 = slab_hit(c, e, pad, o, rc);
        int32_t next = -1;
        if (h0) {
          if (c0 < 0) parity ^= crosses(tris, ~c0, o, fr);
          else next = c0;
        }
        if (h1) {
          if (c1 < 0) parity ^= crosses(tris, ~c1, o, fr);
          else if (next < 0) next = c1;
          else stack[sp++] = c1;
        }
        if (next < 0) {
          if (sp == 0) break;
          next = stack[--sp];
        }
        node = next;
      }
    }
    votes += parity;
  }
  inside[i] = 2 * votes > k_rays;
}

// ---- SPEC S21: the closest point of a triangle.  Every product, sum and difference is rounded on its own (the file
// is built with --fmad=false), dots are ((x x' + y y') + z z'), divisions and the square root are correctly rounded.

constexpr int kDistThreads = 128;

__device__ __forceinline__ float dot3(const float a[3], const float b[3]) {
  return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2];
}

__device__ __forceinline__ void cross3(const float a[3], const float b[3], float c[3]) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}

__device__ __forceinline__ float dist2(const float p[3], const float c[3]) {
  const float dx = p[0] - c[0], dy = p[1] - c[1], dz = p[2] - c[2];
  return (dx * dx + dy * dy) + dz * dz;
}

// candidate on segment (P, Q): P when e.(p - P) <= 0 (a zero-length edge included), Q when it reaches e.e, else
// P + t e with t = e.(p - P) / e.e; it replaces the best one only when its d2 is strictly smaller
__device__ __forceinline__ void closest_on_segment(const float P[3], const float Q[3], const float p[3], float& best,
                                                   float x[3]) {
  float e[3], ap[3], c[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    e[k] = Q[k] - P[k];
    ap[k] = p[k] - P[k];
  }
  const float num = dot3(e, ap), den = dot3(e, e);
  if (!(num > 0.f)) {
#pragma unroll
    for (int k = 0; k < 3; ++k) c[k] = P[k];
  } else if (num >= den) {
#pragma unroll
    for (int k = 0; k < 3; ++k) c[k] = Q[k];
  } else {
    const float t = __fdiv_rn(num, den);
#pragma unroll
    for (int k = 0; k < 3; ++k) c[k] = P[k] + t * e[k];
  }
  const float d2 = dist2(p, c);
  if (d2 < best) {
    best = d2;
#pragma unroll
    for (int k = 0; k < 3; ++k) x[k] = c[k];
  }
}

// SPEC S21 for the lexicographically sorted vertices a <= b <= c: the face candidate (when the projection's scaled
// barycentric weights va = n.(bp x cp), vb = n.(cp x ap), vc = n.(ap x bp), n = ab x ac, are all >= 0 and their sum is
// positive and finite), then the segments ab, ac, bc;
// the smallest d2 wins, the earlier candidate on ties.  Returns d2 and the point in x.
__device__ __forceinline__ float closest_on_triangle(const float a[3], const float b[3], const float c[3],
                                                     const float p[3], float x[3]) {
  float ab[3], ac[3], ap[3], bp[3], cp[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    ab[k] = b[k] - a[k];
    ac[k] = c[k] - a[k];
    ap[k] = p[k] - a[k];
    bp[k] = p[k] - b[k];
    cp[k] = p[k] - c[k];
  }
  float n[3], s[3];
  cross3(ab, ac, n);
  cross3(bp, cp, s);
  const float va = dot3(n, s);
  cross3(cp, ap, s);
  const float vb = dot3(n, s);
  cross3(ap, bp, s);
  const float vc = dot3(n, s);
  float best = INFINITY;
  if (va >= 0.f && vb >= 0.f && vc >= 0.f) {
    const float den = (va + vb) + vc;
    if (den > 0.f && den < INFINITY) {
      const float v = __fdiv_rn(vb, den), w = __fdiv_rn(vc, den);
#pragma unroll
      for (int k = 0; k < 3; ++k) x[k] = (a[k] + v * ab[k]) + w * ac[k];
      best = dist2(p, x);
    }
  }
  closest_on_segment(a, b, p, best, x);
  closest_on_segment(a, c, p, best, x);
  closest_on_segment(b, c, p, best, x);
  return best;
}

// squared distance from p to the box padded by pad on every side, each gap and sum rounded; never above the d2 that
// closest_on_triangle reports for a triangle inside the unpadded box (DESIGN.md section 4.7)
__device__ __forceinline__ float box_bound(const float4 lo, const float4 hi, const float pad, const float p[3]) {
  const float gx = fmaxf(fmaxf((lo.x - pad) - p[0], p[0] - (hi.x + pad)), 0.f);
  const float gy = fmaxf(fmaxf((lo.y - pad) - p[1], p[1] - (hi.y + pad)), 0.f);
  const float gz = fmaxf(fmaxf((lo.z - pad) - p[2], p[2] - (hi.z + pad)), 0.f);
  return (gx * gx + gy * gy) + gz * gz;
}

struct Best {
  float d2;
  int32_t tri;
  float x[3];
};

// the leaf-order triangle j against the best so far: smaller d2, or equal d2 and a lower original index, wins
__device__ __forceinline__ void test_leaf(const float4* __restrict__ tris, const int32_t j, const float p[3],
                                          Best& best) {
  const float4 wa = __ldg(tris + 3 * (int64_t)j), wb = __ldg(tris + 3 * (int64_t)j + 1),
               wc = __ldg(tris + 3 * (int64_t)j + 2);
  const float a[3] = {wa.x, wa.y, wa.z}, b[3] = {wb.x, wb.y, wb.z}, c[3] = {wc.x, wc.y, wc.z};
  float x[3];
  const float d2 = closest_on_triangle(a, b, c, p, x);
  const int32_t t = __float_as_int(wa.w);
  if (d2 < best.d2 || (d2 == best.d2 && t < best.tri)) {
    best.d2 = d2;
    best.tri = t;
#pragma unroll
    for (int k = 0; k < 3; ++k) best.x[k] = x[k];
  }
}

__global__ void __launch_bounds__(kDistThreads)
k_mesh_closest(const float4* __restrict__ nodes, const float4* __restrict__ tris, const float* __restrict__ scene,
               const int64_t n_tri, const float* __restrict__ query, const int64_t m, float* __restrict__ dist,
               float* __restrict__ point, int32_t* __restrict__ tri) {
  const int64_t i = blockIdx.x * (int64_t)kDistThreads + threadIdx.x;
  if (i >= m) return;
  Best best = {INFINITY, INT32_MAX, {NAN, NAN, NAN}};
  if (n_tri > 0) {
    const float p[3] = {__ldg(query + 3 * i), __ldg(query + 3 * i + 1), __ldg(query + 3 * i + 2)};
    if (n_tri == 1) {
      test_leaf(tris, 0, p, best);
    } else {
      // every rounding of a candidate point stays within 2^-18 (M + |q|_inf) of the triangle's box (section 4.7)
      const float pad = (__ldg(scene + 6) + fmaxf(fabsf(p[0]), fmaxf(fabsf(p[1]), fabsf(p[2])))) * 0x1p-18f;
      int32_t stack[kStack];
      float stack_bound[kStack];
      int sp = 0;
      int32_t node = 0;
      for (;;) {
        const float4* nd = nodes + 4 * (int64_t)node;
        const float4 a = __ldg(nd), b = __ldg(nd + 1), c = __ldg(nd + 2), e = __ldg(nd + 3);
        const float lb0 = box_bound(a, b, pad, p), lb1 = box_bound(c, e, pad, p);
        const bool swap = lb1 < lb0;     // nearer child first, child 0 on equal bounds
        const int32_t near = __float_as_int(swap ? b.w : a.w), far = __float_as_int(swap ? a.w : b.w);
        const float near_lb = swap ? lb1 : lb0, far_lb = swap ? lb0 : lb1;
        int32_t next = -1;
        if (!(near_lb > best.d2)) {
          if (near < 0) test_leaf(tris, ~near, p, best);
          else next = near;
        }
        if (!(far_lb > best.d2)) {
          if (far < 0) {
            test_leaf(tris, ~far, p, best);
          } else if (next < 0) {
            next = far;
          } else {
            stack[sp] = far;
            stack_bound[sp++] = far_lb;
          }
        }
        while (next < 0 && sp > 0) {
          --sp;
          if (!(stack_bound[sp] > best.d2)) next = stack[sp];
        }
        if (next < 0) break;
        node = next;
      }
    }
  }
  dist[i] = __fsqrt_rn(best.d2);
  point[3 * i] = best.x[0];
  point[3 * i + 1] = best.x[1];
  point[3 * i + 2] = best.x[2];
  tri[i] = n_tri > 0 ? best.tri : -1;
}

// ---- SPEC S22: the first hit of a ray, the candidates of SPEC S20 ordered by t = T / det.

constexpr int kHitThreads = 128;

// the leaf-order triangle j against the best hit so far: a crossing with 0 < t <= t_max (fp64) replaces it when its
// t is smaller, or equal with a lower original index
__device__ __forceinline__ void test_hit(const float4* __restrict__ tris, const int32_t j, const float o[3],
                                         const RayFrame& fr, const double t_max, double& best_t, int32_t& best_tri) {
  double T, det;
  if (!crossing(tris, j, o, fr, T, det)) return;
  const double t = __ddiv_rn(T, det);
  const int32_t id = __float_as_int(__ldg(&tris[3 * (int64_t)j].w));
  if (t > 0.0 && t <= t_max && (t < best_t || (t == best_t && id < best_tri))) {
    best_t = t;
    best_tri = id;
  }
}

__global__ void __launch_bounds__(kHitThreads)
k_mesh_first_hit(const float4* __restrict__ nodes, const float4* __restrict__ tris, const float* __restrict__ scene,
                 const int64_t n_tri, const float* __restrict__ v, const int32_t* __restrict__ f,
                 const float* __restrict__ origin, const float* __restrict__ dir, const int64_t m,
                 const float* __restrict__ t_max, const float t_max_all, float* __restrict__ t_out,
                 float* __restrict__ point, float* __restrict__ normal, int32_t* __restrict__ tri) {
  const int64_t i = blockIdx.x * (int64_t)kHitThreads + threadIdx.x;
  if (i >= m) return;
  const float o[3] = {__ldg(origin + 3 * i), __ldg(origin + 3 * i + 1), __ldg(origin + 3 * i + 2)};
  const float d[3] = {__ldg(dir + 3 * i), __ldg(dir + 3 * i + 1), __ldg(dir + 3 * i + 2)};
  const double tmax = (double)(t_max ? __ldg(t_max + i) : t_max_all);
  // INT32_MAX: no candidate yet, so a candidate with t = inf (an overflow) still ties in as the brute force's does
  double best_t = INFINITY;
  int32_t best_tri = INT32_MAX;
  if (n_tri > 0) {
    const RayFrame fr = ray_frame(d);
    if (n_tri == 1) {
      test_hit(tris, 0, o, fr, tmax, best_t, best_tri);
    } else {
      const float rc[3] = {__fdiv_rn(1.f, d[0]), __fdiv_rn(1.f, d[1]), __fdiv_rn(1.f, d[2])};
      // S20's padding: the entry distance of the padded box never exceeds the t of a candidate inside (section 4.7)
      const float pad = (__ldg(scene + 6) + fmaxf(fabsf(o[0]), fmaxf(fabsf(o[1]), fabsf(o[2])))) * 0x1p-19f;
      int32_t stack[kStack];
      float stack_tn[kStack];
      int sp = 0;
      int32_t node = 0;
      for (;;) {
        const float4* nd = nodes + 4 * (int64_t)node;
        const float4 a = __ldg(nd), b = __ldg(nd + 1), c = __ldg(nd + 2), e = __ldg(nd + 3);
        float tn0, tn1;
        const bool h0 = slab_entry(a, b, pad, o, rc, tn0), h1 = slab_entry(c, e, pad, o, rc, tn1);
        const bool swap = h1 && (!h0 || tn1 < tn0);     // nearer entry first, child 0 on equal entries
        const int32_t near = __float_as_int(swap ? b.w : a.w), far = __float_as_int(swap ? a.w : b.w);
        const bool near_h = swap ? h1 : h0, far_h = swap ? h0 : h1;
        const float near_tn = swap ? tn1 : tn0, far_tn = swap ? tn0 : tn1;
        // a box is skipped only when its entry is strictly beyond the best t or t_max
        int32_t next = -1;
        if (near_h && !((double)near_tn > fmin(best_t, tmax))) {
          if (near < 0) test_hit(tris, ~near, o, fr, tmax, best_t, best_tri);
          else next = near;
        }
        if (far_h && !((double)far_tn > fmin(best_t, tmax))) {
          if (far < 0) {
            test_hit(tris, ~far, o, fr, tmax, best_t, best_tri);
          } else if (next < 0) {
            next = far;
          } else {
            stack[sp] = far;
            stack_tn[sp++] = far_tn;
          }
        }
        while (next < 0 && sp > 0) {
          --sp;
          if (!((double)stack_tn[sp] > fmin(best_t, tmax))) next = stack[sp];
        }
        if (next < 0) break;
        node = next;
      }
    }
  }
  const bool hit = best_tri != INT32_MAX;
  const float t32 = hit ? __double2float_rn(best_t) : INFINITY;
  float n[3] = {NAN, NAN, NAN};
  if (hit) {
    // the normal in the caller's winding: (v1 - v0) x (v2 - v0), normalised
    float p[3][3], e1[3], e2[3];
    load_tri(v, f, best_tri, p);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      e1[k] = p[1][k] - p[0][k];
      e2[k] = p[2][k] - p[0][k];
    }
    cross3(e1, e2, n);
    const float len = __fsqrt_rn(dot3(n, n));
#pragma unroll
    for (int k = 0; k < 3; ++k) n[k] = __fdiv_rn(n[k], len);
  }
  t_out[i] = t32;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    point[3 * i + k] = hit ? __fadd_rn(o[k], __fmul_rn(t32, d[k])) : NAN;
    normal[3 * i + k] = n[k];
  }
  tri[i] = hit ? best_tri : -1;
}

}  // namespace

extern "C" {

size_t nksr_bvh_workspace_bytes(int64_t n_tri) {
  if (n_tri < 1) return 0;
  return sizeof(int32_t) * (size_t)(3 * n_tri);   // parent[2 n - 1], flags[n - 1], rounded up by one entry
}

int nksr_bvh_keys(const float* v, const int32_t* f, int64_t n_tri, float* scene, int64_t* keys, int32_t* idx,
                  void* stream) {
  if (n_tri < 0 || n_tri > INT32_MAX) return NKSR_E_INVALID;
  if (n_tri == 0) return NKSR_OK;
  if (!v || !f || !scene || !keys || !idx) return NKSR_E_INVALID;
  cudaStream_t st = as_stream(stream);
  k_bvh_scene_init<<<1, 32, 0, st>>>(reinterpret_cast<unsigned*>(scene));
  NKSR_CHECK_LAUNCH();
  const int grid = grid_for(n_tri, kBvhThreads) < 1024 ? grid_for(n_tri, kBvhThreads) : 1024;
  k_bvh_bounds<<<grid, kBvhThreads, 0, st>>>(v, f, n_tri, reinterpret_cast<unsigned*>(scene));
  NKSR_CHECK_LAUNCH();
  k_bvh_keys<<<grid_for(n_tri, kBvhThreads), kBvhThreads, 0, st>>>(v, f, n_tri,
                                                                  reinterpret_cast<const unsigned*>(scene), keys, idx);
  NKSR_CHECK_LAUNCH();
  k_bvh_scene_floats<<<1, 32, 0, st>>>(reinterpret_cast<unsigned*>(scene));
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_bvh_hierarchy(const int64_t* keys, int64_t n_tri, float* nodes, void* ws, size_t ws_bytes, void* stream) {
  if (n_tri < 0 || n_tri > INT32_MAX) return NKSR_E_INVALID;
  if (n_tri <= 1) return NKSR_OK;
  if (!keys || !nodes || !ws) return NKSR_E_INVALID;
  if (ws_bytes < nksr_bvh_workspace_bytes(n_tri)) return NKSR_E_WORKSPACE;
  k_bvh_hierarchy<<<grid_for(n_tri - 1, kBvhThreads), kBvhThreads, 0, as_stream(stream)>>>(
      keys, n_tri, nodes, static_cast<int32_t*>(ws));
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_bvh_refit(const float* v, const int32_t* f, const int32_t* idx, int64_t n_tri, float* nodes, float* tris,
                   void* ws, size_t ws_bytes, void* stream) {
  if (n_tri < 0 || n_tri > INT32_MAX) return NKSR_E_INVALID;
  if (n_tri == 0) return NKSR_OK;
  if (!v || !f || !idx || !tris || !ws || (n_tri > 1 && !nodes)) return NKSR_E_INVALID;
  if (ws_bytes < nksr_bvh_workspace_bytes(n_tri)) return NKSR_E_WORKSPACE;
  cudaStream_t st = as_stream(stream);
  int32_t* parent = static_cast<int32_t*>(ws);
  int32_t* flags = parent + 2 * n_tri - 1;
  if (n_tri > 1 && cudaMemsetAsync(flags, 0, sizeof(int32_t) * (size_t)(n_tri - 1), st) != cudaSuccess)
    return NKSR_E_CUDA;
  k_bvh_refit<<<grid_for(n_tri, kBvhThreads), kBvhThreads, 0, st>>>(v, f, idx, n_tri, parent, flags, nodes,
                                                                     reinterpret_cast<float4*>(tris));
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_occupancy(const float* nodes, const float* tris, const float* scene, int64_t n_tri, const float* query,
                        int64_t m, const float* dirs, int k_rays, uint8_t* inside, void* stream) {
  if (n_tri < 0 || n_tri > INT32_MAX || m < 0 || k_rays < 1 || k_rays > kMaxRays || !(k_rays & 1))
    return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  if (!query || !inside) return NKSR_E_INVALID;
  cudaStream_t st = as_stream(stream);
  if (n_tri == 0) return cudaMemsetAsync(inside, 0, (size_t)m, st) == cudaSuccess ? NKSR_OK : NKSR_E_CUDA;
  if (!tris || !scene || (n_tri > 1 && !nodes)) return NKSR_E_INVALID;
  k_mesh_occupancy<<<grid_for(m, kOccThreads), kOccThreads, 0, st>>>(
      reinterpret_cast<const float4*>(nodes), reinterpret_cast<const float4*>(tris), scene, n_tri, query, m, dirs,
      k_rays, inside);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_closest(const float* nodes, const float* tris, const float* scene, int64_t n_tri, const float* query,
                      int64_t m, float* dist, float* point, int32_t* tri, void* stream) {
  if (n_tri < 0 || n_tri > INT32_MAX || m < 0) return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  if (!query || !dist || !point || !tri) return NKSR_E_INVALID;
  if (n_tri > 0 && (!tris || !scene || (n_tri > 1 && !nodes))) return NKSR_E_INVALID;
  k_mesh_closest<<<grid_for(m, kDistThreads), kDistThreads, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(nodes), reinterpret_cast<const float4*>(tris), scene, n_tri, query, m, dist,
      point, tri);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

int nksr_mesh_first_hit(const float* nodes, const float* tris, const float* scene, int64_t n_tri, const float* v,
                        const int32_t* f, const float* origin, const float* dir, int64_t m, const float* t_max,
                        float t_max_all, float* t, float* point, float* normal, int32_t* tri, void* stream) {
  if (n_tri < 0 || n_tri > INT32_MAX || m < 0) return NKSR_E_INVALID;
  if (m == 0) return NKSR_OK;
  if (!origin || !dir || !t || !point || !normal || !tri) return NKSR_E_INVALID;
  if (n_tri > 0 && (!tris || !scene || !v || !f || (n_tri > 1 && !nodes))) return NKSR_E_INVALID;
  k_mesh_first_hit<<<grid_for(m, kHitThreads), kHitThreads, 0, as_stream(stream)>>>(
      reinterpret_cast<const float4*>(nodes), reinterpret_cast<const float4*>(tris), scene, n_tri, v, f, origin, dir,
      m, t_max, t_max_all, t, point, normal, tri);
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
