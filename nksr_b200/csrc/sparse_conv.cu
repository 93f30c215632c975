// SURVEY 8(f) row 2: the sparse convolution of the NKSRNetwork encoder / U-Net (models/nksr_net.py:73-78 call it,
// configs/default/train.yaml:17-18 size it: unet.f_maps = 32) as ONE gather-GEMM kernel over the hierarchy's index tables:
//
//     y[i, :] = act( bias + res[i, :] + sum_k [idx[i,k] >= 0]  x[idx[i,k], :] . W[k] )          W[k]: Cin x Cout
//
//   * 3x3x3 sparse convolution on level l:     idx = nbr27[l]   (K = 27)
//   * stride-2 convolution level l -> l+1:     idx = child8[l+1] (K = 8: one weight per octant)
// The tables are the ones the Gram assembly already uses (csrc/svh.cu), so no hash lookups happen here.
//
// Tiling: a CTA owns 128 output voxels x TN output channels (TN = 64 or 32); per (k, 32-channel chunk) the 128 gathered
// input rows (128 B each, coalesced) and the 32 x TN slice of W[k] are staged in shared memory.  A (k, tile) pair whose
// 128 sources are all absent is skipped (borders of the hierarchy).
//   k_gather_gemm_f32 : fp32 FFMA, 8 x TN/16 outputs per thread (A tile transposed in smem: two LDS.128 + one LDS.128/64
//                       per 32 / 16 FMAs) -- bit-for-bit an fp32 sum, the parity kernel
//   k_gather_gemm_tf32: mma.sync.m16n8k8 TF32 (fp32 accumulate), one 16 x TN strip per warp, operands staged by a
//                       two-stage cp.async pipeline; inputs are rounded to TF32 (10-bit mantissa, cvt.rna), so results
//                       differ from fp32 by ~1e-3 relative
//   k_gather_gemm_tc  : wgmma.mma_async tf32, two warpgroups x (64 x TN) register accumulators (TN = 32 / 64 / 128),
//                       operands gathered by cp.async into 128-byte-swizzled tiles, four-stage ring -- see below
#include "common.cuh"

namespace {

constexpr int kTM = 128;      // output rows per CTA
constexpr int kKC = 32;       // input channels per staged chunk
constexpr int kThreads = 256;

template <int TN>
__global__ void __launch_bounds__(kThreads, 2)
k_gather_gemm_f32(const float* __restrict__ x, const int32_t* __restrict__ idx, int64_t n_out, int K,
                  const float* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ res,
                  float* __restrict__ y, int Cin, int Cout, int relu) {
  constexpr int CN = TN / 16;                       // output channels per thread
  __shared__ __align__(16) float As[kKC][kTM + 4];  // transposed: [channel][row]
  __shared__ __align__(16) float Bs[kKC][TN];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t row0 = (int64_t)blockIdx.x * kTM;
  const int n0 = blockIdx.y * TN;
  float acc[8][CN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < CN; ++j) acc[i][j] = 0.f;

  for (int k = 0; k < K; ++k) {
    // sources of this warp's 16 rows
    int src_l = -1;
    if (lane < 16) {
      const int64_t r = row0 + wid * 16 + lane;
      if (r < n_out) src_l = __ldg(idx + r * K + k);
    }
    if (!__syncthreads_or(src_l >= 0)) continue;    // nothing to gather for this offset in the whole tile (uniform)
    for (int c0 = 0; c0 < Cin; c0 += kKC) {
#pragma unroll 4
      for (int j = 0; j < 16; ++j) {
        const int s = __shfl_sync(0xffffffffu, src_l, j);
        As[lane][wid * 16 + j] = s >= 0 ? __ldg(x + (int64_t)s * Cin + c0 + lane) : 0.f;
      }
      const float* wp = W + ((int64_t)k * Cin + c0) * Cout + n0;
      for (int t = tid; t < kKC * TN / 4; t += kThreads) {
        const int r = t / (TN / 4), q = t % (TN / 4);
        *reinterpret_cast<float4*>(&Bs[r][q * 4]) = __ldg(reinterpret_cast<const float4*>(wp + (int64_t)r * Cout) + q);
      }
      __syncthreads();
#pragma unroll 8
      for (int c = 0; c < kKC; ++c) {
        const float4 a0 = *reinterpret_cast<const float4*>(&As[c][ty * 8]);
        const float4 a1 = *reinterpret_cast<const float4*>(&As[c][ty * 8 + 4]);
        const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        float b[CN];
        if (CN == 4) {
          const float4 bv = *reinterpret_cast<const float4*>(&Bs[c][tx * 4]);
          b[0] = bv.x; b[1] = bv.y; b[2] = bv.z; b[3] = bv.w;
        } else {
          const float2 bv = *reinterpret_cast<const float2*>(&Bs[c][tx * 2]);
          b[0] = bv.x; b[1] = bv.y;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < CN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
  // epilogue: bias, residual, activation
  float bv[CN];
#pragma unroll
  for (int j = 0; j < CN; ++j) bv[j] = bias ? __ldg(bias + n0 + tx * CN + j) : 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t r = row0 + ty * 8 + i;
    if (r >= n_out) continue;
    float* yp = y + r * Cout + n0 + tx * CN;
    const float* rp = res ? res + r * Cout + n0 + tx * CN : nullptr;
#pragma unroll
    for (int j = 0; j < CN; ++j) {
      float v = acc[i][j] + bv[j];
      if (rp) v += __ldg(rp + j);
      if (relu) v = fmaxf(v, 0.f);
      yp[j] = v;
    }
  }
}

__device__ __forceinline__ uint32_t to_tf32(float v) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(v));
  return r;
}

// D (16x8, fp32) += A (16x8, tf32, row) * B (8x8, tf32, col).  Fragments (g = lane / 4, t = lane % 4):
//   a0 = A[g][t]  a1 = A[g+8][t]  a2 = A[g][t+4]  a3 = A[g+8][t+4];   b0 = B[t][g]  b1 = B[t+4][g]
//   d0 = D[g][2t] d1 = D[g][2t+1] d2 = D[g+8][2t] d3 = D[g+8][2t+1]
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t b0, const uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src, const int src_bytes) {
  // 16-byte asynchronous copy global -> shared (LDGSTS); src_bytes = 0 fills the destination with zeros
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gmem_src), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Two-stage pipeline: while the MMAs of one (offset k, 32-channel chunk) step run, the gathered rows and the weight
// slice of the next step are already on their way into the other shared-memory buffer (cp.async, zero-fill for absent
// sources).  The tile's 128 x K source indices are staged once (they are one contiguous block of `idx`), which also
// tells which offsets have no source in the whole tile -- those steps are skipped.
// WROUNDED: the weights were rounded to TF32 by the caller (no conversion of the B fragments here).
template <int TN, bool WROUNDED>
__global__ void __launch_bounds__(kThreads, 2)
k_gather_gemm_tf32(const float* __restrict__ x, const int32_t* __restrict__ idx, int64_t n_out, int K,
                   const float* __restrict__ W, const float* __restrict__ bias, const float* __restrict__ res,
                   float* __restrict__ y, int Cin, int Cout, int relu) {
  constexpr int NT = TN / 8;                  // 8-column mma tiles per warp strip
  constexpr int AS = kKC + 4;                 // A row stride (floats): fragment loads hit 32 distinct banks
  constexpr int BS = TN + 8;                  // B row stride = 8 mod 32: b0 / b1 loads hit 32 distinct banks
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* As = reinterpret_cast<float*>(smem_raw);                    // [2][kTM][AS]
  float* Bs = As + 2 * kTM * AS;                                     // [2][kKC][BS]
  int32_t* src_s = reinterpret_cast<int32_t*>(Bs + 2 * kKC * BS);    // [kTM][K]
  __shared__ unsigned kmask;                                         // bit k: some row of the tile has a source at k
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int64_t row0 = (int64_t)blockIdx.x * kTM;
  const int n0 = blockIdx.y * TN;
  const int rows_here = (int)min((int64_t)kTM, n_out - row0);
  if (tid == 0) kmask = 0u;
  __syncthreads();
  {
    unsigned mine = 0u;
    const int32_t* ip = idx + row0 * K;
    for (int e = tid; e < kTM * K; e += kThreads) {
      const int r = e / K;
      const int v = r < rows_here ? __ldg(ip + e) : -1;
      src_s[e] = v;
      if (v >= 0) mine |= 1u << (e - r * K);
    }
    mine = __reduce_or_sync(0xffffffffu, mine);
    if (lane == 0 && mine) atomicOr(&kmask, mine);
  }
  __syncthreads();
  const unsigned km = kmask;
  const int nchunk = Cin / kKC;
  const int nsteps = __popc(km) * nchunk;

  float acc[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[j][i] = 0.f;

  // step s -> (k = the (s / nchunk)-th set bit of km, c0 = (s % nchunk) * 32)
  auto issue = [&](const int s, const int buf) {
    const int k = __fns(km, 0, s / nchunk + 1);
    const int c0 = (s - (s / nchunk) * nchunk) * kKC;
    float* a = As + buf * kTM * AS;
#pragma unroll
    for (int j = 0; j < kTM * 8 / kThreads; ++j) {
      const int e = tid + j * kThreads;
      const int r = e >> 3, seg = e & 7;
      const int sidx = src_s[r * K + k];
      const float* gp = x + (int64_t)(sidx >= 0 ? sidx : 0) * Cin + c0 + seg * 4;
      cp_async16(a + r * AS + seg * 4, gp, sidx >= 0 ? 16 : 0);
    }
    float* b = Bs + buf * kKC * BS;
    const float* wp = W + ((int64_t)k * Cin + c0) * Cout + n0;
    for (int e = tid; e < kKC * TN / 4; e += kThreads) {
      const int r = e / (TN / 4), q = e % (TN / 4);
      cp_async16(b + r * BS + q * 4, wp + (int64_t)r * Cout + q * 4, 16);
    }
    cp_async_commit();
  };

  if (nsteps > 0) issue(0, 0);
  for (int s = 0; s < nsteps; ++s) {
    const int buf = s & 1;
    if (s + 1 < nsteps) {
      issue(s + 1, buf ^ 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const float* Aw = As + buf * kTM * AS + wid * 16 * AS;      // this warp's 16 rows
    const float* Bb = Bs + buf * kKC * BS;
#pragma unroll
    for (int ks = 0; ks < kKC; ks += 8) {
      uint32_t a[4];
      a[0] = to_tf32(Aw[g * AS + ks + t]);
      a[1] = to_tf32(Aw[(g + 8) * AS + ks + t]);
      a[2] = to_tf32(Aw[g * AS + ks + t + 4]);
      a[3] = to_tf32(Aw[(g + 8) * AS + ks + t + 4]);
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const float b0 = Bb[(ks + t) * BS + j * 8 + g], b1 = Bb[(ks + t + 4) * BS + j * 8 + g];
        mma_tf32(acc[j], a, WROUNDED ? __float_as_uint(b0) : to_tf32(b0), WROUNDED ? __float_as_uint(b1) : to_tf32(b1));
      }
    }
    __syncthreads();                                            // the buffer is refilled two steps ahead
  }
  // epilogue: rows g / g+8 of the warp's strip, columns 2t / 2t+1 of every 8-column tile
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t r = row0 + wid * 16 + g + 8 * h;
    if (r >= n_out) continue;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      const int cidx = n0 + j * 8 + 2 * t;
      float v0 = acc[j][2 * h], v1 = acc[j][2 * h + 1];
      if (bias) { v0 += __ldg(bias + cidx); v1 += __ldg(bias + cidx + 1); }
      if (res) {
        const float2 rv = __ldg(reinterpret_cast<const float2*>(res + r * Cout + cidx));
        v0 += rv.x; v1 += rv.y;
      }
      if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      *reinterpret_cast<float2*>(y + r * Cout + cidx) = make_float2(v0, v1);
    }
  }
}

template <int TN>
size_t tf32_smem_bytes(int K) {
  return (size_t)(2 * kTM * (kKC + 4) + 2 * kKC * (TN + 8)) * sizeof(float) + (size_t)kTM * K * sizeof(int32_t);
}

template <int TN, bool WROUNDED>
int launch_tf32(dim3 grid, cudaStream_t s, const float* x, const int32_t* idx, int64_t n_out, int K, const float* W,
                const float* bias, const float* res, float* y, int c_in, int c_out, int relu) {
  const size_t smem = tf32_smem_bytes<TN>(K);
  if (smem > 200 * 1024) return NKSR_E_INVALID;
  if (cudaFuncSetAttribute(k_gather_gemm_tf32<TN, WROUNDED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
      cudaSuccess)
    return NKSR_E_CUDA;
  k_gather_gemm_tf32<TN, WROUNDED><<<grid, kThreads, smem, s>>>(x, idx, n_out, K, W, bias, res, y, c_in, c_out, relu);
  return NKSR_OK;
}


// ---------------------------------------------------------------------------------------------------------------------
// k_gather_gemm_tc: the same gather-GEMM on the Hopper tensor cores (wgmma.mma_async kind tf32, fp32 accumulator in
// registers).
//
//   * A tile (128 gathered rows x 32 channels = 128 B per row) and B tile (TN output channels x 32 input channels; the
//     caller passes W transposed to [K][c_out][c_in], "K-major" for the MMA) are written by cp.async straight into the
//     canonical K-major 128-byte-swizzle shared-memory layout: row r at r * 128 B, its 16-byte chunk c at position
//     c ^ (r & 7); 8-row groups 1024 B apart (the descriptor's stride byte offset).  Absent sources are zero-filled.
//   * the two warpgroups of the CTA own rows 0-63 and 64-127; per (offset, 32-channel chunk) step each issues
//     4 x wgmma (M = 64, N = TN, K = 8) on its half of the A tile and the whole B tile.  A four-stage ring keeps two
//     steps of gathers in flight while the MMAs of the previous step may still run (wgmma.wait_group 1).
//   * the accumulator (TN / 2 fp32 registers per thread, the m16n8 fragment layout repeated per 8 columns) goes through
//     bias / residual / ReLU in registers and is stored as float2.
// The operands are fp32 in shared memory; the tensor core reads their upper 19 bits (TF32).  W is rounded by the caller.
constexpr int kTcStages = 4;
constexpr int kTcATile = kTM * kKC * 4;        // 16 KB

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// wgmma shared-memory matrix descriptor, K-major 128-byte swizzle (PTX ISA "matrix descriptor format" of
// wgmma.mma_async): start address >> 4 in bits [0,14), leading byte offset (unused for swizzled K-major; 1) in [16,30),
// stride byte offset 1024 >> 4 in [32,46), base offset 0 (tiles are 1024-byte aligned), swizzle mode 1 = 128 B in [62,64)
__device__ __forceinline__ uint64_t wg_smem_desc(const uint32_t saddr) {
  const uint32_t lo = ((saddr & 0x3FFFFu) >> 4) | (1u << 16);
  const uint32_t hi = (1024u >> 4) | (1u << 30);
  return ((uint64_t)hi << 32) | lo;
}

// D (64 x N, fp32 registers) (+)= A (64 x 8, tf32, smem) * B (8 x N, tf32, smem), N = 32 / 64 / 128
__device__ __forceinline__ void wgmma_tf32(float (&d)[16], const uint64_t adesc, const uint64_t bdesc,
                                           const uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, %16, %17, p, 1, 1;\n\t}\n"
      :
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

__device__ __forceinline__ void wgmma_tf32(float (&d)[32], const uint64_t adesc, const uint64_t bdesc,
                                           const uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1;\n\t}\n"
      :
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

__device__ __forceinline__ void wgmma_tf32(float (&d)[64], const uint64_t adesc, const uint64_t bdesc,
                                           const uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, %64, %65, p, 1, 1;\n\t}\n"
      :
        "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

template <int TN>
__global__ void __launch_bounds__(kThreads, 1)
k_gather_gemm_tc(const float* __restrict__ x, const int32_t* __restrict__ idx, int64_t n_out, int K,
                 const float* __restrict__ Wt, const float* __restrict__ bias, const float* __restrict__ res,
                 float* __restrict__ y, int Cin, int Cout, int relu) {
  constexpr int NS = kTcStages;
  constexpr int kBTile = TN * kKC * 4;
  constexpr int kAHalf = kTcATile / 2;                        // 64 rows of the A tile: one warpgroup's operand
  extern __shared__ unsigned char smem_dyn[];
  // 128-byte swizzle atoms repeat every 1024 bytes and the descriptors carry base offset 0: align the tiles by hand
  const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;
  unsigned char* sm = smem_dyn + (base - smem_u32(smem_dyn));
  const uint32_t a_s = base;                                  // [NS][128 rows][128 B]
  const uint32_t b_s = base + NS * kTcATile;                  // [NS][TN rows][128 B]
  int32_t* src_s = reinterpret_cast<int32_t*>(sm + NS * (kTcATile + kBTile));   // [128][K]
  unsigned* kmask_s = reinterpret_cast<unsigned*>(sm + NS * (kTcATile + kBTile) + ((kTM * K * 4 + 15) & ~15));

  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int wg = wid >> 2;                                    // warpgroup: rows 64 wg .. 64 wg + 63
  const int64_t row0 = (int64_t)blockIdx.x * kTM;
  const int n0 = blockIdx.y * TN;
  const int rows_here = (int)min((int64_t)kTM, n_out - row0);

  if (tid == 0) *kmask_s = 0u;
  __syncthreads();
  {
    unsigned mine = 0u;
    const int32_t* ip = idx + row0 * K;
    for (int e = tid; e < kTM * K; e += kThreads) {
      const int r = e / K;
      const int v = r < rows_here ? __ldg(ip + e) : -1;
      src_s[e] = v;
      if (v >= 0) mine |= 1u << (e - r * K);
    }
    mine = __reduce_or_sync(0xffffffffu, mine);
    if (lane == 0 && mine) atomicOr(kmask_s, mine);
  }
  __syncthreads();
  const unsigned km = *kmask_s;
  const int nchunk = Cin / kKC;
  const int nsteps = __popc(km) * nchunk;

  auto issue = [&](const int s) {
    const int buf = s % NS;
    const int k = __fns(km, 0, s / nchunk + 1);
    const int c0 = (s - (s / nchunk) * nchunk) * kKC;
    const uint32_t a = a_s + buf * kTcATile;
#pragma unroll
    for (int j = 0; j < kTM * 8 / kThreads; ++j) {
      const int e = tid + j * kThreads;
      const int r = e >> 3, seg = e & 7;
      const int sidx = src_s[r * K + k];
      const float* gp = x + (int64_t)(sidx >= 0 ? sidx : 0) * Cin + c0 + seg * 4;
      const uint32_t d = a + r * 128 + ((seg ^ (r & 7)) << 4);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(gp), "r"(sidx >= 0 ? 16 : 0) : "memory");
    }
    const uint32_t b = b_s + buf * kBTile;
    const float* wp = Wt + ((int64_t)k * Cout + n0) * Cin + c0;
#pragma unroll
    for (int j = 0; j < TN * 8 / kThreads; ++j) {
      const int e = tid + j * kThreads;
      const int r = e >> 3, seg = e & 7;
      const uint32_t d = b + r * 128 + ((seg ^ (r & 7)) << 4);
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16, 16;" ::"r"(d), "l"(wp + (int64_t)r * Cin + seg * 4) : "memory");
    }
  };

  float acc[TN / 2];
#pragma unroll
  for (int i = 0; i < TN / 2; ++i) acc[i] = 0.f;

  constexpr int PF = NS - 2;                   // gather distance: stage (s + PF) % NS was last read by step s - 2
  for (int p = 0; p < PF; ++p) {
    if (p < nsteps) issue(p);
    cp_async_commit();
  }
  for (int s = 0; s < nsteps; ++s) {
    cp_async_wait<PF - 1>();                   // this thread's copies of step s have landed ...
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // ... and are visible to the tensor core's proxy
    // every thread's copies of step s are in; both warpgroups have retired the MMAs of step s - 2
    __syncthreads();
    if (s + PF < nsteps) issue(s + PF);
    cp_async_commit();
    const int buf = s % NS;
    const uint64_t ad = wg_smem_desc(a_s + buf * kTcATile + wg * kAHalf), bd = wg_smem_desc(b_s + buf * kBTile);
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (int kk = 0; kk < kKC / 8; ++kk)       // 8 TF32 = 32 bytes along K inside the 128-byte swizzle row
      wgmma_tf32(acc, ad + (uint64_t)(kk * 2), bd + (uint64_t)(kk * 2), (s | kk) != 0);
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");
  }
  asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
  cp_async_wait<0>();
  // epilogue: warp w of the warpgroup holds rows 16 w + g and 16 w + g + 8 (g = lane / 4) of its 64, columns
  // 8 j + 2 t, 8 j + 2 t + 1 (t = lane % 4) in acc[4 j .. 4 j + 3]
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int64_t r = row0 + wg * 64 + (wid & 3) * 16 + g + 8 * h;
    if (r >= n_out) continue;
#pragma unroll
    for (int j = 0; j < TN / 8; ++j) {
      const int cidx = n0 + j * 8 + 2 * t;
      float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
      if (bias) { v0 += __ldg(bias + cidx); v1 += __ldg(bias + cidx + 1); }
      if (res) {
        const float2 rv = __ldg(reinterpret_cast<const float2*>(res + r * Cout + cidx));
        v0 += rv.x; v1 += rv.y;
      }
      if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      *reinterpret_cast<float2*>(y + r * Cout + cidx) = make_float2(v0, v1);
    }
  }
}

template <int TN>
int launch_tc(dim3 grid, cudaStream_t s, const float* x, const int32_t* idx, int64_t n_out, int K, const float* Wt,
              const float* bias, const float* res, float* y, int c_in, int c_out, int relu) {
  const size_t smem = 1024 + (size_t)kTcStages * (kTcATile + TN * kKC * 4) + (((size_t)kTM * K * 4 + 15) & ~(size_t)15) +
                      16;
  if (smem > 227 * 1024) return NKSR_E_INVALID;     // the sm_90 limit per block
  if (cudaFuncSetAttribute(k_gather_gemm_tc<TN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return NKSR_E_CUDA;
  k_gather_gemm_tc<TN><<<grid, kThreads, smem, s>>>(x, idx, n_out, K, Wt, bias, res, y, c_in, c_out, relu);
  return NKSR_OK;
}

}  // namespace

extern "C" {

int nksr_gather_gemm(const float* x, const int32_t* idx, int64_t n_out, int K, const float* W, const float* bias,
                     const float* res, float* y, int c_in, int c_out, int relu, int tf32, void* stream) {
  if (tf32 < 0 || tf32 > 3) return NKSR_E_INVALID;
  if (n_out < 0 || K < 1 || c_in < kKC || c_in % kKC != 0 || c_out < 32 || c_out % 32 != 0) return NKSR_E_INVALID;
  if (n_out == 0) return NKSR_OK;
  if (!x || !idx || !W || !y) return NKSR_E_INVALID;
  cudaStream_t s = as_stream(stream);
  const int tn = c_out % 64 == 0 ? 64 : 32;
  const dim3 grid((unsigned)((n_out + kTM - 1) / kTM), (unsigned)(c_out / tn));
  if (K > 32 && tf32) return NKSR_E_INVALID;           // the tile's offset mask is one 32-bit word
  if (tf32 == 3) {                                     // wgmma: W is [K][c_out][c_in], rounded to TF32
    // 128 output channels per CTA where the layer is that wide: the gathered rows are fetched once per 128 columns
    int rc;
    if (c_out % 128 == 0) {
      const dim3 g128(grid.x, (unsigned)(c_out / 128));
      rc = launch_tc<128>(g128, s, x, idx, n_out, K, W, bias, res, y, c_in, c_out, relu);
    } else {
      rc = tn == 64 ? launch_tc<64>(grid, s, x, idx, n_out, K, W, bias, res, y, c_in, c_out, relu)
                    : launch_tc<32>(grid, s, x, idx, n_out, K, W, bias, res, y, c_in, c_out, relu);
    }
    if (rc != NKSR_OK) return rc;
  } else if (tf32) {
    int rc;
    if (tn == 64)
      rc = tf32 == 2 ? launch_tf32<64, true>(grid, s, x, idx, n_out, K, W, bias, res, y, c_in, c_out, relu)
                     : launch_tf32<64, false>(grid, s, x, idx, n_out, K, W, bias, res, y, c_in, c_out, relu);
    else
      rc = tf32 == 2 ? launch_tf32<32, true>(grid, s, x, idx, n_out, K, W, bias, res, y, c_in, c_out, relu)
                     : launch_tf32<32, false>(grid, s, x, idx, n_out, K, W, bias, res, y, c_in, c_out, relu);
    if (rc != NKSR_OK) return rc;
  } else {
    if (tn == 64)
      k_gather_gemm_f32<64><<<grid, kThreads, 0, s>>>(x, idx, n_out, K, W, bias, res, y, c_in, c_out, relu);
    else
      k_gather_gemm_f32<32><<<grid, kThreads, 0, s>>>(x, idx, n_out, K, W, bias, res, y, c_in, c_out, relu);
  }
  NKSR_CHECK_LAUNCH();
  return NKSR_OK;
}

}  // extern "C"
