// The neural kernel of DESIGN.md SPEC S4, K_l(x, i) = B3((x - c_i)/W_l) * <phi_l(x), z_i>, phi_l(x) = trilinear
// interpolation of z.  This header is the one device definition of the kernel's geometry: voxel_centre and
// local_coord give the fp64-subtracted local coordinate tau, stencil_weights the B-spline and tent weights of a
// stencil slot and their derivatives.  Every kernel that evaluates K or its gradient (row building, field
// evaluation, the backward in field_bwd.cu) takes its geometry from here, so forward and backward cannot disagree;
// each keeps only its own loop over the feature channels.  (The compact gradient rows of the Gram fill use the
// polynomial form in gram_common.cuh, which is not bitwise these weights.)
#pragma once
#include "common.cuh"

// fp64 centre, in level-l voxel units, of the level-l voxel with offset-space coordinate u (SPEC S1)
__device__ __forceinline__ double voxel_centre(int u, int level) { return (double)(u - level_offset(level)) + 0.5; }

// local coordinate tau in [-.5,.5) of p in the voxel with centre c (voxel_centre); inv = 1 / W_l.  The subtraction is
// done in fp64 to avoid cancellation.
__device__ __forceinline__ float local_coord(float p, double inv, double c) { return (float)((double)p * inv - c); }

// weights of neighbour d in {-1,0,1} along one axis at local coordinate tau in [-.5,.5)
// Tent derivative (SPEC S4): one-sided derivative of the trilinear cell containing x, except in
// the snap zone |tau| < 2^-12 around a voxel centre, where the symmetric derivative is used --
// the reference places its normal constraints exactly AT voxel centres (models/nksr_net.py:100),
// where a one-sided rule would depend on the last rounding bit of the coordinate.
#define NKSR_TENT_SNAP 0.000244140625f
__device__ __forceinline__ void axis_weights(float tau, int d, float& b, float& db, float& t, float& dt) {
  const bool mid = fabsf(tau) < NKSR_TENT_SNAP;
  if (d == 0) {
    b = 0.75f - tau * tau;
    db = -2.f * tau;
    t = tau >= 0.f ? 1.f - tau : 1.f + tau;
    dt = mid ? 0.f : (tau >= 0.f ? -1.f : 1.f);
  } else if (d < 0) {
    float h = 0.5f - tau;
    b = 0.5f * h * h;
    db = -h;
    t = tau >= 0.f ? 0.f : -tau;
    dt = mid ? -0.5f : (tau >= 0.f ? 0.f : -1.f);
  } else {
    float h = 0.5f + tau;
    b = 0.5f * h * h;
    db = h;
    t = tau >= 0.f ? tau : 0.f;
    dt = mid ? 0.5f : (tau >= 0.f ? 1.f : 0.f);
  }
}

// weights of the stencil slot at offset (dx,dy,dz) for a location at local coordinate (tx,ty,tz) in its containing
// voxel: per-axis factors, multiplied where they are used; derivatives are with respect to tau (divide by W_l for x)
struct StencilWeights {
  float b[3], db[3], t[3], dt[3];
  __device__ __forceinline__ float B3() const { return b[0] * b[1] * b[2]; }      // B-spline product
  __device__ __forceinline__ float T3() const { return t[0] * t[1] * t[2]; }      // tent (trilinear) product
  __device__ __forceinline__ float dB(int a) const {                              // d B3 / d tau_a
    return a == 0 ? db[0] * b[1] * b[2] : (a == 1 ? b[0] * db[1] * b[2] : b[0] * b[1] * db[2]);
  }
  __device__ __forceinline__ float dT3(int a) const {                             // d T3 / d tau_a
    return a == 0 ? dt[0] * t[1] * t[2] : (a == 1 ? t[0] * dt[1] * t[2] : t[0] * t[1] * dt[2]);
  }
};
__device__ __forceinline__ StencilWeights stencil_weights(float tx, float ty, float tz, int dx, int dy, int dz) {
  StencilWeights w;
  axis_weights(tx, dx, w.b[0], w.db[0], w.t[0], w.dt[0]);
  axis_weights(ty, dy, w.b[1], w.db[1], w.t[1], w.dt[1]);
  axis_weights(tz, dz, w.b[2], w.db[2], w.t[2], w.dt[2]);
  return w;
}

// Per-(location, level) evaluation, one warp per location, lane = stencil slot.  Shared by row building (Gram
// assembly) and field evaluation.
struct LaneKernel {
  int nb;       // neighbour voxel index of this lane's slot (-1: none / lane >= 27)
  float k;      // K_l(x, nb)
  float dk[3];  // grad_x K_l(x, nb)
  float dot;    // <phi_l(x), z_nb>  (0 when nb < 0)
  float tau[3]; // local coordinate of x in the containing voxel
};

// All 32 lanes must call.  base >= 0.  GRAD: also the gradient; FULLGRAD: include the
// grad(phi) term (approx_kernel_grad == false).
// (ux,uy,uz): offset-space coordinates of the containing voxel `base` -- the caller already has them from the
// point's own quantisation (h >> (level+1), SPEC S1), so the key is neither loaded nor decoded;
// inv0 = 1 / voxel_size in fp64, computed once per location (1/(W 2^l) = inv0 * 2^-l exactly).
template <bool GRAD>
__device__ __forceinline__ LaneKernel eval_level_lane(const int32_t* __restrict__ nbr27,
                                                      const float* __restrict__ z, int C, int level,
                                                      float wl, double inv0, float px, float py, float pz, int base,
                                                      int ux, int uy, int uz, bool fullgrad, int lane) {
  LaneKernel r;
  const double inv = inv0 * (1.0 / (double)(1 << level));
  const float tx = local_coord(px, inv, voxel_centre(ux, level));
  const float ty = local_coord(py, inv, voxel_centre(uy, level));
  const float tz = local_coord(pz, inv, voxel_centre(uz, level));
  int dx, dy, dz;
  slot_to_d(lane < 27 ? lane : 13, dx, dy, dz);
  const StencilWeights w = stencil_weights(tx, ty, tz, dx, dy, dz);
  r.nb = lane < 27 ? __ldg(nbr27 + (int64_t)base * 27 + lane) : -1;
  const bool ok = r.nb >= 0;
  const float B3 = w.B3();
  const float T3 = ok ? w.T3() : 0.f;
  float dT3[3];
  if (GRAD) {
    dT3[0] = ok ? w.dT3(0) : 0.f;
    dT3[1] = ok ? w.dT3(1) : 0.f;
    dT3[2] = ok ? w.dT3(2) : 0.f;
  }
  float dot = 0.f, ddot[3] = {0.f, 0.f, 0.f};
  const float* zr = z + (int64_t)(ok ? r.nb : 0) * C;
  auto channel = [&](const float zc) {
    float phi = warp_sum(T3 * zc);
    dot = fmaf(phi, zc, dot);
    if (GRAD && fullgrad) {
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        float dphi = warp_sum(dT3[a] * zc);
        ddot[a] = fmaf(dphi, zc, ddot[a]);
      }
    }
  };
  if ((C & 3) == 0) {
    // the 27 lanes read 27 different feature rows: every load instruction is a 27-wavefront gather in L1, so fetch
    // four channels per instruction (rows of C = 4, 8, 16 ... floats are 16-byte aligned); same arithmetic, same order
    for (int c4 = 0; c4 < C; c4 += 4) {
      const float4 v = ok ? __ldg(reinterpret_cast<const float4*>(zr + c4)) : make_float4(0.f, 0.f, 0.f, 0.f);
      channel(v.x); channel(v.y); channel(v.z); channel(v.w);
    }
  } else {
    for (int c = 0; c < C; ++c) channel(ok ? __ldg(zr + c) : 0.f);
  }
  r.k = ok ? B3 * dot : 0.f;
  r.dot = ok ? dot : 0.f;
  r.tau[0] = tx; r.tau[1] = ty; r.tau[2] = tz;
  if (GRAD) {
    const float iw = 1.f / wl;
    r.dk[0] = ok ? (w.dB(0) * dot + B3 * ddot[0]) * iw : 0.f;
    r.dk[1] = ok ? (w.dB(1) * dot + B3 * ddot[1]) * iw : 0.f;
    r.dk[2] = ok ? (w.dB(2) * dot + B3 * ddot[2]) * iw : 0.f;
  } else {
    r.dk[0] = r.dk[1] = r.dk[2] = 0.f;
  }
  return r;
}
