"""CPU oracle for the NKSR reconstruction hot path -- TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED: the reference ships this path as a closed wheel (SURVEY.md section 0 /
section 8c); the reference tree holds no source, golden vector or known-answer test for it.
This file is therefore a first-principles restatement of the algorithm fixed in
DESIGN.md ("SPEC"), anchored on the reference's *call sites*:

  * voxel quantisation floor(xyz / voxel_size)       models/nksr_net.py:66
  * SVH(voxel_size, depth).build_point_splatting     models/nksr_net.py:57-62
  * KernelField(...).solve_non_fused(pos_xyz, normal_xyz, normal_value,
        pos_weight, normal_weight, reg_weight)        models/nksr_net.py:91-112
  * field.evaluate_f(xyz, grad) -> .value/.gradient  models/loss.py:189-198
  * grad f = -normal  (f > 0 inside)                  models/loss.py:192-196, :99
  * field.extract_dual_mesh(grid_upsample, mise_iter) models/nksr_net.py:214,284;
                                                      examples/recons_simple.py:27

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
may import this module.  The product (nksr_b200/) never does.

Everything is numpy/scipy; integer work follows the exact fp32 formulas the CUDA path
uses (bit-exact contract), floating-point work is done in float64 (tolerance contract).
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

MAX_DEPTH = 8
KEY_BITS = 21
HALF_OFFSET = 1 << 20          # offset of half-voxel coordinates (|h| < 2^20)
TENT_SNAP = 2.0 ** -12         # snap zone of the tent derivative around voxel centres


# --------------------------------------------------------------------------- keys
def _part1by2(v: np.ndarray) -> np.ndarray:
    v = v.astype(np.uint64) & np.uint64(0x1FFFFF)
    v = (v | (v << np.uint64(32))) & np.uint64(0x1F00000000FFFF)
    v = (v | (v << np.uint64(16))) & np.uint64(0x1F0000FF0000FF)
    v = (v | (v << np.uint64(8))) & np.uint64(0x100F00F00F00F00F)
    v = (v | (v << np.uint64(4))) & np.uint64(0x10C30C30C30C30C3)
    v = (v | (v << np.uint64(2))) & np.uint64(0x1249249249249249)
    return v


def _compact1by2(v: np.ndarray) -> np.ndarray:
    v = v.astype(np.uint64) & np.uint64(0x1249249249249249)
    v = (v | (v >> np.uint64(2))) & np.uint64(0x10C30C30C30C30C3)
    v = (v | (v >> np.uint64(4))) & np.uint64(0x100F00F00F00F00F)
    v = (v | (v >> np.uint64(8))) & np.uint64(0x1F0000FF0000FF)
    v = (v | (v >> np.uint64(16))) & np.uint64(0x1F00000000FFFF)
    v = (v | (v >> np.uint64(32))) & np.uint64(0x1FFFFF)
    return v


def morton_encode(u: np.ndarray) -> np.ndarray:
    """u: (n,3) non-negative ints < 2^21 -> int64 key; x is the most significant axis."""
    u = np.asarray(u)
    k = (_part1by2(u[:, 0]) << np.uint64(2)) | (_part1by2(u[:, 1]) << np.uint64(1)) | _part1by2(u[:, 2])
    return k.astype(np.int64)


def morton_decode(k: np.ndarray) -> np.ndarray:
    k = np.asarray(k).astype(np.uint64)
    return np.stack([_compact1by2(k >> np.uint64(2)), _compact1by2(k >> np.uint64(1)),
                     _compact1by2(k)], axis=1).astype(np.int64)


def level_offset(level: int) -> int:
    return 1 << (19 - level)


def voxel_key(ijk: np.ndarray, level: int) -> np.ndarray:
    return morton_encode(np.asarray(ijk, dtype=np.int64) + level_offset(level))


def key_to_ijk(key: np.ndarray, level: int) -> np.ndarray:
    return (morton_decode(key) - level_offset(level)).astype(np.int32)


def quantize_half(xyz: np.ndarray, voxel_size: float) -> np.ndarray:
    """h = floor(x / (W/2)) with IEEE fp32 division (SPEC S1).  Every integer coordinate of
    the hierarchy derives from h: containing voxel at level l is h >> (l+1) -- identical to
    the reference's floor(xyz / voxel_size) (models/nksr_net.py:66) since power-of-two
    scalings of the divisor are exact."""
    half_w = np.float32(np.float32(voxel_size) * np.float32(0.5))
    q = np.asarray(xyz, dtype=np.float32) / half_w
    return np.floor(q).astype(np.int32)


def half_key(h: np.ndarray) -> np.ndarray:
    return morton_encode(np.asarray(h, dtype=np.int64) + HALF_OFFSET)


# --------------------------------------------------------------------------- hierarchy
_OFF8 = np.array([[a, b, c] for a in (0, 1) for b in (0, 1) for c in (0, 1)], dtype=np.int64)
_OFF27 = np.array([[a, b, c] for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)], dtype=np.int64)
_OFF125 = np.array([[a, b, c] for a in range(-2, 3) for b in range(-2, 3) for c in range(-2, 3)], dtype=np.int64)


class OracleSVH:
    """Sparse voxel hierarchy: level l has voxel size W*2^l, voxels sorted by Morton key."""

    def __init__(self, voxel_size: float, depth: int):
        self.voxel_size = float(np.float32(voxel_size))
        self.depth = depth
        self.keys = [np.zeros(0, np.int64) for _ in range(depth)]

    # SPEC S2: trilinear (8-nearest-centre) splatting on every level.
    def build_point_splatting(self, xyz: np.ndarray):
        h0 = quantize_half(xyz, self.voxel_size).astype(np.int64)
        for l in range(self.depth):
            hl = h0 >> l
            base = (hl - 1) >> 1
            cand = (base[:, None, :] + _OFF8[None]).reshape(-1, 3)
            self.keys[l] = np.unique(voxel_key(cand, l))
        return self

    def build_from_keys(self, keys):
        self.keys = [np.asarray(k, np.int64) for k in keys]
        return self

    def n(self, l):
        return self.keys[l].shape[0]

    def ijk(self, l):
        return key_to_ijk(self.keys[l], l)

    def level_w(self, l):
        return float(np.float32(self.voxel_size) * np.float32(2 ** l))

    def centers(self, l):
        return ((self.ijk(l).astype(np.float32) + np.float32(0.5)) * np.float32(self.level_w(l))).astype(np.float32)

    def lookup(self, l, ijk):
        """index of voxel ijk at level l, -1 if inactive."""
        ijk = np.asarray(ijk, np.int64)
        off = level_offset(l)
        ok = np.all((ijk + off >= 0) & (ijk + off < (1 << KEY_BITS)), axis=-1)
        k = voxel_key(np.where(ok[..., None], ijk, 0).reshape(-1, 3), l).reshape(ijk.shape[:-1])
        keys = self.keys[l]
        if keys.shape[0] == 0:
            return np.full(ijk.shape[:-1], -1, np.int64)
        pos = np.searchsorted(keys, k)
        posc = np.minimum(pos, keys.shape[0] - 1)
        hit = ok & (keys[posc] == k)
        return np.where(hit, posc, -1)

    def nbr27(self, l):
        ijk = self.ijk(l).astype(np.int64)
        return self.lookup(l, ijk[:, None, :] + _OFF27[None])

    def offsets(self):
        ns = [self.n(l) for l in range(self.depth)]
        return np.concatenate([[0], np.cumsum(ns)]).astype(np.int64)

    def locate(self, xyz):
        """containing-voxel index per level (L, M), -1 if inactive (SPEC S3)."""
        h0 = quantize_half(xyz, self.voxel_size).astype(np.int64)
        return np.stack([self.lookup(l, h0 >> (l + 1)) for l in range(self.depth)])


# --------------------------------------------------------------------------- basis
def _bspline(tau):
    """quadratic B-spline weights of the 3 neighbours d=-1,0,+1 at local coord tau in [-.5,.5)."""
    w = np.stack([0.5 * (0.5 - tau) ** 2, 0.75 - tau ** 2, 0.5 * (0.5 + tau) ** 2], axis=-1)
    dw = np.stack([-(0.5 - tau), -2.0 * tau, (0.5 + tau)], axis=-1)
    return w, dw


def _tent(tau):
    """trilinear (tent) weights of d=-1,0,+1 (SPEC S4).  Derivative: one-sided (the trilinear
    cell containing x) except in the snap zone |tau| < 2^-12 around a voxel centre, where the
    symmetric derivative (-1/2, 0, +1/2) is used: the reference puts its normal constraints
    exactly at voxel centres (models/nksr_net.py:100)."""
    pos = tau >= 0
    mid = np.abs(tau) < TENT_SNAP
    w = np.stack([np.where(pos, 0.0, -tau), np.where(pos, 1.0 - tau, 1.0 + tau), np.where(pos, tau, 0.0)], axis=-1)
    dw = np.stack([np.where(mid, -0.5, np.where(pos, 0.0, -1.0)), np.where(mid, 0.0, np.where(pos, -1.0, 1.0)),
                   np.where(mid, 0.5, np.where(pos, 1.0, 0.0))], axis=-1)
    return w, dw


def _bspline_abs(tau):
    """_bspline with every signed sum replaced by the sum of the absolute values of its terms: the magnitude scale of
    the weights (running-error analysis; it also covers a rounding of tau, e.g. 0.5 - tau near the support edge)"""
    a = np.abs(tau)
    w = np.stack([0.5 * (0.5 + a) ** 2, 0.75 + tau ** 2, 0.5 * (0.5 + a) ** 2], axis=-1)
    dw = np.stack([0.5 + a, 2.0 * a, 0.5 + a], axis=-1)
    return w, dw


def _tent_abs(tau):
    """_tent as sums of absolute values (see _bspline_abs)"""
    pos = tau >= 0
    a = np.abs(tau)
    w = np.stack([np.where(pos, 0.0, a), 1.0 + a, np.where(pos, a, 0.0)], axis=-1)
    return w, np.abs(_tent(tau)[1])


def _prod3(wx, wy, wz):
    return (wx[:, :, None, None] * wy[:, None, :, None] * wz[:, None, None, :]).reshape(wx.shape[0], 27)


def _level_tau(svh: OracleSVH, l: int, xyz: np.ndarray, base: np.ndarray):
    """neighbour table rows (M,27) (-1 = none) and local coordinates tau (M,3) in the containing voxel of level l"""
    M = xyz.shape[0]
    ok = base >= 0
    b = np.where(ok, base, 0)
    ijk = svh.ijk(l).astype(np.int64)
    nbr = svh.nbr27(l)[b] if svh.n(l) else np.full((M, 27), -1)
    nbr = np.where(ok[:, None], nbr, -1)
    cb = ijk[b] if svh.n(l) else np.zeros((M, 3), np.int64)
    return nbr, xyz.astype(np.float64) / svh.level_w(l) - (cb + 0.5)


def tent_branch_ambiguous(svh: OracleSVH, xyz: np.ndarray, ulps: int = 4) -> np.ndarray:
    """(M,) bool: locations where an fp32 tau within `ulps` ulps of the fp64 one falls on the other side of the snap
    zone |tau| < 2^-12 of the tent derivative on some level.  There an fp32 evaluation may take the other (one-sided vs
    symmetric) derivative, which is a different formula, not a rounding error."""
    base = svh.locate(xyz)
    amb = np.zeros(xyz.shape[0], bool)
    for l in range(svh.depth):
        if svh.n(l) == 0:
            continue
        _, tau = _level_tau(svh, l, xyz, base[l])
        mid = np.abs(tau) < TENT_SNAP
        t32 = tau.astype(np.float32)
        for k in range(-ulps, ulps + 1):
            near = (t32 + np.float32(k) * np.spacing(t32)).astype(np.float64)
            amb |= np.any((np.abs(near) < TENT_SNAP) != mid, axis=1) & (base[l] >= 0)
    return amb


def level_rows(svh: OracleSVH, l: int, xyz: np.ndarray, base: np.ndarray, z: np.ndarray,
               want_grad: bool, approx_kernel_grad: bool, abs_terms: bool = False):
    """Kernel row entries of level l for M locations.

    returns cols (M,27) int (-1 = none), K (M,27), and dK (M,3,27) if want_grad.
    K_l(x, i) = B3((x-c_i)/W_l) * <phi_l(x), z_i>, phi_l = trilinear interpolation of z (SPEC S4).
    Rows whose containing voxel is inactive have no entries at this level (SPEC S3).
    abs_terms: also return Kabs, dKabs -- the same expressions with the B-spline and tent weights, their derivatives
    and z replaced by their sums of absolute values: the scale of the rounding error of any evaluation of K, dK.
    """
    nbr, K, dK = _level_rows(svh, l, xyz, base, z, want_grad, approx_kernel_grad, _bspline, _tent)
    if not abs_terms:
        return nbr, K, dK
    _, Ka, dKa = _level_rows(svh, l, xyz, base, np.abs(z), want_grad, approx_kernel_grad, _bspline_abs, _tent_abs)
    return nbr, K, dK, Ka, dKa


def _level_rows(svh, l, xyz, base, z, want_grad, approx_kernel_grad, bspline, tent):
    M = xyz.shape[0]
    W = svh.level_w(l)
    nbr, tau = _level_tau(svh, l, xyz, base)
    Bw, dBw = zip(*[bspline(tau[:, a]) for a in range(3)])
    Tw, dTw = zip(*[tent(tau[:, a]) for a in range(3)])
    B3 = _prod3(*Bw)
    T3 = _prod3(*Tw)
    zn = np.where((nbr >= 0)[:, :, None], z[np.maximum(nbr, 0)], 0.0).astype(np.float64)  # (M,27,C)
    phi = np.einsum('ms,msc->mc', T3, zn)
    dots = np.einsum('mc,msc->ms', phi, zn)
    K = B3 * dots
    K = np.where(nbr >= 0, K, 0.0)
    if not want_grad:
        return nbr, K, None
    dK = np.zeros((M, 3, 27))
    for a in range(3):
        Bd = list(Bw); Bd[a] = dBw[a]
        dB3 = _prod3(*Bd) / W
        dK[:, a] = dB3 * dots
        if not approx_kernel_grad:
            Td = list(Tw); Td[a] = dTw[a]
            dT3 = _prod3(*Td) / W
            dphi = np.einsum('ms,msc->mc', dT3, zn)
            dK[:, a] += B3 * np.einsum('mc,msc->ms', dphi, zn)
    dK = np.where((nbr >= 0)[:, None, :], dK, 0.0)
    return nbr, K, dK


def build_system(svh: OracleSVH, feats, pos_xyz, normal_xyz, normal_value,
                 pos_weight, normal_weight, reg_weight, approx_kernel_grad=False, abs_terms=False):
    """A = E^T diag(w) E + reg*R,  b = E^T diag(w) t   (SPEC S5).

    E rows: one per position constraint (target 0, weight pos_weight) and three per normal
    constraint (d/dx, d/dy, d/dz of f at normal_xyz; target normal_value; weight normal_weight).
    R is block-diagonal per level: R_ii' = K_l(c_i', i) for |i-i'|_inf <= 1.
    Call site: models/nksr_net.py:100-112.
    abs_terms: also return Aabs = |E|^T diag(w) |E| + reg*|R| and babs = |E|^T diag(w) |t|, where |E| holds the
    abs-term rows (level_rows(abs_terms=True)) and |R| the regulariser of |z|: the per-entry error scales.
    """
    offs = svh.offsets()
    n = int(offs[-1])
    N, Kn = pos_xyz.shape[0], normal_xyz.shape[0]
    rows, cols, vals, avals = [], [], [], []
    base_p = svh.locate(pos_xyz)
    base_n = svh.locate(normal_xyz) if Kn else np.zeros((svh.depth, 0), np.int64)
    for l in range(svh.depth):
        if svh.n(l) == 0:
            continue
        nbr, K, _, *ab = level_rows(svh, l, pos_xyz, base_p[l], feats[l], False, approx_kernel_grad, abs_terms)
        r = np.repeat(np.arange(N), 27).reshape(N, 27)
        m = nbr >= 0
        rows.append(r[m]); cols.append(nbr[m] + offs[l]); vals.append(K[m])
        if abs_terms:
            avals.append(ab[0][m])
        if Kn:
            nbr, _, dK, *ab = level_rows(svh, l, normal_xyz, base_n[l], feats[l], True, approx_kernel_grad, abs_terms)
            m = nbr >= 0
            for a in range(3):
                r = np.repeat(N + 3 * np.arange(Kn) + a, 27).reshape(Kn, 27)
                rows.append(r[m]); cols.append(nbr[m] + offs[l]); vals.append(dK[:, a][m])
                if abs_terms:
                    avals.append(ab[1][:, a][m])
    M = N + 3 * Kn
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    E = sp.csr_matrix((np.concatenate(vals), (rows, cols)), shape=(M, n))
    w = np.concatenate([np.full(N, pos_weight, np.float64), np.full(3 * Kn, normal_weight, np.float64)])
    t = np.concatenate([np.zeros(N), np.asarray(normal_value, np.float64).reshape(-1)])
    EW = E.T.multiply(w[None, :]).tocsr()
    A = (EW @ E).tocsr()
    b = EW @ t
    A = A + reg_weight * build_regulariser(svh, feats)
    if not abs_terms:
        return A.tocsr(), b, E
    Ea = sp.csr_matrix((np.concatenate(avals), (rows, cols)), shape=(M, n))
    EaW = Ea.T.multiply(np.abs(w)[None, :]).tocsr()
    Aabs = (EaW @ Ea).tocsr() + abs(reg_weight) * build_regulariser(svh, [np.abs(f) for f in feats])
    return A.tocsr(), b, E, Aabs.tocsr(), EaW @ np.abs(t)


def build_regulariser(svh: OracleSVH, feats):
    offs = svh.offsets()
    n = int(offs[-1])
    b1 = np.array([0.125, 0.75, 0.125])
    B3c = (b1[:, None, None] * b1[None, :, None] * b1[None, None, :]).reshape(27)
    rows, cols, vals = [], [], []
    for l in range(svh.depth):
        if svh.n(l) == 0:
            continue
        nbr = svh.nbr27(l)
        z = feats[l].astype(np.float64)
        zn = z[np.maximum(nbr, 0)]
        v = B3c[None, :] * np.einsum('nc,nsc->ns', z, zn)
        m = nbr >= 0
        r = np.repeat(np.arange(svh.n(l)), 27).reshape(-1, 27)
        rows.append(r[m] + offs[l]); cols.append(nbr[m] + offs[l]); vals.append(v[m])
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(n, n))


def structural_pattern(svh: OracleSVH):
    """The stored sparsity pattern P of A (SPEC S6): same-level 125-stencil plus, for a fine
    voxel i (level l) and each coarser level l', every active voxel of the 27-stencils of
    (c_i + a) >> (l'-l), a in {-1,0,1}^3; plus the transposes.  Returned as a 0/1 csr."""
    offs = svh.offsets()
    n = int(offs[-1])
    rows, cols = [], []
    for l in range(svh.depth):
        if svh.n(l) == 0:
            continue
        ijk = svh.ijk(l).astype(np.int64)
        nb = svh.lookup(l, ijk[:, None, :] + _OFF125[None])
        r = np.repeat(np.arange(svh.n(l)), 125).reshape(-1, 125)
        m = nb >= 0
        rows.append(r[m] + offs[l]); cols.append(nb[m] + offs[l])
        for lu in range(l + 1, svh.depth):
            if svh.n(lu) == 0:
                continue
            k = lu - l
            lo = ((ijk - 1) >> k) - 1
            off4 = np.array([[a, b, c] for a in range(4) for b in range(4) for c in range(4)], np.int64)
            cand = lo[:, None, :] + off4[None]
            hi = ((ijk + 1) >> k) + 1
            inr = np.all(cand <= hi[:, None, :], axis=-1)
            nb = svh.lookup(lu, cand)
            m = (nb >= 0) & inr
            r = np.repeat(np.arange(svh.n(l)), 64).reshape(-1, 64)
            rows.append(r[m] + offs[l]); cols.append(nb[m] + offs[lu])
            rows.append(nb[m] + offs[lu]); cols.append(r[m] + offs[l])
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    P = sp.csr_matrix((np.ones(rows.shape[0], np.int8), (rows, cols)), shape=(n, n))
    P.sum_duplicates()
    P.data[:] = 1
    return P


# --------------------------------------------------------------------------- solver
def _jacobi_inverse(A, diag, dtype):
    """1/d where d > 0, else 0 (the solver's preconditioner); d = A's diagonal unless given"""
    d = A.diagonal() if diag is None else np.asarray(diag, np.float64)
    return np.where(d > 0, 1.0 / np.where(d > 0, d, 1), 0.0).astype(dtype)


def pcg(A, b, tol=1e-5, max_iter=2000, x0=None, dtype=np.float64, diag=None, history=None):
    """Jacobi-preconditioned CG (SPEC S7); stop at ||r|| <= tol*||b||.  Returns x, iters, relres.
    diag: the preconditioner's diagonal (default: A's).  history: a list that receives (x_k, relres_k) after every
    iteration k = 1, 2, ..."""
    A = A.astype(dtype)
    b = b.astype(dtype)
    dinv = _jacobi_inverse(A, diag, dtype)
    x = np.zeros_like(b) if x0 is None else x0.astype(dtype).copy()
    r = b - A @ x
    z = dinv * r
    p = z.copy()
    rz = float(r.astype(np.float64) @ z.astype(np.float64))
    bn = float(np.linalg.norm(b.astype(np.float64)))
    if bn == 0:
        return x, 0, 0.0
    it = 0
    res = float(np.linalg.norm(r.astype(np.float64))) / bn
    while it < max_iter and res > tol:
        Ap = A @ p
        pAp = float(p.astype(np.float64) @ Ap.astype(np.float64))
        alpha = dtype(rz / pAp)
        x += alpha * p
        r -= alpha * Ap
        z = dinv * r
        rz_new = float(r.astype(np.float64) @ z.astype(np.float64))
        beta = dtype(rz_new / rz)
        rz = rz_new
        p = z + beta * p
        it += 1
        res = float(np.linalg.norm(r.astype(np.float64))) / bn
        if history is not None:
            history.append((x.copy(), res))
    return x, it, res


def pcg_cg(A, b, tol=1e-5, max_iter=2000, dtype=np.float64, diag=None, history=None):
    """The same Jacobi-PCG in the Chronopoulos-Gear arrangement of the distributed solve (csrc/solve.cu, nksr_dcg_*):
    one sweep per iteration forms w = A u and the three dots (r,u), (w,u), (r,r) of the CURRENT iterate, then
        beta = gamma / gamma_prev,  alpha = gamma / (delta - beta gamma / alpha_prev)   (alpha = gamma / delta first)
        p = u + beta p;  s = w + beta s;  x += alpha p;  r -= alpha s;  u = M^-1 r.
    In exact arithmetic its iterates are those of pcg().  Returns x, iters, relres; history as in pcg()."""
    A = A.astype(dtype)
    b = b.astype(dtype)
    dinv = _jacobi_inverse(A, diag, dtype)
    x = np.zeros_like(b)
    r = b.copy()
    u = dinv * r
    p = np.zeros_like(b)
    s = np.zeros_like(b)
    bn = float(np.linalg.norm(b.astype(np.float64)))
    if bn == 0:
        return x, 0, 0.0
    it, gamma_prev, alpha_prev = 0, 0.0, 0.0
    while True:
        w = A @ u
        gamma = float(r.astype(np.float64) @ u.astype(np.float64))
        delta = float(w.astype(np.float64) @ u.astype(np.float64))
        res = float(np.linalg.norm(r.astype(np.float64))) / bn
        if res <= tol or it >= max_iter:
            return x, it, res
        beta = gamma / gamma_prev if it > 0 else 0.0
        alpha = gamma / (delta - beta * gamma / alpha_prev) if it > 0 else gamma / delta
        p = u + dtype(beta) * p
        s = w + dtype(beta) * s
        x += dtype(alpha) * p
        r -= dtype(alpha) * s
        u = dinv * r
        it += 1
        gamma_prev, alpha_prev = gamma, alpha
        if history is not None:
            history.append((x.copy(), float(np.linalg.norm(r.astype(np.float64))) / bn))


# --------------------------------------------------------------------------- field evaluation
def evaluate_f(svh: OracleSVH, feats, alpha, xyz, grad=False, approx_kernel_grad=False, abs_terms=False):
    """f(x) = sum_l [b_l(x) active] sum_{i in N27(b_l(x))} alpha_i K_l(x,i)  (SPEC S3/S4).
    Call site: models/loss.py:189-198,225.
    abs_terms: also return fabs = sum |alpha_i| Kabs_l(x,i) (and gabs from dKabs), the per-query error scales; the
    result is then (f, fabs) or (f, g, fabs, gabs)."""
    offs = svh.offsets()
    base = svh.locate(xyz)
    f = np.zeros(xyz.shape[0])
    g = np.zeros((xyz.shape[0], 3)) if grad else None
    fa = np.zeros(xyz.shape[0])
    ga = np.zeros((xyz.shape[0], 3)) if grad else None
    for l in range(svh.depth):
        if svh.n(l) == 0:
            continue
        nbr, K, dK, *ab = level_rows(svh, l, xyz, base[l], feats[l], grad, approx_kernel_grad, abs_terms)
        a = np.where(nbr >= 0, alpha[np.maximum(nbr, 0) + offs[l]], 0.0)
        f += np.sum(a * K, axis=1)
        if grad:
            g += np.einsum('ms,mas->ma', a, dK)
        if abs_terms:
            fa += np.sum(np.abs(a) * ab[0], axis=1)
            if grad:
                ga += np.einsum('ms,mas->ma', np.abs(a), ab[1])
    if abs_terms:
        return (f, g, fa, ga) if grad else (f, fa)
    return (f, g) if grad else f


# --------------------------------------------------------------------------- marching cubes tables
# corner c = (cx<<2)|(cy<<1)|cz ; edges enumerated axis-major.
MC_CORNERS = np.array([[(c >> 2) & 1, (c >> 1) & 1, c & 1] for c in range(8)], np.int64)
MC_EDGES = []           # (corner_a, corner_b, axis) with a < b along axis
for _ax in range(3):
    for _c in range(8):
        if not (_c >> (2 - _ax)) & 1:
            MC_EDGES.append((_c, _c | (1 << (2 - _ax)), _ax))
MC_EDGES = np.array(MC_EDGES, np.int64)     # 12 edges


def _face_list():
    """six faces, each as 4 corners in cyclic order seen from outside the cube (CCW)."""
    faces = []
    for ax in range(3):
        u, v = (ax + 1) % 3, (ax + 2) % 3
        for side in (0, 1):
            quad = []
            for (a, b) in ((0, 0), (1, 0), (1, 1), (0, 1)):
                p = [0, 0, 0]
                p[ax] = side; p[u] = a; p[v] = b
                quad.append((p[0] << 2) | (p[1] << 1) | p[2])
            if side == 0:
                quad = quad[::-1]
            faces.append(quad)
    return faces


def build_mc_table():
    """Procedural 256-case triangle table (SPEC S9).

    Inside = corner bit set (f > 0).  On every cube face the iso-contour is traced with the
    marching-squares rule "ambiguous faces separate the inside corners"; because that rule
    only looks at the face's own corner signs, neighbouring cells agree and the surface is
    watertight.  Face segments are chained into closed loops around the inside corners and
    fan-triangulated (reversed), so that triangle normals point from inside (f>0) to outside
    (f<0), i.e. along -grad f, matching the reference's outward-normal convention
    (models/loss.py:192-196).
    Returns (tri_table int8 [256, MAXT*3] padded with -1, n_tri int [256]).
    """
    edge_id = {}
    for e, (a, b, _) in enumerate(MC_EDGES):
        edge_id[(int(a), int(b))] = e
        edge_id[(int(b), int(a))] = e
    faces = _face_list()
    tables = []
    for case in range(256):
        inside = [(case >> c) & 1 for c in range(8)]
        nxt = {}
        for quad in faces:
            s = [inside[c] for c in quad]
            # directed segments: walking the face boundary CCW (seen from outside), a segment
            # starts on the edge where we go outside->inside ... we emit it so that the inside
            # region is on the left: from the "leaving inside" edge to the "entering inside" edge
            # around each connected run of inside corners (runs are separated on ambiguous faces).
            k = sum(s)
            if k == 0 or k == 4:
                continue
            # runs of consecutive inside corners in cyclic order
            runs = []
            for i in range(4):
                if s[i] and not s[(i - 1) % 4]:
                    j = i
                    while s[(j + 1) % 4] and (j + 1) % 4 != i:
                        j += 1
                    runs.append((i, j % 4))
            for (i, j) in runs:
                e_in = edge_id[(quad[(i - 1) % 4], quad[i])]      # edge before the run
                e_out = edge_id[(quad[j], quad[(j + 1) % 4])]     # edge after the run
                # inside corners i..j lie CCW from e_in to e_out; the segment e_out -> e_in
                # keeps them on its left when seen from outside.
                assert e_out not in nxt
                nxt[e_out] = e_in
        tris = []
        seen = set()
        for start in sorted(nxt):
            if start in seen:
                continue
            loop = [start]
            seen.add(start)
            cur = nxt[start]
            while cur != start:
                loop.append(cur)
                seen.add(cur)
                cur = nxt[cur]
            for t in range(1, len(loop) - 1):
                tris.append((loop[0], loop[t + 1], loop[t]))
        tables.append(tris)
    maxt = max(len(t) for t in tables)
    tab = np.full((256, maxt * 3), -1, np.int8)
    cnt = np.zeros(256, np.int32)
    for c, tris in enumerate(tables):
        cnt[c] = len(tris)
        for t, tri in enumerate(tris):
            tab[c, 3 * t:3 * t + 3] = tri
    return tab, cnt


# --------------------------------------------------------------------------- dual mesh extraction
def lattice_pos(s, W, R):
    """world position of integer lattice point s at refinement R: W*(0.5 + s/R)  (SPEC S8)."""
    return (np.float32(W) * (np.float32(0.5) + s.astype(np.float32) / np.float32(R))).astype(np.float32)


def extract_dual_mesh(svh: OracleSVH, eval_fn, grid_upsample=1, mise_iter=0, mask_fn=None, coarse_levels=1):
    """Dual marching cubes with MISE refinement (SPEC S8-S10).

    Stage-0 cells are the cubes spanned by the centres of 2x2x2 active finest voxels (the dual
    of the primal grid).  Cells are uniformly split `grid_upsample` times per axis; each MISE
    round evaluates f on the cell corners, keeps the cells whose corner signs are mixed and
    splits them 2x per axis.  The final cells are triangulated with the procedural MC table;
    vertices are welded per lattice edge and ordered by edge key (Morton of the lower end
    relative to the stage-0 minimum, then axis); faces follow cell order then table order.  eval_fn(xyz float32 (M,3)) -> f (M,).  Returns v (V,3) f32, f (T,3) i64.
    """
    W = svh.voxel_size
    R = grid_upsample * (2 ** mise_iter)
    ijk = svh.ijk(0).astype(np.int64)
    if coarse_levels <= 1:
        nb = svh.lookup(0, ijk[:, None, :] + _OFF8[None])
        cells = ijk[np.all(nb >= 0, axis=1)] * R              # min-corner lattice coords
    else:
        # adaptive hierarchies (models/nksr_net.py:175-179,214): a leaf of level 1 .. coarse_levels-1 counts as
        # subdivided down to the finest level ("virtual" finest voxels); cells = cubes between 2x2x2 finest voxels,
        # real or virtual.  Anchors: the real finest voxels, then the virtual ones level by level, leaf by leaf, x-major.
        leaf = {}
        anchors = [ijk]
        for l in range(1, min(coarse_levels, svh.depth)):
            leaf[l] = ~np.isin(svh.keys[l], svh.keys[l - 1] >> 3)
            lij = svh.ijk(l).astype(np.int64)[leaf[l]]
            m = 1 << l
            sub = np.array([[a, b, c] for a in range(m) for b in range(m) for c in range(m)], np.int64)
            anchors.append(((lij << l)[:, None, :] + sub[None]).reshape(-1, 3))
        anchors = np.concatenate(anchors)

        def exists(j):
            ok = svh.lookup(0, j) >= 0
            for l, lf in leaf.items():
                v = svh.lookup(l, j >> l)
                ok |= (v >= 0) & lf[np.maximum(v, 0)]
            return ok
        ok = np.ones(anchors.shape[0], bool)
        for c in range(1, 8):
            ok &= exists(anchors + _OFF8[c][None])
        cells = anchors[ok] * R
    size = R
    if cells.shape[0] == 0:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64)
    cmin = cells.min(axis=0)                                # key origin (SPEC S10)
    # uniform upsample
    if grid_upsample > 1:
        g = grid_upsample
        sub = np.array([[a, b, c] for a in range(g) for b in range(g) for c in range(g)], np.int64) * (size // g)
        cells = (cells[:, None, :] + sub[None]).reshape(-1, 3)
        size //= g
    tab, cnt = build_mc_table()
    rounds = mise_iter
    while True:
        corners = (cells[:, None, :] + _OFF8[None] * size)            # (n,8,3)
        flat = corners.reshape(-1, 3)
        uniq, inv = np.unique(flat, axis=0, return_inverse=True)
        fv = np.asarray(eval_fn(lattice_pos(uniq, W, R)), np.float64)
        cv = fv[inv.reshape(-1)].reshape(-1, 8)
        inside = cv > 0
        case = np.zeros(cells.shape[0], np.int64)
        for c in range(8):
            case |= inside[:, c].astype(np.int64) << c
        cross = (case != 0) & (case != 255)
        cells, cv, case = cells[cross], cv[cross], case[cross]
        if rounds == 0:
            break
        rounds -= 1
        size //= 2
        cells = (cells[:, None, :] + _OFF8[None] * size).reshape(-1, 3)
    if cells.shape[0] == 0:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64)
    # cells keep their natural order: stage-0 voxel order, children x-major (SPEC S10)
    # crossing edges -> vertices
    ea, eb, eax = MC_EDGES[:, 0], MC_EDGES[:, 1], MC_EDGES[:, 2]
    ins = cv > 0
    ecross = ins[:, ea] != ins[:, eb]                                   # (n,12)
    elow = cells[:, None, :] + MC_CORNERS[ea][None] * size              # lattice coord of lower end
    ekey = (morton_encode((elow - cmin).reshape(-1, 3)).reshape(-1, 12) << 2) | eax[None].astype(np.int64)
    fa, fb = cv[:, ea], cv[:, eb]
    with np.errstate(divide='ignore', invalid='ignore'):
        tpar = np.where(ecross, fa / (fa - fb), 0.0)
    uk, first = np.unique(ekey[ecross], return_index=True)
    pa = lattice_pos(elow[ecross][first], W, R).astype(np.float64)
    axv = np.broadcast_to(eax[None], ekey.shape)[ecross][first]
    tp = tpar[ecross][first]
    step = np.float64(np.float32(W) * np.float32(size) / np.float32(R))
    v = pa.copy()
    v[np.arange(v.shape[0]), axv] += tp * step
    # faces
    vid = np.full(ekey.shape, -1, np.int64)
    vid[ecross] = np.searchsorted(uk, ekey[ecross])
    faces = []
    maxt = tab.shape[1] // 3
    for t in range(maxt):
        m = cnt[case] > t
        e = tab[case[m]][:, 3 * t:3 * t + 3].astype(np.int64)
        faces.append((np.nonzero(m)[0], t, np.take_along_axis(vid[m], e, axis=1)))
    cell_idx = np.concatenate([f[0] for f in faces])
    tnum = np.concatenate([np.full(f[0].shape[0], f[1]) for f in faces])
    tri = np.concatenate([f[2] for f in faces])
    o = np.lexsort((tnum, cell_idx))
    tri = tri[o]
    v = v.astype(np.float32)
    if mask_fn is not None:
        keep_v = np.asarray(mask_fn(v), bool)
        tri = tri[np.all(keep_v[tri], axis=1)]
        used = np.zeros(v.shape[0], bool)
        used[tri.reshape(-1)] = True
        remap = np.cumsum(used) - 1
        v, tri = v[used], remap[tri]
    return v, tri
