"""Per-entry error bounds: |got - ref| <= kappa * 2^-24 * scale, element by element.

`scale` is the fp64 magnitude of the computation (the same expression with every signed sum replaced by the sum of
absolute values, oracle/nksr_oracle.py abs_terms=True), so every entry is held to a bound of its own size -- a bound
relative to the largest entry of an output only checks the few entries near that maximum.  kappa is in units of the
fp32 unit roundoff 2^-24; each constant below is set from the worst ratio |got - ref| / (2^-24 scale) measured on an
H100 (stated next to it), with headroom of at most 8x.
"""
import numpy as np
import scipy.sparse as sp

U32 = 2.0 ** -24

# Measured on an NVIDIA H100 80GB HBM3 (power limit 400 W) over the whole GPU suite.
# field.cu / kernel_eval.cuh: kernel rows K, dK.  Worst 4.90 (dK, level 2, C = 4, approx_kernel_grad).
KAPPA_ROWS = 32.0
# assemble.cu: Gram values and diagonal.  Worst 9.49 (values, C = 16, approx, blocks from level 1); diagonal 3.37.
KAPPA_GRAM = 64.0
# assemble.cu: right-hand side.  Worst 5.39 (depth 5, approx).
KAPPA_RHS = 32.0
# field.cu: f and grad f.  Worst 1.72 (f, C = 16, approx); grad f 1.45.
KAPPA_FIELD = 8.0
# sparse_conv.cu, fp32 FFMA kernel against the exact operands.  Worst 16.3 (n_out 129, c_in 64, c_out 256, K 27).
KAPPA_GEMM = 128.0
# sparse_conv.cu, TF32 kernels against their TF32 operands: the tensor cores' fp32 accumulation.  Worst 151 (mma.sync)
# and 147 (wgmma), both at n_out 1000, c_in 256, c_out 192, K 27.  The wgmma output is >= 355 from the rna-x reference.
KAPPA_GEMM_TF32 = 256.0
# TF32 kernels against the unrounded fp32 operands: x truncated (2^-10 = 2^14 u) or rounded (2^13 u) and W rounded
# (2^13 u), plus the accumulation.  Worst 9133 (wgmma).
KAPPA_GEMM_TF32_OPERANDS = 2.0 ** 15

# solve.cu / spmv_stream.cuh: one SpMV (row and streamed kernels) against the scale |A| |x|.  Worst 2.89 (streamed,
# random-graph Laplacian, rows up to ~7000 entries).
KAPPA_SPMV = 16.0
# solve.cu, Jacobi-PCG against fp64 PCG on the same fp32 matrix (tests/test_gpu_solver.py).  First iterate
# x_1 = alpha_0 D^-1 b entry by entry, scale |x_1| (1 + |p|^T |A| |p| / p^T A p).  Worst 1.05 (100^3 Laplacian).
KAPPA_PCG_X1 = 8.0
# Iterate k, normwise: ||x_k - x_k^ref|| <= kappa k u ||x_k^ref||, k = 1 ... 20.  Worst 0.997 (100^3 Laplacian).
KAPPA_PCG_ITER = 7.0
# Reported relative residual info[1] after k iterations against the reference's recursive residual r_k:
# |info[1] - ||r_k|| / ||b||| <= kappa k u ||r_k|| / ||b||.  Worst 0.97 (Chronopoulos-Gear, shapenet); PCG 0.79.
KAPPA_PCG_RES = 6.0
# True fp64 residual of the returned x <= 2 reported + kappa floor, floor = u (|| |A| |x| || + ||b||) / ||b||, for
# tol 1e-3 ... 1e-7.  Worst 1.01 (Chronopoulos-Gear, sphere); PCG 0.93.
KAPPA_PCG_FLOOR = 8.0
# Chronopoulos-Gear kernels (nksr_dcg_*), iterate k normwise against fp64 PCG, and R ranks against one rank.  Worst
# 1.31 (sphere, 2 and 3 ranks, local subsystems).
KAPPA_DCG_ITER = 8.0


def _union(*mats):
    """rows, cols and the values of each sparse matrix on the union of their stored patterns"""
    coos = [sp.coo_matrix(m) for m in mats]
    n_cols = coos[0].shape[1]
    keys = [c.row.astype(np.int64) * n_cols + c.col for c in coos]
    allk = np.unique(np.concatenate(keys))
    vals = []
    for c, k in zip(coos, keys):
        v = np.zeros(allk.shape[0])
        np.add.at(v, np.searchsorted(allk, k), c.data.astype(np.float64))
        vals.append(v)
    return allk // n_cols, allk % n_cols, vals


def level_of(offsets, i):
    return np.searchsorted(np.asarray(offsets), i, side="right") - 1


def level_pair_label(offsets):
    """labels matrix entries (row, col) of a hierarchy system with their level pair"""
    return lambda r, c: f"({r},{c}) levels ({level_of(offsets, r)},{level_of(offsets, c)})"


def ratios(got, ref, scale):
    """|got - ref| / (2^-24 scale) per entry (inf where scale is 0 and got != ref), and the entry indices.  Dense
    arrays of one shape, or scipy sparse matrices compared on the union of their patterns."""
    if sp.issparse(got) or sp.issparse(ref):
        r, c, (g, f, s) = _union(got, ref, scale)
        idx = (r, c)
    else:
        g, f, s = (np.asarray(a, np.float64).reshape(-1) for a in (got, ref, np.broadcast_to(scale, np.shape(ref))))
        idx = None
    d = np.abs(g - f)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(d == 0, 0.0, d / (U32 * s))
    return q, idx, (g, f, s)


def assert_within(got, ref, scale, kappa, what, label=None, worst=8):
    """|got - ref| <= kappa * 2^-24 * scale entry by entry.  On failure lists the `worst` entries with their label
    (label(flat_index) for dense arrays -- default: the index into the array's shape -- or label(row, col) for sparse
    matrices).  Returns the worst ratio |got - ref| / (2^-24 scale), which is printed (pytest -rP shows it)."""
    q, idx, (g, f, s) = ratios(got, ref, scale)
    top = float(q.max()) if q.size else 0.0
    print(f"[bounds] {what}: worst ratio {top:.4g} (kappa {kappa:g}, {q.size} entries)")
    bad = np.nonzero(~(q <= kappa))[0]
    if bad.size == 0:
        return top
    order = bad[np.argsort(-q[bad])][:worst]
    lines = []
    for j in order:
        if idx is not None:
            where = label(int(idx[0][j]), int(idx[1][j])) if label else f"({idx[0][j]},{idx[1][j]})"
        else:
            where = label(int(j)) if label else str(np.unravel_index(j, np.shape(ref)))
        lines.append(f"  {where}: got {g[j]:.9g} ref {f[j]:.9g} scale {s[j]:.3g} ratio {q[j]:.4g}")
    raise AssertionError(f"{what}: {bad.size} of {q.size} entries exceed {kappa:g} * 2^-24 * scale "
                         f"(worst ratio {top:.4g}); worst entries:\n" + "\n".join(lines))


def assert_blockwise(got, ref, offsets, rtol, what):
    """max |got - ref| <= rtol * max |ref| within every level block: level-pair blocks of a sparse system matrix, the
    levels of a vector.  For checks without a per-entry scale: a block of small entries is not judged by the largest
    entry of another.  Returns the worst ratio max |d| / (rtol max |ref|) over the blocks."""
    if sp.issparse(got) or sp.issparse(ref):
        r, c, (g, f) = _union(got, ref)
        blk = level_of(offsets, r) * len(offsets) + level_of(offsets, c)
    else:
        g, f = np.asarray(got, np.float64), np.asarray(ref, np.float64)
        blk = level_of(offsets, np.arange(f.shape[0]))
    d = np.abs(g - f)
    worst, msgs = 0.0, []
    for b in np.unique(blk):
        m = blk == b
        dm, rm = d[m].max(), np.abs(f[m]).max()
        q = dm / (rtol * rm) if rm > 0 else (np.inf if dm > 0 else 0.0)
        name = f"levels ({b // len(offsets)},{b % len(offsets)})" if sp.issparse(ref) else f"level {b}"
        msgs.append(f"{name} {q:.3g}")
        worst = max(worst, q)
    print(f"[bounds] {what}: worst block ratio {worst:.4g} ({', '.join(msgs)})")
    assert worst <= 1.0, f"{what}: max |diff| exceeds {rtol:g} x the block's largest entry: {', '.join(msgs)}"
    return worst


def global_bound_ok(got, ref, rtol):
    """the bound these tests used before: max |got - ref| <= rtol * max |ref| (kept to show what it misses)"""
    d = got - ref
    dmax = abs(d).max() if sp.issparse(d) else np.abs(d).max()
    rmax = abs(ref).max() if sp.issparse(ref) else np.abs(ref).max()
    return bool(dmax <= rtol * rmax)
