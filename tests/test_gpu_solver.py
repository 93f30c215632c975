"""The solver kernels (csrc/solve.cu, csrc/spmv_stream.cuh) through the C-ABI, held to fp64 Jacobi-PCG on the same fp32
matrix: iterate by iterate, in what the solve reports, in what check_every / profile / repeats may not change, at the
edges (b = 0, max_iter 0, tiny n, empty and zero-diagonal rows, NaN, short workspace), and the Chronopoulos-Gear kernels
of the distributed solve run rank by rank in one process.

Systems: the assembled shapenet (4 levels, n 18 230) and sphere (3 levels, n 2 320) systems of test_gpu_parity, a 3-D
7-point Laplacian + shift on a 100^3 grid (n = 10^6: every grid-stride loop of the vector kernels wraps 3 times) and a
random-graph Laplacian with heavy-tailed row lengths 2 ... ~7000 (streamed tiles cut rows, some tiles hold > 512 rows).
Every PCG check runs the row SpMV ('rows'), the streamed SpMV with the split KernelField.solve uses ('stream') and
everything streamed ('stream_all').  The workspace is filled with NaN bytes before every solve, so a kernel that reads
workspace nobody wrote shows as NaN."""
import ctypes as C
import warnings

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import nksr_oracle as O
from tests.bounds import (KAPPA_DCG_ITER, KAPPA_PCG_FLOOR, KAPPA_PCG_ITER, KAPPA_PCG_RES, KAPPA_PCG_X1, KAPPA_SPMV, U32,
                          assert_within)

pytestmark = pytest.mark.gpu

PATHS = ("rows", "stream", "stream_all")
TOLS = (1e-3, 1e-4, 1e-5, 1e-6, 1e-7)
# |iterations - fp64 iterations| <= max(3, margin * fp64 iterations) at tol >= 1e-5.  Measured on an H100 80GB HBM3
# (400 W): worst 6 of 68 (shapenet, everything streamed, tol 1e-3); the others within 5.
PCG_ITER_MARGIN = 0.15
NKSR_E_INVALID, NKSR_E_WORKSPACE = -1, -3


def _lib():
    import nksr_b200._lib as L
    return L


class System:
    """A CSR system on the device (col / val readable 4 entries past nnz, rowptr one entry past n, as the streamed SpMV
    needs) and its fp64 copy: A holds exactly the fp32 values."""

    def __init__(self, A, diag, b, cuda, split=None, rowptr=None, col=None, val=None, tdiag=None, tb=None):
        A = sp.csr_matrix(A)
        self.n, self.nnz = A.shape[0], int(A.indptr[-1])
        self.rp = A.indptr.astype(np.int64)
        if rowptr is None:
            rp = np.zeros(self.n + 2, np.int64)
            rp[:self.n + 1] = self.rp
            rp[self.n + 1] = self.nnz
            cpad = np.zeros(self.nnz + 4, np.int32)
            cpad[:self.nnz] = A.indices
            vpad = np.zeros(self.nnz + 4, np.float32)
            vpad[:self.nnz] = A.data.astype(np.float32)
            t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
            rowptr, col, val = t(rp)[:self.n + 1], t(cpad)[:self.nnz], t(vpad)[:self.nnz]
            tdiag, tb = t(np.asarray(diag, np.float32)), t(np.asarray(b, np.float32))
        self.rowptr, self.col, self.val, self.diag, self.tb = rowptr, col, val, tdiag, tb
        self.A = sp.csr_matrix((A.data.astype(np.float32).astype(np.float64), A.indices, A.indptr), shape=A.shape)
        self.d = np.asarray(diag, np.float32)
        self.b = np.asarray(b, np.float32).astype(np.float64)
        self.split = split if split is not None else (2 * self.n) // 3
        self._hist, self._its = None, {}

    def ref_history(self, kmax):
        """fp64 Jacobi-PCG iterates (x_k, recursive relres_k), k = 1 ... kmax"""
        if self._hist is None or len(self._hist) < kmax:
            self._hist = []
            O.pcg(self.A, self.b, 0.0, kmax, diag=self.d, history=self._hist)
        return self._hist

    def ref_iters(self, tol):
        if tol not in self._its:
            self._its[tol] = O.pcg(self.A, self.b, tol, 20000, diag=self.d)[1]
        return self._its[tol]

    def true_residual(self, x):
        x = np.asarray(x, np.float64)
        bn = np.linalg.norm(self.b)
        true = np.linalg.norm(self.b - self.A @ x) / bn
        floor = U32 * (np.linalg.norm(abs(self.A) @ np.abs(x)) + bn) / bn
        return true, floor


def pcg(S, path, tol, max_iter, check_every=2, profile=0, b=None, ws_short=0):
    """one solve through the C-ABI; returns x (fp32) and info[0:5]"""
    L = _lib()
    dev = S.rowptr.device
    x = torch.full((S.n,), float("nan"), device=dev)
    info = (C.c_double * 5)()
    st = L.stream_ptr(dev)
    b = S.tb if b is None else b
    if path == "rows":
        nb = L.call("nksr_pcg_workspace_bytes", S.n)
    else:
        nb = L.call("nksr_pcg_stream_workspace_bytes", S.n, S.nnz)
    ws = torch.full((nb,), 255, dtype=torch.uint8, device=dev)
    if path == "rows":
        L.call("nksr_pcg_solve", S.rowptr, S.col, S.val, S.diag, b, x, S.n, float(tol), int(max_iter),
               int(check_every), int(profile), ws, nb - ws_short, info, st)
    else:
        split = S.split if path == "stream" else S.n
        split_nnz = int(S.rp[split])
        L.call("nksr_pcg_solve_stream", S.rowptr, S.col, S.val, S.diag, b, x, S.n, S.nnz, split, split_nnz,
               float(tol), int(max_iter), int(check_every), int(profile), ws, nb - ws_short, info, st)
    torch.cuda.synchronize(dev)
    return x.cpu().numpy(), [float(v) for v in info]


def normwise(got, ref, k, what):
    """||got - ref|| / (k u ||ref||)"""
    ref = np.asarray(ref, np.float64)
    d = np.linalg.norm(np.asarray(got, np.float64) - ref)
    rn = np.linalg.norm(ref)
    return d / (k * U32 * rn) if rn > 0 else (0.0 if d == 0 else np.inf)


def report(what, worst, kappa):
    print(f"[bounds] {what}: worst ratio {worst:.4g} (kappa {kappa:g})")
    assert worst <= kappa, f"{what}: worst ratio {worst:.4g} exceeds kappa {kappa:g}"


# ----------------------------------------------------------------------------------------------------- systems
def laplacian3d(m, shift):
    e = np.ones(m)
    T = sp.diags([-e[:-1], 2 * e, -e[:-1]], [-1, 0, 1])
    I = sp.identity(m)
    A = sp.kron(sp.kron(T, I), I) + sp.kron(sp.kron(I, T), I) + sp.kron(sp.kron(I, I), T)
    return (A + shift * sp.identity(m ** 3)).tocsr()


def graph_laplacian(n, seed, max_deg=9000, n_hubs=4):
    """weighted random-graph Laplacian + a positive diagonal; degrees Pareto-distributed in 1 ... max_deg"""
    rng = np.random.default_rng(seed)
    max_deg = max(1, min(max_deg, n - 1))
    deg = np.minimum(np.floor(rng.pareto(1.1, n) + 1).astype(np.int64), max_deg)
    deg[rng.choice(n, min(n_hubs, n), replace=False)] = 2 * max_deg    # about max_deg distinct neighbours
    stubs = np.repeat(np.arange(n), deg)
    rng.shuffle(stubs)
    stubs = stubs[: stubs.size // 2 * 2].reshape(-1, 2)
    stubs = stubs[stubs[:, 0] != stubs[:, 1]]
    w = rng.uniform(0.5, 2.0, stubs.shape[0])
    W = sp.coo_matrix((np.concatenate([w, w]), (np.concatenate([stubs[:, 0], stubs[:, 1]]),
                                                 np.concatenate([stubs[:, 1], stubs[:, 0]]))), shape=(n, n)).tocsr()
    W.sum_duplicates()
    A = (sp.diags(np.asarray(W.sum(axis=1)).ravel() + rng.uniform(0.01, 1.0, n)) - W).tocsr()
    A.sum_duplicates()
    A = sp.csr_matrix(A.astype(np.float32))
    return A, rng.normal(size=n).astype(np.float32)


def holes_system(seed=5):
    """a 24^3 Laplacian with zero-diagonal rows (entries kept, diagonal 0) and empty unknowns (no entry in their row or
    column): the first two rows (they start at entry 0, the start of stream tile 0), one starting exactly at tile 1
    (entry 4096), two at tile 2 (8192), one inside a tile, one last.  Rows before a tile boundary are padded with
    explicit zeros so that the boundary falls between rows."""
    B = laplacian3d(24, 0.05).astype(np.float32).tocsr()
    m = B.shape[0]
    rng = np.random.default_rng(seed)
    zero_diag = rng.choice(m, 40, replace=False)
    layout, count, targets = [["empty", None, 0], ["empty", None, 0]], 0, [(4096, 1), (8192, 2)]
    lens = np.diff(B.indptr)
    zd = set(zero_diag.tolist())
    for i in range(m):
        if targets and count + lens[i] > targets[0][0]:
            layout[-1][2] += targets[0][0] - count      # pad the previous row up to the boundary
            count = targets[0][0]
            layout += [["empty", None, 0] for _ in range(targets.pop(0)[1])]
        layout.append(["row", i, 0])
        count += lens[i]
        if targets and count == targets[0][0]:
            layout += [["empty", None, 0] for _ in range(targets.pop(0)[1])]
        if i == m // 2 + 3:
            layout.append(["empty", None, 0])
    layout.append(["empty", None, 0])
    n = len(layout)
    new = np.zeros(m, np.int64)
    for j, (kind, i, _) in enumerate(layout):
        if kind == "row":
            new[i] = j
    rp, cols, vals = [0], [], []
    for j, (kind, i, pad) in enumerate(layout):
        if kind == "row":
            s, e = B.indptr[i], B.indptr[i + 1]
            c, v = new[B.indices[s:e]], B.data[s:e].copy()
            if i in zd:
                v[c == j] = 0.0
            cols += [c, np.full(pad, j)]
            vals += [v, np.zeros(pad, np.float32)]
            rp.append(rp[-1] + e - s + pad)
        else:
            rp.append(rp[-1])
    A = sp.csr_matrix((np.concatenate(vals).astype(np.float32), np.concatenate(cols), np.array(rp)), shape=(n, n))
    diag = np.zeros(n, np.float32)
    real = np.array([k == "row" for k, _, _ in layout])
    diag[real] = B.diagonal()[[i for k, i, _ in layout if k == "row"]]
    diag[new[zero_diag]] = 0.0
    b = rng.normal(size=n).astype(np.float32)
    b[~real] = 0.0
    frozen = diag <= 0
    empty_at = [j for j, (k, _, _) in enumerate(layout) if k == "empty"]
    return A, diag, b, frozen, empty_at


_CACHE = {}


def _assembled(cuda, which):
    from tests.test_gpu_parity import _solve_setup
    args = {"shapenet": (), "sphere": (4, False, 4000, 0.05, 3, "sphere")}[which]
    field, svh, osvh, feats, xyz, nxyz, nval, (pw, nw, rw) = _solve_setup(cuda, *args)
    field.solver_config.update(keep_system=True, max_iter=0)
    t = lambda a: torch.from_numpy(a).to(cuda)
    with warnings.catch_warnings():
        warnings.simplefilter("error")             # max_iter = 0: no "stopped at max_iter" warning
        field.solve(t(xyz), t(nxyz), t(nval), pw, nw, rw)
    assert field.solve_info["iterations"] == 0 and not field.solve_info["converged"]
    assert float(field.alpha.abs().max()) == 0.0
    s = field.system
    n = s.rowptr.numel() - 1
    np_ = lambda a: a.detach().cpu().numpy()
    A = sp.csr_matrix((np_(s.val), np_(s.col), np_(s.rowptr)), shape=(n, n))
    S = System(A, np_(s.diag), np_(s.rhs), cuda, split=int(field.svh.offsets[2]), rowptr=s.rowptr, col=s.col,
               val=s.val, tdiag=s.diag, tb=s.rhs)
    assert np.array_equal(A.diagonal().astype(np.float32), S.d)      # the preconditioner is the stored diagonal
    offs = list(field.svh.offsets)
    S.xcoord = np.concatenate([osvh.centers(l)[:, 0] for l in range(osvh.depth)]).astype(np.float64)
    assert S.xcoord.shape[0] == n and offs[-1] == n
    S.field = field
    return S


def system(cuda, name):
    if name not in _CACHE:
        if name in ("shapenet", "sphere"):
            _CACHE[name] = _assembled(cuda, name)
        elif name == "lap100":
            A = laplacian3d(100, 0.01).astype(np.float32)
            b = np.random.default_rng(1).normal(size=A.shape[0]).astype(np.float32)
            _CACHE[name] = System(A, A.diagonal(), b, cuda)
        elif name == "ragged":
            A, b = graph_laplacian(60_000, 2)
            _CACHE[name] = System(A, A.diagonal(), b, cuda)
        elif name.startswith("n="):
            n = int(name[2:])
            A, b = graph_laplacian(n, 7 + n, max_deg=min(40, n - 1), n_hubs=1)
            _CACHE[name] = System(A, A.diagonal(), b, cuda)
        elif name == "holes":
            A, diag, b, frozen, empty_at = holes_system()
            S = System(A, diag, b, cuda)
            S.frozen, S.empty_at = frozen, empty_at
            _CACHE[name] = S
    return _CACHE[name]


def test_test_systems_have_the_intended_shapes(cuda):
    """the synthetic systems exercise what they are here for"""
    big = system(cuda, "lap100")
    assert big.n >= 3 * 1056 * 256                    # vector kernels: kGrid * kBlock threads wrap >= 3 times
    rg = system(cuda, "ragged")
    lens = np.diff(rg.rp)
    assert lens.min() <= 2 and lens.max() > 4096                # rows spanning two or more tiles
    starts = rg.rp[:-1]
    tiles = np.arange(4096, rg.nnz, 4096)
    cut = np.searchsorted(rg.rp, tiles, side="right") - 1
    assert (rg.rp[cut] < tiles).any()                  # rows cut by tile boundaries
    assert (np.diff(np.searchsorted(starts, np.arange(0, rg.nnz + 4096, 4096))) > 512).any()   # tiles of > 512 rows
    h = system(cuda, "holes")
    assert h.empty_at[:2] == [0, 1] and h.rp[1] == h.rp[2] == 0
    assert h.rp[h.empty_at[2]] == 4096 and h.rp[h.empty_at[3]] == h.rp[h.empty_at[4]] == 8192
    assert h.empty_at[4] < h.split and h.empty_at[-1] == h.n - 1


# ----------------------------------------------------------------------------------------------------- 1. iterates
ITER_CASES = [(s, p) for s in ("sphere", "shapenet", "ragged", "lap100") for p in PATHS]


@pytest.mark.parametrize("name,path", ITER_CASES)
def test_pcg_iterates_match_fp64(cuda, name, path):
    """x_k (tol 0, max_iter k) against fp64 PCG on the same fp32 matrix, k = 1 ... 12 (and 20 on the small systems):
    ||x_k - x_k^ref|| <= kappa k u ||x_k^ref||; the reported residual against the reference's recursive residual; x_1 =
    alpha_0 D^-1 b entry by entry."""
    S = system(cuda, name)
    ks = list(range(1, 13)) + ([20] if S.n < 100_000 else [])
    hist = S.ref_history(max(ks))
    worst_x, worst_r = 0.0, 0.0
    for k in ks:
        x, info = pcg(S, path, 0.0, k)
        assert info[0] == k and info[4] == 1, (k, info)
        xr, rr = hist[k - 1]
        worst_x = max(worst_x, normwise(x, xr, k, "x"))
        worst_r = max(worst_r, abs(info[1] - rr) / (k * U32 * rr))
        if k == 1:
            z = np.where(S.d > 0, S.b / np.where(S.d > 0, S.d.astype(np.float64), 1.0), 0.0)
            pap = z @ (S.A @ z)
            scale = np.abs(xr) * (1.0 + (np.abs(z) @ (abs(S.A) @ np.abs(z))) / pap)
            assert_within(x, xr, scale, KAPPA_PCG_X1, f"x_1 ({name}, {path})")
    report(f"PCG iterates ({name}, {path}, k <= {max(ks)})", worst_x, KAPPA_PCG_ITER)
    report(f"PCG reported residual ({name}, {path}, k <= {max(ks)})", worst_r, KAPPA_PCG_RES)


# ----------------------------------------------------------------------------------------------------- 2. reporting
@pytest.mark.parametrize("name,path", [(s, p) for s in ("sphere", "shapenet", "ragged") for p in PATHS])
def test_pcg_reports_honestly(cuda, name, path):
    """true fp64 residual <= 2 reported + kappa floor; converged exactly when the reported residual is <= tol; the
    iteration count at tol >= 1e-5 within PCG_ITER_MARGIN of fp64 PCG."""
    S = system(cuda, name)
    worst, lines = 0.0, []
    for tol in TOLS:
        x, info = pcg(S, path, tol, 20000)
        true, floor = S.true_residual(x)
        rep = info[1]
        q = max(true - 2.0 * rep, 0.0) / floor
        worst = max(worst, q)
        tol32 = float(np.float32(tol))
        lines.append(f"tol {tol:g}: iters {int(info[0])} status {int(info[4])} reported {rep:.3e} true {true:.3e} "
                     f"floor {floor:.3e}")
        assert info[4] in (0, 1)
        assert (info[4] == 0) == (rep <= tol32 * (1 + 1e-12)), lines[-1]
        assert info[4] == 0, lines[-1]            # every tol here is reported reached (see DESIGN.md S7)
        if tol >= 1e-5:
            it_ref = S.ref_iters(tol)
            lines[-1] += f" fp64 iters {it_ref}"
            assert abs(info[0] - it_ref) <= max(3, PCG_ITER_MARGIN * it_ref), lines[-1]
        if tol == 1e-7:
            # below the fp32 floor: the recursive residual reaches tol, the true residual stays near the floor (8.8 to
            # 18x the reported one on these systems), and the solve reports convergence
            assert true > tol and true > 5 * rep, lines[-1]
    print(f"[solve] {name} {path}: " + "; ".join(lines))
    report(f"true residual over floor ({name}, {path})", worst, KAPPA_PCG_FLOOR)


# ----------------------------------------------------------------------------------------------------- 3. invariance
@pytest.mark.parametrize("name,path", [(s, p) for s in ("sphere", "shapenet", "ragged") for p in PATHS])
def test_pcg_is_invariant_and_deterministic(cuda, name, path):
    """check_every (odd values round up to pairs) and profile change only how often the host reads back: bitwise the
    same x and the same iterations / residual / status; two runs agree; a solve that converges at iteration j is the
    solve with tol 0 and max_iter j; odd and even max_iter run exactly max_iter iterations."""
    S = system(cuda, name)
    max_iter = 500
    x0, i0 = pcg(S, path, 1e-5, max_iter)
    assert i0[4] == 0 and 0 < i0[0] < max_iter
    j = int(i0[0])
    for ce in (1, 2, 3, 5, 32, max_iter + 7):
        for prof in (0, 1):
            x, info = pcg(S, path, 1e-5, max_iter, ce, prof)
            assert np.array_equal(x, x0) and [info[0], info[1], info[4]] == [i0[0], i0[1], i0[4]], (ce, prof, info, i0)
            if prof:
                assert info[3] == info[0] and info[2] > 0
    xp, ip = pcg(S, path, 0.0, j)
    assert np.array_equal(xp, x0) and ip[0] == j and ip[4] == 1
    for mi in (7, 8):
        ref = None
        for ce in (2, 3, 32):
            for prof in (0, 1):
                x, info = pcg(S, path, 0.0, mi, ce, prof)
                assert info[0] == mi and info[4] == 1, (mi, ce, prof, info)
                if ref is None:
                    ref = (x, info[1])
                assert np.array_equal(x, ref[0]) and info[1] == ref[1]


# ----------------------------------------------------------------------------------------------------- 4. edges
@pytest.mark.parametrize("path", PATHS)
def test_pcg_edge_cases(cuda, path):
    L = _lib()
    S = system(cuda, "sphere")
    # b = 0: x = 0 exactly, no iteration, converged, residual 0
    x, info = pcg(S, path, 1e-6, 100, b=torch.zeros_like(S.tb))
    assert np.all(x == 0) and info[0] == 0 and info[4] == 0 and info[1] == 0
    # max_iter = 0: x = 0, not converged
    for prof in (0, 1):
        x, info = pcg(S, path, 1e-6, 0, profile=prof)
        assert np.all(x == 0) and info[0] == 0 and info[4] == 1
    # NaN in b: status 2
    bn = S.tb.clone()
    bn[S.n // 2] = float("nan")
    x, info = pcg(S, path, 1e-6, 100, b=bn)
    assert info[4] == 2
    # a workspace one byte short; max_iter < 0
    with pytest.raises(L.NksrError, match=f"\\({NKSR_E_WORKSPACE}\\)"):
        pcg(S, path, 1e-6, 10, ws_short=1)
    with pytest.raises(L.NksrError, match=f"\\({NKSR_E_INVALID}\\)"):
        pcg(S, path, 1e-6, -1)


@pytest.mark.parametrize("path", PATHS)
def test_pcg_non_positive_diagonal_never_converges(cuda, path):
    """an unknown whose diagonal is <= 0 is frozen at 0 by the preconditioner; with its own right-hand side its residual
    cannot fall, so the solve must run to max_iter and never report convergence"""
    base = system(cuda, "n=257")
    A = base.A.tolil()
    for i in (5, 100):                       # isolated unknowns: their residual is their right-hand side
        A[i, :] = 0.0
        A[:, i] = 0.0
    A[5, 5], A[100, 100] = -1.0, 2.0
    d = base.d.copy()
    d[[5, 100]] = [-1.0, 0.0]                # a negative diagonal, and a zero one the matrix does not have
    b = base.b.astype(np.float32)
    b[[5, 100]] = 10 * np.abs(b).max()
    S = System(A.tocsr(), d, b, cuda)
    for tol in (1e-1, 1e-3):
        x, info = pcg(S, path, tol, 300)
        assert info[4] == 1 and info[0] == 300 and x[5] == 0 and x[100] == 0
        assert info[1] >= abs(S.b[5]) / np.linalg.norm(S.b) * (1 - 1e-6)


@pytest.mark.parametrize("n", [1, 31, 257, 8449])
@pytest.mark.parametrize("path", PATHS)
def test_pcg_small_n(cuda, n, path):
    """n = 1, one warp, one block, and just past kGrid * 8 warps: iterates against fp64 and convergence at 1e-5"""
    S = system(cuda, f"n={n}")
    hist = S.ref_history(12)
    worst = 0.0
    for k in range(1, min(12, len(hist)) + 1):
        x, info = pcg(S, path, 0.0, k)
        xr, rr = hist[k - 1]
        if info[4] == 0:                # tol 0: converged only on an exactly zero residual (n = 1 may get there)
            assert info[1] == 0 and 1 <= info[0] <= k, (k, info)
        else:
            assert info[4] == 1 and info[0] == k, (k, info)
        worst = max(worst, normwise(x, xr, k, "x"))
    report(f"PCG iterates (n={n}, {path})", worst, KAPPA_PCG_ITER)
    x, info = pcg(S, path, 1e-5, 5000)
    assert info[4] == 0 and info[1] <= float(np.float32(1e-5))
    true, floor = S.true_residual(x)
    assert true <= 2 * info[1] + KAPPA_PCG_FLOOR * floor


@pytest.mark.parametrize("path", PATHS)
def test_pcg_empty_and_zero_diagonal_rows(cuda, path):
    """unknowns with a zero diagonal (their row and column still hold entries) or no entry at all stay exactly 0 and
    the others follow fp64 PCG; one empty row starts exactly at a stream tile boundary, two more at the next one.  The
    fp64 reference itself equals PCG on the reduced system (the other unknowns only)."""
    S = system(cuda, "holes")
    hist = S.ref_history(12)
    keep = ~S.frozen
    red = []
    O.pcg(S.A[keep][:, keep], S.b[keep], 0.0, 12, diag=S.d[keep], history=red)
    for (xf, _), (xr, _) in zip(hist, red):
        assert np.linalg.norm(xf[keep] - xr) <= 1e-10 * np.linalg.norm(xr) and np.all(xf[~keep] == 0)
    worst = 0.0
    for k in range(1, 13):
        x, info = pcg(S, path, 0.0, k)
        assert info[0] == k and info[4] == 1 and np.all(np.isfinite(x)), (k, info)
        assert np.all(x[S.frozen] == 0)
        worst = max(worst, normwise(x, hist[k - 1][0], k, "x"))
        assert abs(info[1] - hist[k - 1][1]) <= KAPPA_PCG_RES * k * U32 * hist[k - 1][1]
    report(f"PCG iterates (empty and zero-diagonal rows, {path})", worst, KAPPA_PCG_ITER)


# ----------------------------------------------------------------------------------------------------- 5. SpMV
@pytest.mark.parametrize("name", ["lap100", "ragged", "holes"])
def test_spmv_per_entry(cuda, name):
    """row SpMV and streamed SpMV (split and all) entry by entry against fp64 with the scale |A| |x|"""
    L = _lib()
    S = system(cuda, name)
    x = torch.randn(S.n, device=cuda)
    xn = x.cpu().numpy().astype(np.float64)
    ref, scale = S.A @ xn, abs(S.A) @ np.abs(xn)
    y = torch.full_like(x, float("nan"))
    L.call("nksr_spmv", S.rowptr, S.col, S.val, x, y, S.n, L.stream_ptr(cuda))
    assert_within(y.cpu().numpy(), ref, scale, KAPPA_SPMV, f"row SpMV ({name})")
    nb = L.call("nksr_spmv_plan_bytes", S.nnz)
    plan = torch.empty(nb, dtype=torch.uint8, device=cuda)
    for split in (S.split, S.n):
        y = torch.full_like(x, float("nan"))
        L.call("nksr_spmv_stream", S.rowptr, S.col, S.val, x, y, S.n, S.nnz, split, int(S.rp[split]), plan, nb,
               L.stream_ptr(cuda))
        assert_within(y.cpu().numpy(), ref, scale, KAPPA_SPMV, f"streamed SpMV ({name}, split {split})")


# ----------------------------------------------------------------------------------------------------- 6. distributed
class Rank:
    """one rank of the distributed solve: its local system, ownership mask and vectors"""

    def __init__(self, S, owner, rank, local, cuda):
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
        own = owner == rank
        if not local:                               # layout (a): the whole system, an ownership mask
            self.g = np.arange(S.n)
            self.rowptr, self.col, self.val, self.diag, self.b = S.rowptr, S.col, S.val, S.diag, S.tb
            self.own = own
        else:                                       # layout (b): owned rows + halo rows of NaN, renumbered
            rows = np.nonzero(own)[0]
            sub = S.A[rows]
            g = np.union1d(rows, np.unique(sub.indices)).astype(np.int64)
            if g.size == 0:                         # a rank that owns nothing still holds a few halo unknowns
                g = np.arange(min(10, S.n), dtype=np.int64)
            self.g = g
            m = g.size
            is_own = own[g]
            counts = np.ones(m, np.int64)           # halo row: one NaN entry on its diagonal
            counts[is_own] = np.diff(sub.indptr)
            rp = np.concatenate([[0], np.cumsum(counts)])
            start = np.zeros(m, np.int64)
            start[is_own] = sub.indptr[:-1]
            er = np.repeat(np.arange(m), counts)
            src = start[er] + np.arange(rp[-1]) - rp[er]
            eo = is_own[er]
            src = np.where(eo, src, 0)
            li = np.searchsorted(g, sub.indices)
            cols = np.where(eo, li[src] if li.size else 0, er)
            vals = np.where(eo, sub.data[src] if li.size else 0.0, np.nan).astype(np.float32)
            A = sp.csr_matrix((vals, cols, rp), shape=(m, m))
            diag = np.where(is_own, S.d[g], np.nan).astype(np.float32)
            b = np.where(is_own, S.b[g], np.nan).astype(np.float32)
            L = System(A, diag, b, cuda, split=m)
            self.rowptr, self.col, self.val, self.diag, self.b = L.rowptr, L.col, L.val, L.diag, L.tb
            self.own = is_own
        self.n = self.g.size
        self.own8 = t(self.own.astype(np.uint8))
        self.owner = owner[self.g]
        self.vec = {k: torch.full((self.n,), float("nan"), device=cuda) for k in "xruwps"}
        L_ = _lib()
        self.nb = L_.call("nksr_dcg_workspace_bytes")
        self.ws = torch.full((self.nb,), 255, dtype=torch.uint8, device=cuda)
        self.red = torch.zeros(3, dtype=torch.float64, device=cuda)

    def status(self):
        info = (C.c_double * 4)()
        _lib().call("nksr_dcg_status", self.ws, info, _lib().stream_ptr(self.red.device))
        return [float(v) for v in info]


def make_ranks(S, owner, R, local, cuda):
    ranks = [Rank(S, owner, r, local, cuda) for r in range(R)]
    # halo exchange plan: for every non-owned local entry, its owner's local index
    for rk in ranks:
        rk.recv = []
        for src in range(R):
            dst = np.nonzero((~rk.own) & (rk.owner == src))[0]
            if dst.size:
                srci = np.searchsorted(ranks[src].g, rk.g[dst])
                assert np.array_equal(ranks[src].g[srci], rk.g[dst])
                dev = rk.red.device
                rk.recv.append((src, torch.from_numpy(dst).to(dev), torch.from_numpy(srci).to(dev)))
    return ranks


def _allreduce(ranks):
    s = ranks[0].red.clone()
    for rk in ranks[1:]:
        s += rk.red
    for rk in ranks:
        rk.red.copy_(s)


def dcg_run(ranks, tol, max_iter, b_zero=False, on_step=None):
    """the host loop of dist_solve.pcg_distributed, every rank in lockstep; returns the per-rank status after the
    last step and the number of steps"""
    L = _lib()
    st = L.stream_ptr(ranks[0].red.device)
    for rk in ranks:
        v = rk.vec
        b = torch.zeros_like(rk.b) if b_zero else rk.b
        L.call("nksr_dcg_init", rk.diag, b, rk.own8, v["x"], v["r"], v["u"], v["p"], v["s"], rk.n, rk.ws, rk.nb,
               rk.red, st)
    _allreduce(ranks)
    for rk in ranks:
        L.call("nksr_dcg_begin", rk.ws, rk.red, float(tol), int(max_iter), st)
    steps = 0
    while True:
        infos = [rk.status() for rk in ranks]
        assert all(i == infos[0] for i in infos), infos                   # every rank reached the same verdict
        it, res, status, done = infos[0]
        assert status == (0 if done == 1 else 2 if done == 2 else 1)
        assert it == min(steps, max_iter) if done in (0, 3) else it <= steps
        if done or steps > max_iter + 2:
            return infos[0], steps
        for rk in ranks:                                                  # halo exchange of u
            for src, dst, srci in rk.recv:
                rk.vec["u"][dst] = ranks[src].vec["u"][srci]
        for rk in ranks:
            v = rk.vec
            L.call("nksr_dcg_spmv_dots", rk.rowptr, rk.col, rk.val, rk.own8, v["r"], v["u"], v["w"], rk.n, rk.ws,
                   rk.red, st)
        _allreduce(ranks)
        for rk in ranks:
            v = rk.vec
            L.call("nksr_dcg_update", rk.diag, rk.own8, v["x"], v["r"], v["u"], v["w"], v["p"], v["s"], rk.n, rk.ws,
                   rk.red, st)
        steps += 1
        if on_step:
            on_step(steps)


def gather_x(ranks, n):
    x = np.full(n, np.nan)
    for rk in ranks:
        xl = rk.vec["x"].cpu().numpy()
        assert np.all(xl[~rk.own] == 0)                                   # the final exchange is the host's job
        x[rk.g[rk.own]] = xl[rk.own]
    assert np.all(np.isfinite(x))
    return x


def ownership(S, R, name):
    """slabs in x for the assembled systems, random for the synthetic ones; R = '3e': three ranks, rank 1 owns nothing"""
    nr = 2 if R == "3e" else R
    if hasattr(S, "xcoord"):
        q = np.quantile(S.xcoord, np.linspace(0, 1, nr + 1)[1:-1])
        owner = np.searchsorted(q, S.xcoord, side="right")
    else:
        owner = np.random.default_rng(17).integers(0, nr, S.n)
    if R == "3e":
        owner = np.where(owner == 1, 2, 0)
    return owner, (3 if R == "3e" else R)


DCG_CASES = ([(s, 1, False) for s in ("sphere", "shapenet", "ragged", "lap100")] +
             [(s, R, loc) for s in ("sphere", "shapenet", "ragged") for R in (2, 3, "3e") for loc in (False, True)] +
             [("lap100", 3, False), ("lap100", 3, True)])
_DCG_ONE = {}


def _dcg_iterates(S, owner, R, local, cuda, kmax):
    """x_k (union of the owned entries) after each step k, the reported residual of x_k, and w on non-owned rows"""
    ranks = make_ranks(S, owner, R, local, cuda)
    xs, res = [], []

    def step(k):
        if k <= kmax:
            xs.append(gather_x(ranks, S.n))
        if k >= 2:
            res.append(ranks[0].status()[1])                             # published with step k: residual of x_{k-1}
        for rk in ranks:
            assert np.all(rk.vec["w"].cpu().numpy()[~rk.own] == 0)

    info, steps = dcg_run(ranks, 0.0, kmax, on_step=step)
    assert info[0] == kmax and info[3] == 3 and info[2] == 1 and steps == kmax + 1
    return xs, res


@pytest.mark.parametrize("name,R,local", DCG_CASES)
def test_dcg_iterates(cuda, name, R, local):
    """the Chronopoulos-Gear step kernels, R ranks emulated in one process (sum of the ranks' partial dots as the
    all-reduce, owners' u copied into the other ranks as the halo exchange).  One rank: x_k against fp64 PCG.  More
    ranks: the union of the owned x_k against one rank.  Non-owned x and w stay 0; halo rows (layout b) are NaN and
    never read."""
    S = system(cuda, name)
    kmax = 20 if S.n < 100_000 else 12
    hist = S.ref_history(kmax)
    owner, nr = ownership(S, R, name)
    xs, res = _dcg_iterates(S, owner, nr, local, cuda, kmax)
    worst_x = worst_r = 0.0
    if R == 1:
        for k in range(1, kmax + 1):
            worst_x = max(worst_x, normwise(xs[k - 1], hist[k - 1][0], k, "x"))
            worst_r = max(worst_r, abs(res[k - 1] - hist[k - 1][1]) / (k * U32 * hist[k - 1][1]))
        _DCG_ONE[name] = xs
        report(f"DCG iterates, one rank ({name})", worst_x, KAPPA_DCG_ITER)
        report(f"DCG reported residual, one rank ({name})", worst_r, KAPPA_PCG_RES)
    else:
        one = _DCG_ONE.get(name) or _dcg_iterates(S, np.zeros(S.n, np.int64), 1, False, cuda, kmax)[0]
        for k in range(1, kmax + 1):
            worst_x = max(worst_x, normwise(xs[k - 1], one[k - 1], k, "x"))
            worst_x = max(worst_x, normwise(xs[k - 1], hist[k - 1][0], k, "x"))
        report(f"DCG iterates, {R} ranks {'local' if local else 'masked'} ({name})", worst_x, KAPPA_DCG_ITER)


@pytest.mark.parametrize("name,local", [(s, loc) for s in ("sphere", "shapenet", "ragged") for loc in (False, True)])
def test_dcg_tolerances_and_max_iter(cuda, name, local):
    """iteration counts at tol within 1 of one rank; true residual <= 2 reported + kappa floor; converged exactly when
    the reported residual is <= tol; odd and even max_iter run exactly max_iter iterations; b = 0 on every rank
    converges at 0 iterations; max_iter 0 stops at once, unconverged"""
    S = system(cuda, name)
    its1 = {}
    worst = 0.0
    for R in (1, 2, 3, "3e"):
        owner, nr = ownership(S, R, name)
        ranks = make_ranks(S, owner, nr, local, cuda)
        for tol in TOLS:
            info, steps = dcg_run(ranks, tol, 20000)
            x = gather_x(ranks, S.n)
            true, floor = S.true_residual(x)
            worst = max(worst, max(true - 2.0 * info[1], 0.0) / floor)
            assert (info[2] == 0) == (info[1] <= float(np.float32(tol)) * (1 + 1e-12)) and info[2] == 0, (R, tol, info)
            if R == 1:
                its1[tol] = info[0]
            else:
                assert abs(info[0] - its1[tol]) <= 1, (R, tol, info[0], its1[tol])
        for mi in (7, 8):
            info, steps = dcg_run(ranks, 0.0, mi)
            assert info[0] == mi and info[2] == 1 and info[3] == 3 and steps == mi + 1
        info, steps = dcg_run(ranks, 1e-6, 100, b_zero=True)
        assert info[0] == 0 and info[2] == 0 and info[1] == 0 and steps == 0
        assert all(np.all(rk.vec["x"].cpu().numpy() == 0) for rk in ranks)
        info, steps = dcg_run(ranks, 1e-6, 0)
        assert info[0] == 0 and info[2] == 1 and info[3] == 3 and steps == 0
    report(f"DCG true residual over floor ({name}, {'local' if local else 'masked'})", worst, KAPPA_PCG_FLOOR)
