"""The matrix-free inference operator (csrc/operator.cu: nksr_op_setup, nksr_op_apply, nksr_pcg_solve_matrix_free)
against the fp64 oracle system (oracle.nksr_oracle.build_system, regulariser included) entry by entry, against the
assembled CSR operator of the same field, bit for bit against itself, and through the PCG.  Edge cases: depths 2 to 8,
C = 1 ... 32, no regulariser, no normal constraints, voxels and whole top-level voxels without locations, and a level
that holds no location."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import nksr_oracle as O
from tests import clouds
from tests.bounds import U32, assert_within

pytestmark = pytest.mark.gpu

# Per-entry bound in units of 2^-24 of the fp64 magnitude scale |E|^T W |E| |x| + |reg| |R| |x| (rhs: |E|^T W |t|,
# diagonal: its own abs-term).  The operator sums per (location, slot) products into per-voxel partials and then 27
# partials per unknown: the same terms as the assembled Gram matrix times x, in another order.
KAPPA_OP = 64.0


def _np(t):
    return t.detach().cpu().numpy()


def _feats(osvh, C, seed):
    rng = np.random.default_rng(seed)
    return [(0.5 + 0.2 * rng.normal(size=(osvh.n(l), C))).astype(np.float32) for l in range(osvh.depth)]


def _setup(cuda, C=4, approx=True, L=4, W=0.02, n_pts=3000, seed=11):
    import nksr_b200
    xyz, _ = clouds.shapenet_like(n_pts)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_point_splatting(torch.from_numpy(xyz).to(cuda))
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    feats = _feats(osvh, C, seed)
    field = nksr_b200.KernelField(svh, None, [torch.from_numpy(f).to(cuda) for f in feats], approx)
    field.solver_config["operator"] = "matrix_free"          # (small systems assemble by default)
    nxyz = np.concatenate([osvh.centers(0), osvh.centers(1)]).astype(np.float32)
    rng = np.random.default_rng(3)
    nval = rng.normal(size=nxyz.shape).astype(np.float32)
    nval /= np.linalg.norm(nval, axis=1, keepdims=True)
    w = (1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * W * W, 1.0)
    return field, osvh, feats, xyz, nxyz, nval, w


def _t(cuda, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _assembled(field, cuda, xyz, nxyz, nval, w):
    field.solver_config.update(operator="assembled", keep_system=True, max_iter=0, compact_rows=field.approx_kernel_grad)
    field.solve(_t(cuda, xyz), None if nxyz is None else _t(cuda, nxyz), None if nval is None else _t(cuda, nval), *w)
    s = field.system
    n = s.rowptr.numel() - 1
    A = sp.csr_matrix((_np(s.val).astype(np.float64), _np(s.col), _np(s.rowptr)), shape=(n, n))
    field.solver_config.update(operator="matrix_free", keep_system=False)
    return A, _np(s.rhs), _np(s.diag)


def _check_against(field, cuda, op, A, A_abs, rhs, b_abs, diag, d_abs, what, seed=0):
    rng = np.random.default_rng(seed)
    assert_within(_np(op.rhs), rhs, b_abs, KAPPA_OP, f"rhs ({what})")
    assert_within(_np(op.diag), diag, d_abs, KAPPA_OP, f"diagonal ({what})")
    for k in range(2):
        x = rng.normal(size=op.n).astype(np.float32)
        y = _np(field.apply_operator(op, _t(cuda, x)))
        assert_within(y, A @ x.astype(np.float64), abs(A_abs) @ np.abs(x).astype(np.float64), KAPPA_OP,
                      f"A x ({what}, vector {k})")


@pytest.mark.parametrize("C,approx", [(4, True), (16, True), (4, False), (1, True), (32, False)])
def test_operator_matches_oracle(cuda, C, approx):
    field, osvh, feats, xyz, nxyz, nval, w = _setup(cuda, C, approx)
    op = field.matrix_free_system(_t(cuda, xyz), _t(cuda, nxyz), _t(cuda, nval), *w)
    A_ref, b_ref, _, A_abs, b_abs = O.build_system(osvh, feats, xyz, nxyz, nval, *w, approx, abs_terms=True)
    _check_against(field, cuda, op, A_ref, A_abs, b_ref, b_abs, A_ref.diagonal(), A_abs.diagonal(),
                   f"oracle, C={C} approx={approx}")


@pytest.mark.parametrize("L", [2, 3, 5, 6, 8])
def test_operator_matches_assembled_across_depths(cuda, L):
    """every depth the assembly supports, against the assembled CSR of the same field (depths > 4 take the
    8-level kernels)"""
    field, osvh, feats, xyz, nxyz, nval, w = _setup(cuda, 4, True, L=L, W=0.03, n_pts=1500)
    A, rhs, diag = _assembled(field, cuda, xyz, nxyz, nval, w)
    op = field.matrix_free_system(_t(cuda, xyz), _t(cuda, nxyz), _t(cuda, nval), *w)
    _, _, _, A_abs, b_abs = O.build_system(osvh, feats, xyz, nxyz, nval, *w, True, abs_terms=True)
    _check_against(field, cuda, op, A, 2 * A_abs, rhs, 2 * b_abs, diag, 2 * A_abs.diagonal(), f"assembled, L={L}")


@pytest.mark.parametrize("case", ["no_regulariser", "positions_only", "sparse_positions", "no_level0_locations"])
def test_operator_edge_cases(cuda, case):
    field, osvh, feats, xyz, nxyz, nval, w = _setup(cuda, 8, True)
    if case == "no_regulariser":
        w = (w[0], w[1], 0.0)
    elif case == "positions_only":
        nxyz = nval = None
    elif case == "sparse_positions":
        # the positions of a corner of the cloud only: voxels and whole top-level voxels without any location
        keep = xyz[:, 0] < np.quantile(xyz[:, 0], 0.2)
        xyz = xyz[keep]
        nxyz, nval = nxyz[: nxyz.shape[0] // 5], nval[: nval.shape[0] // 5]
    else:
        # constraint locations inside level-1 voxels but outside every level-0 voxel: level 0 holds no location
        rng = np.random.default_rng(5)
        c1 = osvh.centers(1)
        cand = (c1[rng.integers(0, c1.shape[0], 20000)] + rng.uniform(-0.02, 0.02, (20000, 3))).astype(np.float32)
        base = osvh.locate(cand)
        cand = cand[(base[0] < 0) & (base[1] >= 0)]
        assert cand.shape[0] > 100
        xyz, nxyz, nval = cand[: cand.shape[0] // 2], cand[cand.shape[0] // 2:], nval[: cand.shape[0] - cand.shape[0] // 2]
    A, rhs, diag = _assembled(field, cuda, xyz, nxyz, nval, w)
    op = field.matrix_free_system(_t(cuda, xyz), None if nxyz is None else _t(cuda, nxyz),
                                  None if nval is None else _t(cuda, nval), *w)
    if case == "no_level0_locations":
        assert (_np(op.base_pos)[0] < 0).all()
    nx = np.zeros((0, 3), np.float32) if nxyz is None else nxyz
    nv = np.zeros((0, 3), np.float32) if nval is None else nval
    _, _, _, A_abs, b_abs = O.build_system(osvh, feats, xyz, nx, nv, *w, True, abs_terms=True)
    _check_against(field, cuda, op, A, 2 * A_abs, rhs, 2 * b_abs + 1e-30, diag, 2 * A_abs.diagonal(), case)


def test_operator_is_bitwise_repeatable(cuda):
    field, osvh, feats, xyz, nxyz, nval, w = _setup(cuda, 4, True)
    args = (_t(cuda, xyz), _t(cuda, nxyz), _t(cuda, nval), *w)
    op1, op2 = field.matrix_free_system(*args), field.matrix_free_system(*args)
    assert torch.equal(op1.rhs, op2.rhs) and torch.equal(op1.diag, op2.diag)
    x = torch.randn(op1.n, device=cuda)
    y1 = field.apply_operator(op1, x)
    assert torch.equal(y1, field.apply_operator(op1, x)) and torch.equal(y1, field.apply_operator(op2, x))
    field.solver_config.update(tol=1e-6)
    a1 = field.solve(*args).alpha.clone()
    a2 = field.solve(*args).alpha
    assert torch.equal(a1, a2) and field.solve_info["operator"] == "matrix_free" and field.solve_info["nnz"] == 0


def test_pcg_iterates_and_solution_follow_fp64(cuda):
    """the first iterates against fp64 Jacobi-PCG on the oracle system, then the converged solve: same iterations
    within the solver tests' margin, and the true fp64 residual of the returned alpha near the tolerance"""
    field, osvh, feats, xyz, nxyz, nval, w = _setup(cuda, 4, True)
    args = (_t(cuda, xyz), _t(cuda, nxyz), _t(cuda, nval), *w)
    A_ref, b_ref, _ = O.build_system(osvh, feats, xyz, nxyz, nval, *w, True)
    hist = []
    O.pcg(A_ref, b_ref, 0.0, 3, history=hist)
    for k in (1, 2, 3):
        field.solver_config.update(max_iter=k, tol=1e-12, check_every=2)
        with pytest.warns(RuntimeWarning):
            field.solve(*args)
        got, ref = _np(field.alpha).astype(np.float64), hist[k - 1][0]
        err = np.linalg.norm(got - ref) / np.linalg.norm(ref)
        print(f"[bounds] matrix-free PCG iterate {k}: relative error {err:.3g}")
        assert err <= 1e-4
    for tol in (1e-4, 1e-6):
        field.solver_config.update(max_iter=2000, tol=tol, check_every=32, profile=True)
        field.solve(*args)
        it_ref = O.pcg(A_ref, b_ref, tol, 20000)[1]
        info = field.solve_info
        assert info["converged"] and abs(info["iterations"] - it_ref) <= max(3, 0.15 * it_ref), (info, it_ref)
        assert info["spmv_launches"] == info["iterations"] and info["spmv_ms"] > 0
        x = _np(field.alpha).astype(np.float64)
        true = np.linalg.norm(b_ref - A_ref @ x) / np.linalg.norm(b_ref)
        assert true <= 3 * tol + 1e3 * U32, (tol, true)
