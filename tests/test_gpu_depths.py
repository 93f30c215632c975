"""Hierarchy depths other than the default 4: depth 1 (no cross-level blocks) and depth 5
(exercises the MAXL = 8 kernel instantiations), plus a hierarchy adopted from explicit keys
(the decoder hierarchy of the reference is not the encoder's, models/nksr_net.py:74-78)."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import nksr_oracle as O
from tests import clouds
from tests.bounds import KAPPA_FIELD, KAPPA_GRAM, KAPPA_RHS, assert_within, level_pair_label

pytestmark = pytest.mark.gpu


def _np(t):
    return t.detach().cpu().numpy()


@pytest.mark.parametrize("L,W,approx", [(1, 0.06, False), (5, 0.02, False), (5, 0.02, True)])
def test_assembly_solve_mesh_at_depth(cuda, L, W, approx):
    import nksr_b200
    xyz, nrm = clouds.sphere(3000, seed=L)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_point_splatting(t(xyz))
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    for l in range(L):
        assert np.array_equal(_np(svh.keys[l]), osvh.keys[l])
        assert np.array_equal(_np(svh.nbr27[l]).astype(np.int64), osvh.nbr27(l))
    rng = np.random.default_rng(L)
    feats = [(0.5 + 0.2 * rng.normal(size=(osvh.n(l), 4))).astype(np.float32) for l in range(L)]
    ad = min(2, L)
    nxyz = np.concatenate([osvh.centers(d) for d in range(ad)])
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True)).astype(np.float32)
    pw, nw = 1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * W * W
    field = nksr_b200.KernelField(svh, None, [t(f) for f in feats], approx)
    field.solver_config.update(keep_system=True, tol=1e-6, max_iter=4000, check_every=1)
    field.solve(t(xyz), t(nxyz), t(nval), pw, nw, 1.0)
    s = field.system
    A = sp.csr_matrix((_np(s.val).astype(np.float64), _np(s.col), _np(s.rowptr)), shape=(s.n, s.n))
    # no constraint or query location within a few ulps of the tent derivative's snap-zone edge (none left out)
    q = (xyz[:300] + 0.003).astype(np.float32)
    assert int(O.tent_branch_ambiguous(osvh, nxyz).sum()) == 0 and int(O.tent_branch_ambiguous(osvh, q).sum()) == 0
    A_ref, b_ref, _, A_abs, b_abs = O.build_system(osvh, feats, xyz, nxyz, nval, pw, nw, 1.0, approx, abs_terms=True)
    P = O.structural_pattern(osvh)
    assert A.nnz == P.nnz
    what = f"L={L} approx={approx}"
    assert_within(A, A_ref, A_abs, KAPPA_GRAM, f"Gram values ({what})", level_pair_label(osvh.offsets()))
    assert_within(_np(s.rhs), b_ref, b_abs, KAPPA_RHS, f"rhs ({what})")
    assert_within(_np(s.diag), A_ref.diagonal(), A_abs.diagonal(), KAPPA_GRAM, f"diagonal ({what})")
    alpha = _np(field.alpha).astype(np.float64)
    assert np.linalg.norm(A_ref @ alpha - b_ref) <= 2e-4 * np.linalg.norm(b_ref)
    fo, go, fa, ga = O.evaluate_f(osvh, feats, alpha, q, grad=True, approx_kernel_grad=approx, abs_terms=True)
    r = field.evaluate_f(t(q), grad=True)
    assert_within(_np(r.value), fo, fa, KAPPA_FIELD, f"f ({what})")
    assert_within(_np(r.gradient), go, ga, KAPPA_FIELD, f"grad f ({what})")
    mesh = field.extract_dual_mesh(mise_iter=1)
    rad = np.linalg.norm(_np(mesh.v), axis=1)
    # (a single coarse level cannot place the surface accurately; parity with the oracle is asserted above)
    assert mesh.f.shape[0] > 200 and abs(np.median(rad) - 0.35) < (0.02 if L > 1 else 0.1)


def test_hierarchy_from_explicit_keys(cuda):
    """build_from_keys with a pruned finest level (an 'adaptive' decoder hierarchy): tables and the
    Gram pattern still match the oracle on the same key sets."""
    import nksr_b200
    xyz, _ = clouds.shapenet_like(2000)
    W, L = 0.03, 3
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    keep0 = osvh.keys[0][O.key_to_ijk(osvh.keys[0], 0)[:, 0] >= 0]          # drop the x < 0 half on level 0
    okeys = [keep0, osvh.keys[1], osvh.keys[2]]
    osvh2 = O.OracleSVH(W, L).build_from_keys(okeys)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_from_keys([torch.from_numpy(k).to(cuda) for k in okeys])
    for l in range(L):
        assert np.array_equal(_np(svh.nbr27[l]).astype(np.int64), osvh2.nbr27(l))
    rng = np.random.default_rng(0)
    feats = [(0.5 + 0.2 * rng.normal(size=(osvh2.n(l), 4))).astype(np.float32) for l in range(L)]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    field = nksr_b200.KernelField(svh, None, [t(f) for f in feats])
    field.solver_config.update(keep_system=True, max_iter=0)
    nxyz = osvh2.centers(0)
    nval = np.tile(np.array([[0.0, 0.0, 1.0]], np.float32), (nxyz.shape[0], 1))
    assert int(O.tent_branch_ambiguous(osvh2, nxyz).sum()) == 0          # no location left out (test_gpu_parity)
    field.solve(t(xyz), t(nxyz), t(nval), 3.0, 0.02, 1.0)
    s = field.system
    A = sp.csr_matrix((_np(s.val).astype(np.float64), _np(s.col), _np(s.rowptr)), shape=(s.n, s.n))
    A_ref, b_ref, _, A_abs, b_abs = O.build_system(osvh2, feats, xyz, nxyz, nval, 3.0, 0.02, 1.0, abs_terms=True)
    assert A.nnz == O.structural_pattern(osvh2).nnz
    assert_within(A, A_ref, A_abs, KAPPA_GRAM, "Gram values (explicit keys)", level_pair_label(osvh2.offsets()))
    assert_within(_np(s.rhs), b_ref, b_abs, KAPPA_RHS, "rhs (explicit keys)")
    assert_within(_np(s.diag), A_ref.diagonal(), A_abs.diagonal(), KAPPA_GRAM, "diagonal (explicit keys)")
    # points in the pruned half have no level-0 term (SPEC S3) on both sides
    q = xyz[xyz[:, 0] < -0.05][:200]
    field.alpha = t(rng.normal(size=s.n).astype(np.float32))
    fo, fa = O.evaluate_f(osvh2, feats, _np(field.alpha).astype(np.float64), q, abs_terms=True)
    assert_within(_np(field.evaluate_f(t(q)).value), fo, fa, KAPPA_FIELD, "f (explicit keys)")
