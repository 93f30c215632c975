"""The per-entry Gram bound of tests/bounds.py against the old global one, on the numpy oracle alone.

The system is the one the GPU assembly tests compare (tests/test_gpu_parity.py::_solve_setup: shapenet_like(3000),
W = 0.02, 4 levels, C = 4, normal constraints at the centres of levels 0 and 1).  Each mutation below is a local kernel
bug of the kind a ragged tile, a skipped row or a wrong placement slot produces.  The per-entry bound rejects all of
them; the old bound (max |A - A_ref| <= 5e-4 max |A_ref|) accepts two, which is why the parity tests no longer use it.
An fp32 rebuild of the same system (rows and products rounded to fp32) passes the per-entry bound.
"""
import numpy as np
import pytest
import scipy.sparse as sp

from oracle import nksr_oracle as O
from tests import clouds
from tests.bounds import KAPPA_GRAM, KAPPA_RHS, assert_within, global_bound_ok, level_pair_label

OLD_RTOL_GRAM = 5e-4


@pytest.fixture(scope="module")
def system():
    xyz, _ = clouds.shapenet_like(3000)
    W, L, C = 0.02, 4, 4
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    rng = np.random.default_rng(11)
    feats = [(0.5 + 0.2 * rng.normal(size=(osvh.n(l), C))).astype(np.float32) for l in range(L)]
    nxyz = np.concatenate([osvh.centers(0), osvh.centers(1)])
    rng = np.random.default_rng(3)
    nval = rng.normal(size=nxyz.shape).astype(np.float32)
    nval /= np.linalg.norm(nval, axis=1, keepdims=True)
    args = (osvh, feats, xyz, nxyz, nval, 1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * W * W, 1.0)
    A, b, E, Aabs, babs = O.build_system(*args, abs_terms=True)
    return dict(args=args, A=A, b=b, E=E, Aabs=Aabs, babs=babs, offs=osvh.offsets())


def _new_ok(s, A):
    try:
        assert_within(A, s["A"], s["Aabs"], KAPPA_GRAM, "Gram", level_pair_label(s["offs"]))
        return True
    except AssertionError:
        return False


def _weights(s):
    osvh, feats, xyz, nxyz, nval, pw, nw, rw = s["args"]
    return np.concatenate([np.full(xyz.shape[0], pw), np.full(3 * nxyz.shape[0], nw)])


def test_abs_scale_bounds_the_entries(system):
    s = system
    assert s["A"].shape == s["Aabs"].shape
    D = abs(s["A"]) - s["Aabs"]
    assert D.max() <= 1e-12 * s["Aabs"].max()                       # |A| <= Aabs entry by entry
    assert np.all(np.abs(s["b"]) <= s["babs"] * (1 + 1e-12))
    assert s["Aabs"].min() >= 0


def test_fp32_rebuild_is_accepted(system):
    """rows rounded to fp32, E^T W E and E^T W t multiplied and summed in fp32, the regulariser rounded to fp32"""
    s = system
    osvh, feats, xyz, nxyz, nval, pw, nw, rw = s["args"]
    E32 = s["E"].astype(np.float32)
    EW32 = E32.T.multiply(_weights(s).astype(np.float32)[None, :]).tocsr().astype(np.float32)
    A32 = (EW32 @ E32).astype(np.float32) + np.float32(rw) * O.build_regulariser(osvh, feats).astype(np.float32)
    assert A32.dtype == np.float32
    t32 = np.concatenate([np.zeros(xyz.shape[0], np.float32), nval.reshape(-1)])
    b32 = EW32 @ t32
    assert b32.dtype == np.float32
    worst = assert_within(A32, s["A"], s["Aabs"], KAPPA_GRAM, "Gram (fp32 rebuild)", level_pair_label(s["offs"]))
    assert worst > 0.5                                               # the rounding is seen at all
    assert_within(b32, s["b"], s["babs"], KAPPA_RHS, "rhs (fp32 rebuild)")


def test_zeroed_small_entries_are_rejected(system):
    s = system
    A = s["A"].copy()
    tol = OLD_RTOL_GRAM * abs(A).max()
    small = np.abs(A.data) < 0.9 * tol
    assert small.mean() > 0.8                                        # most entries lie below the old tolerance
    A.data[small] = 0.0
    assert global_bound_ok(A, s["A"], OLD_RTOL_GRAM)
    assert not _new_ok(s, A)


def test_bspline_tail_weights_off_by_half_a_percent_are_rejected(system, monkeypatch):
    s = system
    exact = O._bspline

    def off(tau):
        w, dw = exact(tau)
        return w * np.array([1.005, 1.0, 1.005]), dw
    monkeypatch.setattr(O, "_bspline", off)
    A, _, _ = O.build_system(*s["args"])
    assert not _new_ok(s, A)


def test_one_median_cross_level_entry_off_by_ten_percent_is_rejected(system):
    s = system
    offs = s["offs"]
    C = s["A"].tocoo()
    blk = (C.row < offs[1]) & (C.col >= offs[3]) & (C.data != 0)
    med = np.median(np.abs(C.data[blk]))
    assert med < 1e-4 * abs(C).max()                                 # the block's entries are far below the old bound
    cand = np.nonzero(blk & (np.abs(C.data) > 0.9 * med) & (np.abs(C.data) < 1.1 * med))[0]
    # the entries of this block cancel heavily (Aabs / |A| is ~1e3 at the median): take the candidate whose
    # |A| / Aabs is the median one among them, neither the easiest nor the hardest to see
    rel = np.abs(C.data[cand]) / np.asarray(s["Aabs"][C.row[cand], C.col[cand]]).ravel()
    j = cand[np.argsort(rel)[rel.shape[0] // 2]]
    r, c = int(C.row[j]), int(C.col[j])
    A = s["A"].tolil()
    A[r, c] *= 1.1
    A[c, r] *= 1.1
    A = A.tocsr()
    assert global_bound_ok(A, s["A"], OLD_RTOL_GRAM)
    assert not _new_ok(s, A)


def test_one_normal_location_missing_from_one_level_is_rejected(system):
    s = system
    osvh, feats, xyz, nxyz, nval, pw, nw, rw = s["args"]
    offs = s["offs"]
    E = s["E"].tocoo()
    k = 0                                                             # normal constraint 0, on the coarsest level
    drop = (E.row >= xyz.shape[0] + 3 * k) & (E.row < xyz.shape[0] + 3 * k + 3) & (E.col >= offs[3])
    assert drop.sum() > 0
    Em = sp.csr_matrix((E.data[~drop], (E.row[~drop], E.col[~drop])), shape=E.shape)
    EW = Em.T.multiply(_weights(s)[None, :]).tocsr()
    A = (EW @ Em).tocsr() + rw * O.build_regulariser(osvh, feats)
    assert not _new_ok(s, A)


def test_failure_report_names_the_level_pair(system):
    s = system
    A = s["A"].tolil()
    r, c = int(s["offs"][1]) + 5, int(s["offs"][1]) + 5                # a level-1 diagonal entry
    A[r, c] *= 1.01
    with pytest.raises(AssertionError, match=r"levels \(1,1\)"):
        assert_within(A.tocsr(), s["A"], s["Aabs"], KAPPA_GRAM, "Gram", level_pair_label(s["offs"]))
