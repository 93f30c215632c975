"""The work items of the matrix-free gather-scatter (csrc/operator.cu): the merged location order and the items cut from
it against a numpy restatement of the rule, and the operator against the fp64 oracle for item sizes from one location
to whole top-level voxels, on a cloud with one very dense cluster (one top-level voxel spans many items, level-2 voxels hold
more locations than an item) and top-level voxels that hold only positions or only normal
locations."""
import numpy as np
import pytest
import torch

from oracle import nksr_oracle as O
from tests import clouds
from tests.test_gpu_matrix_free import _check_against, _feats, _np, _t

pytestmark = pytest.mark.gpu

CUT_LEVEL = 2          # items never split a voxel of levels 0 to 2
HUGE = 1 << 30


def _cloud():
    xyz, _ = clouds.shapenet_like(3000)
    rng = np.random.default_rng(7)
    c = xyz[np.argsort(xyz[:, 0])[xyz.shape[0] // 5]]     # on the side that keeps its positions
    cluster = (c + rng.normal(scale=0.006, size=(4000, 3))).astype(np.float32)
    return np.concatenate([xyz, cluster]).astype(np.float32)


def _system(cuda, W=0.02, L=4, C=4, approx=True):
    import nksr_b200
    xyz = _cloud()
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_point_splatting(torch.from_numpy(xyz).to(cuda))
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    feats = _feats(osvh, C, 11)
    field = nksr_b200.KernelField(svh, None, [torch.from_numpy(f).to(cuda) for f in feats], approx)
    centers = np.concatenate([osvh.centers(0), osvh.centers(1)]).astype(np.float32)
    # positions on the low-x side, normal locations on the high-x side: top-level voxels with one kind only
    pos = xyz[xyz[:, 0] < np.quantile(xyz[:, 0], 0.7)]
    nxyz = centers[centers[:, 0] > np.quantile(centers[:, 0], 0.3)]
    rng = np.random.default_rng(3)
    nval = rng.normal(size=nxyz.shape).astype(np.float32)
    nval /= np.linalg.norm(nval, axis=1, keepdims=True)
    w = (1e4 / pos.shape[0], 1e4 / nxyz.shape[0] * W * W, 1.0)
    return field, osvh, feats, pos, nxyz, nval, w


def _expected_items(vox, S):
    """the cutting rule restated: per top-level voxel run, greedy items of at most S locations cut only where no voxel
    of a level <= CUT_LEVEL continues; without such a cut within S locations, the item runs to the next cut"""
    T, m = vox.shape[0] - 1, vox.shape[1]
    legal = np.ones(m + 1, bool)
    for l in range(CUT_LEVEL + 1):
        legal[1:m] &= ~((vox[l, :-1] >= 0) & (vox[l, 1:] == vox[l, :-1]))
    top = vox[T]
    out = []
    k = 0
    while k < m:
        if top[k] < 0:
            k += 1
            continue
        s = k
        while k < m and top[k] == top[s]:
            k += 1
        e, a = k, s
        while a < e:
            if a + S >= e:
                b = e
            else:
                cand = [c for c in range(a + S, a, -1) if legal[c]]
                b = cand[0] if cand else next(c for c in range(a + S + 1, e + 1) if c == e or legal[c])
            out.append((a, b, (1 if a == s else 0) | (2 if b == e else 0), 0))
            a = b
    return np.array(out, np.int32).reshape(-1, 4)


def _check_order(op, order, vox):
    """the merged order is a permutation of both location lists, carries their containing voxels, and keeps every
    voxel's locations contiguous at every level"""
    bp, bn = _np(op.base_pos), _np(op.base_nrm)
    n_pos, n_nrm = bp.shape[1], bn.shape[1]
    pos = order[order >= 0]
    nrm = ~order[order < 0]
    assert np.array_equal(pos, np.arange(n_pos)) and np.array_equal(nrm, np.arange(n_nrm))
    ref = np.where(order >= 0, bp[:, np.maximum(order, 0)], bn[:, np.maximum(~order, 0)])
    assert np.array_equal(vox, ref)
    for l in range(vox.shape[0]):
        v = vox[l][vox[l] >= 0]
        starts = np.flatnonzero(np.r_[True, v[1:] != v[:-1]])
        assert np.unique(v[starts]).size == starts.size, f"a level-{l} voxel's locations are not contiguous"


@pytest.mark.parametrize("S", [1, 8, 64, HUGE])
def test_items_follow_the_cutting_rule(cuda, S):
    field, osvh, feats, xyz, nxyz, nval, w = _system(cuda)
    op = field.matrix_free_system(_t(cuda, xyz), _t(cuda, nxyz), _t(cuda, nval), *w, item_size=S)
    order, vox, items = (_np(t) for t in field.operator_items(op))
    _check_order(op, order, vox)
    T = vox.shape[0] - 1
    exp = _expected_items(vox, S)
    assert np.array_equal(items, exp), (items.shape, exp.shape)
    # the properties the rule promises
    covered = np.zeros(order.size, np.int32)
    for b, e, _, _ in items:
        covered[b:e] += 1
        assert (vox[T, b:e] == vox[T, b]).all(), "an item crosses a top-level voxel"
        if e - b > S:
            assert (vox[CUT_LEVEL, b:e] == vox[CUT_LEVEL, b]).all() and vox[CUT_LEVEL, b] >= 0
        for l in range(CUT_LEVEL + 1):
            if b > 0 and vox[T, b - 1] == vox[T, b]:
                assert vox[l, b] < 0 or vox[l, b] != vox[l, b - 1], f"a cut inside a level-{l} voxel"
    assert (covered == (vox[T] >= 0)).all(), "every location in exactly one item"
    # the scene: a top voxel over many items, level-2 voxels larger than an item, voxels of one kind only
    kinds = {}
    for k in range(order.size):
        kinds.setdefault(vox[T, k], set()).add(order[k] >= 0)
    assert any(s == {True} for s in kinds.values()) and any(s == {False} for s in kinds.values())
    if S == 8:
        # one top voxel over several items (its level-2 voxels are whole items at this size): top-level edge sums
        assert np.bincount(vox[T, items[:, 0]]).max() > 4
        assert (items[:, 1] - items[:, 0] > S).any()
    if S == HUGE:
        assert items.shape[0] == np.unique(vox[T][vox[T] >= 0]).size


@pytest.mark.parametrize("S", [1, 64, HUGE])
def test_operator_matches_oracle_for_item_sizes(cuda, S):
    field, osvh, feats, xyz, nxyz, nval, w = _system(cuda)
    op = field.matrix_free_system(_t(cuda, xyz), _t(cuda, nxyz), _t(cuda, nval), *w, item_size=S)
    A_ref, b_ref, _, A_abs, b_abs = O.build_system(osvh, feats, xyz, nxyz, nval, *w, True, abs_terms=True)
    _check_against(field, cuda, op, A_ref, A_abs, b_ref, b_abs, A_ref.diagonal(), A_abs.diagonal(), f"item size {S}")


@pytest.mark.parametrize("L,approx,S", [(8, True, 1), (8, True, 16), (4, False, 1), (4, False, 16), (8, False, 4)])
def test_deep_and_full_row_walks_match_oracle(cuda, L, approx, S):
    """the 8-level walk and the 3-line gradient rows with items split many times (edge sums on every level above 2)"""
    field, osvh, feats, xyz, nxyz, nval, w = _system(cuda, L=L, approx=approx)
    op = field.matrix_free_system(_t(cuda, xyz), _t(cuda, nxyz), _t(cuda, nval), *w, item_size=S)
    items = _np(field.operator_items(op)[2])
    assert (items[:, 2] & 1 == 0).sum() > 100          # items that continue a top voxel's run
    A_ref, b_ref, _, A_abs, b_abs = O.build_system(osvh, feats, xyz, nxyz, nval, *w, approx, abs_terms=True)
    _check_against(field, cuda, op, A_ref, A_abs, b_ref, b_abs, A_ref.diagonal(), A_abs.diagonal(),
                   f"L={L} approx={approx} item size {S}")


def test_items_are_bitwise_repeatable(cuda):
    field, osvh, feats, xyz, nxyz, nval, w = _system(cuda)
    args = (_t(cuda, xyz), _t(cuda, nxyz), _t(cuda, nval), *w)
    op1, op2 = field.matrix_free_system(*args, item_size=4), field.matrix_free_system(*args, item_size=4)
    assert torch.equal(op1.rhs, op2.rhs) and torch.equal(op1.diag, op2.diag)
    assert all(torch.equal(a, b) for a, b in zip(field.operator_items(op1), field.operator_items(op2)))
    x = torch.randn(op1.n, device=cuda)
    y1 = field.apply_operator(op1, x)
    for _ in range(3):
        assert torch.equal(y1, field.apply_operator(op1, x)) and torch.equal(y1, field.apply_operator(op2, x))
