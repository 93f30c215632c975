"""CPU only: the host reference for the sort-free placement of the transposed cross-level Gram entries
(oracle/placement_proto.py, DESIGN.md SPEC S6b) -- its table formula and its vectorised storage order reproduce a
brute-force sort exactly."""
import numpy as np
import pytest

from oracle import nksr_oracle as O
from oracle import placement_proto as P
from tests import clouds


def _hierarchy(prune):
    xyz, _ = clouds.sphere(600, radius=0.3, noise=0.01, seed=3)
    blob = np.random.default_rng(1).normal(0, 0.08, (150, 3)).astype(np.float32) + np.float32([0.9, 0.1, -0.2])
    svh = O.OracleSVH(0.06, 3).build_point_splatting(np.concatenate([xyz, blob]))
    if prune:       # an adaptive hierarchy: half of level 0 removed, so some level-1 voxels have no children
        keys = list(svh.keys)
        keys[0] = keys[0][O.key_to_ijk(keys[0], 0)[:, 0] >= 0]
        svh = O.OracleSVH(0.06, 3).build_from_keys(keys)
    return svh


@pytest.mark.parametrize("l,k,prune", [(0, 1, False), (0, 2, False), (1, 1, False), (0, 1, True), (0, 2, True)])
def test_structural_placement_equals_sorted_placement(l, k, prune):
    svh = _hierarchy(prune)
    by_formula, seg_len = P.placement_by_structure(svh, l, k)
    by_sort = P.placement_by_sort(svh, l, k)
    assert by_formula == by_sort
    # the positions of every coarse voxel are a permutation of 0..len-1 and the prefix total is the length
    per_c = {}
    for (c, _), pos in by_formula.items():
        per_c.setdefault(c, []).append(pos)
    for c, lst in per_c.items():
        assert sorted(lst) == list(range(len(lst))) and seg_len[c] == len(lst)


@pytest.mark.parametrize("prune", [False, True])
def test_transposed_order_is_the_sorted_placement(prune):
    """transposed_order (vectorised, the whole hierarchy) against placement_by_sort (brute force, one level pair):
    every row's transposed segment is its level pairs' sorted entries, finer levels first"""
    svh = _hierarchy(prune)
    offs = svh.offsets()
    rows, cols = P.transposed_order(svh)
    want_r, want_c = [], []
    for lu in range(1, svh.depth):
        seg = {}
        for l in range(lu):
            for (c, j), pos in P.placement_by_sort(svh, l, lu - l).items():
                seg.setdefault(c, []).append((l, pos, j + offs[l]))
        for c in sorted(seg):
            for _, _, col in sorted(seg[c]):
                want_r.append(c + offs[lu])
                want_c.append(col)
    assert len(want_r) > 0
    assert np.array_equal(rows, want_r) and np.array_equal(cols, want_c)
