"""SPEC S20's ray-parity occupancy (tests/occupancy_oracle.py) on meshes with a known inside: an icosphere, a union of
unit cubes hit exactly through its vertices and edges, and the invariances the rule promises; the direction constants
of csrc/raycast.cu; the 'o3d-iou' opt-in of both evaluators.  No GPU."""
import itertools
import math
import os
import re

import numpy as np
import pytest

from tests import occupancy_oracle as OO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def icosphere(level, R=1.0):
    t = (1.0 + 5 ** 0.5) / 2
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
         [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10],
         [8, 6, 7], [9, 8, 1]]
    v = [np.array(p, dtype=np.float64) / np.linalg.norm(p) for p in v]
    for _ in range(level):
        mid, nf = {}, []

        def m(a, b):
            k = (min(a, b), max(a, b))
            if k not in mid:
                p = v[a] + v[b]
                v.append(p / np.linalg.norm(p))
                mid[k] = len(v) - 1
            return mid[k]
        for a, b, c in f:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    return (np.array(v) * R).astype(np.float32), np.array(f, dtype=np.int32)


def inscribed_radius(v, f):
    a, b, c = (v[f[:, k]].astype(np.float64) for k in range(3))
    n = np.cross(b - a, c - a)
    return float(np.min(np.abs((n * a).sum(1)) / np.linalg.norm(n, axis=1)))


def shell_queries(rng, n, r_lo, r_hi):
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (d * (r_lo + (r_hi - r_lo) * rng.random((n, 1)))).astype(np.float32)


CUBES = {(0, 0, 0), (1, 0, 0), (2, 0, 0), (0, 1, 0), (0, 2, 0), (0, 0, 1), (1, 1, 1)}   # an L plus two on top


def cube_union(cells=CUBES, rng=None):
    """the boundary of a union of unit cubes as triangles (each boundary square split along a diagonal; with rng,
    random diagonals and windings)"""
    v, f, index = [], [], {}

    def vid(p):
        if p not in index:
            index[p] = len(v)
            v.append(p)
        return index[p]
    for c in sorted(cells):
        for ax in range(3):
            for side in (0, 1):
                nb = list(c)
                nb[ax] += 1 if side else -1
                if tuple(nb) in cells:
                    continue
                u, w = [a for a in range(3) if a != ax]
                corners = []
                for du, dw in ((0, 0), (1, 0), (1, 1), (0, 1)):
                    p = list(c)
                    p[ax] += side
                    p[u] += du
                    p[w] += dw
                    corners.append(vid(tuple(p)))
                a, b, cc, d = corners
                tris = [[a, b, cc], [a, cc, d]] if rng is None or rng.random() < 0.5 else [[a, b, d], [b, cc, d]]
                for t in tris:
                    f.append(t[::-1] if rng is not None and rng.random() < 0.5 else t)
    return np.array(v, dtype=np.float32), np.array(f, dtype=np.int32)


def lattice_labels(cells=CUBES):
    """queries on the integer and half-integer lattice around the union, with the analytic occupancy; points on the
    surface (touching both an occupied and a free cell) are left out"""
    g = np.arange(-1.0, 4.01, 0.5)
    pts, lab = [], []
    for p in itertools.product(g, g, g):
        touch = [range(int(math.floor(x)) - (1 if x == math.floor(x) else 0), int(math.floor(x)) + 1) for x in p]
        occ = [c in cells for c in itertools.product(*touch)]
        if all(occ) or not any(occ):
            pts.append(p)
            lab.append(all(occ))
    return np.array(pts, dtype=np.float32), np.array(lab)


DYADIC = np.array([[1, 1, 1], [1, 2, 4], [-4, 1, 2], [2, -4, -1], [-1, -1, 1]], dtype=np.float32)


def test_icosphere_inside_and_outside_for_every_direction_and_k():
    v, f = icosphere(4)
    r_in = inscribed_radius(v, f)
    rng = np.random.default_rng(0)
    q = np.concatenate([shell_queries(rng, 150, 0.0, 0.999 * r_in), shell_queries(rng, 150, 1.001, 2.0)])
    want = np.arange(300) < 150
    for d in OO.DEFAULT_DIRECTIONS:
        assert np.array_equal(OO.occupancy(v, f, q, directions=d[None]), want)
    for k in range(1, OO.MAX_RAYS + 1, 2):
        assert np.array_equal(OO.occupancy(v, f, q, n_rays=k), want)


def test_cube_union_ties_match_the_voxel_occupancy():
    """dyadic shears are exact, so rays pass exactly through vertices and edges of the grid-aligned surface"""
    q, want = lattice_labels()
    assert want.sum() > 0 and (~want).sum() > 0
    for seed in (None, 1, 2):
        v, f = cube_union(rng=None if seed is None else np.random.default_rng(seed))
        for d in DYADIC:
            got = OO.occupancy(v, f, q, directions=d[None])
            assert np.array_equal(got, want), (seed, d, q[got != want][:5])


def test_invariant_under_permutation_rotation_and_winding():
    v, f = icosphere(3, 0.8)
    rng = np.random.default_rng(3)
    v = v + (rng.normal(size=v.shape) * 0.02).astype(np.float32)       # not a sphere any more: an irregular closed mesh
    q = (rng.random((400, 3)) * 2.0 - 1.0).astype(np.float32)
    base = [OO.ray_crossings(v, f, q, d) for d in OO.DEFAULT_DIRECTIONS[:3]]
    g = f[rng.permutation(f.shape[0])]
    rot = rng.integers(0, 3, size=g.shape[0])
    g = np.stack([np.roll(row, r) for row, r in zip(g, rot)])
    flip = rng.random(g.shape[0]) < 0.5
    g[flip] = g[flip][:, ::-1]
    for d, b in zip(OO.DEFAULT_DIRECTIONS[:3], base):
        assert np.array_equal(OO.ray_crossings(v, g, q, d), b)
    assert np.array_equal(OO.occupancy(v, g, q, n_rays=3), OO.occupancy(v, f, q, n_rays=3))


def test_default_directions_match_the_cuda_constants():
    src = open(os.path.join(ROOT, "nksr_b200", "csrc", "raycast.cu")).read()
    body = re.search(r"kDefaultDirs\[kMaxRays\]\[3\] = \{(.*?)\};", src, re.S).group(1)
    lits = re.findall(r"(-?0x[0-9a-fA-F.]+p[-+]?\d+)f", body)
    got = np.array([float.fromhex(x) for x in lits], dtype=np.float64).reshape(-1, 3)
    assert got.shape == (OO.MAX_RAYS, 3)
    assert np.array_equal(got, OO.DEFAULT_DIRECTIONS.astype(np.float64))
    assert np.array_equal(got.astype(np.float32).astype(np.float64), got)        # exact fp32 values
    a = np.sort(np.abs(got), axis=1)
    assert a.min() >= 0.15 and np.diff(a, axis=1).min() >= 0.05
    from nksr_b200 import metrics as M
    assert M.MAX_RAYS == OO.MAX_RAYS


def test_oracle_evaluator_iou_and_refusals():
    assert OO.occupancy_iou([1, 1, 0, 0], [1, 0, 0, 0]) == 1.0 / (2.0 + 1e-6)
    assert OO.occupancy_iou([0, 0], np.array([0, 0], np.uint8)) == 0.0
    v, f = icosphere(2, 0.5)
    rng = np.random.default_rng(4)
    gt = rng.normal(size=(3000, 3))
    gt /= np.linalg.norm(gt, axis=1, keepdims=True)
    pts = (rng.random((2000, 3)) * 1.4 - 0.7).astype(np.float32)
    occ = np.linalg.norm(pts, axis=1) < 0.5
    names = ["chamfer-L1", "o3d-iou"]
    ev = OO.OracleOccupancyEvaluator(n_points=5000, metric_names=names, occupancy_rays=3)
    out = ev.eval_mesh((v, f), gt * 0.5, gt, onet_samples=(pts, occ))
    pred = OO.occupancy(v, f, pts, n_rays=3)
    assert out["o3d-iou"] == OO.occupancy_iou(pred, occ) and 0.9 < out["o3d-iou"] < 1.0
    plain = OO.OracleOccupancyEvaluator(n_points=5000, metric_names=["chamfer-L1"]).eval_mesh((v, f), gt * 0.5, gt)
    assert plain["chamfer-L1"] == out["chamfer-L1"]
    empty = ev.eval_mesh((v, np.zeros((0, 3), np.int32)), gt, gt, onet_samples=(pts, occ))
    assert all(math.isnan(x) for x in empty.values())
    for k in (0, 2, 4, 11, -1):
        with pytest.raises(ValueError):
            OO.OracleOccupancyEvaluator(metric_names=names, occupancy_rays=k)
    with pytest.raises(ValueError, match="o3d-iou"):
        ev.eval_mesh((v, f), gt, gt)
    with pytest.raises(ValueError, match="o3d-iou"):
        OO.OracleOccupancyEvaluator(metric_names=names)


def test_product_opt_in_checks_without_a_gpu():
    from nksr_b200.metrics import MeshEvaluator
    with pytest.raises(ValueError, match="occupancy_rays"):
        MeshEvaluator(metric_names=["chamfer-L1", "o3d-iou"])
    for k in (0, 2, 10):
        with pytest.raises(ValueError):
            MeshEvaluator(metric_names=["o3d-iou"], occupancy_rays=k)
    ev = MeshEvaluator(metric_names=MeshEvaluator.ALL_METRICS + ["o3d-iou"], occupancy_rays=5)
    assert ev.metric_names[-1] == "o3d-iou" and ev.occupancy_rays == 5
    with pytest.raises(ValueError, match="unknown"):
        MeshEvaluator(metric_names=["o3d-iou", "bogus"], occupancy_rays=3)
    with pytest.raises(ValueError, match="onet_samples"):
        ev._evaluate(np.zeros((0, 3)), np.zeros((1, 3)))
