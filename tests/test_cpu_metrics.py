"""The mesh-quality metric definitions (DESIGN.md SPEC S18) on their numpy / scipy restatement, oracle/metrics.py."""
import math

import numpy as np
import pytest

from oracle import metrics as OM


def _plane(n_side, offset=0.0, spacing=0.001):
    g = (np.arange(n_side) - (n_side - 1) / 2.0) * spacing
    x, y = np.meshgrid(g, g, indexing="ij")
    xyz = np.stack([x.ravel(), y.ravel(), np.full(x.size, offset)], axis=1)
    return xyz, np.tile([0.0, 0.0, 1.0], (xyz.shape[0], 1))


def test_cloud_against_itself_is_perfect():
    rng = np.random.default_rng(0)
    xyz = rng.normal(size=(2000, 3))
    nrm = rng.normal(size=(2000, 3))
    out = OM.OracleMeshEvaluator(metric_names=OM.ALL_METRICS)._evaluate(xyz, xyz, nrm, nrm)
    for k in ("completeness", "accuracy", "chamfer-L1", "chamfer-L2", "completeness2", "accuracy2"):
        assert out[k] == 0.0, k
    for k in ("f-score", "f-score-15", "f-score-20", "f-precision", "f-recall"):
        assert out[k] == 1.0, k
    assert out["normals"] == pytest.approx(1.0, abs=1e-12)


@pytest.mark.parametrize("delta", [0.004, 0.008, 0.03, 0.07])
def test_offset_plane_distances_and_fscores(delta):
    """a dense patch against the same patch shifted by delta along its normal: every distance is delta (the patches
    are identical in x-y, so no rim effect), and the F-scores switch at the thresholds"""
    src, nsrc = _plane(200)
    tgt, ntgt = _plane(200, offset=delta)
    out = OM.summarise(*_both(src, nsrc, tgt, ntgt))
    assert out["completeness"] == pytest.approx(delta, rel=1e-12)
    assert out["accuracy"] == pytest.approx(delta, rel=1e-12)
    assert out["chamfer-L2"] == pytest.approx(delta * delta, rel=1e-12)
    assert out["normals"] == pytest.approx(1.0)
    if delta < 0.01:
        assert out["f-score"] == 1.0
    if 0.02 < delta < 0.1:
        assert math.isnan(out["f-score"]) and math.isnan(out["f-score-20"])   # p + r = 0: numpy's 0/0
        assert out["f-precision"] == 0.0 and out["f-recall"] == 0.0
        assert out["f-score-outdoor"] == 1.0


def _both(src, nsrc, tgt, ntgt):
    comp, _, comp_dot = OM.nearest(tgt, src, ntgt, nsrc)
    acc, _, acc_dot = OM.nearest(src, tgt, nsrc, ntgt)
    return comp, comp_dot, acc, acc_dot


def test_empty_mesh_missing_normals_and_name_filter():
    ev = OM.OracleMeshEvaluator(metric_names=OM.ESSENTIAL_METRICS)
    out = ev.eval_mesh((np.zeros((0, 3)), np.zeros((0, 3), dtype=np.int64)), np.zeros((5, 3)), None)
    assert sorted(out) == sorted(OM.ESSENTIAL_METRICS) and all(math.isnan(x) for x in out.values())
    xyz, _ = _plane(20)
    out = OM.OracleMeshEvaluator(metric_names=["chamfer-L1", "normals", "normals accuracy"])._evaluate(
        xyz, xyz, np.ones_like(xyz), None)
    assert sorted(out) == ["chamfer-L1", "normals", "normals accuracy"]
    assert out["chamfer-L1"] == 0.0 and math.isnan(out["normals"]) and math.isnan(out["normals accuracy"])
    with pytest.raises(ValueError, match="o3d-iou"):
        OM.OracleMeshEvaluator(metric_names=["chamfer-L1", "o3d-iou"])


def test_product_refuses_o3d_iou_and_unknown_names():
    from nksr_b200.metrics import METRIC_KEYS, MeshEvaluator
    assert MeshEvaluator.ESSENTIAL_METRICS == OM.ESSENTIAL_METRICS
    assert MeshEvaluator.ALL_METRICS == OM.ALL_METRICS
    assert set(OM.summarise(np.zeros(1), np.zeros(1), np.zeros(1), np.zeros(1))) == set(METRIC_KEYS)
    with pytest.raises(ValueError, match="o3d-iou"):
        MeshEvaluator(metric_names=["o3d-iou"])
    with pytest.raises(ValueError, match="unknown"):
        MeshEvaluator(metric_names=["chamfer-L3"])


def test_sampler_counts_and_positions():
    rng = np.random.default_rng(1)
    v = rng.normal(size=(60, 3)).astype(np.float32)
    f = rng.integers(0, 60, size=(100, 3))
    f[7] = [3, 3, 5]                      # zero area: repeated vertex
    v[50] = v[51]
    f[8] = [50, 51, 9]                    # zero area: coincident vertices
    f[9] = [10, 11, 10]
    n = 12345
    start = OM.sample_starts(v, f, n)
    counts = np.diff(start)
    assert start[0] == 0 and start[-1] == n and counts.sum() == n and (counts >= 0).all()
    area = OM.triangle_areas(v, f)
    assert (counts[area == 0] == 0).all() and (area == 0).sum() >= 3
    xyz, nrm, tri = OM.sample_surface(v, f, n, seed=3)
    assert xyz.shape == (n, 3) and np.array_equal(np.bincount(tri, minlength=100), counts)
    # on its triangle: in the plane, and the barycentrics of the in-plane solve are in [0, 1]
    vd = v.astype(np.float64)
    p0, p1, p2 = vd[f[tri, 0]], vd[f[tri, 1]], vd[f[tri, 2]]
    assert np.abs(((xyz - p0) * nrm).sum(1)).max() < 1e-9
    assert np.allclose(np.linalg.norm(nrm, axis=1), 1.0)
    e1, e2, d = p1 - p0, p2 - p0, xyz - p0
    g11, g12, g22 = (e1 * e1).sum(1), (e1 * e2).sum(1), (e2 * e2).sum(1)
    b1, b2 = (d * e1).sum(1), (d * e2).sum(1)
    det = g11 * g22 - g12 * g12
    u, w = (g22 * b1 - g12 * b2) / det, (g11 * b2 - g12 * b1) / det
    tol = 1e-7
    assert (u > -tol).all() and (w > -tol).all() and (u + w < 1 + tol).all()
    # a different seed moves the samples, the same seed does not
    assert np.array_equal(OM.sample_surface(v, f, n, seed=3)[0], xyz)
    assert not np.allclose(OM.sample_surface(v, f, n, seed=4)[0], xyz)


def test_sampler_area_ratio():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [3, 0, 0], [0, 3, 0], [0, 0, 0]], dtype=np.float32)
    v[3:] += 5.0
    f = np.array([[0, 1, 2], [5, 3, 4]])          # areas 0.5 and 4.5: ratio 1:9
    for n in (10, 1000, 99999):
        c = np.diff(OM.sample_starts(v, f, n))
        assert abs(c[0] - n / 10) <= 1 and c.sum() == n
    v2 = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [3, 0, 1], [0, 1, 1]], dtype=np.float32)
    f2 = np.array([[0, 1, 2], [3, 4, 5]])         # areas 0.5 and 1.5: ratio 1:3
    for n in (4, 1001, 777777):
        c = np.diff(OM.sample_starts(v2, f2, n))
        assert abs(3 * c[0] - c[1]) <= 3 and abs(c[0] - n / 4) <= 1 and c.sum() == n


def test_hash_is_uniform_and_on_the_fp32_grid():
    u = OM.hash_uniform(0, np.arange(200000, dtype=np.uint64))
    assert u.dtype == np.float32 and u.min() >= 0.0 and u.max() < 1.0
    assert np.array_equal(u * np.float32(16777216.0), np.floor(u * np.float32(16777216.0)))
    hist = np.bincount((u * 10).astype(int), minlength=10)
    assert np.abs(hist - 20000).max() < 600
