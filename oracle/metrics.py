"""numpy / scipy restatement of the mesh-quality metrics (DESIGN.md SPEC S18), for the tests and tools/metrics_bench.py.

The sampler uses the same count rule and the same counter hash as csrc/metrics.cu (bit for bit for the random draws;
positions in fp64 from the same fp32 draws); nearest neighbours come from scipy's cKDTree in fp64.  The product never
imports this module.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

THRESHOLDS = (0.01, 0.015, 0.02, 0.002, 0.1)
ESSENTIAL_METRICS = ["chamfer-L1", "f-score", "normals"]
ALL_METRICS = ["completeness", "accuracy", "normals completeness", "normals accuracy", "normals", "completeness2",
               "accuracy2", "chamfer-L2", "chamfer-L1", "f-precision", "f-recall", "f-score", "f-score-15",
               "f-score-20"]

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def mix64(z):
    """splitmix64's output mix on uint64 arrays (wrapping arithmetic)"""
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def hash_uniform(seed: int, counter):
    """u = (mix64(mix64(seed) + counter) >> 40) * 2^-24 as fp32: uniform in [0, 1) on a 2^-24 grid"""
    hs = mix64(np.array([int(seed) & 0xFFFFFFFFFFFFFFFF], dtype=np.uint64))[0]
    with np.errstate(over="ignore"):
        z = mix64(np.asarray(counter, dtype=np.uint64) + hs)
    return ((z >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)).astype(np.float32)


def triangle_areas(v, f):
    v = np.asarray(v, dtype=np.float32).astype(np.float64)
    f = np.asarray(f, dtype=np.int64).reshape(-1, 3)
    return 0.5 * np.linalg.norm(np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]), axis=1)


def sample_starts(v, f, n: int):
    """int64[T + 1]: triangle t receives the samples [start[t], start[t+1]) with start[t] = round(n S_{t-1} / A)"""
    S = np.cumsum(triangle_areas(v, f))
    T = S.shape[0]
    start = np.zeros(T + 1, dtype=np.int64)
    if T == 0 or not S[-1] > 0 or n <= 0:
        return start
    start[1:] = np.clip(np.round(n * S / S[-1]).astype(np.int64), 0, n)
    start[-1] = n
    return start


def sample_surface(v, f, n: int, seed: int = 0):
    """(xyz (n, 3) fp64, unit triangle normal (n, 3), source triangle (n,)): SPEC S18's sampler"""
    v32 = np.asarray(v, dtype=np.float32)
    f = np.asarray(f, dtype=np.int64).reshape(-1, 3)
    start = sample_starts(v32, f, n)
    total = int(start[-1])
    if total == 0:
        return np.zeros((0, 3)), np.zeros((0, 3)), np.zeros(0, dtype=np.int64)
    tri = np.repeat(np.arange(f.shape[0]), np.diff(start))
    i = np.arange(total, dtype=np.uint64)
    r1 = hash_uniform(seed, 2 * i)
    r2 = hash_uniform(seed, 2 * i + np.uint64(1))
    s = np.sqrt(r1.astype(np.float64))
    w = np.stack([1.0 - s, s * (1.0 - r2), s * r2], axis=1)
    vd = v32.astype(np.float64)
    p0, p1, p2 = vd[f[tri, 0]], vd[f[tri, 1]], vd[f[tri, 2]]
    xyz = w[:, :1] * p0 + w[:, 1:2] * p1 + w[:, 2:] * p2
    nrm = np.cross(p1 - p0, p2 - p0)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    return xyz, nrm, tri


def nearest(query, target, query_normal=None, target_normal=None):
    """(distance, index, |n_q . n_t| of unit normals or NaN) of every query's nearest target point, cKDTree in fp64"""
    query = np.asarray(query, dtype=np.float64).reshape(-1, 3)
    tree = cKDTree(np.asarray(target, dtype=np.float64).reshape(-1, 3))
    dist, idx = tree.query(query, workers=-1)
    if query_normal is None or target_normal is None:
        return dist, idx, np.full(query.shape[0], np.nan)
    with np.errstate(invalid="ignore", divide="ignore"):
        qn = np.asarray(query_normal, dtype=np.float64)
        tn = np.asarray(target_normal, dtype=np.float64)
        qn = qn / np.linalg.norm(qn, axis=-1, keepdims=True)
        tn = tn / np.linalg.norm(tn, axis=-1, keepdims=True)
        dot = np.abs((tn[idx] * qn).sum(axis=-1))
    return dist, idx, dot


def summarise(completeness, completeness_dot, accuracy, accuracy_dot, thresholds=THRESHOLDS):
    """the metric dict from the two distance / normal-agreement arrays (SPEC S18 formulas)"""
    c, a = np.asarray(completeness, np.float64), np.asarray(accuracy, np.float64)
    recall = [float(np.mean(c <= t)) for t in thresholds]
    precision = [float(np.mean(a <= t)) for t in thresholds]
    with np.errstate(invalid="ignore"):
        fs = [float(np.float64(2.0 * p * r) / np.float64(p + r)) for p, r in zip(precision, recall)]
    comp, acc = float(c.mean()), float(a.mean())
    comp2, acc2 = float((c * c).mean()), float((a * a).mean())
    comp_n, acc_n = float(np.mean(completeness_dot)), float(np.mean(accuracy_dot))
    return {
        "completeness": comp, "accuracy": acc,
        "normals completeness": comp_n, "normals accuracy": acc_n, "normals": 0.5 * comp_n + 0.5 * acc_n,
        "completeness2": comp2, "accuracy2": acc2, "chamfer-L2": 0.5 * (comp2 + acc2), "chamfer-L1": 0.5 * (comp + acc),
        "f-precision": precision[0], "f-recall": recall[0], "f-score": fs[0], "f-score-15": fs[1], "f-score-20": fs[2],
        "f-precision-outdoor": precision[4], "f-recall-outdoor": recall[4], "f-score-outdoor": fs[4],
    }


class OracleMeshEvaluator:
    """The evaluator's interface on the definitions above (no 'o3d-iou')."""

    ESSENTIAL_METRICS = ESSENTIAL_METRICS
    ALL_METRICS = ALL_METRICS

    def __init__(self, n_points=100000, metric_names=ALL_METRICS, seed=0):
        if "o3d-iou" in metric_names:
            raise ValueError("'o3d-iou' is not provided")
        self.n_points, self.metric_names, self.seed = int(n_points), list(metric_names), int(seed)

    def eval_mesh(self, mesh, pointcloud_tgt, normals_tgt, onet_samples=None):
        v, f = mesh
        xyz, nrm, _ = sample_surface(v, f, self.n_points, self.seed)
        return self._evaluate(xyz, pointcloud_tgt, nrm, normals_tgt)

    def _evaluate(self, pointcloud, pointcloud_tgt, normals=None, normals_tgt=None, onet_samples=None, mesh=None):
        if np.asarray(pointcloud).shape[0] == 0:
            return {k: float("nan") for k in self.metric_names}
        comp, _, comp_dot = nearest(pointcloud_tgt, pointcloud, normals_tgt, normals)
        acc, _, acc_dot = nearest(pointcloud, pointcloud_tgt, normals, normals_tgt)
        out = summarise(comp, comp_dot, acc, acc_dot)
        return {k: out[k] for k in self.metric_names}
