"""MeshEvaluator on the GPU (csrc/metrics.cu, nksr_b200/metrics.py; DESIGN.md SPEC S18) against its numpy / scipy
restatement oracle/metrics.py: the sampler, the exact nearest neighbours (including the far-query pass), the metrics
end to end on a reconstructed mesh, an analytic bound, the accepted input types and a 5e6-sample run."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import metrics as OM
from tests import clouds

pytestmark = pytest.mark.gpu

REL = 1e-6       # fp32 distance from fp32 coordinates: a few roundings of the squared distance, relative


def _np(t):
    return t.detach().cpu().numpy()


def _icosphere(level, R=1.0):
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


def _random_mesh(rng, V=400, T=3000):
    v = (rng.normal(size=(V, 3)) * [2.0, 1.0, 0.5]).astype(np.float32)
    f = rng.integers(0, V, size=(T, 3)).astype(np.int32)
    f[::97, 1] = f[::97, 0]                              # zero-area triangles
    return v, f


def test_sampler_matches_oracle(cuda):
    from nksr_b200.metrics import sample_surface
    rng = np.random.default_rng(5)
    v, f = _random_mesh(rng)
    n = 300_000
    tv, tf = torch.from_numpy(v).to(cuda), torch.from_numpy(f).to(cuda)
    xyz, nrm, tri = (_np(a) for a in sample_surface(tv, tf, n, seed=11))
    assert xyz.shape == (n, 3) and tri.shape == (n,)
    oxyz, onrm, otri = OM.sample_surface(v, f, n, seed=11)
    # the count boundaries: equal except where n S_t / A lies within fp64 rounding of .5 (the GPU's prefix sum is
    # associated differently from numpy's)
    start = np.concatenate([[0], np.cumsum(np.bincount(tri, minlength=f.shape[0]))])
    ostart = OM.sample_starts(v, f, n)
    assert start[-1] == n
    diff = np.nonzero(start != ostart)[0]
    S = np.cumsum(OM.triangle_areas(v, f))
    frac = (n * S / S[-1]) % 1.0
    assert len(diff) <= 3 and all(abs(frac[t - 1] - 0.5) < 1e-7 for t in diff)
    same = tri == otri
    assert same.sum() >= n - 3 * len(diff)
    assert (OM.triangle_areas(v, f)[tri] > 0).all()
    scale = np.abs(v).max()
    assert np.abs(xyz[same] - oxyz[same]).max() <= 16 * 2.0 ** -24 * scale
    assert np.abs(nrm[same] - onrm[same]).max() <= 1e-6
    again = _np(sample_surface(tv, tf, n, seed=11)[0])
    assert np.array_equal(again, xyz)
    other = _np(sample_surface(tv, tf, n, seed=12)[0])
    assert not np.allclose(other, xyz)


def _check_nn(cuda, q, t, qn=None, tn=None):
    from nksr_b200.metrics import nearest_neighbours
    q, t = q.astype(np.float32), t.astype(np.float32)
    g = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(cuda)
    d, i, dot = (_np(a) for a in nearest_neighbours(g(q), g(t), g(qn), g(tn)))
    rd, ri, rdot = OM.nearest(q, t, qn, tn)
    assert np.all(np.abs(d - rd) <= REL * rd + 1e-30), np.abs(d - rd).max()
    # the same point, or one tied with it to within the fp32 rounding
    alt = np.linalg.norm(t[i].astype(np.float64) - q, axis=1)
    assert np.all((i == ri) | (alt <= rd * (1 + 2 * REL) + 1e-30))
    if qn is not None and tn is not None:
        ok = ~np.isnan(rdot)
        assert np.array_equal(np.isnan(dot), ~ok)
        with np.errstate(invalid="ignore"):
            want = np.abs((tn[i] / np.linalg.norm(tn[i], axis=1, keepdims=True) *
                           qn / np.linalg.norm(qn, axis=1, keepdims=True)).sum(1))
        assert np.abs(dot[ok] - want[ok]).max() < 1e-5
    return d, i, dot


def test_nearest_matches_ckdtree(cuda):
    rng = np.random.default_rng(0)
    t = rng.random((60_000, 3))
    q = rng.random((30_000, 3)) * 1.2 - 0.1
    tn, qn = rng.normal(size=t.shape), rng.normal(size=q.shape)
    qn[:50] = 0.0                                        # zero-length normal: NaN, as the reference's division
    _check_nn(cuda, q, t, qn, tn)
    # a surface-like cloud (the bunny) against noisy copies of itself
    xyz, nrm = clouds.bunny()
    _check_nn(cuda, xyz + rng.normal(size=xyz.shape) * 0.01, xyz, nrm, nrm)
    _check_nn(cuda, xyz, xyz + rng.normal(size=xyz.shape) * 0.002)


def test_nearest_outside_the_cloud(cuda):
    """queries below the target's box, and queries further than the coarsest cell (the far-query pass)"""
    rng = np.random.default_rng(1)
    t = rng.random((40_000, 3))
    below = rng.random((5_000, 3)) - 1.3                 # entirely below the box: the hash origin moves with them
    far = rng.normal(size=(5_000, 3)) * 100.0            # far beyond the coarsest cell (~0.5)
    mixed = np.concatenate([below, far, rng.random((5_000, 3)), t[:100] + 1e-4])
    _check_nn(cuda, mixed, t)
    _check_nn(cuda, rng.normal(size=(3000, 3)) * 1e6, t)  # outside the key frame entirely
    # a thin, elongated cloud and queries off its ends
    line = np.stack([np.linspace(0, 50, 20_000), np.zeros(20_000), rng.random(20_000) * 1e-3], axis=1)
    _check_nn(cuda, np.concatenate([line[::7] + [0, 3.0, 0], [[-100, 0, 0], [200, 5, 5]]]), line)


def test_nearest_ties_and_degenerate_sizes(cuda):
    from nksr_b200.metrics import nearest_neighbours
    rng = np.random.default_rng(2)
    base = rng.random((5_000, 3)).astype(np.float32)
    t = np.repeat(base, 3, axis=0)                       # each point three times: ties go to the lower index
    q = np.concatenate([rng.random((8_000, 3)), rng.normal(size=(500, 3)) * 30]).astype(np.float32)
    d, i, _ = _check_nn(cuda, q, t)
    assert np.all(i % 3 == 0)
    g = lambda a: torch.from_numpy(a.astype(np.float32)).to(cuda)
    d, i, dot = nearest_neighbours(g(np.zeros((0, 3))), g(t))
    assert d.shape == (0,) and i.shape == (0,)
    one = np.array([[0.3, -2.0, 5.0]], dtype=np.float32)
    d, i, _ = _check_nn(cuda, q, one)
    assert np.all(i == 0)
    d, i, _ = _check_nn(cuda, one, one)
    assert d[0] == 0.0


def _bunny_mesh(cuda):
    import nksr_b200
    xyz, nrm = clouds.bunny()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    rec = nksr_b200.Reconstructor(cuda)
    field = rec.reconstruct(t(xyz), t(nrm), detail_level=1.0, solver_tol=1e-6)
    return field.extract_dual_mesh(mise_iter=1), xyz, nrm


def test_bunny_metrics_match_oracle(cuda):
    from nksr_b200.metrics import MeshEvaluator, sample_surface
    mesh, xyz, nrm = _bunny_mesh(cuda)
    names = MeshEvaluator.ALL_METRICS + ["f-precision-outdoor", "f-recall-outdoor", "f-score-outdoor"]
    n = 200_000
    out = MeshEvaluator(n_points=n, metric_names=names, seed=3).eval_mesh(mesh, xyz, nrm)
    sx, sn, _ = (_np(a) for a in sample_surface(mesh.v, mesh.f, n, seed=3))
    comp, _, cdot = OM.nearest(xyz, sx, nrm, sn)
    acc, _, adot = OM.nearest(sx, xyz, sn, nrm)
    ref = OM.summarise(comp, cdot, acc, adot)
    assert sorted(out) == sorted(names)
    for k in ("completeness", "accuracy", "chamfer-L1"):
        assert out[k] == pytest.approx(ref[k], rel=2e-6), k
    for k in ("completeness2", "accuracy2", "chamfer-L2"):
        assert out[k] == pytest.approx(ref[k], rel=4e-6), k
    for k in ("normals completeness", "normals accuracy", "normals"):
        assert out[k] == pytest.approx(ref[k], abs=1e-6), k
    # threshold fractions: only samples within rounding of a threshold may fall on the other side
    for k, th in (("f-precision", 0.01), ("f-recall", 0.01), ("f-precision-outdoor", 0.1), ("f-recall-outdoor", 0.1)):
        d = acc if "precision" in k else comp
        slack = np.mean(np.abs(d - th) <= 4 * REL * th)
        assert abs(out[k] - ref[k]) <= slack + 1e-12, k
    for k in ("f-score", "f-score-15", "f-score-20", "f-score-outdoor"):
        assert out[k] == pytest.approx(ref[k], abs=1e-4), k
    diag = float(np.linalg.norm(xyz.max(0) - xyz.min(0)))
    assert out["chamfer-L1"] < 0.01 * diag and out["normals"] > 0.9


def test_sphere_chamfer_below_sagitta(cuda):
    from nksr_b200.metrics import MeshEvaluator
    R = 1.0
    v, f = _icosphere(2, R)
    a, b, c = (v[f[:, k]].astype(np.float64) for k in range(3))
    la, lb, lc = (np.linalg.norm(x, axis=1) for x in (b - c, c - a, a - b))
    area = 0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1)
    rc = (la * lb * lc / (4 * area)).max()               # the largest circumradius
    sagitta = R - math.sqrt(R * R - rc * rc)
    rng = np.random.default_rng(4)
    gt = rng.normal(size=(2_000_000, 3))
    gt /= np.linalg.norm(gt, axis=1, keepdims=True)
    out = MeshEvaluator(n_points=2_000_000).eval_mesh((torch.from_numpy(v).to(cuda), torch.from_numpy(f).to(cuda)),
                                                      gt * R, gt)
    assert 0 < out["chamfer-L1"] < sagitta, (out["chamfer-L1"], sagitta)
    assert out["normals"] > 0.99


def test_accepted_inputs_give_the_same_dict(cuda):
    from nksr_b200.meshing import DualMesh
    from nksr_b200.metrics import MeshEvaluator
    v, f = _icosphere(2, 0.5)
    rng = np.random.default_rng(6)
    gt = rng.normal(size=(20_000, 3))
    gt /= np.linalg.norm(gt, axis=1, keepdims=True)
    gt_n = gt.copy()
    gt *= 0.5
    ev = MeshEvaluator(n_points=50_000)
    tv, tf = torch.from_numpy(v).to(cuda), torch.from_numpy(f).to(cuda)
    base = ev.eval_mesh(DualMesh(v=tv, f=tf), torch.from_numpy(gt).to(cuda), torch.from_numpy(gt_n).to(cuda))
    for mesh, p, n in (((tv, tf), gt, gt_n), ((v, f), gt, gt_n),
                       (SimpleNamespace(vertices=v.astype(np.float64), triangles=f.astype(np.int64)), gt, gt_n),
                       (DualMesh(v=tv, f=tf.long()), torch.from_numpy(gt), torch.from_numpy(gt_n))):
        assert ev.eval_mesh(mesh, p, n) == base
    assert sorted(base) == sorted(MeshEvaluator.ALL_METRICS)
    ess = MeshEvaluator(n_points=50_000, metric_names=MeshEvaluator.ESSENTIAL_METRICS).eval_mesh((v, f), gt, gt_n)
    assert ess == {k: base[k] for k in MeshEvaluator.ESSENTIAL_METRICS}
    empty = MeshEvaluator(metric_names=MeshEvaluator.ESSENTIAL_METRICS).eval_mesh(
        (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int32)), gt, gt_n)
    assert sorted(empty) == sorted(MeshEvaluator.ESSENTIAL_METRICS) and all(math.isnan(x) for x in empty.values())
    no_n = ev.eval_mesh((v, f), gt, None)
    assert math.isnan(no_n["normals"]) and no_n["chamfer-L1"] == base["chamfer-L1"]


def test_cfg4_crop_against_5e6_samples(cuda):
    import nksr_b200
    from nksr_b200.metrics import MeshEvaluator, nearest_neighbours, sample_surface
    from tests import scenes
    xyz, sensor, W = scenes.crop("cfg4_outdoor", 1_000_000, with_sensor=True)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    rec = nksr_b200.Reconstructor(cuda)
    field = rec.reconstruct(t(xyz), sensor=t(sensor), voxel_size=W,
                            preprocess_fn=nksr_b200.get_estimate_normal_preprocess_fn(64, 85.0),
                            approx_kernel_grad=True, solver_tol=1e-4, fused_mode=True)
    mesh = field.extract_dual_mesh(mise_iter=1)
    n = 5_000_000
    out = MeshEvaluator(n_points=n, metric_names=MeshEvaluator.ALL_METRICS).eval_mesh(mesh, t(xyz), None)
    assert math.isfinite(out["chamfer-L1"]) and math.isnan(out["normals"])
    sx = sample_surface(mesh.v, mesh.f, n, seed=0)[0]
    comp = _np(nearest_neighbours(t(xyz), sx)[0])
    acc = _np(nearest_neighbours(sx, t(xyz))[0])
    assert out["completeness"] == pytest.approx(comp.astype(np.float64).mean(), rel=1e-12)
    assert out["accuracy"] == pytest.approx(acc.astype(np.float64).mean(), rel=1e-12)
    rng = np.random.default_rng(7)
    sxn = _np(sx).astype(np.float64)
    qi = rng.choice(xyz.shape[0], 100_000, replace=False)
    rd = cKDTree(sxn).query(xyz[qi].astype(np.float64), workers=-1)[0]
    assert np.all(np.abs(comp[qi] - rd) <= REL * rd + 1e-30)
    si = rng.choice(n, 100_000, replace=False)
    rd = cKDTree(xyz.astype(np.float64)).query(sxn[si], workers=-1)[0]
    assert np.all(np.abs(acc[si] - rd) <= REL * rd + 1e-30)
