"""Mesh occupancy on the GPU (csrc/raycast.cu, nksr_b200.metrics.MeshOccupancy; DESIGN.md SPEC S20) against the
brute-force rule of tests/occupancy_oracle.py, bit for bit: a random triangle soup, exact vertex / edge hits on a cube
union, a reconstructed dual-MC mesh, a 1.3 M-triangle icosphere, degenerate builds; then 'o3d-iou' end to end."""
import math

import numpy as np
import pytest
import torch

from tests import clouds
from tests import occupancy_oracle as OO
from tests.test_cpu_occupancy import DYADIC, cube_union, icosphere, inscribed_radius, lattice_labels

pytestmark = pytest.mark.gpu


def _occ(cuda, v, f):
    from nksr_b200.metrics import MeshOccupancy
    return MeshOccupancy(torch.from_numpy(np.ascontiguousarray(v)).to(cuda),
                         torch.from_numpy(np.ascontiguousarray(f)).to(cuda))


def _along(occ, q, dirs):
    from nksr_b200.metrics import occupancy_along
    return occupancy_along(occ, torch.from_numpy(np.ascontiguousarray(q, dtype=np.float32)).to(occ.device),
                           dirs).cpu().numpy()


def _contains(occ, q, k):
    return occ.contains(torch.from_numpy(np.ascontiguousarray(q, dtype=np.float32)).to(occ.device), k).cpu().numpy()


def _check_against_oracle(cuda, v, f, q, ks=(1, 3, 5)):
    """per-direction parity and the K-ray vote, both bitwise against the oracle"""
    occ = _occ(cuda, v, f)
    parity = [OO.ray_crossings(v, f, q, d) & 1 for d in OO.DEFAULT_DIRECTIONS[:max(ks)]]
    for i, p in enumerate(parity):
        assert np.array_equal(_along(occ, q, OO.DEFAULT_DIRECTIONS[i:i + 1]), p.astype(bool)), i
    for k in ks:
        want = 2 * sum(parity[:k]) > k
        assert np.array_equal(_contains(occ, q, k), want), k
    return occ


def test_random_soup_bitwise(cuda):
    rng = np.random.default_rng(0)
    V, T = 400, 3000
    v = (rng.normal(size=(V, 3)) * [2.0, 1.0, 0.5]).astype(np.float32)
    f = rng.integers(0, V, size=(T, 3)).astype(np.int32)
    f[::97, 1] = f[::97, 0]                                  # zero-area triangles
    f[1::89] = f[2::89][: len(f[1::89])]                     # duplicates
    flip = rng.random(T) < 0.5
    f[flip] = f[flip][:, ::-1]                               # mixed winding
    q = (rng.normal(size=(20_000, 3)) * [2.5, 1.3, 0.7]).astype(np.float32)
    q[:500] = v[rng.integers(0, V, 500)]                     # queries on vertices
    _check_against_oracle(cuda, v, f, q)


def test_cube_union_ties_on_the_kernel(cuda):
    q, want = lattice_labels()
    for seed in (None, 1):
        v, f = cube_union(rng=None if seed is None else np.random.default_rng(seed))
        occ = _occ(cuda, v, f)
        for d in DYADIC:
            got = _along(occ, q, d[None])
            assert np.array_equal(got, want), (seed, d)
            assert np.array_equal(got, OO.occupancy(v, f, q, directions=d[None]))
        got = _along(occ, q, DYADIC)
        assert np.array_equal(got, want)


def test_dual_mc_sphere(cuda):
    import nksr_b200
    R, W = 0.35, 0.02
    xyz, nrm = clouds.sphere(40_000, radius=R, noise=0.001, seed=3)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    field = nksr_b200.Reconstructor(cuda).reconstruct(t(xyz), t(nrm), voxel_size=W, solver_tol=1e-6)
    mesh = field.extract_dual_mesh(mise_iter=1)
    v, f = mesh.v.cpu().numpy(), mesh.f.cpu().numpy().astype(np.int32)
    rng = np.random.default_rng(5)
    q = (rng.random((200_000, 3)) * 1.0 - 0.5).astype(np.float32)
    from nksr_b200.metrics import MeshOccupancy
    occ = MeshOccupancy(mesh.v, mesh.f)
    got = {k: _contains(occ, q, k) for k in (1, 3, 5)}
    sub = rng.choice(q.shape[0], 1000, replace=False)
    parity = [OO.ray_crossings(v, f, q[sub], d) & 1 for d in OO.DEFAULT_DIRECTIONS[:5]]
    for k in (1, 3, 5):
        assert np.array_equal(got[k][sub], 2 * sum(parity[:k]) > k), k
    r = np.linalg.norm(q.astype(np.float64), axis=1)
    far = np.abs(r - R) > 2 * W
    gt = r < R
    iou = {k: OO.occupancy_iou(got[k][far], gt[far]) for k in (1, 3, 5)}
    # The mesh is open (sub-cell holes: about 2 k edges with one triangle), so a single ray mislabels some samples
    # and the vote repairs them.  Measured on an H100: IoU 0.97363 (K = 1), 0.99968 (K = 3), 1.0 (K = 5); the bounds
    # leave a margin of about 1e-2, 5e-4 and 1e-4.
    for k, bound in ((1, 0.96), (3, 0.999), (5, 0.9999)):
        assert iou[k] >= bound, (k, iou[k])


def test_large_icosphere(cuda):
    v, f = icosphere(8)
    assert f.shape[0] > 1_000_000
    r_in = inscribed_radius(v, f)
    rng = np.random.default_rng(6)
    q = (rng.random((1_000_000, 3)) * 2.4 - 1.2).astype(np.float32)
    r = np.linalg.norm(q.astype(np.float64), axis=1)
    occ = _occ(cuda, v, f)
    for k in (1, 3):
        got = _contains(occ, q, k)
        assert np.array_equal(got[r < r_in], np.ones((r < r_in).sum(), bool))
        assert not got[r > 1.0].any()
    sub = rng.choice(q.shape[0], 40, replace=False)
    assert np.array_equal(_contains(occ, q[sub], 1), OO.occupancy(v, f, q[sub], n_rays=1))


def test_degenerate_builds(cuda):
    rng = np.random.default_rng(7)
    # every triangle has its centroid at the origin: all Morton keys equal, the hierarchy splits on the index alone
    u = rng.integers(-8, 9, size=(5000, 3)).astype(np.float32)
    w = rng.integers(-8, 9, size=(5000, 3)).astype(np.float32)
    v = np.concatenate([u, w, -(u + w)]).astype(np.float32)
    f = np.stack([np.arange(5000), 5000 + np.arange(5000), 10000 + np.arange(5000)], axis=1).astype(np.int32)
    q = (rng.normal(size=(3000, 3)) * 6).astype(np.float32)
    _check_against_oracle(cuda, v, f, q, ks=(1, 3))
    # one triangle
    v1 = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0.5]], np.float32)
    f1 = np.array([[0, 1, 2]], np.int32)
    q1 = (rng.random((5000, 3)) * 3 - 1).astype(np.float32)
    _check_against_oracle(cuda, v1, f1, q1)
    # queries far outside the box of a closed mesh
    vs, fs = icosphere(3, 0.5)
    far = (rng.normal(size=(4000, 3)) * 1e4).astype(np.float32)
    occ = _check_against_oracle(cuda, vs, fs, far, ks=(1, 3))
    assert not _contains(occ, far, 3).any()
    # no triangles, no queries
    none = _occ(cuda, vs, np.zeros((0, 3), np.int32))
    assert not _contains(none, far[:10], 3).any()
    assert _contains(occ, np.zeros((0, 3), np.float32), 3).shape == (0,)
    assert _contains(none, np.zeros((0, 3), np.float32), 1).shape == (0,)


def test_evaluator_o3d_iou_end_to_end(cuda):
    from nksr_b200.metrics import MeshEvaluator
    v, f = icosphere(3, 0.5)
    rng = np.random.default_rng(8)
    gt = rng.normal(size=(20_000, 3))
    gt /= np.linalg.norm(gt, axis=1, keepdims=True)
    gt_n = gt.copy()
    gt *= 0.5
    pts = (rng.random((10_000, 3)) * 1.2 - 0.6).astype(np.float32)
    occ = np.linalg.norm(pts, axis=1) < 0.5
    mesh = (torch.from_numpy(v).to(cuda), torch.from_numpy(f).to(cuda))
    names = MeshEvaluator.ALL_METRICS + ["o3d-iou"]
    ev = MeshEvaluator(n_points=50_000, metric_names=names, occupancy_rays=3)
    out = ev.eval_mesh(mesh, gt, gt_n, onet_samples=(pts, occ))
    plain = MeshEvaluator(n_points=50_000).eval_mesh(mesh, gt, gt_n, onet_samples=(pts, occ))
    assert sorted(out) == sorted(names)
    assert {k: out[k] for k in plain} == plain
    want = OO.occupancy_iou(OO.occupancy(v, f, pts, n_rays=3), occ)
    assert out["o3d-iou"] == want and 0.95 < want < 1.0
    for sample in ((pts, occ.astype(np.uint8)), (torch.from_numpy(pts).to(cuda), torch.from_numpy(occ).to(cuda)),
                   (torch.from_numpy(pts), torch.from_numpy(occ.astype(np.uint8)))):
        assert ev.eval_mesh(mesh, gt, gt_n, onet_samples=sample) == out
    with pytest.raises(ValueError, match="onet_samples"):
        ev.eval_mesh(mesh, gt, gt_n)
    empty = ev.eval_mesh((v, np.zeros((0, 3), np.int32)), gt, gt_n, onet_samples=(pts, occ))
    assert all(math.isnan(x) for x in empty.values())


def test_rejections(cuda):
    from nksr_b200._lib import NksrError
    from nksr_b200.metrics import MeshOccupancy
    v, f = icosphere(1)
    tv, tf = torch.from_numpy(v).to(cuda), torch.from_numpy(f).to(cuda)
    bad = tf.clone()
    bad[3, 1] = v.shape[0]
    with pytest.raises(NksrError):
        MeshOccupancy(tv, bad)
    bad[3, 1] = -1
    with pytest.raises(NksrError):
        MeshOccupancy(tv, bad)
    nan = tv.clone()
    nan[2, 0] = float("nan")
    with pytest.raises(NksrError):
        MeshOccupancy(nan, tf)
    with pytest.raises(NksrError):
        MeshOccupancy(tv.cpu(), tf)
    occ = MeshOccupancy(tv, tf)
    with pytest.raises(NksrError):
        occ.contains(torch.zeros((4, 3)), 1)
    with pytest.raises(NksrError):
        occ.contains(torch.full((4, 3), float("inf"), device=cuda), 1)
    for k in (0, 2, 11):
        with pytest.raises(ValueError):
            occ.contains(torch.zeros((4, 3), device=cuda), k)
