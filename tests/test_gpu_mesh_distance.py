"""The closest-triangle query on the GPU (csrc/raycast.cu k_mesh_closest, MeshOccupancy.closest / signed_distance;
DESIGN.md SPEC S21) against the brute force of tests/distance_oracle.py, bit for bit, and training against a mesh
(gt_geometry.MeshGroundTruth with TrainingScene(gt=...))."""
import math

import numpy as np
import pytest
import torch

from tests import clouds
from tests import distance_oracle as D
from tests.test_cpu_occupancy import icosphere, inscribed_radius

pytestmark = pytest.mark.gpu


def _occ(cuda, v, f):
    from nksr_b200.metrics import MeshOccupancy
    return MeshOccupancy(torch.from_numpy(np.ascontiguousarray(v)).to(cuda),
                         torch.from_numpy(np.ascontiguousarray(f)).to(cuda))


def _closest(occ, q):
    d, x, t = occ.closest(torch.from_numpy(np.ascontiguousarray(q, dtype=np.float32)).to(occ.device))
    assert d.dtype == torch.float32 and x.dtype == torch.float32 and t.dtype == torch.int64
    return d.cpu().numpy(), x.cpu().numpy(), t.cpu().numpy()


def _bitwise(got, want):
    for g, w in zip(got, want):
        if g.dtype == np.float32:
            g, w = g.view(np.uint32), w.view(np.uint32)
        assert np.array_equal(g, w)


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
    q[500:600] = (v[f[500:600, 0]] + v[f[500:600, 1]]) / 2   # and on edges
    occ = _occ(cuda, v, f)
    _bitwise(_closest(occ, q), D.mesh_closest(v, f, q))
    # the occupancy is untouched by the query, and the two queries share one build
    from tests import occupancy_oracle as OO
    inside = occ.contains(torch.from_numpy(q).to(cuda), 3).cpu().numpy()
    assert np.array_equal(inside, OO.occupancy(v, f, q, n_rays=3))


def test_icosphere_signed_distance(cuda):
    v, f = icosphere(4, 0.5)
    rng = np.random.default_rng(1)
    q = (rng.random((200_000, 3)) * 1.6 - 0.8).astype(np.float32)
    occ = _occ(cuda, v, f)
    d, x, t = _closest(occ, q)
    r = np.linalg.norm(q.astype(np.float64), axis=1)
    gap = 0.5 - inscribed_radius(v, f)                       # the polygon lies between the two spheres
    assert np.all(np.abs(d - np.abs(r - 0.5)) <= gap + 1e-6)
    tq = torch.from_numpy(q).to(cuda)
    sd = occ.signed_distance(tq, 3)
    inside = occ.contains(tq, 3)
    assert torch.equal(sd < 0, inside)
    assert torch.equal(sd.abs(), torch.from_numpy(d).to(cuda))
    assert bool(inside[torch.from_numpy(r < 0.5 - gap).to(cuda)].all())
    sub = rng.choice(q.shape[0], 2000, replace=False)
    _bitwise((d[sub], x[sub], t[sub]), D.mesh_closest(v, f, q[sub]))


def test_large_icosphere_subsample(cuda):
    v, f = icosphere(8)
    assert f.shape[0] > 1_000_000
    rng = np.random.default_rng(2)
    q = (rng.random((1_000_000, 3)) * 2.4 - 1.2).astype(np.float32)
    occ = _occ(cuda, v, f)
    d, x, t = _closest(occ, q)
    r = np.linalg.norm(q.astype(np.float64), axis=1)
    gap = 1.0 - inscribed_radius(v, f)
    assert np.all(np.abs(d - np.abs(r - 1.0)) <= gap + 1e-6)
    sub = rng.choice(q.shape[0], 24, replace=False)
    _bitwise((d[sub], x[sub], t[sub]), D.mesh_closest(v, f, q[sub]))


def test_degenerate_builds(cuda):
    rng = np.random.default_rng(3)
    q = (rng.normal(size=(4000, 3)) * 3).astype(np.float32)
    # all centroids at the origin: equal Morton keys
    u = rng.integers(-8, 9, size=(3000, 3)).astype(np.float32)
    w = rng.integers(-8, 9, size=(3000, 3)).astype(np.float32)
    v = np.concatenate([u, w, -(u + w)]).astype(np.float32)
    f = np.stack([np.arange(3000), 3000 + np.arange(3000), 6000 + np.arange(3000)], axis=1).astype(np.int32)
    _bitwise(_closest(_occ(cuda, v, f), q), D.mesh_closest(v, f, q))
    # every triangle on one coincident point, and zero-area triangles (segments)
    pt = np.float32([[0.5, -0.25, 0.125]])
    f0 = np.zeros((50, 3), np.int32)
    _bitwise(_closest(_occ(cuda, pt, f0), q), D.mesh_closest(pt, f0, q))
    seg = rng.normal(size=(30, 3)).astype(np.float32)
    fs = np.stack([np.arange(10), 10 + np.arange(10), np.arange(10)], axis=1).astype(np.int32)
    fs2 = np.stack([np.arange(10), 20 + np.arange(10), 20 + np.arange(10)], axis=1)
    fs = np.concatenate([fs, fs2]).astype(np.int32)
    _bitwise(_closest(_occ(cuda, seg, fs), q), D.mesh_closest(seg, fs, q))
    # one and two triangles
    v1 = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0.5], [2, 2, 2]], np.float32)
    for f1 in (np.int32([[0, 1, 2]]), np.int32([[0, 1, 2], [1, 3, 2]])):
        _bitwise(_closest(_occ(cuda, v1, f1), q), D.mesh_closest(v1, f1, q))
    # no triangles, no queries
    none = _occ(cuda, v1, np.zeros((0, 3), np.int32))
    d, x, t = _closest(none, q[:7])
    assert np.all(np.isinf(d)) and np.all(np.isnan(x)) and np.all(t == -1)
    assert torch.equal(none.signed_distance(torch.from_numpy(q[:7]).to(cuda)),
                       torch.full((7,), math.inf, device=cuda))
    one = _occ(cuda, v1, np.int32([[0, 1, 2]]))
    for occ in (one, none):
        d, x, t = _closest(occ, np.zeros((0, 3), np.float32))
        assert d.shape == (0,) and x.shape == (0, 3) and t.shape == (0,)


def test_rejections(cuda):
    from nksr_b200._lib import NksrError
    v, f = icosphere(1)
    occ = _occ(cuda, v, f)
    with pytest.raises(NksrError):
        occ.closest(torch.zeros((4, 3)))
    with pytest.raises(NksrError):
        occ.signed_distance(torch.zeros((4, 3)))
    for bad in (float("inf"), float("nan")):
        with pytest.raises(NksrError):
            occ.closest(torch.full((4, 3), bad, device=cuda))
        with pytest.raises(NksrError):
            occ.signed_distance(torch.full((4, 3), bad, device=cuda))
    for k in (0, 2, 11):
        with pytest.raises(ValueError):
            occ.signed_distance(torch.zeros((4, 3), device=cuda), k)


def _mesh_gt(cuda, W=0.02, level=5):
    from nksr_b200.gt_geometry import MeshGroundTruth
    v, f = icosphere(level, 0.35)
    return MeshGroundTruth(torch.from_numpy(v).to(cuda), torch.from_numpy(f).to(cuda), tau=2 * W)


def test_mesh_ground_truth_sign_and_classes(cuda):
    from nksr_b200.sdfgen import sdf_from_points
    W = 0.02
    gt = _mesh_gt(cuda, W)
    xyz, nrm, vol = gt.torch_attr()
    assert vol is None and xyz.shape == (100_000, 3) and nrm.shape == (100_000, 3)
    assert torch.allclose(nrm.norm(dim=1), torch.ones(1, device=cuda), atol=1e-5)
    assert float((nrm * xyz).sum(1).min()) > 0              # outward winding gives outward normals
    g = torch.Generator(device=cuda).manual_seed(4)
    q = torch.rand((100_000, 3), generator=g, device=cuda) * 1.2 - 0.6
    sdf = gt.query_sdf(q)
    r = q.double().norm(dim=1)
    far = (r - 0.35).abs() > 2 * W
    ref = -sdf_from_points(q, xyz, nrm, 8, 3.0, adaptive_knn=8)[0]
    assert int(far.sum()) > 50_000
    assert torch.equal(torch.sign(sdf[far]), torch.sign(ref[far]))
    assert torch.equal(sdf[far] > 0, r[far] < 0.35)
    cls = gt.query_classification(q)
    # the (distance, inside) kept for q is the fresh answer, and an in-place change of q is noticed
    assert torch.equal(sdf, -gt.mesh.signed_distance(q, 3))
    q2 = q.clone()
    q2.mul_(0.5)
    assert torch.equal(gt.query_sdf(q2), -gt.mesh.signed_distance(q2, 3))
    q2.add_(0.25)
    assert torch.equal(gt.query_sdf(q2), -gt.mesh.signed_distance(q2, 3))
    assert torch.equal(gt.query_classification(q), cls)
    assert cls.dtype == torch.int64 and set(torch.unique(cls).tolist()) == {0, 1}
    assert torch.equal(cls == 1, (sdf < 0) & (sdf.abs() >= 2 * W))
    assert torch.equal(gt.query_classification(q, band=0.5) == 1, (sdf < 0) & (sdf.abs() >= W))


class _Field:
    """an analytic field on the scene's hierarchy: |x| - 0.33 + a ripple"""

    def __init__(self, svh):
        self.svh = svh

    def evaluate_f(self, q, grad=False):
        from types import SimpleNamespace
        return SimpleNamespace(value=q.norm(dim=1) - 0.33 + 0.01 * torch.sin(17.0 * q[:, 0]))


def test_training_with_mesh_ground_truth(cuda):
    from nksr_b200 import training as T
    from nksr_b200.network import NKSRNetwork
    W = 0.02
    gt = _mesh_gt(cuda, W)
    xyz, nrm = clouds.sphere(30_000, noise=0.001)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(cuda)
    scene = T.TrainingScene(t(xyz), t(nrm), W, 4, gt=gt)
    assert scene.ref_xyz is gt.xyz
    field = _Field(scene.enc_svh)
    gen = lambda: torch.Generator(device=cuda).manual_seed(5)
    got = T.spatial_loss(field, scene.ref_xyz, scene.ref_normal, W, generator=gen(), gt=gt)
    # models/loss.py:227-248 restated on the mesh's SDF and classes
    q = T.udf_samples(scene.enc_svh, gt.xyz, gt.normal, W, T.SPATIAL_SAMPLERS, gen())
    pd = field.evaluate_f(q).value
    tr = lambda f: torch.tanh(f / W) * W
    gt_tsdf = tr(gt.query_sdf(q))
    cls = gt.query_classification(q)
    near, empty = cls == 0, cls == 1
    assert int(near.sum()) > 0 and int(empty.sum()) > 0
    want = (torch.abs((tr(pd)[near] - gt_tsdf[near]) / W).sum() + (0.1 * torch.exp(pd[empty] / (2 * W))).sum()) \
        / q.shape[0]
    torch.testing.assert_close(got, want, rtol=1e-5, atol=0)
    torch.testing.assert_close(T.udf_gt(q, gt.xyz, gt.normal, W, gt=gt), tr(gt.query_sdf(q)).abs(), rtol=0, atol=0)
    net = NKSRNetwork(dict(backbone="unet", tree_depth=4, kernel_dim=4, trainable=True, seed=3)).to(cuda)
    opt = T.make_optimizer(net)
    gen = torch.Generator(device=cuda).manual_seed(3)
    for _ in range(3):
        l_struct, l_udf, k = T.train_step(net, opt, scene, gen, kernel=True)
        assert math.isfinite(float(l_struct)) and math.isfinite(float(l_udf))
        assert all(math.isfinite(float(v)) for v in k.values())
        grads = [p.grad for p in net.parameters() if p.grad is not None]
        assert grads and all(bool(torch.isfinite(g).all()) for g in grads)
