"""The PointTSDFVolume ray builder on the GPU (csrc/tsdf_volume.cu, DESIGN.md SPEC S19) against the fp64 oracle
(oracle/gt_volume.py), its repeatability and ray-order independence, its edge cases, and training with volume ground
truth (nksr_b200/training.py with TrainingScene(gt=...))."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import gt_volume as O
from tests import clouds

pytestmark = pytest.mark.gpu


def _kernel(xyz, sensor, lo, h, dims, tau, dev):
    """the entry point on a given grid"""
    from nksr_b200 import _lib
    x = torch.as_tensor(np.ascontiguousarray(xyz, np.float32)).to(dev)
    s = torch.as_tensor(np.ascontiguousarray(sensor, np.float32)).to(dev)
    vmin3 = (C.c_float * 3)(*[float(v) for v in np.asarray(lo, np.float32)])
    dims3 = (C.c_int64 * 3)(*dims)
    vol = torch.empty(tuple(dims), dtype=torch.float32, device=dev)
    nb = _lib.call("nksr_tsdf_volume_workspace_bytes", C.addressof(dims3))
    ws = _lib._ws(nb, dev)
    _lib.call("nksr_tsdf_volume", x, s, x.shape[0], C.addressof(vmin3), float(np.float32(h)), C.addressof(dims3),
              float(np.float32(tau)), vol, ws, nb, _lib.stream_ptr(dev))
    return vol.cpu().numpy()


def _classes(v):
    return np.where(np.isnan(v), 2, np.where(np.abs(v) < 1.0, 0, 1))


def _agree(name, got, xyz, sensor, lo, h, dims, tau):
    """classes equal and near values within fp32 rounding at every node the oracle does not flag; returns the number
    of flagged nodes"""
    want, amb = O.tsdf_volume(xyz, sensor, lo, h, dims, tau)
    ok = ~amb
    cg, cw = _classes(got), _classes(want)
    bad = ok & (cg != cw)
    assert not bad.any(), f"{name}: {int(bad.sum())} nodes differ in class, first at {np.argwhere(bad)[:3].tolist()}"
    near = ok & (cw == 0)
    if near.any():
        np.testing.assert_allclose(got[near], want[near], rtol=0, atol=2e-6)
    n_amb = int(amb.sum())
    print(f"[gt_volume] {name}: {np.prod(dims)} nodes, near {int((cw == 0).sum())} free {int((cw == 1).sum())} "
          f"unknown {int((cw == 2).sum())}; ambiguous in the oracle {n_amb}; agree elsewhere")
    return n_amb


def _plane(lo, h, z_surface, z_sensor, n_side, tilt=0.0):
    ij = np.stack(np.meshgrid(np.arange(n_side), np.arange(n_side), indexing="ij"), -1).reshape(-1, 2)
    xy = lo[:2] + (ij + 0.5 + math.sqrt(2) / 10) * h
    xyz = np.c_[xy, z_surface + tilt * xy[:, 0]].astype(np.float32)
    sensor = np.c_[xy[:, 0] * (1 - tilt) + tilt, xy[:, 1], np.full(len(xy), z_sensor)].astype(np.float32)
    return xyz, sensor


def test_plane_at_irrational_offsets_matches_the_oracle_exactly(cuda):
    h = math.sqrt(2) / 20
    lo = np.full(3, math.pi / 1000)
    xyz, sensor = _plane(lo, h, 1.0 + math.e / 100, 0.1 + math.sqrt(3) / 100, 10)
    dims = (12, 12, 16)
    got = _kernel(xyz, sensor, lo, h, dims, 2 * h, cuda)
    assert _agree("plane, vertical rays", got, xyz, sensor, lo, h, dims, 2 * h) == 0
    want, _ = O.tsdf_volume(xyz, sensor, lo, h, dims, 2 * h)
    assert np.array_equal(got, want, equal_nan=True)


def test_tilted_plane_sphere_and_occlusion_match_the_oracle(cuda):
    h = math.sqrt(2) / 20
    lo = np.full(3, math.pi / 1000)
    xyz, sensor = _plane(lo, h, 0.9 + math.e / 100, 0.1, 24, tilt=0.3)
    _agree("tilted plane, slanted rays", _kernel(xyz, sensor, lo, h, (30, 30, 24), 2 * h, cuda), xyz, sensor, lo, h,
           (30, 30, 24), 2 * h)
    # a sphere seen from outside: every point's sensor 1.5 out along its normal
    p, n = clouds.sphere(20000, noise=0.0)
    s = (p + 1.5 * n).astype(np.float32)
    h, lo = 0.02, np.full(3, -0.41)
    dims = (42, 42, 42)
    _agree("sphere, outward sensors", _kernel(p, s, lo, h, dims, 2 * h, cuda), p, s, lo, h, dims, 2 * h)
    # two parallel planes: the rays to the back one stop at the front one and leave the gap unknown
    h = math.sqrt(2) / 20
    lo = np.full(3, math.pi / 1000)
    f, s1 = _plane(lo, h, 0.8 + math.e / 100, 0.1 + math.sqrt(3) / 100, 10)
    b, s2 = _plane(lo, h, 1.6 + math.e / 100, 0.1 + math.sqrt(3) / 100, 10)
    xyz, sensor, dims = np.r_[f, b], np.r_[s1, s2], (12, 12, 24)
    got = _kernel(xyz, sensor, lo, h, dims, 2 * h, cuda)
    assert _agree("two planes", got, xyz, sensor, lo, h, dims, 2 * h) == 0
    z = np.float32(lo[2]) + np.arange(24) * np.float32(h)
    gap = (z > f[0, 2] + 2 * h) & (z < b[0, 2] - 2 * h)
    assert gap.any() and np.isnan(got[5, 5][gap]).all()


def test_cfg4_crop_matches_the_oracle(cuda):
    from nksr_b200.gt_geometry import PointTSDFVolume
    from tests import scenes
    xyz, sensor, W = scenes.crop("cfg4_outdoor", 200_000, with_sensor=True)
    t = lambda a: torch.from_numpy(a).to(cuda)
    gt = PointTSDFVolume.from_sensor_rays(t(xyz), t(xyz), t(sensor), h=W, tau=2 * W, margin=8 * W)
    got = gt.volume.cpu().numpy()
    n_amb = _agree("cfg4 crop 200k", got, xyz, sensor, gt.volume_min, W, got.shape, 2 * W)
    assert n_amb < 0.02 * got.size
    fr = gt.class_fractions()
    assert fr["near"] > 0 and fr["free"] > 0 and fr["unknown"] > 0


def test_repeatable_and_ray_order_independent(cuda):
    from nksr_b200.gt_geometry import PointTSDFVolume
    from tests import scenes
    xyz, sensor, W = scenes.crop("cfg4_outdoor", 100_000, with_sensor=True)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    build = lambda x, s: PointTSDFVolume.from_sensor_rays(t(x), t(x), t(s), h=W, tau=2 * W, margin=4 * W).volume
    a, b = build(xyz, sensor), build(xyz, sensor)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    perm = np.random.default_rng(0).permutation(xyz.shape[0])
    c = build(xyz[perm], sensor[perm])
    assert np.array_equal(_classes(a.cpu().numpy()), _classes(c.cpu().numpy()))
    # values may differ only where two rays tie on |sdf| with opposite signs or different last bits
    fin = torch.isfinite(a)
    assert float((a[fin] - c[fin]).abs().max()) < 2e-6 or int((a[fin] != c[fin]).sum()) < 1e-4 * int(fin.sum())


def test_edge_cases(cuda):
    h, lo, dims = 0.1, np.zeros(3), (8, 8, 8)
    # no rays: all unknown
    got = _kernel(np.zeros((0, 3)), np.zeros((0, 3)), lo, h, dims, 0.2, cuda)
    assert np.isnan(got).all()
    # rays that never enter the box, and degenerate rays
    xyz = np.array([[5.0, 5.0, 5.0], [-3.0, 0.2, 0.2], [0.3, 0.3, 0.3], [np.nan, 0.3, 0.3]], np.float32)
    sensor = np.array([[6.0, 5.0, 5.0], [-3.0, 5.0, 0.2], [0.3, 0.3, 0.3], [0.0, 0.0, 0.0]], np.float32)
    got = _kernel(xyz, sensor, lo, h, dims, 0.2, cuda)
    assert np.isnan(got).all()
    # r <= tau: the sensor inside the band
    rng = np.random.default_rng(3)
    p = rng.uniform(0.2, 0.5, (200, 3)).astype(np.float32)
    s = (p + rng.normal(size=(200, 3)).astype(np.float32) * 0.05).astype(np.float32)
    got = _kernel(p, s, lo + math.pi / 1000, h, dims, 0.2, cuda)
    _agree("r <= tau", got, p, s, lo + math.pi / 1000, h, dims, 0.2)
    assert (np.abs(got[np.isfinite(got)]) < 1.0).mean() > 0.5


def _sphere_scene(cuda, n=30_000, W=0.02, depth=4):
    from nksr_b200.gt_geometry import PointTSDFVolume
    from nksr_b200 import training as T
    xyz, nrm = clouds.sphere(n, noise=0.001)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(cuda)
    sensor = xyz + 1.0 * nrm
    gt = PointTSDFVolume.from_sensor_rays(t(xyz), t(nrm), t(sensor), h=W, tau=2 * W, margin=W * 2 ** (depth - 1))
    return T.TrainingScene(t(xyz), t(nrm), W, depth, gt=gt), gt


class _Field:
    """an analytic field on the scene's hierarchy: |x| - 0.33 + a ripple"""

    def __init__(self, svh):
        self.svh = svh

    def evaluate_f(self, q, grad=False):
        from types import SimpleNamespace
        return SimpleNamespace(value=q.norm(dim=1) - 0.33 + 0.01 * torch.sin(17.0 * q[:, 0]))


def test_losses_with_volume_ground_truth_match_a_torch_restatement(cuda):
    from nksr_b200 import training as T
    from nksr_b200.sdfgen import sdf_from_points
    scene, gt = _sphere_scene(cuda)
    W = scene.voxel_size
    field = _Field(scene.enc_svh)
    g1 = torch.Generator(device=cuda).manual_seed(5)
    got = T.spatial_loss(field, scene.ref_xyz, scene.ref_normal, W, generator=g1, gt=gt)
    # models/loss.py:227-248 restated
    g2 = torch.Generator(device=cuda).manual_seed(5)
    q = T.udf_samples(scene.enc_svh, gt.xyz, gt.normal, W, T.SPATIAL_SAMPLERS, g2)
    pd = field.evaluate_f(q).value
    tr = lambda f: torch.tanh(f / W) * W
    gt_tsdf = tr(-sdf_from_points(q, gt.xyz, gt.normal, 8, 3.0, adaptive_knn=8)[0])
    cls = gt.query_classification(q)
    near, empty = cls == 0, cls == 1
    assert int(near.sum()) > 0 and int(empty.sum()) > 0 and int((cls == 2).sum()) > 0
    want = (torch.abs((tr(pd)[near] - gt_tsdf[near]) / W).sum() + (0.1 * torch.exp(pd[empty] / (2 * W))).sum()) \
        / q.shape[0]
    torch.testing.assert_close(got, want, rtol=1e-5, atol=0)
    # the UDF ground truth (models/loss.py:111-117)
    torch.testing.assert_close(T.udf_gt(q, gt.xyz, gt.normal, W, gt=gt), tr(gt.query_sdf(q)).abs(), rtol=0, atol=0)
    # without gt the loss is the dense-points one
    g3, g4 = (torch.Generator(device=cuda).manual_seed(5) for _ in range(2))
    a = T.spatial_loss(field, scene.xyz, scene.normal, W, generator=g3)
    q = T.udf_samples(scene.enc_svh, scene.xyz, scene.normal, W, T.SPATIAL_SAMPLERS, g4)
    b = torch.abs((tr(field.evaluate_f(q).value) - tr(-sdf_from_points(q, scene.xyz, scene.normal, 8, 0.02)[0])) / W)
    torch.testing.assert_close(a, b.sum() / q.shape[0], rtol=1e-5, atol=0)


def test_training_with_volume_ground_truth_lowers_the_empty_space_term(cuda):
    from nksr_b200 import training as T
    from nksr_b200.network import NKSRNetwork
    scene, gt = _sphere_scene(cuda)
    print(f"[gt_volume] sphere volume {tuple(gt.volume.shape)}, fractions {gt.class_fractions()}")
    net = NKSRNetwork(dict(backbone="unet", tree_depth=4, kernel_dim=4, trainable=True, seed=3)).to(cuda)
    opt = T.make_optimizer(net)
    gen = torch.Generator(device=cuda).manual_seed(3)
    curve = []
    for step in range(8):
        _, _, k = T.train_step(net, opt, scene, gen, kernel=True)
        curve.append({key: float(v) for key, v in k.items()})
        grads = [p.grad for p in net.parameters() if p.grad is not None]
        assert grads and all(bool(torch.isfinite(g).all()) for g in grads)
    print(f"[gt_volume] spatial_empty {[round(c['spatial_empty'], 5) for c in curve]}")
    assert all(math.isfinite(v) for c in curve for v in c.values())
    assert np.mean([c["spatial_empty"] for c in curve[-3:]]) < np.mean([c["spatial_empty"] for c in curve[:3]])
