"""Volume ground truth without a GPU (DESIGN.md SPEC S19): the fp64 oracle of the ray builder (oracle/gt_volume.py) on
hand-made rays, the PointTSDFVolume's groundtruth.bin round trip and classification rule (nksr_b200/gt_geometry.py),
and the argument checks of the host class and of the C-ABI entry point."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from oracle import gt_volume as O


def _plane_rays(z_surface, z_sensor, n_side, lo, h):
    """vertical rays to a lattice of points on the plane z = z_surface, one per column, at irrational offsets"""
    ij = np.stack(np.meshgrid(np.arange(n_side), np.arange(n_side), indexing="ij"), -1).reshape(-1, 2)
    xy = lo[:2] + (ij + 0.5 + math.sqrt(2) / 10) * h
    xyz = np.c_[xy, np.full(len(xy), z_surface)].astype(np.float32)
    return xyz, np.c_[xy, np.full(len(xy), z_sensor)].astype(np.float32)


def test_oracle_free_nodes_lie_in_front_of_the_hit():
    h = math.sqrt(2) / 20
    tau = 2 * h
    lo = np.array([0.0, 0.0, 0.0]) + math.pi / 1000
    xyz, sensor = _plane_rays(1.0 + math.e / 100, 0.1 + math.sqrt(3) / 100, 10, lo, h)
    vol, amb = O.tsdf_volume(xyz, sensor, lo, h, (12, 12, 16), tau)
    assert not amb.any()
    z = np.float32(lo[2]) + np.arange(16) * float(np.float32(h))
    zs = float(xyz[0, 2])
    col = vol[3, 4]                                  # a column with a ray through it
    free, near, unknown = col == 1.0, np.abs(col) < 1.0, np.isnan(col)
    assert free.any() and near.any() and unknown.any()
    assert np.all(zs - z[free] >= float(np.float32(tau)) * (1 - 1e-6))          # in front of the hit by >= tau
    assert np.all(np.abs(zs - z[near]) < float(np.float32(tau)))
    np.testing.assert_allclose(col[near], (zs - z[near]) / np.float32(tau), atol=1e-6)
    # below the first sensor-side node nothing is observed, nor beyond the band behind the surface
    assert np.all(unknown[z > zs + tau])
    # columns no ray passes stay unknown
    assert np.isnan(vol[11, 11]).all()


def test_oracle_two_parallel_planes_leave_the_gap_unknown():
    h = math.sqrt(2) / 20
    tau = 2 * h
    lo = np.array([0.0, 0.0, 0.0]) + math.pi / 1000
    zs = 0.1 + math.sqrt(3) / 100
    front, s1 = _plane_rays(0.8 + math.e / 100, zs, 10, lo, h)
    back, s2 = _plane_rays(1.6 + math.e / 100, zs, 10, lo, h)
    vol, amb = O.tsdf_volume(np.r_[front, back], np.r_[s1, s2], lo, h, (12, 12, 24), tau)
    assert not amb.any()
    z = np.float32(lo[2]) + np.arange(24) * float(np.float32(h))
    col = vol[5, 5]
    gap = (z > front[0, 2] + tau) & (z < back[0, 2] - tau)
    assert gap.any() and np.isnan(col[gap]).all()             # the back rays stop at the front surface
    assert np.all(col[(z < front[0, 2] - tau) & (z >= zs + h)] == 1.0)
    assert np.all(np.abs(col[np.abs(z - back[0, 2]) < tau]) < 1.0)   # the back surface is still observed
    # without the front plane the same rays carve the gap
    alone, _ = O.tsdf_volume(back, s2, lo, h, (12, 12, 24), tau)
    assert np.all(alone[5, 5][gap] == 1.0)


def test_oracle_flags_rays_along_cell_boundaries():
    h = 0.25
    lo = np.zeros(3)
    # a ray along the boundary plane x = lo + h/2 enters cells with zero overlap on one side
    xyz = np.array([[0.125, 0.3, 1.0]], np.float32)
    sensor = np.array([[0.125, 0.3, 0.05]], np.float32)
    _, amb = O.tsdf_volume(xyz, sensor, lo, h, (4, 4, 8), 0.5)
    assert amb.any()


def _make(volume, lo, hi, device="cpu"):
    from nksr_b200.gt_geometry import PointTSDFVolume
    xyz = torch.rand(7, 3)
    return PointTSDFVolume(xyz, torch.nn.functional.normalize(torch.randn(7, 3), dim=1), torch.as_tensor(volume),
                           lo, hi)


def test_groundtruth_bin_round_trip(tmp_path):
    from nksr_b200.gt_geometry import PointTSDFVolume
    rng = np.random.default_rng(0)
    vol = rng.uniform(-1, 1, (4, 5, 6)).astype(np.float32)
    vol[0, 0, 0] = np.nan
    gt = _make(vol, [0.5, -1.0, 2.0], [2.0, 1.0, 4.5])
    path = tmp_path / "groundtruth.bin"
    gt.save(path)
    with np.load(path) as z:
        assert set(z.files) == {"xyz", "normal", "volume", "volume_min", "volume_max"}
        np.testing.assert_array_equal(z["volume"], vol)
    back = PointTSDFVolume.load(path, device="cpu")
    for a, b in zip(back.torch_attr(), gt.torch_attr()):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    np.testing.assert_array_equal(back.volume_min, gt.volume_min)
    np.testing.assert_array_equal(back.volume_max, gt.volume_max)


def _classify_loop(q, vol, lo, hi, band):
    """the rule restated one query at a time: inclusive box, nearest node of linspace(lo, hi, dims) with ties to the
    even index (Python's round), NaN -> 2, |v| < band -> 0, else 1; outside -> 2"""
    out = []
    dims = vol.shape
    for p in q:
        if not all(lo[a] <= p[a] <= hi[a] for a in range(3)):
            out.append(2)
            continue
        idx = [min(max(round((float(p[a]) - lo[a]) / (hi[a] - lo[a]) * (dims[a] - 1)), 0), dims[a] - 1)
               for a in range(3)]
        v = vol[idx[0], idx[1], idx[2]]
        out.append(2 if not np.isfinite(v) else (0 if abs(v) < band else 1))
    return np.array(out)


def test_classification_matches_the_loop_restatement():
    # dims - 1 and the box are powers of two, so every normalised coordinate below is exact in fp32
    dims, lo, hi = (5, 3, 9), np.array([0.0, -1.0, 2.0]), np.array([2.0, 0.0, 6.0])
    rng = np.random.default_rng(1)
    vol = rng.choice([-0.5, 0.25, 0.99, 1.0, -1.0, 1.5, np.nan], size=dims).astype(np.float32)
    gt = _make(vol, lo, hi)
    step = (hi - lo) / (np.array(dims) - 1)
    q = [rng.uniform(lo - 0.3, hi + 0.3, (400, 3))]
    half = lo + (rng.integers(0, np.array(dims) - 1, (300, 3)) + 0.5) * step          # exactly between two nodes
    q.append(half)
    face = rng.uniform(lo, hi, (300, 3))
    axis = rng.integers(0, 3, 300)
    face[np.arange(300), axis] = np.where(rng.random(300) < 0.5, lo[axis], hi[axis])
    q.append(face)
    q.append(np.array([lo, hi, [lo[0], hi[1], lo[2]], lo - 1e-3, hi + 1e-3]))
    q = np.concatenate(q).astype(np.float32)
    for band in (1.0, 0.5):
        got = gt.query_classification(torch.from_numpy(q), band=band).numpy()
        want = _classify_loop(q, vol, lo, hi, band)
        np.testing.assert_array_equal(got, want)
    got = gt.query_classification(torch.from_numpy(q)).numpy()
    assert {0, 1, 2} <= set(got.tolist())
    nan_nodes = np.argwhere(np.isnan(vol))[:5]
    at_nan = (lo + nan_nodes * step).astype(np.float32)
    assert (gt.query_classification(torch.from_numpy(at_nan)).numpy() == 2).all()


def test_argument_validation():
    from nksr_b200.gt_geometry import PointTSDFVolume
    vol = np.zeros((2, 2, 2), np.float32)
    with pytest.raises(ValueError):
        _make(vol, [0, 0, 0], [1, 0, 1])                 # empty box
    with pytest.raises(ValueError):
        _make(vol, [0, 0, 0], [1, np.nan, 1])
    with pytest.raises(ValueError):
        _make(np.zeros((2, 2), np.float32), [0, 0, 0], [1, 1, 1])
    with pytest.raises(ValueError):
        PointTSDFVolume(torch.zeros(3, 3), torch.zeros(4, 3), torch.zeros(2, 2, 2), [0, 0, 0], [1, 1, 1])
    p = torch.rand(10, 3)
    s = p + 1.0
    for kw in (dict(h=0.0, tau=0.1, margin=0.0), dict(h=0.1, tau=-1.0, margin=0.0),
               dict(h=float("nan"), tau=0.1, margin=0.0), dict(h=0.1, tau=0.1, margin=-1.0),
               dict(h=1e-4, tau=0.1, margin=10.0)):                                      # 2^31 nodes or more
        with pytest.raises(ValueError):
            PointTSDFVolume.from_sensor_rays(p, p, s, **kw)
    with pytest.raises(ValueError):
        PointTSDFVolume.from_sensor_rays(p, p, s[:5], h=0.1, tau=0.2, margin=0.0)
    with pytest.raises(ValueError):
        PointTSDFVolume.from_sensor_rays(p[:0], p[:0], s[:0], h=0.1, tau=0.2, margin=0.0)
    bad = p.clone()
    bad[3, 1] = float("inf")
    with pytest.raises(ValueError):
        PointTSDFVolume.from_sensor_rays(bad, p, s, h=0.1, tau=0.2, margin=0.0)
    from nksr_b200._lib import NksrError
    with pytest.raises(NksrError):                       # CUDA only
        PointTSDFVolume.from_sensor_rays(p, p, s, h=0.1, tau=0.2, margin=0.0)


def test_entry_point_rejects_bad_arguments():
    """the C-ABI checks its arguments before it touches the device"""
    from nksr_b200 import _lib
    lib = _lib.load()
    d = lambda *v: (C.c_int64 * 3)(*v)
    assert lib.nksr_tsdf_volume_workspace_bytes(C.addressof(d(4, 5, 6))) == 8 * 120
    for bad in (d(1, 5, 6), d(4, 0, 6), d(2 ** 11, 2 ** 10, 2 ** 10)):
        assert lib.nksr_tsdf_volume_workspace_bytes(C.addressof(bad)) == 0
    vmin = (C.c_float * 3)(0.0, 0.0, 0.0)
    fake = 1 << 20                                      # never dereferenced: the checks fail first
    dims = d(4, 5, 6)

    def rc(n=1, h=0.1, dims=dims, tau=0.2, ws_bytes=8 * 120, vmin=vmin):
        return lib.nksr_tsdf_volume(fake, fake, n, C.addressof(vmin), h, C.addressof(dims), tau, fake, fake, ws_bytes,
                                    None)
    assert rc(h=0.0) == -1 and rc(tau=0.0) == -1 and rc(h=float("inf")) == -1 and rc(n=-1) == -1
    assert rc(dims=d(4, 1, 6)) == -1
    assert rc(vmin=(C.c_float * 3)(0.0, float("nan"), 0.0)) == -1
    assert rc(ws_bytes=8 * 120 - 1) == -3
