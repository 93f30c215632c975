"""The first hit of a ray on the GPU (csrc/raycast.cu k_mesh_first_hit, MeshOccupancy.intersect; DESIGN.md SPEC S22)
against the brute force of tests/hit_oracle.py, bit for bit; the guarantee that rays from inside a closed mesh never
miss; and simulated LiDAR scans of a closed room (gt_geometry.scan_mesh) checked against the mesh, against the S19
volume builder, and run end to end through reconstruction, evaluation and training."""
import math

import numpy as np
import pytest
import torch

from tests import distance_oracle as D
from tests import hit_oracle as H
from tests.test_cpu_occupancy import cube_union, icosphere, inscribed_radius

pytestmark = pytest.mark.gpu


def box_mesh(lo, hi, inward=False):
    """the 12 triangles of the box [lo, hi], wound so that the normals point out of it (into it with inward)"""
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    v, f = [], []
    for a in range(3):
        u, w = (a + 1) % 3, (a + 2) % 3
        for side in (0, 1):
            base = len(v)
            for du, dw in ((0, 0), (1, 0), (1, 1), (0, 1)):
                p = lo.copy()
                p[a] = hi[a] if side else lo[a]
                p[u] = hi[u] if du else lo[u]
                p[w] = hi[w] if dw else lo[w]
                v.append(p)
            quad = [[base, base + 1, base + 2], [base, base + 2, base + 3]]     # e_u x e_w = +e_a
            out = side == 1
            f += [t if out != inward else t[::-1] for t in quad]
    return np.array(v, np.float32), np.array(f, np.int32)


ROOM_INNER = ((-2.0, -2.0, 0.0), (2.0, 2.0, 2.5))
ROOM_FURNITURE = (((0.5, -1.5, 0.05), (1.2, -0.8, 0.8)), ((-1.5, 0.4, 0.05), (-0.6, 1.4, 1.1)),
                  ((-0.3, 0.8, 1.4), (0.3, 1.2, 1.8)))
ROOM_POSES = np.float32([[0.0, 0.0, 1.2], [-1.2, -1.0, 1.5], [1.0, 1.2, 0.6]])


def room_mesh():
    """a closed room: walls 0.2 thick (an outward outer box around an inward inner box) and three boxes standing
    clear of the floor and walls.  The solid is walls and boxes; the air is outside it by ray parity, enclosed."""
    parts = [box_mesh((-2.2, -2.2, -0.2), (2.2, 2.2, 2.7)), box_mesh(*ROOM_INNER, inward=True)]
    parts += [box_mesh(lo, hi) for lo, hi in ROOM_FURNITURE]
    v, f, off = [], [], 0
    for pv, pf in parts:
        v.append(pv)
        f.append(pf + off)
        off += pv.shape[0]
    return np.concatenate(v), np.concatenate(f).astype(np.int32)


def in_room_air(p, margin=0.0):
    """bool: p lies in the room's air, at least margin from the inner walls and the boxes"""
    p = np.asarray(p, np.float64)
    lo, hi = np.asarray(ROOM_INNER[0]), np.asarray(ROOM_INNER[1])
    ok = np.all((p > lo + margin) & (p < hi - margin), axis=1)
    for blo, bhi in ROOM_FURNITURE:
        ok &= ~np.all((p > np.asarray(blo) - margin) & (p < np.asarray(bhi) + margin), axis=1)
    return ok


def _occ(cuda, v, f):
    from nksr_b200.metrics import MeshOccupancy
    return MeshOccupancy(torch.from_numpy(np.ascontiguousarray(v)).to(cuda),
                         torch.from_numpy(np.ascontiguousarray(f)).to(cuda))


def _hit(occ, o, d, t_max=None):
    c = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(occ.device)
    out = occ.intersect(c(o), c(d), c(t_max) if isinstance(t_max, np.ndarray) else t_max)
    assert [x.dtype for x in out] == [torch.float32] * 3 + [torch.int64]
    return tuple(x.cpu().numpy() for x in out)


def _bitwise(got, want):
    for g, w in zip(got, want):
        if g.dtype == np.float32:
            g, w = g.view(np.uint32), w.view(np.uint32)
        assert np.array_equal(g, w)


def _unit(rng, n):
    d = rng.normal(size=(n, 3))
    return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def test_icosphere_bitwise(cuda):
    v, f = icosphere(3, 0.5)
    rng = np.random.default_rng(0)
    n = 6000
    inside = _unit(rng, n) * (rng.random((n, 1)) * 0.45).astype(np.float32)
    outside = _unit(rng, n) * (0.6 + rng.random((n, 1))).astype(np.float32)
    aimed = -outside + (0.1 * rng.normal(size=(n, 3))).astype(np.float32)        # mostly towards the sphere
    surface = v[rng.integers(0, v.shape[0], n)]                                  # on vertices
    w = rng.random((n, 3)).astype(np.float32)
    w /= w.sum(1, keepdims=True)
    on_face = np.einsum("nk,nkc->nc", w, v[f[rng.integers(0, f.shape[0], n)]]).astype(np.float32)
    o = np.concatenate([inside, outside, outside, surface, on_face])
    d = np.concatenate([_unit(rng, n), _unit(rng, n), aimed, _unit(rng, n), _unit(rng, n)])
    d[:50] = np.float32([0, 0, 1])                                               # axis rays, zero components
    d[50:100] = np.float32([0.5, -2.0, 0])
    occ = _occ(cuda, v, f)
    got = _hit(occ, o, d)
    _bitwise(got, H.first_hit(v, f, o, d))
    assert np.all(got[3][:n] >= 0)                                               # from inside: always a hit
    assert np.mean(got[3][2 * n:3 * n] >= 0) > 0.9 and np.mean(got[3][n:2 * n] >= 0) < 1.0


def test_box_vertices_and_edges_bitwise(cuda):
    """the grid-aligned cube union with rays aimed exactly at its vertices and edge midpoints, and along the axes"""
    v, f = cube_union()
    rng = np.random.default_rng(1)
    targets = np.concatenate([v, (v[f[:, 0]] + v[f[:, 1]]) / 2, (v[f[:, 1]] + v[f[:, 2]]) / 2]).astype(np.float32)
    o = ((rng.integers(-4, 12, size=(targets.shape[0] * 4, 3))) * 0.5).astype(np.float32)
    tg = targets[rng.integers(0, targets.shape[0], o.shape[0])]
    d = tg - o
    keep = np.any(d != 0, axis=1)
    o, d = o[keep], d[keep]
    axis_o = (rng.integers(-2, 8, size=(3000, 3)) * 0.5).astype(np.float32)
    axis_d = np.eye(3, dtype=np.float32)[rng.integers(0, 3, 3000)] * rng.choice([-1.0, 1.0], (3000, 1)).astype(
        np.float32)
    o, d = np.concatenate([o, axis_o]), np.concatenate([d, axis_d])
    occ = _occ(cuda, v, f)
    got = _hit(occ, o, d)
    _bitwise(got, H.first_hit(v, f, o, d))
    # random diagonals and windings
    v2, f2 = cube_union(rng=np.random.default_rng(2))
    _bitwise(_hit(_occ(cuda, v2, f2), o, d), H.first_hit(v2, f2, o, d))


def test_soup_t_max_and_empty(cuda):
    rng = np.random.default_rng(3)
    V, T = 300, 2000
    v = (rng.normal(size=(V, 3)) * [2.0, 1.0, 0.5]).astype(np.float32)
    f = rng.integers(0, V, size=(T, 3)).astype(np.int32)
    f[::97, 1] = f[::97, 0]                                      # zero-area triangles
    f[1::89] = f[2::89][: len(f[1::89])]                         # duplicates
    f[3::71] = f[3::71][:, ::-1]
    m = 20_000
    o = (rng.normal(size=(m, 3)) * [2.5, 1.3, 0.7]).astype(np.float32)
    o[:500] = v[rng.integers(0, V, 500)]
    d = _unit(rng, m)
    d[500:700] = v[f[:200, 0]] - o[500:700]                      # aimed at vertices
    d[700:900] *= np.float32([1, 0, 1])                          # zero components
    occ = _occ(cuda, v, f)
    full = _hit(occ, o, d)
    _bitwise(full, H.first_hit(v, f, o, d))
    tm = (rng.random(m) * 3.0).astype(np.float32)
    tm[:100] = full[0][:100]                 # a cut at the hit's fp32 t: the fp64 comparison keeps or drops it
    _bitwise(_hit(occ, o, d, tm), H.first_hit(v, f, o, d, tm))
    _bitwise(_hit(occ, o, d, 0.75), H.first_hit(v, f, o, d, np.float32(0.75)))
    one = _occ(cuda, v, f[:1])
    _bitwise(_hit(one, o, d), H.first_hit(v, f[:1], o, d))
    none = _occ(cuda, v, np.zeros((0, 3), np.int32))
    t, x, n, tri = _hit(none, o[:9], d[:9])
    assert np.all(np.isinf(t)) and np.isnan(x).all() and np.isnan(n).all() and np.all(tri == -1)
    t, x, n, tri = _hit(occ, o[:0], d[:0])
    assert t.shape == (0,) and x.shape == (0, 3) and n.shape == (0, 3) and tri.shape == (0,)


def test_rejections(cuda):
    from nksr_b200._lib import NksrError
    v, f = icosphere(1)
    occ = _occ(cuda, v, f)
    z = torch.zeros((4, 3), device=cuda)
    one = torch.ones((4, 3), device=cuda)
    with pytest.raises(NksrError):
        occ.intersect(torch.zeros((4, 3)), one)
    with pytest.raises(NksrError):
        occ.intersect(torch.full((4, 3), math.nan, device=cuda), one)
    with pytest.raises(NksrError):
        occ.intersect(z, torch.full((4, 3), math.inf, device=cuda))
    with pytest.raises(ValueError):
        occ.intersect(z, z)
    with pytest.raises(ValueError):
        occ.intersect(z, one[:3])
    with pytest.raises(ValueError):
        occ.intersect(z, one, math.nan)
    with pytest.raises(ValueError):
        occ.intersect(z, one, torch.ones(3, device=cuda))


@pytest.mark.parametrize("mesh", ["icosphere3", "icosphere6", "room"])
def test_rays_from_inside_never_miss(cuda, mesh):
    rng = np.random.default_rng(4)
    n = 200_000
    if mesh == "room":
        v, f = room_mesh()
        p = (rng.random((3 * n, 3)) * [4.0, 4.0, 2.5] + [-2.0, -2.0, 0.0]).astype(np.float32)
        o = p[in_room_air(p, 1e-3)][:n]
    else:
        v, f = icosphere(3 if mesh == "icosphere3" else 6, 0.5)
        o = _unit(rng, n) * (rng.random((n, 1)) * 0.999 * inscribed_radius(v, f)).astype(np.float32)
    d = _unit(rng, o.shape[0])
    d[: o.shape[0] // 10] = np.eye(3, dtype=np.float32)[rng.integers(0, 3, o.shape[0] // 10)]
    occ = _occ(cuda, v, f)
    t, x, nrm, tri = _hit(occ, o, d)
    assert np.all(tri >= 0) and np.all(np.isfinite(t)) and np.all(t > 0)
    sub = rng.choice(o.shape[0], 300, replace=False)
    _bitwise((t[sub], x[sub], nrm[sub], tri[sub]), H.first_hit(v, f, o[sub], d[sub]))


def test_large_icosphere_subsample(cuda):
    v, f = icosphere(8)
    assert f.shape[0] > 1_000_000
    rng = np.random.default_rng(5)
    m = 1_000_000
    o = np.concatenate([_unit(rng, m // 2) * (rng.random((m // 2, 1)) * 0.99).astype(np.float32),
                        _unit(rng, m // 2) * (1.05 + rng.random((m // 2, 1))).astype(np.float32)])
    d = np.concatenate([_unit(rng, m // 2), -o[m // 2:] / np.linalg.norm(o[m // 2:], axis=1, keepdims=True)
                        + (0.3 * rng.normal(size=(m // 2, 3))).astype(np.float32)]).astype(np.float32)
    occ = _occ(cuda, v, f)
    t, x, n, tri = _hit(occ, o, d)
    hit = tri >= 0
    assert np.all(hit[: m // 2])
    r = np.linalg.norm(x[hit].astype(np.float64), axis=1)
    assert np.all((r > inscribed_radius(v, f) - 1e-5) & (r < 1.0 + 1e-5))
    assert np.all((n[hit] * x[hit]).sum(1) > 0)                  # outward winding: outward normals
    sub = rng.choice(m, 24, replace=False)
    _bitwise((t[sub], x[sub], n[sub], tri[sub]), H.first_hit(v, f, o[sub], d[sub]))


def _room_scan(cuda, noise=0.0, gen=None):
    from nksr_b200.gt_geometry import lidar_directions, scan_mesh
    v, f = room_mesh()
    occ = _occ(cuda, v, f)
    dirs = lidar_directions(64, 1024, (-45.0, 45.0))
    return v, f, occ, scan_mesh(occ, torch.from_numpy(ROOM_POSES).to(cuda), dirs, range_noise=noise, generator=gen)


def test_room_scan_lies_on_the_mesh(cuda):
    v, f, occ, scan = _room_scan(cuda)
    xyz, sensor, normal, tri = scan
    P, R = ROOM_POSES.shape[0], 64 * 1024
    assert xyz.shape[0] == P * R                                 # a closed room: every ray returns
    assert tri.dtype == torch.int64 and bool((tri >= 0).all())
    assert torch.equal(sensor, torch.from_numpy(ROOM_POSES).to(cuda).repeat_interleave(R, 0))
    # the hit point's own rounding (section 4.7: within 2^-18 (M + |o|) of the triangle) plus S21's error
    M = float(np.abs(v).max())
    S = max(M, float(xyz.abs().max()))
    a, b, c = (v[f[:, k]].astype(np.float64) for k in range(3))
    h = np.linalg.norm(np.cross(b - a, c - a), axis=1) / np.max(
        [np.linalg.norm(b - a, axis=1), np.linalg.norm(c - a, axis=1), np.linalg.norm(c - b, axis=1)], axis=0)
    bound = 2.0 ** -18 * (M + float(np.abs(ROOM_POSES).max())) + 2.0 ** -20 * S + 2.0 ** -21 * S * S / h.min()
    dist, _, ctri = occ.closest(xyz)
    assert float(dist.max()) <= bound
    from tests.occupancy_oracle import lex_sorted
    fs = lex_sorted(v, f)[tri.cpu().numpy()]
    d2, _, _ = D.closest_on_triangle(v[fs[:, 0]], v[fs[:, 1]], v[fs[:, 2]], xyz.cpu().numpy())
    assert float(np.sqrt(d2).max()) <= bound                     # the reported triangle is the one it lies on
    print(f"[scan] {xyz.shape[0]} points, closest triangle = hit triangle for "
          f"{float((ctri == tri).double().mean()):.6f}")
    want = torch.from_numpy(H.triangle_normals(v, f)).to(cuda)[tri]
    assert torch.equal(normal, want)
    # into the air: every normal faces its sensor
    assert bool(((sensor - xyz) * normal).sum(1).gt(0).all())
    # reproducible, and nothing is drawn without noise
    g = torch.Generator(device=cuda).manual_seed(7)
    state = g.get_state()
    again = _room_scan(cuda, 0.0, g)[3]
    assert torch.equal(g.get_state(), state)
    for a1, a2 in zip(scan, again):
        assert torch.equal(a1, a2)
    noisy = _room_scan(cuda, 0.01, g)[3]
    assert not torch.equal(g.get_state(), state)
    moved = noisy.xyz - xyz
    u = (xyz - sensor) / (xyz - sensor).norm(dim=1, keepdim=True)
    assert float(torch.linalg.cross(moved, u, dim=1).norm(dim=1).max()) < 1e-5      # along the ray
    assert 0.0099 < float((moved * u).sum(1).std()) < 0.0101 and torch.equal(noisy.tri, tri)
    # max_range keeps the hits with t <= max_range, in ray order
    from nksr_b200.gt_geometry import lidar_directions, scan_mesh
    near = scan_mesh(occ, ROOM_POSES, lidar_directions(64, 1024, (-45.0, 45.0)), max_range=2.0)
    keep = (xyz - sensor).norm(dim=1) <= 2.0 + 1e-5
    assert abs(near.xyz.shape[0] - int(keep.sum())) <= 0.001 * xyz.shape[0]
    assert float((near.xyz - near.sensor).norm(dim=1).max()) <= 2.0 + 1e-5


def test_room_scan_against_the_volume_builder(cuda):
    """S19 from the scan: free space is carved only between a sensor and its first hit, so every node the volume calls
    empty (class 1) lies within sqrt(3) h of air; one more than 2 h from the mesh is therefore in the air itself --
    outside the solid by ray parity.  The sign agreement at the near-surface nodes is reported, not asserted."""
    from nksr_b200.gt_geometry import MeshGroundTruth, PointTSDFVolume
    v, f, occ, scan = _room_scan(cuda)
    h = 0.05
    vol = PointTSDFVolume.from_sensor_rays(scan.xyz, scan.normal, scan.sensor, h=h, tau=2 * h, margin=2 * h)
    dims = vol.volume.shape
    axes = [torch.tensor(vol.volume_min[a] + np.arange(dims[a]) * h, dtype=torch.float32, device=cuda)
            for a in range(3)]
    nodes = torch.stack(torch.meshgrid(*axes, indexing="ij"), dim=-1).reshape(-1, 3)
    cls = vol.query_classification(nodes)
    dist, inside = occ.distance_and_inside(nodes, 3)
    far_free = (cls == 1) & (dist > 2 * h)
    assert int(far_free.sum()) > 10_000
    assert not bool(inside[far_free].any())
    assert bool(torch.from_numpy(in_room_air(nodes[far_free].cpu().numpy())).all())
    near = cls == 0
    gt = MeshGroundTruth(torch.from_numpy(v).to(cuda), torch.from_numpy(f).to(cuda), tau=2 * h)
    agree = (torch.sign(vol.query_sdf(nodes[near])) == torch.sign(gt.query_sdf(nodes[near]))).double().mean()
    print(f"[scan] S19 near-surface nodes {int(near.sum())}: sign agrees with the mesh at {float(agree):.4f}")


def test_room_scan_end_to_end(cuda):
    import nksr_b200
    from nksr_b200 import _lib
    from nksr_b200 import training as T
    from nksr_b200.gt_geometry import MeshGroundTruth
    from nksr_b200.metrics import MeshEvaluator, sample_surface
    from nksr_b200.network import NKSRNetwork
    from nksr_b200.reconstructor import estimate_normals_knn
    v, f, occ, scan = _room_scan(cuda)
    W = 0.05
    rec = nksr_b200.Reconstructor(cuda)
    field = rec.reconstruct(scan.xyz, sensor=scan.sensor, voxel_size=W,
                            preprocess_fn=nksr_b200.get_estimate_normal_preprocess_fn(64, 85.0))
    mesh = field.extract_dual_mesh(mise_iter=1)
    assert mesh.f.shape[0] > 1000 and bool(torch.isfinite(mesh.v).all())
    tv, tf = torch.from_numpy(v).to(cuda), torch.from_numpy(f).to(cuda)
    gx, gn, _ = sample_surface(tv, tf, 200_000, seed=0)
    out = MeshEvaluator(n_points=100_000).eval_mesh(mesh, gx, gn)
    assert all(math.isfinite(x) for x in out.values())
    print(f"[scan] room reconstruction: chamfer-L1 {out['chamfer-L1']:.4f}, f-score {out['f-score']:.4f}")
    r = estimate_normals_knn(scan.xyz, scan.sensor, 64, 85.0)
    s = _lib.exclusive_scan32(r.keep)
    cnt = int(s[-1].item())
    px, pn = (_lib.compact_rows(a, r.keep, s, cnt) for a in (r.xyz, r.normal))
    gt = MeshGroundTruth(tv, tf, tau=2 * W)
    scene = T.TrainingScene(px, pn, W, 4, gt=gt)
    net = NKSRNetwork(dict(backbone="unet", tree_depth=4, kernel_dim=4, trainable=True, seed=3)).to(cuda)
    opt = T.make_optimizer(net)
    gen = torch.Generator(device=cuda).manual_seed(3)
    for _ in range(5):
        l_struct, l_udf, k = T.train_step(net, opt, scene, gen, kernel=True)
        assert math.isfinite(float(l_struct)) and math.isfinite(float(l_udf))
        assert all(math.isfinite(float(x)) for x in k.values())
        grads = [p.grad for p in net.parameters() if p.grad is not None]
        assert grads and all(bool(torch.isfinite(g).all()) for g in grads)
