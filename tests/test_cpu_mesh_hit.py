"""SPEC S22, the first hit of a ray (tests/hit_oracle.py, which csrc/raycast.cu restates), on the CPU: hits exactly
where S20 counts crossings, analytic t on axis-aligned quads and a tilted plane, the t_max cut and the tie rule, and
the scanner pattern of gt_geometry.lidar_directions."""
import numpy as np

from tests import hit_oracle as H
from tests import occupancy_oracle as OO
from tests.test_cpu_occupancy import cube_union, icosphere


def test_hit_iff_the_ray_crosses():
    rng = np.random.default_rng(0)
    v, f = icosphere(2, 0.5)
    sv = rng.normal(size=(80, 3)).astype(np.float32)
    sf = rng.integers(0, 80, size=(150, 3)).astype(np.int32)
    sf[::13, 2] = sf[::13, 0]                                  # zero-area triangles
    cv, cf = cube_union(rng=rng)
    dirs = list(OO.DEFAULT_DIRECTIONS[:3]) + [np.float32([0, 0, 1]), np.float32([0.5, -1.0, 0]),
                                              np.float32([-0.125, 0.25, -1])]
    for vv, ff, q in ((v, f, rng.normal(size=(300, 3)).astype(np.float32) * 0.6),
                      (sv, sf, rng.normal(size=(300, 3)).astype(np.float32)),
                      (cv, cf, (rng.integers(-2, 8, size=(300, 3)) * 0.5).astype(np.float32))):
        for d in dirs:
            count = OO.ray_crossings(vv, ff, q, d)
            t, x, n, tri = H.first_hit(vv, ff, q, np.broadcast_to(d, q.shape))
            assert np.array_equal(tri >= 0, count > 0)
            assert np.all(t[tri >= 0] > 0) and np.all(np.isinf(t[tri < 0]))
            assert np.all(np.isfinite(x[tri >= 0])) and np.all(np.isnan(x[tri < 0]))


def _quad(axis, at, s=1.0):
    """the square |u|, |w| <= s in the plane x[axis] = at, two triangles wound counter-clockwise seen from +axis"""
    u, w = (axis + 1) % 3, (axis + 2) % 3
    v = np.zeros((4, 3), np.float32)
    for i, (a, b) in enumerate(((-s, -s), (s, -s), (s, s), (-s, s))):
        v[i, axis], v[i, u], v[i, w] = at, a, b
    return v, np.int32([[0, 1, 2], [0, 2, 3]])


def test_analytic_t_on_quads_and_a_tilted_plane():
    for axis in range(3):
        v, f = _quad(axis, 2.0)
        o = np.zeros((3, 3), np.float32)
        o[:, (axis + 1) % 3] = [0.25, -0.5, 0.0]
        d = np.zeros((3, 3), np.float32)
        d[:, axis] = [1.0, 0.5, -1.0]
        d[1, (axis + 2) % 3] = 0.125                          # an oblique ray with a zero component
        t, x, n, tri = H.first_hit(v, f, o, d)
        assert np.array_equal(t, np.float32([2.0, 4.0, np.inf]))
        assert np.array_equal(x[:2, axis], [2.0, 2.0]) and np.isnan(x[2]).all() and tri[2] == -1
        want_n = np.zeros(3, np.float32)
        want_n[axis] = 1.0
        assert np.array_equal(n[:2], [want_n, want_n])
        assert np.allclose(x[:2], o[:2] + t[:2, None] * d[:2], atol=0)
    # the plane x + z = 2 through a large triangle: its normal is (1, 0, 1) / sqrt(2)
    v = np.float32([[2, -8, 0], [-6, 8, 8], [10, 8, -8]])
    f = np.int32([[0, 2, 1]])
    o = np.zeros((4, 3), np.float32)
    d = np.float32([[0, 0, 1], [1, 0, 0], [1, 0, 1], [0.5, 0, 0.5]])
    t, x, n, tri = H.first_hit(v, f, o, d)
    assert np.array_equal(t, np.float32([2, 2, 1, 2])) and np.array_equal(tri, [0, 0, 0, 0])
    assert np.array_equal(x, np.float32([[0, 0, 2], [2, 0, 0], [1, 0, 1], [1, 0, 1]]))
    s = np.float32(1.0) / np.sqrt(np.float32(2.0))
    assert np.allclose(n, [[s, 0, s]] * 4, rtol=0, atol=1e-7)
    # the opposite winding flips the normal, and only the normal
    t2, x2, n2, tri2 = H.first_hit(v, f[:, ::-1], o, d)
    assert np.array_equal(t2, t) and np.array_equal(x2, x) and np.array_equal(n2, -n)


def test_t_max_ties_and_empty_mesh():
    v1, f1 = _quad(2, 1.0)
    v2, f2 = _quad(2, 3.0)
    v = np.concatenate([v2, v1, v1])                         # the far quad first, the near one twice
    f = np.concatenate([f2, f1 + 4, f1[:, ::-1] + 8])
    o = np.float32([[0.25, 0.5, 0.0]] * 4)
    d = np.float32([[0, 0, 1]] * 4)
    t, x, n, tri = H.first_hit(v, f, o, d, t_max=np.float32([np.inf, 1.0, 0.5, 2.0]))
    assert np.array_equal(t, np.float32([1.0, 1.0, np.inf, 1.0]))
    assert np.array_equal(tri, [3, 3, -1, 3])                  # the lower of the two equal hits (3 and 5)
    _, _, _, tri = H.first_hit(v, f, np.float32([[0.25, 0.5, 2.0]]), np.float32([[0, 0, 1]]))
    assert tri[0] == 1                                          # the near quad lies behind the origin
    t, x, n, tri = H.first_hit(v, np.zeros((0, 3), np.int32), o, d)
    assert np.all(np.isinf(t)) and np.isnan(x).all() and np.isnan(n).all() and np.all(tri == -1)


def test_lidar_directions():
    from nksr_b200.gt_geometry import lidar_directions
    d = lidar_directions(64, 1024).numpy()
    assert d.shape == (64 * 1024, 3) and d.dtype == np.float32
    assert np.all(np.abs(np.linalg.norm(d.astype(np.float64), axis=1) - 1.0) < 1e-6)
    el = np.rad2deg(np.arcsin(d[:, 2].astype(np.float64)))
    assert abs(el.min() + 24.8) < 1e-4 and abs(el.max() - 2.0) < 1e-4
    assert np.allclose(el[:64], np.linspace(-24.8, 2.0, 64), atol=1e-4)      # the beams of the first azimuth step
    az = np.rad2deg(np.arctan2(d[::64, 1], d[::64, 0]).astype(np.float64)) % 360.0
    assert np.allclose(az, (np.arange(1024) + 0.5) * 360.0 / 1024, atol=1e-4)
    one = lidar_directions(1, 4, (10.0, 10.0)).numpy()
    assert one.shape == (4, 3) and np.allclose(np.rad2deg(np.arcsin(one[:, 2])), 10.0, atol=1e-5)
