"""SPEC S21, the fp32 closest point of a triangle (tests/distance_oracle.py, which csrc/raycast.cu restates), on the
CPU: its error against an independent fp64 distance on random, sliver and degenerate triangles over all seven Voronoi
regions, its invariance under vertex rotation and winding, and the tie rule of the mesh query."""
import numpy as np

from tests import distance_oracle as D
from tests.test_cpu_occupancy import icosphere


def _lex(a, b, c):
    t = np.stack([a, b, c], 1)
    order = np.lexsort((t[..., 2], t[..., 1], t[..., 0]), axis=1)
    t = np.take_along_axis(t, order[..., None], 1)
    return t[:, 0], t[:, 1], t[:, 2]


U = 2.0 ** -24


def _check_bound(a, b, c, p, sliver=False):
    """SPEC S21's accuracy bound against the independent fp64 distance: |d32 - d64| <= 2^-20 S, S the largest
    |coordinate| of the triangle and the query; for slivers and needles plus min(h, 2^-21 S^2 / h), h the triangle's
    smallest height (2 area / longest edge, in fp64).  Returns the fp64 regions and the largest error in units of
    2^-24 S."""
    a, b, c = _lex(*(np.asarray(z, np.float32) for z in (a, b, c)))
    p = np.asarray(p, np.float32)
    d2, x, _ = D.closest_on_triangle(a, b, c, p)
    d32 = np.sqrt(d2).astype(np.float64)
    d64, region = D.exact_closest(a, b, c, p)
    assert np.all(np.isfinite(d32)) and np.all(np.isfinite(x))
    s = np.max(np.abs(np.concatenate([a, b, c, p], axis=1)), axis=1).astype(np.float64)
    bound = 2.0 ** -20 * s
    if sliver:
        a64, b64, c64 = (z.astype(np.float64) for z in (a, b, c))
        area2 = np.linalg.norm(np.cross(b64 - a64, c64 - a64), axis=1)
        longest = np.max([np.linalg.norm(b64 - a64, axis=1), np.linalg.norm(c64 - a64, axis=1),
                          np.linalg.norm(c64 - b64, axis=1)], axis=0)
        h = area2 / longest                                  # 0 where rounding to fp32 made the sliver a segment
        with np.errstate(divide="ignore"):
            bound = bound + np.where(h > 0, np.minimum(h, 2.0 ** -21 * s * s / h), 0.0)
    err = np.abs(d32 - d64)
    assert np.all(err <= bound), float(np.max(err / bound))
    # the point is the one whose distance is reported
    assert np.array_equal(np.sqrt(D.closest_on_triangle(x, x, x, p)[0]), np.sqrt(d2))
    return region, float(np.max(err / (U * s)))


def test_error_bound_and_all_seven_regions():
    rng = np.random.default_rng(0)
    n = 60_000
    a, b, c = rng.normal(size=(3, n, 3))
    w = rng.random((n, 3))
    w /= w.sum(1, keepdims=True)
    on = lambda c2: w[:, :1] * a + w[:, 1:2] * b + w[:, 2:] * c2
    seen, worst = np.zeros(7, np.int64), 0.0
    # well-shaped triangles: far queries, and queries within 1e-4 of the face
    for q in (rng.normal(size=(n, 3)) * 1.5, on(c) + 1e-4 * rng.normal(size=(n, 3))):
        region, e = _check_bound(a, b, c, q)
        seen += np.bincount(region, minlength=7)
        worst = max(worst, e)
    # degenerate: two coincident vertices, a segment with its midpoint, a point -- no face region, no h term
    p = rng.normal(size=(n, 3)) * 1.5
    for deg in ((a, b, a.copy()), (a, b, ((a + b) / 2).astype(np.float32)), (a, a.copy(), a.copy())):
        region, e = _check_bound(*deg, p)
        assert not np.any(region == 0)
        worst = max(worst, e)
    print(f"[distance] well-shaped and degenerate: largest error {worst:.2f} x 2^-24 S")
    # slivers (c within 1e-7 .. 1e-2 of the line ab) and needles (c within that of b): far, near and on the face
    s = 10.0 ** rng.uniform(-7, -2, (n, 1))
    sliver = a + rng.random((n, 1)) * (b - a) + s * rng.normal(size=(n, 3))
    needle = b + s * rng.normal(size=(n, 3))
    for c2 in (sliver, needle):
        for q in (rng.normal(size=(n, 3)) * 1.5, on(c2) + 1e-4 * rng.normal(size=(n, 3)), on(c2)):
            seen += np.bincount(_check_bound(a, b, c2, q, sliver=True)[0], minlength=7)
    assert np.all(seen > 100), seen


def test_exact_on_axis_aligned_cases():
    """distances that are exact in fp32: the face (at asymmetric barycentrics, so swapped weights fail), an edge and
    a vertex of the unit right triangle"""
    a, b, c = np.float32([[0, 0, 0]]), np.float32([[0, 1, 0]]), np.float32([[1, 0, 0]])
    p = np.float32([[0.25, 0.5, 2.0], [0.125, 0.75, -0.5], [0.5, -3.0, 0.0], [-1.0, -1.0, 0.0], [2.0, 0.0, 0.0]])
    d2, x, region = D.closest_on_triangle(a, b, c, p)
    assert np.array_equal(np.sqrt(d2), np.float32([2.0, 0.5, 3.0, np.sqrt(np.float32(2.0)), 1.0]))
    assert np.array_equal(x, np.float32([[0.25, 0.5, 0], [0.125, 0.75, 0], [0.5, 0, 0], [0, 0, 0], [1, 0, 0]]))
    assert np.array_equal(region, [0, 0, 2, 1, 2])
    d64, r64 = D.exact_closest(a, b, c, p)
    assert np.array_equal(d64, [2.0, 0.5, 3.0, np.sqrt(2.0), 1.0]) and np.array_equal(r64, [0, 0, 2, 4, 6])


def test_rotation_and_winding_do_not_change_a_bit():
    rng = np.random.default_rng(1)
    v = (rng.normal(size=(300, 3)) * [2.0, 1.0, 0.5]).astype(np.float32)
    f = rng.integers(0, 300, size=(500, 3)).astype(np.int32)
    f[::37, 2] = f[::37, 0]                                   # zero-area triangles
    q = (rng.normal(size=(3000, 3)) * 2.0).astype(np.float32)
    q[:100] = v[rng.integers(0, 300, 100)]
    want = D.mesh_closest(v, f, q)
    for perm in ((1, 2, 0), (2, 0, 1), (0, 2, 1), (2, 1, 0), (1, 0, 2)):
        got = D.mesh_closest(v, f[:, perm], q)
        for g, w in zip(got, want):
            assert np.array_equal(g.view(np.uint32) if g.dtype == np.float32 else g,
                                  w.view(np.uint32) if w.dtype == np.float32 else w), perm


def test_ties_go_to_the_lower_index():
    rng = np.random.default_rng(2)
    v = rng.normal(size=(60, 3)).astype(np.float32)
    f = rng.integers(0, 60, size=(40, 3)).astype(np.int32)
    dup = np.concatenate([f, f[:, ::-1], np.roll(f, 1, axis=1)])  # every triangle three times, rotated and flipped
    q = rng.normal(size=(2000, 3)).astype(np.float32)
    d, x, t = D.mesh_closest(v, f, q)
    d2, x2, t2 = D.mesh_closest(v, dup, q)
    assert np.array_equal(d, d2) and np.array_equal(x, x2) and np.array_equal(t, t2)
    assert t.max() < 40
    # a query equidistant from two mirrored triangles
    v = np.float32([[0, 0, 1], [1, 0, 1], [0, 1, 1], [0, 0, -1], [1, 0, -1], [0, 1, -1]])
    for f in (np.int32([[3, 4, 5], [0, 1, 2]]), np.int32([[0, 1, 2], [3, 4, 5]])):
        _, _, t = D.mesh_closest(v, f, np.float32([[0.2, 0.2, 0.0]]))
        assert t[0] == 0


def test_icosphere_against_the_radius_and_empty_meshes():
    v, f = icosphere(3, 0.5)
    rng = np.random.default_rng(3)
    q = (rng.normal(size=(500, 3)) * 0.6).astype(np.float32)
    d, x, t = D.mesh_closest(v, f, q)
    r = np.linalg.norm(q.astype(np.float64), axis=1)
    # the polygon lies between the inscribed and circumscribed spheres, so d is within their gap of |r - R|
    from tests.test_cpu_occupancy import inscribed_radius
    gap = 0.5 - inscribed_radius(v, f)
    assert np.all(np.abs(d - np.abs(r - 0.5)) <= gap + 1e-6)
    assert np.all((t >= 0) & (t < f.shape[0]))
    d, x, t = D.mesh_closest(v, np.zeros((0, 3), np.int32), q[:5])
    assert np.all(np.isinf(d)) and np.all(np.isnan(x)) and np.all(t == -1)
