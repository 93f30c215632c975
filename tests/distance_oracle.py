"""numpy restatement of SPEC S21 (DESIGN.md), the closest point of a triangle mesh behind MeshOccupancy.closest: every
triangle for every query, with each fp32 operation of csrc/raycast.cu written out in the same order (numpy rounds
every float32 product, sum, division and square root on its own).  The GPU result (an LBVH traversal) is held to it bit
for bit.  `exact_closest`, the yardstick for the fp32 routine's error, computes the distance in fp64 by a different
formulation (the plane's normal equations and clamped edge projections), so an error in S21's algebra shows up."""
import numpy as np

from tests.occupancy_oracle import lex_sorted

F32 = np.float32


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], axis=-1)


def _segment(P, Q, p, best, x):
    """candidate on (P, Q): P when e.(p - P) <= 0, Q when it reaches e.e, else P + t e; replaces where strictly
    closer"""
    e, ap = Q - P, p - P
    num, den = _dot(e, ap), _dot(e, e)
    t = num / den
    c = P + t[..., None] * e
    c = np.where((num >= den)[..., None], Q, c)
    c = np.where((~(num > 0))[..., None], P, c)
    d = p - c
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    better = d2 < best
    return np.where(better, d2, best), np.where(better[..., None], c, x), better


def closest_on_triangle(a, b, c, p, dtype=F32):
    """S21 for vertices a <= b <= c (lexicographic) and query p, broadcast over leading axes: (d2, point, region) with
    region 0 the face, 1 / 2 / 3 the segments ab / ac / bc (the candidate that won, vertices included).  With
    dtype=np.float64 the same steps in fp64."""
    a, b, c, p = (np.asarray(z, dtype) for z in (a, b, c, p))
    a, b, c, p = np.broadcast_arrays(a, b, c, p)
    with np.errstate(all="ignore"):
        ab, ac, ap, bp, cp = b - a, c - a, p - a, p - b, p - c
        n = _cross(ab, ac)
        va, vb, vc = _dot(n, _cross(bp, cp)), _dot(n, _cross(cp, ap)), _dot(n, _cross(ap, bp))
        den = (va + vb) + vc
        face = (va >= 0) & (vb >= 0) & (vc >= 0) & (den > 0) & np.isfinite(den)
        v, w = vb / den, vc / den
        x = (a + v[..., None] * ab) + w[..., None] * ac
        d = p - x
        best = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
        best = np.where(face, best, np.array(np.inf, dtype))
        x = np.where(face[..., None], x, np.array(np.nan, dtype))
        region = np.zeros(best.shape, np.int64)
        for r, (P, Q) in enumerate(((a, b), (a, c), (b, c)), start=1):
            best, x, better = _segment(P, Q, p, best, x)
            region[better] = r
    return best, x, region


def mesh_closest(v, f, q, chunk_elems=1 << 21):
    """S21 brute force: (distance fp32 (m,), point fp32 (m, 3), triangle int64 (m,)) over every triangle of (v, f);
    the lowest d2 wins, ties to the lower triangle index; no triangles: inf, NaN, -1"""
    v = np.asarray(v, F32).reshape(-1, 3)
    q = np.asarray(q, F32).reshape(-1, 3)
    f = lex_sorted(v, f)
    m, t = q.shape[0], f.shape[0]
    dist = np.full(m, np.inf, F32)
    point = np.full((m, 3), np.nan, F32)
    tri = np.full(m, -1, np.int64)
    if t == 0:
        return dist, point, tri
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    step = max(1, chunk_elems // t)
    for s in range(0, m, step):
        p = q[s:s + step, None, :]
        d2, x, _ = closest_on_triangle(a[None], b[None], c[None], p)
        j = np.argmin(d2, axis=1)                          # the first minimum: the lower index on ties
        rows = np.arange(d2.shape[0])
        dist[s:s + step] = np.sqrt(d2[rows, j])
        point[s:s + step] = x[rows, j]
        tri[s:s + step] = j
    return dist, point, tri


def exact_closest(a, b, c, p):
    """fp64 distance from p to triangle (a, b, c) and the Voronoi region of the closest point (0 face, 1 / 2 / 3 the
    open edges ab / ac / bc, 4 / 5 / 6 the vertices a / b / c), by a formulation independent of S21's: the face point
    solves the 2 x 2 normal equations of the plane parametrisation a + s ab + t ac (Cramer's rule), each edge is the
    clamped parametric projection, and the nearest of these wins.  A triangle without area has no face region."""
    a, b, c, p = (np.asarray(z, np.float64) for z in (a, b, c, p))
    a, b, c, p = np.broadcast_arrays(a, b, c, p)
    dot = lambda x, y: np.sum(x * y, axis=-1)
    ab, ac, ap = b - a, c - a, p - a
    g00, g01, g11, r0, r1 = dot(ab, ab), dot(ab, ac), dot(ac, ac), dot(ab, ap), dot(ac, ap)
    det = g00 * g11 - g01 * g01
    with np.errstate(all="ignore"):
        s = (g11 * r0 - g01 * r1) / det
        t = (g00 * r1 - g01 * r0) / det
        face = (det > 0) & (s >= 0) & (t >= 0) & (s + t <= 1)
        dist = np.where(face, np.linalg.norm(ap - s[..., None] * ab - t[..., None] * ac, axis=-1), np.inf)
    region = np.zeros(dist.shape, np.int64)
    for r, (P, Q, iP, iQ) in enumerate(((a, b, 4, 5), (a, c, 4, 6), (b, c, 5, 6)), start=1):
        e = Q - P
        ee = dot(e, e)
        with np.errstate(all="ignore"):
            u = np.where(ee > 0, np.clip(dot(p - P, e) / np.where(ee > 0, ee, 1.0), 0.0, 1.0), 0.0)
        d = np.linalg.norm(p - P - u[..., None] * e, axis=-1)
        better = d < dist
        dist = np.where(better, d, dist)
        region[better] = np.where(u[better] == 0, iP, np.where(u[better] == 1, iQ, r))
    return dist, region
