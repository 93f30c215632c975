"""numpy restatement of SPEC S22 (DESIGN.md), the first hit of a ray behind MeshOccupancy.intersect: every triangle for
every ray.  The candidates are S20's crossings, with the frame, the lexicographic vertex order and the edge ownership
taken from tests/occupancy_oracle.py; each candidate's t = T / det is one fp64 division, and the output is rounded as
csrc/raycast.cu rounds it (numpy rounds every float32 and float64 operation on its own, with no fused multiply-add).
The GPU result (an LBVH traversal) is held to it bit for bit."""
import numpy as np

from tests.distance_oracle import _cross, _dot
from tests.occupancy_oracle import _owns, lex_sorted, ray_frame

F32 = np.float32


def _candidate_t(vu, f, o, kx, ky, kz, sx, sy, sz):
    """fp64 t (c, T) of every triangle for rays from o (c, 3) sharing the axes (kx, ky, kz), with per-ray shears
    sx, sy, sz (c,) fp32; NaN where S20 counts no crossing"""
    a = vu[None] - o[:, None, :]                                   # fp32 (c, V, 3): vertex - origin
    az = a[..., kz]
    Xv = a[..., kx] - sx[:, None] * az                             # fp32: rounded product, rounded difference
    Yv = a[..., ky] - sy[:, None] * az
    Zv = sz[:, None] * az
    X, Y, Z = Xv[:, f], Yv[:, f], Zv[:, f]                         # (c, T, 3)
    Xd, Yd = X.astype(np.float64), Y.astype(np.float64)
    U = Xd[..., 2] * Yd[..., 1] - Yd[..., 2] * Xd[..., 1]
    V = Xd[..., 0] * Yd[..., 2] - Yd[..., 0] * Xd[..., 2]
    W = Xd[..., 1] * Yd[..., 0] - Yd[..., 1] * Xd[..., 0]
    mixed = ((U < 0) | (V < 0) | (W < 0)) & ((U > 0) | (V > 0) | (W > 0))
    det = U + V + W
    pos = det > 0
    hit = ~mixed & (det != 0)
    hit &= (U != 0) | _owns(X[..., 1], Y[..., 1], X[..., 2], Y[..., 2], pos)
    hit &= (V != 0) | _owns(X[..., 2], Y[..., 2], X[..., 0], Y[..., 0], pos)
    hit &= (W != 0) | _owns(X[..., 0], Y[..., 0], X[..., 1], Y[..., 1], pos)
    Zd = Z.astype(np.float64)
    T = U * Zd[..., 0] + V * Zd[..., 1] + W * Zd[..., 2]
    hit &= np.where(pos, T > 0, T < 0)
    with np.errstate(all="ignore"):
        return np.where(hit, T / det, np.nan)


def triangle_normals(v, f):
    """fp32 unit normals (v1 - v0) x (v2 - v0) / |.| in the given winding; NaN for a zero cross product"""
    v = np.asarray(v, F32).reshape(-1, 3)
    f = np.asarray(f, np.int64).reshape(-1, 3)
    with np.errstate(all="ignore"):
        n = _cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
        return n / np.sqrt(_dot(n, n))[:, None]


def first_hit(v, f, o, d, t_max=np.inf, chunk_elems=1 << 21):
    """S22 brute force: (t fp32 (m,), point fp32 (m, 3), normal fp32 (m, 3), triangle int64 (m,)) of the rays from
    o along d over every triangle of (v, f): the candidate with the smallest fp64 t in (0, t_max], ties to the lower
    index; a miss gives inf, NaN, NaN, -1"""
    v = np.asarray(v, F32).reshape(-1, 3)
    o = np.asarray(o, F32).reshape(-1, 3)
    d = np.asarray(d, F32).reshape(-1, 3)
    m = o.shape[0]
    tmax = np.broadcast_to(np.asarray(t_max, F32).astype(np.float64), (m,))
    f0 = np.asarray(f, np.int64).reshape(-1, 3)
    t_out = np.full(m, np.inf, F32)
    point = np.full((m, 3), np.nan, F32)
    normal = np.full((m, 3), np.nan, F32)
    tri = np.full(m, -1, np.int64)
    if f0.shape[0] == 0 or m == 0:
        return t_out, point, normal, tri
    used, fs = np.unique(lex_sorted(v, f0), return_inverse=True)
    fs = fs.reshape(-1, 3)
    vu = v[used]
    frames = [ray_frame(x) for x in d]
    axes = np.array([fr[:3] for fr in frames], np.int64)
    shear = np.array([fr[3:] for fr in frames], F32)
    best = np.full(m, np.inf)
    step = max(1, chunk_elems // fs.shape[0])
    for key in np.unique(axes, axis=0):
        rays = np.nonzero((axes == key).all(axis=1))[0]
        for s in range(0, rays.shape[0], step):
            r = rays[s:s + step]
            t = _candidate_t(vu, fs, o[r], *key, shear[r, 0], shear[r, 1], shear[r, 2])
            cand = (t > 0) & (t <= tmax[r, None])
            key_t = np.where(cand, t, np.inf)
            j = np.argmin(key_t, axis=1)                           # the first minimum: the lower index on ties
            rows = np.arange(r.shape[0])
            # every candidate at t = inf (an overflow): the first candidate, as the kernel's tie rule gives
            j = np.where(cand.any(axis=1) & np.isinf(key_t[rows, j]), np.argmax(cand, axis=1), j)
            found = cand[rows, j]
            best[r] = np.where(found, t[rows, j], np.inf)
            tri[r] = np.where(found, j, -1)
    hit = tri >= 0
    t_out[hit] = best[hit].astype(F32)
    point[hit] = o[hit] + t_out[hit, None] * d[hit]
    normal[hit] = triangle_normals(v, f0[tri[hit]])
    return t_out, point, normal, tri
