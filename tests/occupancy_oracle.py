"""numpy restatement of SPEC S20 (DESIGN.md), the ray-parity mesh occupancy behind the evaluator's 'o3d-iou': every
triangle for every query, vectorised over triangles, with the fp32 and fp64 roundings of csrc/raycast.cu written out.
The GPU result (an LBVH traversal) is held to it bit for bit.  OracleOccupancyEvaluator is oracle/metrics.py's
evaluator with the same `occupancy_rays` opt-in as nksr_b200.metrics.MeshEvaluator."""
import numpy as np

from oracle import metrics as OM

# SPEC S20's built-in ray directions (fp32), the first K of which vote; csrc/raycast.cu holds the same constants
MAX_RAYS = 9
DEFAULT_DIRECTIONS = np.array([[float.fromhex(x) for x in row] for row in (
    ("-0x1.8815a2p-3", "0x1.480a34p-1", "0x1.7cb0ecp-1"),
    ("0x1.c613e2p-2", "0x1.286306p-1", "-0x1.5e5c32p-1"),
    ("-0x1.3433a6p-2", "-0x1.42e6aap-3", "-0x1.e18a22p-1"),
    ("0x1.2ed1f8p-1", "-0x1.69843ep-1", "-0x1.8ebf20p-2"),
    ("-0x1.9f3f84p-1", "0x1.c1902cp-3", "0x1.15a29ep-1"),
    ("0x1.ac4238p-2", "-0x1.62a6b6p-1", "-0x1.2cdb7cp-1"),
    ("-0x1.b7da02p-1", "0x1.3c78c4p-3", "0x1.f3a8dap-2"),
    ("0x1.3037d2p-2", "-0x1.35be2ep-1", "0x1.7a3dacp-1"),
    ("-0x1.1448b4p-1", "-0x1.78b382p-1", "-0x1.a314ecp-2"),
)], dtype=np.float32)


def check_rays(k) -> int:
    k = int(k)
    if k < 1 or k > MAX_RAYS or k % 2 == 0:
        raise ValueError(f"the number of rays must be odd and in [1, {MAX_RAYS}], got {k}")
    return k


def ray_frame(d):
    """(kx, ky, kz, Sx, Sy, Sz) of direction d: kz = the first index of max |d|, kx, ky the next two cyclically,
    swapped when d[kz] < 0; the shears are correctly rounded fp32 divisions"""
    d = np.asarray(d, dtype=np.float32)
    kz = int(np.argmax(np.abs(d)))
    kx, ky = (kz + 1) % 3, (kz + 2) % 3
    if d[kz] < 0:
        kx, ky = ky, kx
    return kx, ky, kz, d[kx] / d[kz], d[ky] / d[kz], np.float32(1.0) / d[kz]


def _owns(px, py, qx, qy, pos):
    """edge (P, Q) owns a zero edge function: its inward normal s (Qy - Py, Px - Qx) points to +x, or along +y"""
    a = (qy > py) | ((qy == py) & (px > qx))
    b = (qy < py) | ((qy == py) & (px < qx))
    return np.where(pos, a, b)


def lex_sorted(v, f):
    """every triangle's vertex indices with the vertices in lexicographic (x, y, z) order, by the kernel's three
    compare-and-swaps"""
    f = np.array(f, dtype=np.int64).reshape(-1, 3)

    def less(a, b):
        return (a[:, 0] < b[:, 0]) | ((a[:, 0] == b[:, 0]) & ((a[:, 1] < b[:, 1]) |
                                                              ((a[:, 1] == b[:, 1]) & (a[:, 2] < b[:, 2]))))

    for i, j in ((0, 1), (1, 2), (0, 1)):
        sw = less(v[f[:, j]], v[f[:, i]])
        f[sw, i], f[sw, j] = f[sw, j], f[sw, i]
    return f


def ray_crossings(v, f, q, d):
    """int (m,): how many triangles of (v, f) the ray from each query along d crosses (SPEC S20, brute force)"""
    v = np.asarray(v, dtype=np.float32).reshape(-1, 3)
    q = np.asarray(q, dtype=np.float32).reshape(-1, 3)
    f = lex_sorted(v, f)
    kx, ky, kz, sx, sy, sz = ray_frame(d)
    out = np.zeros(q.shape[0], dtype=np.int64)
    if f.shape[0] == 0:
        return out
    used, f = np.unique(f, return_inverse=True)
    f = f.reshape(-1, 3)
    vu = v[used]
    chunk = max(1, (1 << 20) // f.shape[0])
    for s in range(0, q.shape[0], chunk):
        a = vu[None] - q[s:s + chunk, None, :]                     # fp32 (c, V, 3): vertex - query
        az = a[..., kz]
        Xv = a[..., kx] - sx * az                                  # fp32: rounded product, rounded difference
        Yv = a[..., ky] - sy * az
        Zv = sz * az
        X, Y, Z = Xv[:, f], Yv[:, f], Zv[:, f]                     # (c, T, 3)
        Xd, Yd = X.astype(np.float64), Y.astype(np.float64)
        U = Xd[..., 2] * Yd[..., 1] - Yd[..., 2] * Xd[..., 1]      # exact products, one rounded difference
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
        T = U * Zd[..., 0] + V * Zd[..., 1] + W * Zd[..., 2]      # left to right, every step rounded
        hit &= np.where(pos, T > 0, T < 0)
        out[s:s + chunk] = hit.sum(axis=1)
    return out


def occupancy(v, f, q, directions=None, n_rays=3):
    """bool (m,): more than K/2 of the K rays cross the mesh an odd number of times; the directions default to the
    first n_rays of DEFAULT_DIRECTIONS"""
    dirs = DEFAULT_DIRECTIONS[:check_rays(n_rays)] if directions is None else np.asarray(directions, np.float32)
    check_rays(dirs.shape[0])
    votes = sum((ray_crossings(v, f, q, d) & 1) for d in dirs)
    return 2 * np.asarray(votes) > dirs.shape[0]


def occupancy_iou(pred, gt):
    """the reference's IoU: integer counts, fp64 division, + 1e-6 in the denominator"""
    pred, gt = np.asarray(pred).astype(bool), np.asarray(gt) != 0
    return float(np.sum(pred & gt)) / (float(np.sum(pred | gt)) + 1e-6)


class OracleOccupancyEvaluator(OM.OracleMeshEvaluator):
    """oracle/metrics.py's evaluator plus 'o3d-iou' when occupancy_rays=K is given"""

    def __init__(self, n_points=100000, metric_names=OM.ALL_METRICS, seed=0, occupancy_rays=None):
        names = list(metric_names)
        if occupancy_rays is None:
            super().__init__(n_points, names, seed)        # refuses 'o3d-iou'
        else:
            super().__init__(n_points, [k for k in names if k != "o3d-iou"], seed)
            self.metric_names = names
        self.occupancy_rays = None if occupancy_rays is None else check_rays(occupancy_rays)

    def eval_mesh(self, mesh, pointcloud_tgt, normals_tgt, onet_samples=None):
        v, f = mesh
        xyz, nrm, _ = OM.sample_surface(v, f, self.n_points, self.seed)
        return self._evaluate(xyz, pointcloud_tgt, nrm, normals_tgt, onet_samples, mesh)

    def _evaluate(self, pointcloud, pointcloud_tgt, normals=None, normals_tgt=None, onet_samples=None, mesh=None):
        names = self.metric_names
        if "o3d-iou" not in names:
            return super()._evaluate(pointcloud, pointcloud_tgt, normals, normals_tgt, onet_samples, mesh)
        if onet_samples is None or mesh is None:
            raise ValueError("'o3d-iou' needs the mesh and onet_samples")
        self.metric_names = [k for k in names if k != "o3d-iou"]
        try:
            out = super()._evaluate(pointcloud, pointcloud_tgt, normals, normals_tgt, onet_samples, mesh)
        finally:
            self.metric_names = names
        v, f = mesh
        f = np.asarray(f).reshape(-1, 3)
        if np.asarray(pointcloud).shape[0] == 0 or f.shape[0] == 0:
            out["o3d-iou"] = float("nan")
        else:
            out["o3d-iou"] = occupancy_iou(occupancy(v, f, onet_samples[0], n_rays=self.occupancy_rays),
                                           onet_samples[1])
        return {k: out[k] for k in names}
