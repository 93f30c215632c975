"""Mesh-quality metrics -- host mirror of the reference's metrics.MeshEvaluator.

Reference contract:
  MeshEvaluator(n_points=5e6 or 5e5, metric_names=MeshEvaluator.ESSENTIAL_METRICS)   models/nksr_net.py:298-312
  .eval_mesh(mesh, ref_xyz, ref_normal, onet_samples=None) -> {name: value}

The mesh is sampled area-uniformly (csrc/metrics.cu: k_sample_surface) and both nearest-neighbour passes are exact
(k_metric_nearest on the multi-level voxel hash, k_metric_far for the queries the hierarchy does not resolve); the
means and threshold fractions are fp64 reductions in torch.  DESIGN.md SPEC S18 defines every step.

`o3d-iou` (opt-in, MeshEvaluator(occupancy_rays=K)) is the volumetric IoU of the reference's ONet occupancy samples
against MeshOccupancy, a ray-parity occupancy of the mesh on an LBVH (csrc/raycast.cu; SPEC S20).  The reference takes
its occupancy from a package outside its tree, so the value is this project's rule, not a reproduction.  The same BVH
answers the closest-triangle query (`MeshOccupancy.closest`, `signed_distance`; SPEC S21) and the first hit of a ray
(`MeshOccupancy.intersect`; SPEC S22).
"""
from __future__ import annotations

import ctypes as C
import logging
import math
from typing import Optional

import numpy as np
import torch

from ._lib import MAX_DEPTH, NksrError, _ws, call, require_cuda, sort_pairs, stream_ptr

_log = logging.getLogger(__name__)

THRESHOLDS = (0.01, 0.015, 0.02, 0.002, 0.1)
START_LEVEL = 2         # first level of the nearest-point search, as for PCNNField
MAX_RAYS = 9            # KMAX of SPEC S20: the number of built-in ray directions (csrc/raycast.cu)
_NAN = float("nan")


def _as_tensor(a, device, dtype) -> torch.Tensor:
    if isinstance(a, torch.Tensor):
        return a.detach().to(device=device, dtype=dtype).contiguous()
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a))).to(device=device, dtype=dtype).contiguous()


def sample_surface(v: torch.Tensor, f: torch.Tensor, n: int, seed: int = 0):
    """n area-uniform samples of the triangle mesh (v, f) on its device: (xyz (n, 3), unit triangle normal (n, 3),
    source triangle (n,) int32).  Triangle t receives the samples [round(n S_{t-1} / A), round(n S_t / A)) of the fp64
    area prefix S (A = S_T); a mesh without area gives none."""
    require_cuda(v, "v")
    dev = v.device
    v = v.detach().to(torch.float32).contiguous()
    f = f.detach().to(device=dev, dtype=torch.int32).reshape(-1, 3).contiguous()
    n = int(n)
    t = f.shape[0]
    if t:
        vd = v.double()
        area = 0.5 * torch.linalg.vector_norm(torch.linalg.cross(vd[f[:, 1].long()] - vd[f[:, 0].long()],
                                                                  vd[f[:, 2].long()] - vd[f[:, 0].long()]), dim=1)
        prefix = torch.cumsum(area, 0)
        total = float(prefix[-1].item())
    if n <= 0 or t == 0 or not total > 0.0:
        return (torch.empty((0, 3), dtype=torch.float32, device=dev), torch.empty((0, 3), dtype=torch.float32, device=dev),
                torch.empty(0, dtype=torch.int32, device=dev))
    start = torch.zeros(t + 1, dtype=torch.int64, device=dev)
    start[1:] = torch.round(n * prefix / total).long().clamp_(0, n)
    start[-1] = n
    xyz = torch.empty((n, 3), dtype=torch.float32, device=dev)
    nrm = torch.empty((n, 3), dtype=torch.float32, device=dev)
    tri = torch.empty(n, dtype=torch.int32, device=dev)
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    call("nksr_sample_surface", v, f, t, start, n, seed - (1 << 64) if seed >= 1 << 63 else seed, xyz, nrm, tri,
         stream_ptr(dev))
    return xyz, nrm, tri


def nearest_neighbours(query: torch.Tensor, target: torch.Tensor, query_normal: Optional[torch.Tensor] = None,
                       target_normal: Optional[torch.Tensor] = None):
    """Exact nearest target point of every query: (distance (m,) fp32, index into `target` (m,) int64, |n_q . n_t| of the
    unit normals (m,), NaN unless both normal sets are given).  Ties go to the lower index of the hash's sorted order,
    which for coincident target points is their input order.  An empty target gives distance inf and index -1."""
    from .reconstructor import _knn_hash
    require_cuda(target, "target")
    dev = target.device
    target = target.detach().to(torch.float32).contiguous()
    query = query.detach().to(dev, torch.float32).contiguous()
    m, n = query.shape[0], target.shape[0]
    dot = torch.full((m,), _NAN, dtype=torch.float32, device=dev)
    if n == 0 or m == 0:
        return (torch.full((m,), math.inf, dtype=torch.float32, device=dev),
                torch.full((m,), -1, dtype=torch.int64, device=dev), dot)
    origin = torch.minimum(target.min(dim=0).values, query.min(dim=0).values)
    perm, svh, _, ranges, origin = _knn_hash(target, levels=MAX_DEPTH, origin=origin)
    xs = target[perm].contiguous()
    both = query_normal is not None and target_normal is not None
    tn = target_normal.detach().to(dev, torch.float32)[perm].contiguous() if both else None
    qn = query_normal.detach().to(dev, torch.float32).contiguous() if both else None
    origin_host = (C.c_float * 3)(*[float(x) for x in origin.tolist()])
    box = torch.empty((svh.num_voxels(svh.depth - 1), 6), dtype=torch.float32, device=dev)
    far_list = torch.empty(m, dtype=torch.int32, device=dev)
    far_count = torch.empty(1, dtype=torch.int32, device=dev)
    dist = torch.empty(m, dtype=torch.float32, device=dev)
    idx = torch.empty(m, dtype=torch.int32, device=dev)
    call("nksr_metric_nearest", svh.view(), xs, tn, ranges, box, n, query, qn, m, C.addressof(origin_host), START_LEVEL,
         dist, idx, dot if both else None, far_list, far_count, stream_ptr(dev))
    return dist, perm[idx.long()], dot


def summarise(completeness: torch.Tensor, completeness_dot: torch.Tensor, accuracy: torch.Tensor,
              accuracy_dot: torch.Tensor, thresholds=THRESHOLDS) -> dict:
    """Every metric of the evaluator from the two distance and normal-agreement arrays, in fp64 (SPEC S18)."""
    c, a = completeness.double(), accuracy.double()
    th = torch.tensor(thresholds, dtype=torch.float64, device=c.device)
    recall = (c[None, :] <= th[:, None]).double().mean(dim=1)
    precision = (a[None, :] <= th[:, None]).double().mean(dim=1)
    stats = torch.stack([c.mean(), (c * c).mean(), completeness_dot.double().mean(), a.mean(), (a * a).mean(),
                         accuracy_dot.double().mean()])
    comp, comp2, comp_n, acc, acc2, acc_n = stats.tolist()         # the one host read
    p, r = precision.tolist(), recall.tolist()
    fs = [2.0 * p[i] * r[i] / (p[i] + r[i]) if p[i] + r[i] > 0 else _NAN for i in range(len(p))]
    return {
        "completeness": comp, "accuracy": acc,
        "normals completeness": comp_n, "normals accuracy": acc_n, "normals": 0.5 * comp_n + 0.5 * acc_n,
        "completeness2": comp2, "accuracy2": acc2, "chamfer-L2": 0.5 * (comp2 + acc2),
        "chamfer-L1": 0.5 * (comp + acc),
        "f-precision": p[0], "f-recall": r[0], "f-score": fs[0], "f-score-15": fs[1], "f-score-20": fs[2],
        "f-precision-outdoor": p[4], "f-recall-outdoor": r[4], "f-score-outdoor": fs[4],
    }


def _check_rays(k) -> int:
    k = int(k)
    if k < 1 or k > MAX_RAYS or k % 2 == 0:
        raise ValueError(f"the number of rays must be odd and in [1, {MAX_RAYS}], got {k}")
    return k


class MeshOccupancy:
    """Inside / outside of a triangle mesh by ray parity (SPEC S20): a query is inside when more than half of its K
    rays cross the mesh an odd number of times.  Winding never enters, so triangle soups and mixed orientations are
    fine; on a closed mesh every ray agrees, on an open one the vote is a definition.  The BVH is built once here;
    `contains` answers any number of query batches, `closest` / `signed_distance` the distance to the mesh on the
    same BVH (SPEC S21) and `intersect` the first hit of a ray (SPEC S22).  CUDA only."""

    def __init__(self, v: torch.Tensor, f: torch.Tensor):
        require_cuda(v, "v")
        require_cuda(f, "f")
        dev = v.device
        v = v.detach().to(torch.float32).reshape(-1, 3).contiguous()
        f = f.detach().to(dev).reshape(-1, 3)
        n_v, t = v.shape[0], f.shape[0]
        if t >= 2 ** 31:
            raise NksrError(f"{t} triangles: the occupancy BVH holds fewer than 2^31")
        if t and (int(f.min()) < 0 or int(f.max()) >= n_v):
            raise NksrError(f"face indices must lie in [0, {n_v})")
        if not bool(torch.isfinite(v).all()):
            raise NksrError("mesh vertices must be finite")
        f = f.to(torch.int32).contiguous()
        self.device, self.n_tri = dev, t
        self.v, self.f = v, f               # the first hit's normal is taken in the caller's winding

        self.scene = torch.zeros(8, dtype=torch.float32, device=dev)
        self.nodes = torch.empty((max(t - 1, 0), 16), dtype=torch.float32, device=dev)
        self.tris = torch.empty((t, 12), dtype=torch.float32, device=dev)
        if t == 0:
            return
        st = stream_ptr(dev)
        keys = torch.empty(t, dtype=torch.int64, device=dev)
        idx = torch.empty(t, dtype=torch.int32, device=dev)
        call("nksr_bvh_keys", v, f, t, self.scene, keys, idx, st)
        keys, idx = sort_pairs(keys, idx)
        nb = call("nksr_bvh_workspace_bytes", t)
        ws = _ws(nb, dev)
        if t > 1:
            call("nksr_bvh_hierarchy", keys, t, self.nodes, ws, nb, st)
        call("nksr_bvh_refit", v, f, idx, t, self.nodes if t > 1 else None, self.tris, ws, nb, st)

    def contains(self, points, n_rays: int = 3) -> torch.Tensor:
        """bool (m,): inside by the vote of the first n_rays built-in directions (odd, 1 <= n_rays <= 9)"""
        return occupancy_along(self, points, None, _check_rays(n_rays))

    def closest(self, points):
        """the closest point of the mesh to every query (SPEC S21): (distance (m,) fp32, closest point (m, 3) fp32,
        original triangle index (m,) int64).  Equal squared distances go to the lower triangle index; a mesh without
        triangles gives distance inf, point NaN and index -1.  Bitwise the brute force over every triangle."""
        dist, point, tri = _closest(self, _queries(self, points))
        return dist, point, tri.long()

    def signed_distance(self, points, n_rays: int = 3) -> torch.Tensor:
        """fp32 (m,): the distance of `closest`, negated where `contains(points, n_rays)` is true -- negative inside, as
        open3d's convention.  The sign is ray parity, not winding."""
        dist, inside = self.distance_and_inside(points, n_rays)
        return torch.where(inside, -dist, dist)

    def distance_and_inside(self, points, n_rays: int = 3):
        """(the distance of `closest`, the bool of `contains(points, n_rays)`) from one validation of the queries"""
        k = _check_rays(n_rays)
        q = _queries(self, points)
        return _closest(self, q)[0], _occupancy(self, q, None, k)

    def intersect(self, origins, directions, t_max=None):
        """the first hit of every ray from origins[i] along directions[i] (SPEC S22; (m, 3) each, finite, no direction
        all zero): (t (m,) fp32, point = origin + t * direction (m, 3) fp32, unit normal of the hit triangle in its
        (v1 - v0) x (v2 - v0) winding (m, 3) fp32, original triangle index (m,) int64).  Only hits at 0 < t <= t_max
        count (None: +inf; a number, or one value per ray); t is in units of the direction's length.  Equal t go to
        the lower triangle index.  A miss, and every ray of a mesh without triangles, gives t inf, point and normal
        NaN and index -1.  Bitwise the brute force over every triangle."""
        o = _ray_array(self, origins, "origins")
        d = _ray_array(self, directions, "directions")
        m = o.shape[0]
        if d.shape[0] != m:
            raise ValueError(f"{m} origins but {d.shape[0]} directions")
        if m and not bool((d != 0).any(dim=1).all()):
            raise ValueError("every ray direction needs a nonzero component")
        t_all, t_ray = math.inf, None
        if t_max is not None:
            if isinstance(t_max, torch.Tensor) and t_max.dim() > 0 or isinstance(t_max, (np.ndarray, list, tuple)):
                if isinstance(t_max, torch.Tensor):
                    require_cuda(t_max, "t_max")
                t_ray = _as_tensor(t_max, self.device, torch.float32).reshape(-1)
                if t_ray.shape[0] != m:
                    raise ValueError(f"t_max has {t_ray.shape[0]} values for {m} rays")
                if bool(torch.isnan(t_ray).any()):
                    raise ValueError("t_max must not be NaN")
            else:
                t_all = float(np.float32(float(t_max)))
                if math.isnan(t_all):
                    raise ValueError("t_max must not be NaN")
        t = torch.empty(m, dtype=torch.float32, device=self.device)
        point = torch.empty((m, 3), dtype=torch.float32, device=self.device)
        normal = torch.empty((m, 3), dtype=torch.float32, device=self.device)
        tri = torch.empty(m, dtype=torch.int32, device=self.device)
        if m:
            has = self.n_tri > 0
            call("nksr_mesh_first_hit", self.nodes if self.n_tri > 1 else None, self.tris if has else None,
                 self.scene, self.n_tri, self.v if has else None, self.f if has else None, o, d, m, t_ray, t_all, t,
                 point, normal, tri, stream_ptr(self.device))
        return t, point, normal, tri.long()

    def __repr__(self):
        return f"MeshOccupancy(triangles={self.n_tri}, device={self.device})"


def _queries(occ: MeshOccupancy, points) -> torch.Tensor:
    """the query points as a contiguous fp32 (m, 3) tensor on the mesh's device: CUDA tensors or host arrays,
    finite"""
    if isinstance(points, torch.Tensor):
        require_cuda(points, "points")
    q = _as_tensor(points, occ.device, torch.float32).reshape(-1, 3)
    if not bool(torch.isfinite(q).all()):
        raise NksrError("query points must be finite")
    return q


def _ray_array(occ: MeshOccupancy, a, what: str) -> torch.Tensor:
    """ray origins or directions as a contiguous fp32 (m, 3) tensor on the mesh's device, checked as _queries does"""
    if isinstance(a, torch.Tensor):
        require_cuda(a, what)
    x = _as_tensor(a, occ.device, torch.float32).reshape(-1, 3)
    if not bool(torch.isfinite(x).all()):
        raise NksrError(f"ray {what} must be finite")
    return x


def _closest(occ: MeshOccupancy, q: torch.Tensor):
    """nksr_mesh_closest on checked queries (_queries): distance, point, int32 triangle"""
    m = q.shape[0]
    dist = torch.empty(m, dtype=torch.float32, device=occ.device)
    point = torch.empty((m, 3), dtype=torch.float32, device=occ.device)
    tri = torch.empty(m, dtype=torch.int32, device=occ.device)
    if m:
        call("nksr_mesh_closest", occ.nodes if occ.n_tri > 1 else None, occ.tris if occ.n_tri else None, occ.scene,
             occ.n_tri, q, m, dist, point, tri, stream_ptr(occ.device))
    return dist, point, tri


def _occupancy(occ: MeshOccupancy, q: torch.Tensor, dirs: Optional[torch.Tensor], k: int) -> torch.Tensor:
    """nksr_mesh_occupancy on checked queries and ray settings"""
    m = q.shape[0]
    inside = torch.empty(m, dtype=torch.uint8, device=occ.device)
    if m:
        call("nksr_mesh_occupancy", occ.nodes if occ.n_tri > 1 else None, occ.tris, occ.scene, occ.n_tri, q, m, dirs,
             k, inside, stream_ptr(occ.device))
    return inside.bool()


def occupancy_along(occ: MeshOccupancy, points, directions=None, n_rays: Optional[int] = None) -> torch.Tensor:
    """MeshOccupancy.contains with explicit ray directions ((K, 3), K odd in [1, 9], every component nonzero and
    finite) or, with directions None, the first n_rays built-in ones"""
    q = _queries(occ, points)
    dirs = None
    if directions is not None:
        dirs = _as_tensor(directions, occ.device, torch.float32).reshape(-1, 3)
        k = _check_rays(dirs.shape[0])
        if not bool((torch.isfinite(dirs) & (dirs != 0)).all()):
            raise ValueError("every ray direction component must be finite and nonzero")
    else:
        k = _check_rays(n_rays)
    return _occupancy(occ, q, dirs, k)


def occupancy_iou(pred: torch.Tensor, gt: torch.Tensor) -> float:
    """the reference's volumetric IoU: |pred & gt| / (|pred | gt| + 1e-6), integer counts, fp64 division"""
    both = torch.stack([(pred & gt).sum(), (pred | gt).sum()]).tolist()
    return float(both[0]) / (float(both[1]) + 1e-6)


METRIC_KEYS = ("completeness", "accuracy", "normals completeness", "normals accuracy", "normals", "completeness2",
               "accuracy2", "chamfer-L2", "chamfer-L1", "f-precision", "f-recall", "f-score", "f-score-15",
               "f-score-20", "f-precision-outdoor", "f-recall-outdoor", "f-score-outdoor")


def mesh_arrays(mesh):
    """(v, f) of a DualMesh (.v, .f), a (v, f) pair or an object with `vertices` / `triangles` (an open3d mesh)."""
    if isinstance(mesh, (tuple, list)) and len(mesh) == 2:
        return mesh[0], mesh[1]
    if hasattr(mesh, "v") and hasattr(mesh, "f"):
        return mesh.v, mesh.f
    if hasattr(mesh, "vertices") and hasattr(mesh, "triangles"):
        return mesh.vertices, mesh.triangles
    raise TypeError("mesh must be a DualMesh, a (v, f) pair or have `vertices` and `triangles`")


class MeshEvaluator:
    """Drop-in for the reference's metrics.MeshEvaluator: same constructor, class attributes, methods, keys and
    definitions; CUDA only.  `o3d-iou` (the volumetric IoU on the ONet occupancy samples) is computed only when
    `occupancy_rays` (odd, 1..9) is given: it uses this project's ray-parity rule (MeshOccupancy, SPEC S20), not the
    package the reference takes it from, so a caller opts in knowingly."""

    ESSENTIAL_METRICS = ["chamfer-L1", "f-score", "normals"]
    ALL_METRICS = ["completeness", "accuracy", "normals completeness", "normals accuracy", "normals",
                   "completeness2", "accuracy2", "chamfer-L2",
                   "chamfer-L1", "f-precision", "f-recall", "f-score", "f-score-15", "f-score-20"]

    def __init__(self, n_points=100000, metric_names=ALL_METRICS, device=None, seed: int = 0,
                 occupancy_rays: Optional[int] = None):
        names = list(metric_names)
        if occupancy_rays is not None:
            occupancy_rays = _check_rays(occupancy_rays)
        elif "o3d-iou" in names:
            raise ValueError("'o3d-iou' needs occupancy_rays=K (odd, 1..9): its mesh occupancy is this project's "
                             "ray-parity rule (SPEC S20), not the package the reference takes it from")
        unknown = [k for k in names if k not in METRIC_KEYS and not (k == "o3d-iou" and occupancy_rays)]
        if unknown:
            raise ValueError(f"unknown metric names {unknown}; known: {list(METRIC_KEYS)}")
        self.n_points = int(n_points)
        self.thresholds = np.array(THRESHOLDS)
        self.fidx = [0, 1, 2, 3, 4]
        self.metric_names = names
        self.device = torch.device(device) if device is not None else None
        self.seed = int(seed)
        self.occupancy_rays = occupancy_rays

    def _device_for(self, a) -> torch.device:
        if self.device is not None:
            return self.device
        if isinstance(a, torch.Tensor) and a.is_cuda:
            return a.device
        return torch.device("cuda", 0)

    def eval_mesh(self, mesh, pointcloud_tgt, normals_tgt, onet_samples=None):
        """Samples n_points on the mesh (area-uniform, triangle normals) and evaluates them against the target."""
        v, f = mesh_arrays(mesh)
        dev = self._device_for(v)
        v = _as_tensor(v, dev, torch.float32).reshape(-1, 3)
        f = _as_tensor(f, dev, torch.int32).reshape(-1, 3)
        xyz, nrm, _ = sample_surface(v, f, self.n_points, self.seed)
        return self._evaluate(xyz, pointcloud_tgt, nrm, normals_tgt, onet_samples, (v, f))

    def _evaluate(self, pointcloud, pointcloud_tgt, normals=None, normals_tgt=None, onet_samples=None, mesh=None):
        dev = self._device_for(pointcloud)
        want_iou = "o3d-iou" in self.metric_names
        if want_iou and (onet_samples is None or mesh is None):
            raise ValueError("'o3d-iou' needs the mesh and onet_samples = (points (N, 3), occupancy (N,))")
        if int(pointcloud.shape[0]) == 0:
            _log.warning("Empty pointcloud / mesh detected! Return NaN metric!")
            return {k: _NAN for k in self.metric_names}
        pts = _as_tensor(pointcloud, dev, torch.float32).reshape(-1, 3)
        tgt = _as_tensor(pointcloud_tgt, dev, torch.float32).reshape(-1, 3)
        if tgt.shape[0] == 0:
            raise NksrError("the target point cloud is empty")
        nrm = _as_tensor(normals, dev, torch.float32).reshape(-1, 3) if normals is not None else None
        nrm_t = _as_tensor(normals_tgt, dev, torch.float32).reshape(-1, 3) if normals_tgt is not None else None
        comp, _, comp_dot = nearest_neighbours(tgt, pts, nrm_t, nrm)
        acc, _, acc_dot = nearest_neighbours(pts, tgt, nrm, nrm_t)
        out = summarise(comp, comp_dot, acc, acc_dot, tuple(self.thresholds.tolist()))
        if want_iou:
            out["o3d-iou"] = self._occupancy_iou(mesh, onet_samples, dev)
        return {k: out[k] for k in self.metric_names}

    def _occupancy_iou(self, mesh, onet_samples, dev) -> float:
        """o3d-iou of the reference (metrics.py:180-188): occupancy of onet_samples[0] against onet_samples[1] != 0"""
        v, f = mesh_arrays(mesh)
        v = _as_tensor(v, dev, torch.float32).reshape(-1, 3)
        f = _as_tensor(f, dev, torch.int64).reshape(-1, 3)
        if f.shape[0] == 0:
            return _NAN
        pts = _as_tensor(onet_samples[0], dev, torch.float32).reshape(-1, 3)
        gt = onet_samples[1]
        gt = (gt.detach().to(dev) if isinstance(gt, torch.Tensor) else torch.from_numpy(np.asarray(gt)).to(dev))
        gt = gt.reshape(-1) != 0
        if gt.shape[0] != pts.shape[0]:
            raise ValueError(f"onet_samples: {pts.shape[0]} points but {gt.shape[0]} occupancy values")
        pred = MeshOccupancy(v, f).contains(pts, self.occupancy_rays)
        return occupancy_iou(pred, gt)


__all__ = ["MeshEvaluator", "MeshOccupancy", "sample_surface", "nearest_neighbours", "summarise", "mesh_arrays",
           "occupancy_iou", "THRESHOLDS", "MAX_RAYS"]
