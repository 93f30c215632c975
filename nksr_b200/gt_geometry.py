"""Volume ground truth for training: the reference's PointTSDFVolume (dataset/av_gt_geometry.py:110-187), the
supervision its default configs train with (configs/default/train.yaml: supervision.gt_type "PointTSDFVolume").

    gt = PointTSDFVolume.from_sensor_rays(xyz, normal, sensor, h, tau, margin)   # csrc/tsdf_volume.cu, SPEC S19
    gt = PointTSDFVolume.load("groundtruth.bin")          # an npz: xyz, normal, volume, volume_min, volume_max
    xyz, normal, volume = gt.torch_attr()
    sdf = gt.query_sdf(q)                                 # -sdf_from_points(q, xyz, normal, 8, 3.0, adaptive_knn=8)
    cls = gt.query_classification(q)                      # 0 near surface, 1 empty, 2 unknown / outside

The reference ships such volumes as data only; `from_sensor_rays` builds one from a LiDAR-like cloud whose points
carry their sensor position.

Mesh ground truth for object datasets (a closed mesh such as ShapeNet's), SPEC S21:

    gt = MeshGroundTruth(v, f, tau)                       # the BVH of metrics.MeshOccupancy, surface samples
    sdf = gt.query_sdf(q)                                 # -signed_distance: positive inside
    cls = gt.query_classification(q)                      # 1 outside with |sdf| >= band tau, else 0

Simulated LiDAR scans of a mesh, for sensor-bearing input with exact ground truth (SPEC S22, the first hit on the
same BVH):

    dirs = lidar_directions(64, 1024)                     # a spinning scanner's unit directions, our pattern
    xyz, sensor, normal, tri = scan_mesh(gt.mesh, sensors, dirs, max_range=...)
"""
from __future__ import annotations

import ctypes as C
import math
from typing import NamedTuple

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from ._lib import call, stream_ptr
from .metrics import MeshOccupancy, _check_rays, sample_surface
from .sdfgen import sdf_from_points

_NODE_BYTES = 4 + 8       # the fp32 volume and the builder's 64-bit key per node


class PointTSDFVolume:
    """oriented points (xyz, normal: N x 3 fp32 tensors) and a dense volume (X x Y x Z fp32 tensor) over the box
    [volume_min, volume_max] (float64 arrays), whose node (i, j, k) sits at volume_min + (i, j, k) (max - min) /
    (dims - 1): the ticks of linspace(min, max, dims), as grid_sample's align_corners=True reads them.  Node values:
    sdf / tau near the surface, +1 in observed free space, NaN unknown."""

    def __init__(self, xyz: torch.Tensor, normal: torch.Tensor, volume: torch.Tensor, volume_min, volume_max):
        self.xyz = xyz.to(torch.float32).contiguous()
        self.normal = normal.to(self.xyz.device, torch.float32).contiguous()
        self.volume = volume.to(self.xyz.device, torch.float32).contiguous()
        self.volume_min = np.asarray(volume_min, np.float64).reshape(3)
        self.volume_max = np.asarray(volume_max, np.float64).reshape(3)
        if self.xyz.dim() != 2 or self.xyz.shape[1] != 3 or self.normal.shape != self.xyz.shape:
            raise ValueError("xyz and normal must both be N x 3")
        if self.volume.dim() != 3:
            raise ValueError("volume must be X x Y x Z")
        if not (np.all(np.isfinite(self.volume_min)) and np.all(np.isfinite(self.volume_max))
                and np.all(self.volume_min < self.volume_max)):
            raise ValueError("the box needs finite volume_min < volume_max on every axis")

    # ------------------------------------------------------------------ the reference's contract
    def torch_attr(self):
        return self.xyz, self.normal, self.volume

    def query_sdf(self, queries: torch.Tensor) -> torch.Tensor:
        """the ground-truth SDF of the reference's volume supervision (dataset/av_gt_geometry.py:63-78)"""
        return -sdf_from_points(queries, self.xyz, self.normal, 8, 3.0, adaptive_knn=8)[0]

    def query_classification(self, queries: torch.Tensor, band: float = 1.0) -> torch.Tensor:
        """int64 class per query: 0 near surface (|v| < band at the nearest node), 1 empty (any other finite value),
        2 unknown (a NaN node, or a query outside [volume_min, volume_max]; the bounds are inclusive).  The nearest
        node is grid_sample's: align_corners=True, border padding, ties rounded half to even."""
        q = queries.to(self.volume.device, torch.float32)
        lo, hi = self.volume_min, self.volume_max
        inside = torch.ones(q.shape[0], dtype=torch.bool, device=q.device)
        for a in range(3):
            inside &= (q[:, a] >= lo[a]) & (q[:, a] <= hi[a])
        qi = q[inside]
        # grid_sample's x indexes the last volume axis: (z, y, x) normalised to [-1, 1]
        g = torch.stack([(qi[:, a] - lo[a]) / (hi[a] - lo[a]) * 2.0 - 1.0 for a in (2, 1, 0)], dim=1)
        v = F.grid_sample(self.volume[None, None], g[None, None, None], mode="nearest", padding_mode="border",
                          align_corners=True)[0, 0, 0, 0]
        cls_in = torch.ones_like(v, dtype=torch.long)
        cls_in[~torch.isfinite(v)] = 2
        cls_in[v.abs() < band] = 0
        cls = torch.full((q.shape[0],), 2, dtype=torch.long, device=q.device)
        cls[inside] = cls_in
        return cls

    def save(self, path):
        """an npz in the key set of the reference's groundtruth.bin"""
        with open(path, "wb") as fh:
            np.savez_compressed(fh, xyz=self.xyz.cpu().numpy(), normal=self.normal.cpu().numpy(),
                                volume=self.volume.cpu().numpy(), volume_min=self.volume_min,
                                volume_max=self.volume_max)

    @classmethod
    def load(cls, path, device="cuda"):
        with np.load(path) as z:
            t = lambda k: torch.from_numpy(np.ascontiguousarray(z[k], dtype=np.float32)).to(device)
            return cls(t("xyz"), t("normal"), t("volume"), z["volume_min"], z["volume_max"])

    # ------------------------------------------------------------------ the builder
    @classmethod
    def from_sensor_rays(cls, xyz: torch.Tensor, normal: torch.Tensor, sensor: torch.Tensor, h: float, tau: float,
                         margin: float):
        """the volume of SPEC S19 over the points' bounds grown by `margin`, node spacing `h`, truncation `tau`: one
        ray per point from its sensor position (csrc/tsdf_volume.cu).  xyz, normal, sensor: N x 3 on one CUDA device."""
        if xyz.dim() != 2 or xyz.shape[1] != 3 or sensor.shape != xyz.shape or normal.shape != xyz.shape:
            raise ValueError("xyz, normal and sensor must all be N x 3")
        dev = xyz.device
        xyz = xyz.detach().to(torch.float32).contiguous()
        sensor = sensor.detach().to(dev, torch.float32).contiguous()
        n = xyz.shape[0]
        if n == 0:
            raise ValueError("from_sensor_rays needs at least one point for the box")
        h32, tau32 = float(np.float32(h)), float(np.float32(tau))
        if not (np.isfinite(h32) and h32 > 0.0) or not (np.isfinite(tau32) and tau32 > 0.0):
            raise ValueError(f"h and tau must be finite and > 0 (h={h}, tau={tau})")
        if not (np.isfinite(margin) and margin >= 0.0):
            raise ValueError(f"margin must be finite and >= 0 (margin={margin})")
        if not bool(torch.isfinite(xyz).all()):
            raise ValueError("xyz must be finite: its bounds give the box")
        lo = xyz.min(dim=0).values.double().cpu().numpy() - margin
        hi = xyz.max(dim=0).values.double().cpu().numpy() + margin
        vmin = lo.astype(np.float32)                             # node 0, as the kernel reads it
        dims = [max(int(np.ceil((hi[a] - float(vmin[a])) / h32)) + 1, 2) for a in range(3)]
        n_nodes = dims[0] * dims[1] * dims[2]
        if n_nodes >= 2 ** 31:
            raise ValueError(f"a {dims[0]} x {dims[1]} x {dims[2]} grid has 2^31 nodes or more: raise h or crop")
        _lib.require_cuda(xyz, "xyz")
        need = n_nodes * _NODE_BYTES
        free_bytes = torch.cuda.mem_get_info(dev)[0]
        if need > free_bytes:
            raise MemoryError(f"a {dims[0]} x {dims[1]} x {dims[2]} grid needs {need / 2**30:.2f} GiB, "
                              f"{free_bytes / 2**30:.2f} GiB free on {dev}")
        vmin3 = (C.c_float * 3)(*[float(v) for v in vmin])
        dims3 = (C.c_int64 * 3)(*dims)
        volume = torch.empty(dims, dtype=torch.float32, device=dev)
        nb = call("nksr_tsdf_volume_workspace_bytes", C.addressof(dims3))
        ws = _lib._ws(nb, dev)
        call("nksr_tsdf_volume", xyz, sensor, n, C.addressof(vmin3), h32, C.addressof(dims3), tau32, volume, ws, nb,
             stream_ptr(dev))
        vmin64 = vmin.astype(np.float64)
        vmax64 = vmin64 + (np.asarray(dims, np.float64) - 1.0) * h32
        return cls(xyz, normal.detach().to(dev), volume, vmin64, vmax64)

    def class_fractions(self):
        """fractions of the nodes that are near (|v| < 1), free (v = 1) and unknown (NaN)"""
        v = self.volume
        fin = torch.isfinite(v)
        near = fin & (v.abs() < 1.0)
        n = max(v.numel(), 1)
        return dict(near=float(near.sum()) / n, free=float((fin & ~near).sum()) / n, unknown=float((~fin).sum()) / n)


class MeshGroundTruth:
    """exact SDF supervision from a triangle mesh (SPEC S21), with the three methods TrainingScene and the losses use.
    The surface samples are `n_surface` area-uniform points of sample_surface with their unit triangle normals
    (oriented by the winding); the SDF is the distance to the closest triangle on the BVH, signed by the ray-parity
    occupancy of `n_rays` rays (SPEC S20), so the sign is right on a closed mesh whatever its winding.  `tau` is the
    truncation that separates near-surface from empty space in query_classification.  The losses ask query_sdf and
    query_classification about the same samples, so the last query tensor's (distance, inside) is kept and reused
    while that tensor is unchanged (same object, same in-place version counter)."""

    def __init__(self, v: torch.Tensor, f: torch.Tensor, tau: float, n_surface: int = 100_000, n_rays: int = 3,
                 seed: int = 0):
        tau = float(tau)
        if not (np.isfinite(tau) and tau > 0.0):
            raise ValueError(f"tau must be finite and > 0 (tau={tau})")
        self.tau, self.n_rays = tau, _check_rays(n_rays)
        self.mesh = MeshOccupancy(v, f)
        self.xyz, self.normal, _ = sample_surface(v, f, n_surface, seed)
        self._last = None

    def _distance_and_inside(self, queries):
        last = self._last
        if last is not None and last[0] is queries and last[1] == queries._version:
            return last[2]
        out = self.mesh.distance_and_inside(queries, self.n_rays)
        self._last = (queries, queries._version, out) if isinstance(queries, torch.Tensor) else None
        return out

    def torch_attr(self):
        """(surface samples, their unit normals, None): a mesh has no volume"""
        return self.xyz, self.normal, None

    def query_sdf(self, queries: torch.Tensor) -> torch.Tensor:
        """-signed_distance: the distance to the mesh, positive inside and negative on the side the normals of a
        consistently wound closed mesh point to (PointTSDFVolume.query_sdf's convention)"""
        dist, inside = self._distance_and_inside(queries)
        return torch.where(inside, dist, -dist)

    def query_classification(self, queries: torch.Tensor, band: float = 1.0) -> torch.Tensor:
        """int64 class per query: 1 (empty space) where the query is outside and its distance is >= band * tau (an fp32
        comparison), 0 everywhere else -- inside a closed mesh the truncated SDF is known, so the near-surface term
        applies there too.  2 (unknown) is never returned."""
        dist, inside = self._distance_and_inside(queries)
        return (~inside & (dist >= band * self.tau)).long()

    def __repr__(self):
        return f"MeshGroundTruth(triangles={self.mesh.n_tri}, samples={self.xyz.shape[0]}, tau={self.tau})"


def lidar_directions(n_beams: int = 64, n_azimuth: int = 1024, elevation_deg=(-24.8, 2.0)) -> torch.Tensor:
    """unit fp32 directions of a spinning scanner, (n_beams * n_azimuth, 3) on the host: azimuth step k (the outer
    index) at 2 pi (k + 1/2) / n_azimuth from +x towards +y, beam j (the inner index) at the elevation
    lo + (hi - lo) j / (n_beams - 1) above the xy plane (lo alone for one beam), each direction
    (cos e cos a, cos e sin a, sin e) formed in fp64 and rounded once.  The default is a 64-beam sensor's vertical field
    of view; the pattern is this project's definition, not any vendor's firing order."""
    n_beams, n_azimuth = int(n_beams), int(n_azimuth)
    if n_beams < 1 or n_azimuth < 1:
        raise ValueError(f"n_beams and n_azimuth must be >= 1 (got {n_beams}, {n_azimuth})")
    lo, hi = (float(x) for x in elevation_deg)
    if not (np.isfinite(lo) and np.isfinite(hi) and -90.0 <= lo <= hi <= 90.0):
        raise ValueError(f"elevation_deg must be finite with -90 <= lo <= hi <= 90 (got {elevation_deg})")
    e = np.deg2rad(lo + (hi - lo) * np.arange(n_beams) / max(n_beams - 1, 1))
    a = 2.0 * np.pi * (np.arange(n_azimuth) + 0.5) / n_azimuth
    ce = np.cos(e)[None, :]
    d = np.stack([ce * np.cos(a)[:, None], ce * np.sin(a)[:, None],
                  np.broadcast_to(np.sin(e)[None, :], (n_azimuth, n_beams))], axis=-1)
    return torch.from_numpy(np.ascontiguousarray(d.reshape(-1, 3).astype(np.float32)))


class MeshScan(NamedTuple):
    """the returns of scan_mesh, in ray order: point, the sensor position it was seen from, the unit normal of the hit
    triangle (its winding) and the original triangle index (int64)"""
    xyz: torch.Tensor
    sensor: torch.Tensor
    normal: torch.Tensor
    tri: torch.Tensor


SCAN_BATCH = 1 << 22      # rays per intersect call in scan_mesh: about 200 MB of ray and hit buffers


def scan_mesh(mesh: MeshOccupancy, sensors, directions, max_range: float = math.inf, range_noise: float = 0.0,
              generator=None) -> MeshScan:
    """a simulated scan of the mesh: every direction ((R, 3), e.g. lidar_directions()) cast from every sensor position
    ((P, 3)), ray p R + r from sensors[p] along directions[r] (pose-major), in batches of SCAN_BATCH rays.  The returns
    are the first hits (MeshOccupancy.intersect, SPEC S22) with t <= max_range -- t is in units of the direction, so
    with unit directions it is the range -- kept in ray order.  With range_noise > 0 each point moves along its unit
    ray by range_noise times a standard normal drawn from `generator` (one draw per return, in order); with 0 nothing
    is drawn and the scan is bitwise reproducible.  Sensors and directions may be host arrays or tensors."""
    dev = mesh.device
    max_range, range_noise = float(max_range), float(range_noise)
    if math.isnan(max_range):
        raise ValueError("max_range must not be NaN")
    if not (math.isfinite(range_noise) and range_noise >= 0.0):
        raise ValueError(f"range_noise must be finite and >= 0 (got {range_noise})")
    s = torch.as_tensor(sensors).detach().to(dev, torch.float32).reshape(-1, 3).contiguous()
    d = torch.as_tensor(directions).detach().to(dev, torch.float32).reshape(-1, 3).contiguous()
    P, R = s.shape[0], d.shape[0]
    parts = []
    for start in range(0, P * R, SCAN_BATCH):
        ray = torch.arange(start, min(start + SCAN_BATCH, P * R), device=dev)
        o, dr = s[ray // R], d[ray % R]
        t, point, normal, tri = mesh.intersect(o, dr, max_range)
        keep = (tri >= 0).to(torch.int32)
        scan = _lib.exclusive_scan32(keep)
        cnt = int(scan[-1].item())
        rows = [point, o, normal, tri] + ([dr] if range_noise > 0.0 else [])
        parts.append([_lib.compact_rows(a.contiguous(), keep, scan, cnt) for a in rows])
    if not parts:
        e3 = torch.empty((0, 3), dtype=torch.float32, device=dev)
        return MeshScan(e3, e3.clone(), e3.clone(), torch.empty(0, dtype=torch.int64, device=dev))
    cols = [torch.cat(c) for c in zip(*parts)]
    xyz, sensor, normal, tri = cols[:4]
    if range_noise > 0.0:
        u = cols[4] / torch.linalg.vector_norm(cols[4], dim=1, keepdim=True)
        eps = torch.randn((xyz.shape[0], 1), generator=generator, device=dev, dtype=torch.float32)
        xyz = xyz + (range_noise * eps) * u
    return MeshScan(xyz, sensor, normal, tri)
