"""Reconstructor -- host mirror of nksr.Reconstructor.

Reference contract (closed wheel; call sites only):
  Reconstructor(device); .chunk_tmp_device; .network       examples/recons_simple.py:25,
                                                            examples/recons_by_chunk.py:26-27
  .reconstruct(xyz, normal=None, sensor=None, detail_level=0.0, voxel_size=None,
               chunk_size=None, preprocess_fn=None, approx_kernel_grad=, solver_tol=,
               fused_mode=)                                  examples/recons_waymo.py:30-37,
                                                            NKSR-USAGE.md:126-137
  get_estimate_normal_preprocess_fn(knn, max_angle_deg)     examples/recons_waymo.py:36
The wiring of one reconstruction (SVH -> network -> KernelField -> solve -> mask) follows the
open training model, models/nksr_net.py:57-133, including its constraint weights.
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import Callable, List, Optional

import torch

from . import _lib
from ._lib import call, stream_ptr
from .fields import BaseField, EvaluationResult, KernelField, LayerField, NeuralField
from .meshing import DualMesh
from .network import NKSRNetwork
from .svh import SparseFeatureHierarchy

DEFAULT_VOXEL_SIZE = 0.1          # configs/default/train.yaml:11
POS_WEIGHT = 1.0e4                # configs/default/train.yaml:27-29 (solver.pos_weight)
NORMAL_WEIGHT = 1.0e4             # solver.normal_weight


def _count_voxels(xyz: torch.Tensor, w: float) -> int:
    n = xyz.shape[0]
    hk = torch.empty(n, dtype=torch.int64, device=xyz.device)
    status = torch.zeros(1, dtype=torch.int32, device=xyz.device)
    call("nksr_point_half_keys", xyz, n, float(w), hk, status, stream_ptr(xyz.device))
    count = int(_lib.unique_sorted(_lib.sort_keys(hk), 3).numel())
    if int(status.item()) & 1:
        # |x| / w outside the 2^19-voxel key range: keys collapse; report "finer than representable" so that the
        # bisections that call this move towards larger voxels (ADVICE r1)
        return n
    return count


def voxel_size_from_detail(xyz: torch.Tensor, detail_level: float) -> float:
    """detail_level in [0,1] -> finest voxel size such that the cloud has on average
    8 * 4^-detail points per occupied voxel (our definition; the reference only documents the
    knob's direction, NKSR-USAGE.md:129-131).  Log-bisection on the occupied-voxel count."""
    d = min(max(float(detail_level), 0.0), 1.0)
    target = 8.0 * (0.25 ** d)
    ext = float((xyz.max(dim=0).values - xyz.min(dim=0).values).max().item())
    lo, hi = max(ext * 1e-5, 1e-9), max(ext, 1e-6)
    n = xyz.shape[0]
    for _ in range(24):
        mid = math.sqrt(lo * hi)
        if n / max(_count_voxels(xyz, mid), 1) > target:
            hi = mid
        else:
            lo = mid
    return math.sqrt(lo * hi)


KNN_LEVELS = 7        # levels of the voxel hash behind the kNN search (cell size doubles per level)


def _knn_hash(xyz: torch.Tensor, levels: int = KNN_LEVELS, origin: Optional[torch.Tensor] = None):
    """Multi-level voxel hash of a cloud for neighbour searches: returns (perm, svh, base, ranges, origin) with the points
    Morton-sorted by `perm`, the hierarchy of their containing voxels (finest cell ~ a sixth of the mean point
    spacing, doubling per level), base[l][i] = containing voxel of sorted point i, ranges[offset_l + v] = [first,
    last) sorted point of voxel v.  Keys are taken on coordinates shifted to the bounding-box corner, or to `origin`
    (a point at or below that corner, e.g. the corner of the cloud and its queries together) where given; an origin
    further than 2^18 finest cells below the corner is raised to that distance, so that the cloud stays in the key
    range."""
    dev, st = xyz.device, stream_ptr(xyz.device)
    n = xyz.shape[0]
    lo = xyz.min(dim=0).values
    ext = (xyz.max(dim=0).values - lo).tolist()                      # the one host read of the set-up
    emax = max(max(ext), 1e-12)
    dims = [max(e, 1e-3 * emax) for e in ext]
    h0 = 0.15 * (dims[0] * dims[1] * dims[2] / max(n, 1)) ** (1.0 / 3.0)
    h0 = float(torch.tensor(max(h0, emax / 2.0 ** 17), dtype=torch.float32).item())
    if origin is not None:
        lo = torch.maximum(torch.minimum(origin.to(lo), lo), lo - 2.0 ** 18 * h0)
    shifted = (xyz - lo).contiguous()
    hk = torch.empty(n, dtype=torch.int64, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    call("nksr_point_half_keys", shifted, n, h0, hk, status, st)
    hk_sorted, perm = _lib.sort_pairs(hk, torch.arange(n, dtype=torch.int32, device=dev))
    perm = perm.long()
    shifted = shifted[perm].contiguous()
    keys = [_lib.unique_sorted(hk_sorted, 3 * (l + 1)) for l in range(levels)]
    svh = SparseFeatureHierarchy(h0, levels, dev).build_from_keys(keys)
    base = svh.locate(shifted)
    offs = svh.offsets
    ranges = torch.empty((svh.num_unknowns, 2), dtype=torch.int32, device=dev)
    for l in range(levels):
        call("nksr_row_ranges", base[l], n, ranges[offs[l]:], svh.num_voxels(l), st)
    return perm, svh, base, ranges, lo


def estimate_normals_knn(xyz: torch.Tensor, sensor: Optional[torch.Tensor], knn: int = 64,
                         max_angle_deg: float = 85.0, want_eig: bool = False):
    """Exact kNN-PCA normals (csrc/normals.cu: k_knn_normals).  Returns the Morton permutation, the normals (in
    permuted order, flipped towards `sensor` when given), the keep flags of the grazing-angle filter, optionally
    the covariance eigenvalues, and the number of points whose neighbourhood could not be proven exact."""
    _lib.require_cuda(xyz, "xyz")
    xyz = xyz.detach().to(torch.float32).contiguous()
    n = xyz.shape[0]
    k = min(int(knn), 64, n)
    if k < 3:
        raise _lib.NksrError("normal estimation needs at least 3 points")
    dev, st = xyz.device, stream_ptr(xyz.device)
    perm, svh, base, ranges, _ = _knn_hash(xyz)
    xs = xyz[perm].contiguous()
    ss = sensor.detach().to(torch.float32)[perm].contiguous() if sensor is not None else None
    nrm = torch.empty((n, 3), dtype=torch.float32, device=dev)
    keep = torch.empty(n, dtype=torch.int32, device=dev)
    eig = torch.empty((n, 3), dtype=torch.float32, device=dev) if want_eig else None
    inexact = torch.zeros(1, dtype=torch.int32, device=dev)
    call("nksr_knn_normals", svh.view(), xs, ss, base, ranges, n, k, math.cos(math.radians(max_angle_deg)), nrm, keep,
         eig, inexact, st)
    return SimpleNamespace(perm=perm, xyz=xs, sensor=ss, normal=nrm, keep=keep, eig=eig, inexact=inexact)


def get_estimate_normal_preprocess_fn(knn: int = 64, max_angle_deg: float = 85.0, mode: str = "knn") -> Callable:
    """Normal estimation + sensor-side orientation + grazing-angle filter, following the open CPU twin
    examples/recons_waymo_cpu.py:21-41 line by line: k-nearest-neighbour PCA normals (:26), unit view direction
    (:32-33), flip (:34-36), |cos| > cos(max_angle) filter (:38-39).  mode='knn' (default): exact kNN on a
    multi-level voxel hash, one warp per point; mode='voxel': the round-1 approximation (PCA over the 27 voxels
    around the point of a grid sized to hold ~knn points; every point of a voxel gets the same normal)."""
    if mode not in ("knn", "voxel"):
        raise ValueError("mode must be 'knn' or 'voxel'")

    def fn_knn(xyz: torch.Tensor, normal: Optional[torch.Tensor], sensor: Optional[torch.Tensor]):
        assert normal is None, "normal already exists"
        assert sensor is not None, "please provide sensor positions for consistent orientations"
        r = estimate_normals_knn(xyz, sensor, knn, max_angle_deg)
        scan = _lib.exclusive_scan32(r.keep)
        cnt = int(scan[-1].item())
        return _lib.compact_rows(r.xyz, r.keep, scan, cnt), _lib.compact_rows(r.normal, r.keep, scan, cnt), None

    def fn(xyz: torch.Tensor, normal: Optional[torch.Tensor], sensor: Optional[torch.Tensor]):
        assert normal is None, "normal already exists"
        assert sensor is not None, "please provide sensor positions for consistent orientations"
        n = xyz.shape[0]
        # voxel size such that a 27-neighbourhood holds ~knn points
        ext = float((xyz.max(dim=0).values - xyz.min(dim=0).values).max().item())
        lo, hi = max(ext * 1e-5, 1e-9), max(ext, 1e-6)
        for _ in range(12):                                         # log-bisection to ~0.3 %
            mid = math.sqrt(lo * hi)
            ratio = n / max(_count_voxels(xyz, mid), 1) * 9.0       # ~9 occupied voxels of 27 on a surface
            if ratio > knn:
                hi = mid
            else:
                lo = mid
            if abs(ratio - knn) < 0.05 * knn:
                lo = hi = mid
                break
        h = float(torch.tensor(math.sqrt(lo * hi), dtype=torch.float32).item())
        dev, st = xyz.device, stream_ptr(xyz.device)
        # Morton-sort the points so that every voxel owns one contiguous range
        hk = torch.empty(n, dtype=torch.int64, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        call("nksr_point_half_keys", xyz, n, h, hk, status, st)
        _, perm = _lib.sort_pairs(hk, torch.arange(n, dtype=torch.int32, device=dev))
        perm = perm.long()
        xs, ss = xyz[perm].contiguous(), sensor[perm].contiguous()
        svh = SparseFeatureHierarchy(h, 1, dev).build_point_splatting(xs)
        nv = svh.num_voxels(0)
        base = svh.locate(xs)
        ranges = torch.empty((nv, 2), dtype=torch.int32, device=dev)
        call("nksr_row_ranges", base[0], n, ranges, nv, st)
        mom = torch.empty((nv, 10), dtype=torch.float32, device=dev)
        call("nksr_voxel_moments", svh.keys[0], nv, ranges, xs, h, mom, st)
        vox_normal = torch.empty((nv, 3), dtype=torch.float32, device=dev)
        call("nksr_voxel_pca_normals", svh.nbr27[0], mom, nv, h, vox_normal, st)
        nrm = torch.empty((n, 3), dtype=torch.float32, device=dev)
        keep = torch.empty(n, dtype=torch.int32, device=dev)
        call("nksr_orient_normals", xs, ss, base[0], vox_normal, n, math.cos(math.radians(max_angle_deg)), nrm,
             keep, st)
        scan = _lib.exclusive_scan32(keep)
        cnt = int(scan[-1].item())
        return _lib.compact_rows(xs, keep, scan, cnt), _lib.compact_rows(nrm, keep, scan, cnt), None

    return fn_knn if mode == "knn" else fn


class ChunkedField(BaseField):
    """Cubic chunks reconstructed one after the other (examples/recons_by_chunk.py:27-29, NKSR-USAGE.md:88-120).

    Every chunk is solved on the points of its core cube plus a margin of two coarsest voxels.  With all chunks at
    hand (`union_svh` given) the field is their partition-of-unity blend: the weight of chunk k is 1 in its core
    shrunk by the margin, falls linearly to 0 at core + margin, and the weights are normalised -- so neighbouring
    solutions cross-fade over the 2-margin band around a seam and `extract_dual_mesh` runs ONCE, on the hierarchy of the
    whole cloud, over the blended field (a single welded mesh, no cracks along chunk faces).  Without it (a rank of the
    multi-GPU chunk mapping holds only its own chunks) a query belongs to the chunk whose core contains it and the
    chunk meshes are clipped to their cores and concatenated.

    `chunk_tmp_device = cpu` (NKSR-USAGE.md:101,151): the solved chunk fields wait in host memory and visit
    `compute_device` one at a time while they are evaluated -- this build has no CPU evaluator."""

    def __init__(self, fields: List[KernelField], cores: torch.Tensor, chunk_size: float, margin: float = 0.0,
                 union_svh=None, compute_device=None, adaptive_depth: int = 2):
        super().__init__(union_svh if union_svh is not None else fields[0].svh)
        self.fields = fields
        self.cores = cores                       # (n_chunks, 3) integer chunk coordinates
        self.chunk_size = chunk_size
        self.margin = float(margin)
        self.blended = union_svh is not None and margin > 0
        self.compute_device = torch.device(compute_device) if compute_device is not None else fields[0].svh.device
        if self.blended:
            self.set_mask_field(LayerField(union_svh, min(adaptive_depth, union_svh.depth)))

    # a chunk field parked on the host visits the GPU for the duration of one evaluation
    def _visit(self, f):
        parked = f.svh.device.type != "cuda"
        if parked:
            f.to_(self.compute_device)
        return parked

    def _owner(self, xyz):
        c = torch.floor(xyz / self.chunk_size).long()
        owner = torch.full((xyz.shape[0],), -1, dtype=torch.long, device=xyz.device)
        for k in range(self.cores.shape[0]):
            owner[(c == self.cores[k].to(xyz.device)[None]).all(dim=1)] = k
        return owner

    def _weights(self, xyz, k):
        """partition-of-unity weight of chunk k before normalisation: product over the axes of a ramp that is 0 at
        core -+ margin and 1 from core +- margin inwards"""
        lo = self.cores[k].to(xyz.device).float() * self.chunk_size - self.margin
        hi = (self.cores[k].to(xyz.device).float() + 1.0) * self.chunk_size + self.margin
        ramp = torch.minimum((xyz - lo[None]) / (2.0 * self.margin), (hi[None] - xyz) / (2.0 * self.margin))
        return ramp.clamp(0.0, 1.0).prod(dim=1)

    def evaluate_f(self, xyz, grad=False):
        dev = xyz.device
        val = torch.zeros(xyz.shape[0], device=dev)
        g = torch.zeros((xyz.shape[0], 3), device=dev) if grad else None
        if not self.blended:
            owner = self._owner(xyz)
        else:
            wsum = torch.zeros(xyz.shape[0], device=dev)
        for k, f in enumerate(self.fields):
            if self.blended:
                w = self._weights(xyz, k)
                m = w > 0
            else:
                m = owner == k
            if not bool(m.any()):
                continue
            parked = self._visit(f)
            r = f.evaluate_f(xyz[m].to(f.svh.device), grad=grad)
            wk = w[m] if self.blended else 1.0
            val[m] += wk * r.value.to(dev)
            if grad:                              # (the gradient of the weights is left out: it vanishes off the seams)
                g[m] += (wk[:, None] if self.blended else 1.0) * r.gradient.to(dev)
            if self.blended:
                wsum[m] += wk
            if parked:
                f.to_("cpu")
        if self.blended:
            inv = 1.0 / wsum.clamp(min=1e-12)
            val = val * inv
            if grad:
                g = g * inv[:, None]
        return EvaluationResult(value=val, gradient=g)

    def mask(self, xyz):
        return self.mask_field.mask(xyz) if self.mask_field is not None else torch.ones(
            xyz.shape[0], dtype=torch.bool, device=xyz.device)

    def extract_dual_mesh(self, grid_upsample: int = 1, mise_iter: int = 0, max_points: int = -1):
        if self.blended:
            from .meshing import extract_dual_mesh
            return extract_dual_mesh(self, grid_upsample=grid_upsample, mise_iter=mise_iter, max_points=max_points)
        vs, fs, off = [], [], 0
        dev = self.compute_device
        for k, f in enumerate(self.fields):
            parked = self._visit(f)
            m = f.extract_dual_mesh(grid_upsample=grid_upsample, mise_iter=mise_iter, max_points=max_points)
            if parked:
                f.to_("cpu")
            if m.f.shape[0] == 0:
                continue
            cen = m.v[m.f].mean(dim=1)
            inside = (torch.floor(cen / self.chunk_size).long() == self.cores[k].to(cen.device)[None]).all(dim=1)
            tri = m.f[inside]
            used = torch.zeros(m.v.shape[0], dtype=torch.bool, device=cen.device)
            used[tri.reshape(-1)] = True
            remap = torch.cumsum(used.long(), 0) - 1
            vs.append(m.v[used].to(dev))
            fs.append((remap[tri] + off).to(dev))
            off += int(used.sum().item())
        if not vs:
            return DualMesh(v=torch.zeros((0, 3), device=dev), f=torch.zeros((0, 3), dtype=torch.int64, device=dev), c=None)
        return DualMesh(v=torch.cat(vs), f=torch.cat(fs), c=None)

    def to_(self, device):
        for f in self.fields:
            f.to_(device)
        if torch.device(device).type == "cuda":
            self.compute_device = torch.device(device)
            if self.blended:
                self.svh.to_(device)
                self.mask_field.to_(device)
        return self


def mask_field(network, feats, dec_svh, udf_svh, adaptive_depth: int, voxel_size: float) -> BaseField:
    """the mask of a reconstruction (models/nksr_net.py:124-133): with udf.enabled the UDF NeuralField over every level
    of the decoder's udf_svh, keeping f <= 2 voxel_size; else the LayerField of dec_svh's `adaptive_depth` finest
    levels"""
    if getattr(network, "udf_enabled", False):
        nf = NeuralField(udf_svh, network.udf_decoder, feats.udf_features)
        nf.set_level_set(2.0 * voxel_size)
        return nf
    return LayerField(dec_svh, adaptive_depth)


class Reconstructor:
    def __init__(self, device, network: Optional[NKSRNetwork] = None, tree_depth: int = 4, adaptive_depth: int = 2,
                 kernel_dim: int = 4):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.NksrError("nksr_b200.Reconstructor needs a CUDA device (CUDA-only build, no CPU path)")
        _lib.load()
        self.chunk_tmp_device = self.device
        self.tree_depth, self.adaptive_depth = tree_depth, adaptive_depth
        self._timer = _lib.StageTimer(self.device, enabled=False)
        self.network = (network or NKSRNetwork(dict(kernel_dim=kernel_dim, tree_depth=tree_depth,
                                                    adaptive_depth=adaptive_depth))).to(self.device)
        self.last_stats = {}

    # one chunk / the whole cloud: models/nksr_net.py:41-133 without the Lightning plumbing
    def _reconstruct_one(self, xyz, normal, sensor, voxel_size, approx_kernel_grad, solver_tol, fused_mode,
                         solver_max_iter) -> BaseField:
        if normal is not None:
            feat = normal
        elif sensor is not None:
            view = sensor - xyz
            feat = view / (torch.linalg.norm(view, dim=-1, keepdim=True) + 1e-6)     # models/nksr_net.py:48-52
        else:
            raise ValueError("either normal or sensor (with a normal-estimating preprocess_fn) is required")
        with torch.no_grad():        # reconstruction is inference: no graph, no system kept, even for a trainable network
            return self._reconstruct_field(xyz, feat, voxel_size, approx_kernel_grad, solver_tol, fused_mode,
                                           solver_max_iter)

    def _reconstruct_field(self, xyz, feat, voxel_size, approx_kernel_grad, solver_tol, fused_mode, solver_max_iter):
        tm = self._timer
        svh = SparseFeatureHierarchy(voxel_size, self.tree_depth, self.device).build_point_splatting(xyz)
        tm.mark("svh_build")
        enc = self.network.encoder(xyz, feat, svh, 0)
        feats, dec_svh, udf_svh = self.network.unet(enc, svh, adaptive_depth=self.adaptive_depth)
        if getattr(self.network, "structure", "encoder") == "predicted" and dec_svh.num_unknowns == 0:
            raise _lib.NksrError("predicted structure is empty: the network kept no voxel, there is nothing to solve")
        ad = min(self.adaptive_depth, dec_svh.depth)
        if getattr(self.network, "geometry", "kernel") == "neural":
            # models/nksr_net.py:114-119: the output field is the SDF decoder over the basis features, no solve
            field = NeuralField(dec_svh, self.network.sdf_decoder, feats.basis_features, position_gradient=True)
            tm.mark("network")
            field.set_mask_field(mask_field(self.network, feats, dec_svh, udf_svh, ad, voxel_size))
            return field
        field = KernelField(dec_svh, self.network.interpolators, feats.basis_features, approx_kernel_grad)
        field._timer = tm
        tm.mark("network")
        field.solver_config["tol"] = float(solver_tol)
        field.solver_config["max_iter"] = int(solver_max_iter)
        normal_xyz = torch.cat([dec_svh.get_voxel_centers(d) for d in range(ad)])
        normal_value = torch.cat([feats.normal_features[d] for d in range(ad)])
        normal_weight = NORMAL_WEIGHT / normal_xyz.shape[0] * (voxel_size ** 2)        # models/nksr_net.py:103-104
        field.solve(xyz, normal_xyz, -normal_value, POS_WEIGHT / xyz.shape[0], normal_weight, 1.0,
                    fused_mode=fused_mode)
        field.set_mask_field(mask_field(self.network, feats, dec_svh, udf_svh, ad, voxel_size))
        field._n_normal = int(normal_xyz.shape[0])
        return field

    def reconstruct(self, xyz: torch.Tensor, normal: Optional[torch.Tensor] = None,
                    sensor: Optional[torch.Tensor] = None, detail_level: Optional[float] = 0.0,
                    voxel_size: Optional[float] = None, chunk_size: Optional[float] = None,
                    preprocess_fn: Optional[Callable] = None, approx_kernel_grad: bool = False,
                    solver_tol: float = 1.0e-5, fused_mode: bool = True, solver_max_iter: int = 2000):
        _lib.require_cuda(xyz, "xyz")
        xyz = xyz.detach().to(self.device, torch.float32).contiguous()
        normal = normal.detach().to(self.device, torch.float32).contiguous() if normal is not None else None
        sensor = sensor.detach().to(self.device, torch.float32).contiguous() if sensor is not None else None
        if chunk_size is not None and chunk_size > 0:
            if getattr(self.network, "structure", "encoder") == "predicted":
                # the blended field is meshed on one union hierarchy built from the points (SPEC S14), which a grown
                # per-chunk hierarchy would not match
                raise _lib.NksrError("chunk mode needs structure='encoder': chunked reconstruction on hierarchies grown "
                                     "from the predicted structure is not supported")
            # NKSR-USAGE.md:137: detail_level / voxel_size are not tunable in chunk mode
            voxel_size = DEFAULT_VOXEL_SIZE
            return self._reconstruct_chunks(xyz, normal, sensor, voxel_size, float(chunk_size), preprocess_fn,
                                            approx_kernel_grad, solver_tol, fused_mode, solver_max_iter)
        self._timer = _lib.StageTimer(self.device)
        if preprocess_fn is not None:
            xyz, normal, sensor = preprocess_fn(xyz, normal, sensor)
            xyz = xyz.contiguous()
            self._timer.mark("preprocess")
        if voxel_size is None:
            voxel_size = DEFAULT_VOXEL_SIZE if detail_level is None else voxel_size_from_detail(xyz, detail_level)
        field = self._reconstruct_one(xyz, normal, sensor, float(voxel_size), approx_kernel_grad, solver_tol,
                                      fused_mode, solver_max_iter)
        if isinstance(field, NeuralField):
            self.last_stats = dict(voxel_size=float(voxel_size), points=int(xyz.shape[0]), geometry="neural")
        else:
            self.last_stats = dict(field.solve_info, voxel_size=float(voxel_size), points=int(xyz.shape[0]),
                                   normal_locations=int(getattr(field, "_n_normal", 0)))
        return field

    def stage_times(self) -> dict:
        """CUDA-event time per stage (ms) of the last `reconstruct` call when NKSR_STAGE_TIMES=1 (synchronises)."""
        return self._timer.report()

    def _reconstruct_chunks(self, xyz, normal, sensor, voxel_size, chunk_size, preprocess_fn, approx_kernel_grad,
                            solver_tol, fused_mode, solver_max_iter, chunk_filter=None):
        if getattr(self.network, "geometry", "kernel") == "neural":
            # (also reached from dist.reconstruct_distributed) the chunks are blended as solved kernel fields
            raise _lib.NksrError("chunk mode does not support geometry='neural': the blended chunk field is built from "
                                 "kernel solves; build the network with geometry='kernel' or reconstruct without "
                                 "chunk_size")
        if getattr(self.network, "udf_enabled", False):
            # (also reached from dist.reconstruct_distributed) the blended field has no UDF hierarchy to mask with
            raise _lib.NksrError("chunk mode does not support udf.enabled: the blended chunk field has no UDF "
                                 "hierarchy; build the network with udf=dict(enabled=False) or reconstruct without "
                                 "chunk_size")
        self._timer = _lib.StageTimer(self.device, enabled=False)
        margin = voxel_size * (2 ** (self.tree_depth - 1)) * 2.0       # two coarsest voxels of overlap
        cidx = torch.floor(xyz / chunk_size).long()
        cores = torch.unique(cidx, dim=0)
        fields, kept, core_pts = [], [], []
        for k in range(cores.shape[0]):
            if chunk_filter is not None and not chunk_filter(k, cores.shape[0]):
                continue
            lo = cores[k].float() * chunk_size - margin
            hi = (cores[k].float() + 1.0) * chunk_size + margin
            m = ((xyz >= lo[None]) & (xyz < hi[None])).all(dim=1)
            cx = xyz[m]
            cn = normal[m] if normal is not None else None
            cs = sensor[m] if sensor is not None else None
            if preprocess_fn is not None:
                cx, cn, cs = preprocess_fn(cx, cn, cs)
            if cx.shape[0] < 16:
                continue
            f = self._reconstruct_one(cx.contiguous(), cn, cs, voxel_size, approx_kernel_grad, solver_tol, fused_mode,
                                      solver_max_iter)
            if torch.device(self.chunk_tmp_device) != self.device:
                f.to_(self.chunk_tmp_device)         # another GPU, or host memory (NKSR-USAGE.md:101)
            fields.append(f)
            kept.append(cores[k])
            inner = (torch.floor(cx / chunk_size).long() == cores[k][None]).all(dim=1)
            core_pts.append(cx[inner])
        if not fields:
            raise _lib.NksrError("no chunk contained enough points")
        union = None
        if chunk_filter is None:
            # all chunks are here: one hierarchy over the points the chunks kept, for the blended field's single mesh
            union = SparseFeatureHierarchy(voxel_size, self.tree_depth, self.device).build_point_splatting(
                torch.cat(core_pts).contiguous())
        return ChunkedField(fields, torch.stack(kept), chunk_size, margin=margin, union_svh=union,
                            compute_device=self.device, adaptive_depth=self.adaptive_depth)
