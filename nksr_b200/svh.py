"""SparseFeatureHierarchy -- host mirror of nksr.SparseFeatureHierarchy.

Reference contract (closed wheel; call sites only):
  ctor (voxel_size, depth, device)            models/nksr_net.py:57-61
  build_point_splatting(xyz)                  models/nksr_net.py:62
  grids[d] (None when empty)                  models/nksr_net.py:80, models/loss.py:34
  get_voxel_centers(d)                        models/nksr_net.py:100
  grid.active_grid_coords/grid_to_world/voxel_size   models/loss.py:36,45,46
All arithmetic runs in libnksr_b200.so (csrc/svh.cu); this file only owns tensors.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import _lib
from ._lib import call, stream_ptr


class SparseIndexGrid:
    """One level of the hierarchy (what the reference exposes as `svh.grids[d]`)."""

    def __init__(self, svh: "SparseFeatureHierarchy", level: int):
        self._svh = svh
        self.level = level
        self.voxel_size = float(svh.voxel_size * (2 ** level))

    @property
    def num_voxels(self) -> int:
        return int(self._svh.keys[self.level].numel())

    def active_grid_coords(self) -> torch.Tensor:
        """(n,3) int32 voxel ijk (models/loss.py:36)."""
        keys = self._svh.keys[self.level]
        ijk = torch.empty((keys.numel(), 3), dtype=torch.int32, device=keys.device)
        call("nksr_decode_ijk", keys, keys.numel(), self.level, ijk, stream_ptr(keys.device))
        return ijk

    def grid_to_world(self, ijk: torch.Tensor) -> torch.Tensor:
        """voxel index space -> world; integer ijk maps to the voxel CENTRE (models/loss.py:45-50)."""
        return (ijk.to(torch.float32) + 0.5) * self.voxel_size

    def world_to_grid(self, xyz: torch.Tensor) -> torch.Tensor:
        return xyz / self.voxel_size - 0.5


class SparseFeatureHierarchy:
    def __init__(self, voxel_size: float, depth: int, device):
        if not (1 <= depth <= _lib.MAX_DEPTH):
            raise ValueError(f"depth must be in 1..{_lib.MAX_DEPTH}")
        self.voxel_size = float(torch.tensor(voxel_size, dtype=torch.float32).item())
        self.depth = depth
        self.device = torch.device(device)
        self.keys: List[torch.Tensor] = [torch.zeros(0, dtype=torch.int64, device=self.device) for _ in range(depth)]
        # tables have one extra slot: index `depth` is the virtual level above the coarsest one
        self.parent: List[Optional[torch.Tensor]] = [None] * (depth + 1)
        self.child8: List[Optional[torch.Tensor]] = [None] * (depth + 1)
        self.nbr27: List[Optional[torch.Tensor]] = [None] * (depth + 1)
        self.top_keys: Optional[torch.Tensor] = None
        self.nbr125_top: Optional[torch.Tensor] = None
        self._view = None

    # ------------------------------------------------------------------ construction
    def build_point_splatting(self, xyz: torch.Tensor):
        """Activate, on every level, the 8 voxels whose centres surround each point
        (DESIGN.md SPEC S2).  Replaces models/nksr_net.py:62."""
        _lib.require_cuda(xyz, "xyz")
        xyz = xyz.detach().to(torch.float32).contiguous()
        dev, st = xyz.device, stream_ptr(xyz.device)
        n = xyz.shape[0]
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        hk = torch.empty(n, dtype=torch.int64, device=dev)
        call("nksr_point_half_keys", xyz, n, self.voxel_size, hk, status, st)
        uh = _lib.unique_sorted(_lib.sort_keys(hk))
        if int(status.item()) & 1:
            raise _lib.NksrError("point coordinates outside the supported range (|x| < 2^19 voxels) or non-finite")
        keys = []
        # one extra, VIRTUAL level on top (no unknowns): it parents the coarsest real level so that
        # every level finds its 125-neighbourhood through parent tables and can be grouped by parent
        for l in range(self.depth + 1):
            cand = torch.empty(uh.numel() * 8, dtype=torch.int64, device=dev)
            call("nksr_splat_candidates", uh, uh.numel(), cand, st)
            keys.append(_lib.unique_sorted(_lib.sort_keys(cand)))
            if l < self.depth:
                uh = _lib.unique_sorted(uh, 3)
        return self.build_from_keys(keys[:self.depth], top_keys=keys[self.depth])

    def build_adaptive_normal_variation(self, xyz: torch.Tensor, normal: torch.Tensor, tau: float = 0.2,
                                        adaptive_depth: int = 2):
        """Adaptive hierarchy for ground-truth decoders (models/nksr_net.py:175-179): start from the
        splatted hierarchy; a voxel of one of the finest `adaptive_depth` levels (but not level 0)
        whose points have consistent normals -- variation 1 - |mean normal| below `tau` -- or that holds
        no point at all (splat-only) becomes a leaf and every finer voxel below it is dropped.  Coarser levels are always subdivided.
        Training-side helper: plain torch on top of the CUDA tables (outside the hot path)."""
        self.build_point_splatting(xyz)
        normal = normal.detach().to(self.device, torch.float32)
        base = self.locate(xyz.detach().to(self.device, torch.float32).contiguous()).long()
        keys = [k.clone() for k in self.keys]
        drop = [torch.zeros(k.numel(), dtype=torch.bool, device=self.device) for k in keys]
        for l in range(min(adaptive_depth, self.depth) - 1, 0, -1):
            n = keys[l].numel()
            acc = torch.zeros((n, 4), device=self.device)
            ok = base[l] >= 0
            acc.index_add_(0, base[l][ok], torch.cat([normal[ok], torch.ones((int(ok.sum()), 1), device=self.device)], 1))
            variation = 1.0 - acc[:, :3].norm(dim=1) / acc[:, 3].clamp(min=1.0)
            leaf = ((variation < tau) | (acc[:, 3] == 0)) & ~drop[l]      # point-free (splat-only) voxels are leaves too
            stop = leaf | drop[l]                           # everything below a leaf (or a dropped voxel) goes
            drop[l - 1] |= stop[self.parent[l - 1].long()]
        out = self.build_from_keys([k[~d] for k, d in zip(keys, drop)], top_keys=self.top_keys)
        # leaves exist on the levels below `adaptive_depth`: extract_dual_mesh meshes them as if subdivided
        self.adaptive_depth = min(int(adaptive_depth), self.depth)
        return out

    def build_from_structure(self, enc_svh: "SparseFeatureHierarchy", classes_by_level, adaptive_depth: int):
        """The decoder hierarchy grown from explicit structure classes over an encoder hierarchy (DESIGN.md SPEC S16):
        classes_by_level[l] (0 empty, 1 leaf, 2 subdivide) for every voxel of level l of the grown hierarchy T, or a
        function (T, l) -> those classes, for the levels 0 .. self.depth - 1 (T's coarsest level is enc_svh's).  This
        hierarchy becomes the kept voxels of T; `adaptive_depth` says below which level a leaf stays a leaf."""
        from .structure import grow_from_classes
        if len(classes_by_level) != self.depth:
            raise ValueError(f"{len(classes_by_level)} levels of classes for a depth-{self.depth} hierarchy")
        grow_from_classes(enc_svh, classes_by_level, adaptive_depth, dec=self)
        return self

    def build_from_keys(self, keys, top_keys=None):
        """Adopt sorted, unique, parent-closed Morton keys per level and build the tables.
        `top_keys`: keys of the virtual level above the coarsest one (default: its parents)."""
        self.keys = [k.to(self.device, torch.int64).contiguous() for k in keys]
        dev, st = self.device, stream_ptr(self.device)
        L = self.depth
        if top_keys is None:
            top_keys = _lib.unique_sorted(self.keys[L - 1], 3)
        self.top_keys = top_keys.to(dev, torch.int64).contiguous()
        allk = self.keys + [self.top_keys]
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        for l in range(L):
            n, nu = allk[l].numel(), allk[l + 1].numel()
            self.parent[l] = torch.empty(n, dtype=torch.int32, device=dev)
            call("nksr_parent_index", allk[l], n, allk[l + 1], nu, self.parent[l], status, st)
            self.child8[l + 1] = torch.empty((nu, 8), dtype=torch.int32, device=dev)
            call("nksr_child_table", allk[l], self.parent[l], n, self.child8[l + 1], nu, st)
        self.nbr27[L] = torch.empty((self.top_keys.numel(), 27), dtype=torch.int32, device=dev)
        call("nksr_nbr27_search", self.top_keys, self.top_keys.numel(), self.nbr27[L], st)
        if L >= _lib.MAX_DEPTH:        # no room for the virtual level in the C view: explicit 5^3 table instead
            top = self.keys[L - 1]
            self.nbr125_top = torch.empty((top.numel(), 125), dtype=torch.int32, device=dev)
            call("nksr_nbr125_search", top, top.numel(), self.nbr125_top, st)
        else:
            self.nbr125_top = None
        for l in range(L - 1, -1, -1):
            n = self.keys[l].numel()
            self.nbr27[l] = torch.empty((n, 27), dtype=torch.int32, device=dev)
            call("nksr_nbr27_from_parent", self.keys[l], self.parent[l], n, self.nbr27[l + 1], self.child8[l + 1],
                 self.nbr27[l], st)
        if int(status.item()) & 2:
            raise _lib.NksrError("hierarchy is not parent-closed (a voxel has no parent on the next level)")
        self._view = None
        return self

    # ------------------------------------------------------------------ accessors
    @property
    def grids(self):
        return [SparseIndexGrid(self, l) if self.keys[l].numel() > 0 else None for l in range(self.depth)]

    def num_voxels(self, l: int) -> int:
        return int(self.keys[l].numel())

    @property
    def offsets(self):
        out, acc = [], 0
        for l in range(self.depth):
            out.append(acc)
            acc += self.num_voxels(l)
        return out + [acc]

    @property
    def num_unknowns(self) -> int:
        return self.offsets[-1]

    def get_voxel_centers(self, d: int) -> torch.Tensor:
        g = SparseIndexGrid(self, d)
        return g.grid_to_world(g.active_grid_coords())

    def view(self) -> _lib.SvhT:
        """C struct handed to the kernels (pointers stay valid while this object lives)."""
        if torch.device(self.device).type != "cuda":
            raise _lib.NksrError("this hierarchy is parked in host memory: move it back with to_(<cuda device>) "
                                 "(nksr_b200 has no CPU path)")
        if self._view is None:
            v = _lib.SvhT()
            v.depth = self.depth
            v.voxel_size = self.voxel_size
            offs = self.offsets
            for l in range(self.depth):
                v.n[l] = self.num_voxels(l)
                v.offset[l] = offs[l]
                v.keys[l] = self.keys[l].data_ptr()
                v.parent[l] = self.parent[l].data_ptr() if self.parent[l] is not None else None
                v.child8[l] = self.child8[l].data_ptr() if self.child8[l] is not None else None
                v.nbr27[l] = self.nbr27[l].data_ptr() if self.nbr27[l] is not None else None
            v.nbr125_top = self.nbr125_top.data_ptr() if self.nbr125_top is not None else None
            L = self.depth
            if L < _lib.MAX_DEPTH and self.top_keys is not None:          # virtual level at index L
                v.n[L] = self.top_keys.numel()
                v.offset[L] = offs[L]
                v.keys[L] = self.top_keys.data_ptr()
                v.child8[L] = self.child8[L].data_ptr()
                v.nbr27[L] = self.nbr27[L].data_ptr()
            else:
                v.parent[L - 1] = None
            self._view = v
        return self._view

    def locate(self, xyz: torch.Tensor) -> torch.Tensor:
        """(depth, M) int32 containing-voxel index per level, -1 when inactive."""
        xyz = xyz.to(torch.float32).contiguous()
        base = torch.empty((self.depth, xyz.shape[0]), dtype=torch.int32, device=xyz.device)
        call("nksr_locate", self.view(), xyz, xyz.shape[0], base, stream_ptr(xyz.device))
        return base

    def evaluate_voxel_status(self, grid: SparseIndexGrid, d: int) -> torch.Tensor:
        """Training target of the structure head (models/loss.py:155): for every voxel of `grid`
        (level d of another hierarchy) 0 = absent here, 1 = present as a leaf, 2 = present with
        children.  Plain torch (training-only, outside the hot path)."""
        other = grid._svh.keys[d]
        mine = self.keys[d]
        if mine.numel() == 0:
            return torch.zeros(other.numel(), dtype=torch.long, device=other.device)
        pos = torch.searchsorted(mine, other).clamp(max=mine.numel() - 1)
        present = mine[pos] == other
        status = present.long()
        if d > 0 and self.child8[d] is not None:
            has_child = (self.child8[d] >= 0).any(dim=1)
            status = torch.where(present & has_child[pos], torch.full_like(status, 2), status)
        return status

    def get_visualization(self):
        return [self.get_voxel_centers(l) for l in range(self.depth) if self.num_voxels(l)]

    def to_(self, device):
        device = torch.device(device)
        # a CPU device only PARKS the tables in host memory (chunk_tmp_device = cpu, NKSR-USAGE.md:101): nothing can be
        # computed there -- view() refuses until the hierarchy is moved back to a CUDA device
        self.device = device
        self.keys = [k.to(device) for k in self.keys]
        for name in ("parent", "child8", "nbr27"):
            setattr(self, name, [t.to(device) if t is not None else None for t in getattr(self, name)])
        if self.nbr125_top is not None:
            self.nbr125_top = self.nbr125_top.to(device)
        if self.top_keys is not None:
            self.top_keys = self.top_keys.to(device)
        self._view = None
        return self
