"""The structure-grown decoder hierarchy (DESIGN.md SPEC S16).

The reference's decoder does not run on the encoder hierarchy: level by level, top down, the structure head of the
decoder classifies every voxel it predicted for as empty (0), leaf (1) or subdivided (2), and the next finer level holds
the 8 children of every subdivided voxel (models/nksr_net.py:74-86; `dec_tmp_svh`).  `StructureGrowth` builds that
hierarchy T one level per step, from the logits of the level just decoded or from forced classes (teacher forcing:
`G.evaluate_voxel_status` of a ground-truth hierarchy G), and at the end the decoder hierarchy `dec_svh` of the kept
voxels.

    g = StructureGrowth(enc_svh, depth, adaptive_depth)
    for l in range(depth - 1, -1, -1):
        ...                                   # decode level l on g.T (skip input through g.skip27(l))
        g.step(l, logits=structure_logits_l)  # classifies T_l, appends T_{l-1}
    dec_svh = g.finish()

impl='cuda' runs the kernels of csrc/structure.cu (classification, the child emission with its tables, the table
composition) plus the existing scan / compaction / neighbour-table kernels; one host read-back per level sizes the
children.  impl='torch' is the plain-torch restatement of the same SPEC (argmax, keys by shift, join and neighbours by
searchsorted) that the tests compare the kernels with bit for bit; it runs on CPU tensors too.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import _lib
from ._lib import NksrError, call, stream_ptr
from .svh import SparseFeatureHierarchy

# children a level may hold, as a multiple of the encoder voxels of that level, before growth refuses
# (`structure_max_ratio`).  A surface's splat hierarchy occupies about half of the children of its voxels, so the full
# 8-child closure of a correct prediction (teacher forcing) is about 2x the encoder level; 4 leaves room for that and
# stops a random-weight network, which subdivides nearly everything (8^k times the coarsest count k levels down), long
# before it runs out of memory.
DEFAULT_MAX_RATIO = 4.0


# ---------------------------------------------------------------------------------------------------- torch helpers
def _spread3(v: torch.Tensor) -> torch.Tensor:
    out = torch.zeros_like(v)
    for b in range(21):
        out |= ((v >> b) & 1) << (3 * b)
    return out


def _compact3(k: torch.Tensor) -> torch.Tensor:
    out = torch.zeros_like(k)
    for b in range(21):
        out |= ((k >> (3 * b)) & 1) << b
    return out


def morton_encode(x, y, z):
    """63-bit Morton key of int64 voxel coordinates (SPEC S1: x in the highest bit of each triple)"""
    return (_spread3(x) << 2) | (_spread3(y) << 1) | _spread3(z)


def morton_decode(k):
    return _compact3(k >> 2), _compact3(k >> 1), _compact3(k)


def nbr27_torch(keys: torch.Tensor) -> torch.Tensor:
    """(n, 27) int32 same-level neighbour table of sorted keys by search (slot s: d = (s/9, s/3 % 3, s % 3) - 1)"""
    n = keys.numel()
    if n == 0:
        return torch.zeros((0, 27), dtype=torch.int32, device=keys.device)
    x, y, z = morton_decode(keys)
    s = torch.arange(27, device=keys.device)
    nx, ny, nz = x[:, None] + s // 9 - 1, y[:, None] + (s // 3) % 3 - 1, z[:, None] + s % 3 - 1
    lim = 1 << 21
    ok = (nx >= 0) & (ny >= 0) & (nz >= 0) & (nx < lim) & (ny < lim) & (nz < lim)
    nk = morton_encode(nx.clamp(0, lim - 1), ny.clamp(0, lim - 1), nz.clamp(0, lim - 1))
    return _lookup(keys, nk, ok)


def _lookup(keys, query, ok=None):
    """int32 index of every query key in the sorted keys, -1 when absent (or not ok)"""
    if keys.numel() == 0:
        return torch.full(query.shape, -1, dtype=torch.int32, device=query.device)
    pos = torch.searchsorted(keys, query.reshape(-1)).view(query.shape).clamp(max=keys.numel() - 1)
    hit = keys[pos] == query
    if ok is not None:
        hit &= ok
    return torch.where(hit, pos, torch.full_like(pos, -1)).to(torch.int32)


def classify_torch(logits: torch.Tensor, level: int, adaptive_depth: int, forced: Optional[torch.Tensor] = None):
    """SPEC S16 classes, keep and subdivide flags: c = torch.argmax of the logits (or the forced classes)"""
    c = forced.to(torch.int64) if forced is not None else torch.argmax(logits, dim=1)
    keep = c >= 1
    sub = (c == 2) | ((c == 1) & (level >= adaptive_depth)) if level >= 1 else torch.zeros_like(keep)
    return c.to(torch.int8), keep, sub


# ---------------------------------------------------------------------------------------------------- growth
class StructureGrowth:
    """Top-down construction of the grown hierarchy T (SPEC S16) over the encoder hierarchy `enc_svh`, `depth` levels
    (D <= enc_svh.depth).  T is a SparseFeatureHierarchy whose levels below the current one are empty until `step`
    appends them.  After `step(l)`: `classes[l]` (int8), `kept[l]` (int64 indices into T_l of the kept voxels),
    `join[l-1]` (int32 index into E_{l-1} of every voxel of T_{l-1}, or -1)."""

    def __init__(self, enc_svh: SparseFeatureHierarchy, depth: int, adaptive_depth: int,
                 max_ratio: Optional[float] = DEFAULT_MAX_RATIO, impl: str = "cuda"):
        E, D = enc_svh, int(depth)
        if not 1 <= D <= E.depth:
            raise ValueError(f"depth must be in 1..{E.depth}")
        self.E, self.D, self.adaptive_depth, self.impl = E, D, int(adaptive_depth), impl
        self.max_ratio = max_ratio
        dev = E.keys[0].device
        self.device = dev
        T = SparseFeatureHierarchy(E.voxel_size, D, dev)
        T.device = torch.device(dev)
        # the top level and everything above it are E's
        T.keys[D - 1] = E.keys[D - 1]
        T.parent[D - 1] = E.parent[D - 1]
        T.child8[D] = E.child8[D]
        T.nbr27[D] = E.nbr27[D]
        T.nbr27[D - 1] = E.nbr27[D - 1]
        T.top_keys = E.top_keys if D == E.depth else E.keys[D]
        T.nbr125_top = E.nbr125_top if D == E.depth else None
        for l in range(D - 1):
            T.parent[l] = torch.zeros(0, dtype=torch.int32, device=dev)
            T.child8[l + 1] = torch.zeros((0, 8), dtype=torch.int32, device=dev)
            T.nbr27[l] = torch.zeros((0, 27), dtype=torch.int32, device=dev)
        self.T = T
        self.join: Dict[int, torch.Tensor] = {
            D - 1: torch.arange(E.num_voxels(D - 1), dtype=torch.int32, device=dev)}
        self.classes: Dict[int, torch.Tensor] = {}
        self.kept: Dict[int, torch.Tensor] = {}
        self._kept_keys: Dict[int, torch.Tensor] = {}
        self._skip: Dict[int, torch.Tensor] = {}

    # ------------------------------------------------------------------ tables
    def skip27(self, l: int) -> torch.Tensor:
        """(|T_l|, 27) int32: join_l of every neighbour of T.nbr27[l] -- the gather table of E's encoder output x_l onto
        T_l (-1 where the neighbour is absent or not in E).  Injective per tap, since join is."""
        if l not in self._skip:
            nbr, join = self.T.nbr27[l], self.join[l]
            if self.impl == "torch":
                out = torch.where(nbr >= 0, join.long()[nbr.long().clamp(min=0)], torch.full_like(nbr.long(), -1))
                self._skip[l] = out.to(torch.int32)
            else:
                out = torch.empty_like(nbr)
                call("nksr_compose_taps", nbr, nbr.shape[0], 27, join, out, stream_ptr(nbr.device))
                self._skip[l] = out
        return self._skip[l]

    # ------------------------------------------------------------------ one level
    def step(self, l: int, logits: Optional[torch.Tensor] = None, forced: Optional[torch.Tensor] = None):
        """classify T_l from its structure logits (n, 3) -- any row stride -- or from forced classes (n,), record the
        kept voxels and, for l >= 1, append T_{l-1}.  An empty T_l leaves every finer level empty."""
        T, E = self.T, self.E
        keys = T.keys[l]
        n = keys.numel()
        if forced is None and logits is None:
            raise ValueError("step needs the structure logits or forced classes")
        src = forced if forced is not None else logits
        if src.shape[0] != n:
            raise ValueError(f"level {l}: {src.shape[0]} classes / logits for {n} voxels")
        dev = self.device
        if self.impl == "torch":
            cls, keep, sub = classify_torch(logits, l, self.adaptive_depth, forced)
            kept = torch.nonzero(keep).squeeze(1)
            sub_idx = torch.nonzero(sub).squeeze(1)
            n_sub = int(sub_idx.numel())
        else:
            st = stream_ptr(dev)
            cls = torch.empty(n, dtype=torch.int8, device=dev)
            keep = torch.empty(n, dtype=torch.int32, device=dev)
            sub = torch.empty(n, dtype=torch.int32, device=dev)
            if forced is not None:
                call("nksr_structure_classify", None, 0, forced.to(torch.int32).contiguous(), n, l,
                     self.adaptive_depth, cls, keep, sub, st)
            else:
                lg = logits.detach()
                if lg.dtype != torch.float32 or lg.stride(1) != 1:
                    lg = lg.to(torch.float32).contiguous()
                call("nksr_structure_classify", lg, lg.stride(0) if n else 3, None, n, l, self.adaptive_depth, cls,
                     keep, sub, st)
            keep_scan = _lib.exclusive_scan32(keep)
            sub_scan = _lib.exclusive_scan32(sub)
            n_kept, n_sub = (int(v) for v in torch.stack([keep_scan[-1], sub_scan[-1]]).tolist())   # the read-back
            kept = _lib.compact_rows(torch.arange(n, dtype=torch.int64, device=dev), keep, keep_scan, n_kept)
            self._kept_keys[l] = _lib.compact_rows(keys, keep, keep_scan, n_kept)
        self.classes[l], self.kept[l] = cls, kept
        if l == 0:
            return
        n_child = 8 * n_sub
        n_enc = E.num_voxels(l - 1)
        if self.max_ratio is not None and n_child > self.max_ratio * max(n_enc, 1):
            raise NksrError(f"predicted structure: level {l - 1} would hold {n_child} voxels, more than "
                            f"structure_max_ratio = {self.max_ratio} x its {n_enc} encoder voxels")
        enc_child8 = E.child8[l]
        if self.impl == "torch":
            o = torch.arange(8, device=dev)
            ckeys = ((keys[sub_idx][:, None] << 3) | o).reshape(-1)
            cparent = sub_idx.repeat_interleave(8).to(torch.int32)
            child8 = torch.full((n, 8), -1, dtype=torch.int32, device=dev)
            child8[sub_idx] = torch.arange(n_child, dtype=torch.int32, device=dev).view(n_sub, 8)
            cjoin = _lookup(E.keys[l - 1], ckeys)
            cnbr = nbr27_torch(ckeys)
        else:
            ckeys = torch.empty(n_child, dtype=torch.int64, device=dev)
            cparent = torch.empty(n_child, dtype=torch.int32, device=dev)
            cjoin = torch.empty(n_child, dtype=torch.int32, device=dev)
            child8 = torch.empty((n, 8), dtype=torch.int32, device=dev)
            call("nksr_structure_grow", keys, sub, sub_scan, n, self.join[l], enc_child8, ckeys, cparent, cjoin,
                 child8, st)
            cnbr = torch.empty((n_child, 27), dtype=torch.int32, device=dev)
            call("nksr_nbr27_from_parent", ckeys, cparent, n_child, T.nbr27[l], child8, cnbr, st)
        T.keys[l - 1], T.parent[l - 1], T.child8[l], T.nbr27[l - 1] = ckeys, cparent, child8, cnbr
        self.join[l - 1] = cjoin
        T._view = None

    # ------------------------------------------------------------------ result
    def finish(self, dec: Optional[SparseFeatureHierarchy] = None) -> SparseFeatureHierarchy:
        """dec_svh: build_from_keys of the kept keys of every level (above them E's virtual level), with
        adaptive_depth set so that meshing treats its leaves as SPEC S8b says.  `dec`: the (depth-D) hierarchy
        object to build into, else a new one."""
        keys = []
        for l in range(self.D):
            if l not in self.kept:
                raise NksrError(f"level {l} of the grown hierarchy was never classified")
            keys.append(self._kept_keys[l] if l in self._kept_keys else self.T.keys[l][self.kept[l]])
        if dec is None:
            dec = SparseFeatureHierarchy(self.E.voxel_size, self.D, self.device)
        elif dec.depth != self.D:
            raise ValueError(f"the decoder hierarchy has depth {dec.depth}, the grown one {self.D}")
        dec.build_from_keys(keys, top_keys=self.T.top_keys)
        dec.adaptive_depth = min(self.adaptive_depth, self.D)
        return dec


def grow_from_classes(enc_svh: SparseFeatureHierarchy, classes_by_level, adaptive_depth: int, impl: str = "cuda",
                      max_ratio: Optional[float] = None, dec: Optional[SparseFeatureHierarchy] = None):
    """(dec_svh, growth) for explicit classes: classes_by_level[l] is a tensor of T_l's classes or a function
    (T, l) -> classes, for l = D-1 .. 0 with D = len(classes_by_level)"""
    D = len(classes_by_level)
    g = StructureGrowth(enc_svh, D, adaptive_depth, max_ratio=max_ratio, impl=impl)
    for l in range(D - 1, -1, -1):
        c = classes_by_level[l]
        g.step(l, forced=c(g.T, l) if callable(c) else c)
    return g.finish(dec), g


def teacher_classes(gt_svh: SparseFeatureHierarchy):
    """the forced classes of teacher forcing: (T, l) -> gt_svh.evaluate_voxel_status of T_l"""
    from .svh import SparseIndexGrid
    return lambda T, l: gt_svh.evaluate_voxel_status(SparseIndexGrid(T, l), l)
