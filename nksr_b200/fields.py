"""Implicit fields -- host mirror of nksr.fields.{KernelField, NeuralField, LayerField, PCNNField}.

Reference contract (closed wheel; call sites only):
  KernelField(svh, interpolator, features, approx_kernel_grad)      models/nksr_net.py:91-96
  .solver_config['verbose']                                          models/nksr_net.py:97-98
  .solve_non_fused(pos_xyz, normal_xyz, normal_value, pos_weight,
                   normal_weight, reg_weight)                        models/nksr_net.py:105-112
  .evaluate_f(xyz, grad) -> .value / .gradient ; .evaluate_f_bar     models/loss.py:99,189-198,225
  .set_mask_field / .set_texture_field / .to_ / .extract_dual_mesh   models/nksr_net.py:133,214,284
  NeuralField(svh, decoder, features).set_level_set(v)               models/nksr_net.py:115-130
  LayerField(svh, adaptive_depth)                                    models/nksr_net.py:132
  PCNNField(xyz, color)                                              examples/recons_colored_mesh.py:28
The arithmetic is in libnksr_b200.so; the algorithm is fixed in DESIGN.md (SPEC S3-S7).
"""
from __future__ import annotations

import ctypes as C
import os
import warnings
from types import SimpleNamespace
from typing import Optional

import torch

from . import _lib
from ._lib import call, stream_ptr
from .svh import SparseFeatureHierarchy

# where the transposed (finer-level) Gram entries go: "sorted" = atomic cursor + per-row segment sort,
# "structural" = straight to the final slot from prefix tables (SPEC S6b).  solver_config['placement'] or the
# NKSR_PLACEMENT environment variable override it.
DEFAULT_PLACEMENT = "structural"
# the layout every parity test runs on unless a test selects the other
DEFAULT_ROW_LAYOUT = "levels"
# the Gram fill (solver_config['fill'] or the NKSR_FILL environment variable override it): "brick", "rows", "grouped"
DEFAULT_FILL = "brick"
# 'brick' bricks a fine level only when it holds at least this many constraint locations per voxel (measured on H100:
# faster at 18 per voxel, slower at 1.7 and 4.9; DESIGN 4.1)
BRICK_MIN_LOCATIONS_PER_VOXEL = 8.0


_TOTAL_MEMORY = {}


def _total_memory(dev) -> int:
    key = torch.device(dev).index or 0
    if key not in _TOTAL_MEMORY:
        _TOTAL_MEMORY[key] = int(torch.cuda.get_device_properties(dev).total_memory * 0.94)   # driver / context reserve
    return _TOTAL_MEMORY[key]


class EvaluationResult(SimpleNamespace):
    """`.value` (M,) and `.gradient` (M,3) as consumed at models/loss.py:189-198."""


class BaseField:
    def __init__(self, svh: SparseFeatureHierarchy):
        self.svh = svh
        self.mask_field: Optional["BaseField"] = None
        self.texture_field = None
        self.level_set = 0.0

    def set_mask_field(self, mask_field):
        self.mask_field = mask_field

    def set_texture_field(self, texture_field):
        self.texture_field = texture_field

    def set_level_set(self, v: float):
        self.level_set = float(v)

    def evaluate_f(self, xyz: torch.Tensor, grad: bool = False) -> EvaluationResult:
        raise NotImplementedError

    def mask(self, xyz: torch.Tensor) -> torch.Tensor:
        """bool (M,): True where geometry is kept by this field used as a mask."""
        raise NotImplementedError

    def to_(self, device):
        self.svh.to_(device)
        if self.mask_field is not None:
            self.mask_field.to_(device)
        return self

    def extract_dual_mesh(self, grid_upsample: int = 1, mise_iter: int = 0, max_points: int = -1, cell_filter=None):
        from .meshing import extract_dual_mesh
        return extract_dual_mesh(self, grid_upsample=grid_upsample, mise_iter=mise_iter, max_points=max_points,
                                 cell_filter=cell_filter)


def _as_level_list(features, depth):
    if isinstance(features, dict):
        return [features.get(d, None) for d in range(depth)]
    return [features[d] if d < len(features) else None for d in range(depth)]


_SIDE_STREAMS = {}


def _side_stream(dev):
    """one side stream per device for the life of the process (the caching allocator keeps a pool per stream)"""
    key = torch.device(dev).index if torch.device(dev).index is not None else torch.cuda.current_device()
    if key not in _SIDE_STREAMS:
        _SIDE_STREAMS[key] = torch.cuda.Stream(torch.device("cuda", key))
    return _SIDE_STREAMS[key]


class KernelField(BaseField):
    def __init__(self, svh: SparseFeatureHierarchy, interpolator=None, features=None,
                 approx_kernel_grad: bool = False):
        super().__init__(svh)
        self.approx_kernel_grad = bool(approx_kernel_grad)
        # check_every = iterations per CUDA-graph launch (one host read-back of the device-side verdict each)
        self.solver_config = {"verbose": False, "tol": 1.0e-5, "max_iter": 2000, "check_every": 32}
        self.interpolator = interpolator
        self.alpha: Optional[torch.Tensor] = None
        self.solve_info = {}
        self.system = None          # kept for inspection / tests when solver_config['keep_system']
        self._set_features(features)

    # -- features: z_l = interpolator_l(basis_features_l), one (n_l, C) fp32 block per level
    def _set_features(self, features):
        depth, dev = self.svh.depth, self.svh.device
        feats = _as_level_list(features, depth)
        z, C_ = [], None
        for l in range(depth):
            f = feats[l]
            n = self.svh.num_voxels(l)
            if f is None:
                z.append(None)
                continue
            if f.shape[0] != n:
                raise ValueError(f"features[{l}] has {f.shape[0]} rows but level {l} has {n} voxels")
            f = f.detach().to(dev, torch.float32)
            if self.interpolator is not None:
                mod = self.interpolator[l] if not isinstance(self.interpolator, dict) else self.interpolator[str(l)]
                with torch.no_grad():
                    f = mod(f)
            f = f.contiguous()
            if f.data_ptr() % 16:                     # the kernels fetch four channels per 128-bit load
                f = f.clone()
            C_ = f.shape[1] if C_ is None else C_
            if f.shape[1] != C_:
                raise ValueError("all levels must share one kernel_dim")
            z.append(f)
        if C_ is None:
            raise ValueError("KernelField needs basis features on at least one level")
        if not (1 <= C_ <= 32):
            raise ValueError("kernel_dim must be in 1..32")
        self.z = [t if t is not None else torch.zeros((self.svh.num_voxels(l), C_), device=dev)
                  for l, t in enumerate(z)]
        self.channels = C_
        self._feat_view = None

    def feat_view(self) -> _lib.FeatT:
        if self._feat_view is None:
            v = _lib.FeatT()
            v.channels = self.channels
            for l in range(self.svh.depth):
                v.z[l] = self.z[l].data_ptr()
            self._feat_view = v
        return self._feat_view

    # ------------------------------------------------------------------ solve
    def _sorted_rows(self, xyz: torch.Tensor, mode: int, extra: Optional[torch.Tensor] = None,
                     interleaved: bool = False):
        """Morton-sort locations, locate them on every level, build their kernel rows.
        `interleaved` (depth <= 4, modes 0 / 1): rows as (m, rows, 32, 4 levels) -- the four levels of a slot are one
        float4 -- instead of (m, depth, rows * 32)."""
        svh, dev = self.svh, xyz.device
        st = stream_ptr(dev)
        m = xyz.shape[0]
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        hk = torch.empty(m, dtype=torch.int64, device=dev)
        call("nksr_point_half_keys", xyz, m, svh.voxel_size, hk, status, st)
        if int(status.item()) & 1:
            raise _lib.NksrError("constraint locations outside the supported range (|x| < 2^19 voxels) or non-finite")
        _, perm = _lib.sort_pairs(hk, torch.arange(m, dtype=torch.int32, device=dev))
        perm = perm.long()
        xs = xyz[perm].contiguous()
        ex = extra[perm].contiguous() if extra is not None else None
        base = svh.locate(xs)
        n_total = svh.num_unknowns
        ranges = torch.empty((n_total, 2), dtype=torch.int32, device=dev)
        offs = svh.offsets
        for l in range(svh.depth):
            call("nksr_row_ranges", base[l], m, ranges[offs[l]:], svh.num_voxels(l), st)
        width = _lib.ROW_STRIDE * (3 if mode == 1 else 1)
        if interleaved:
            if svh.depth > 4 or mode == 2:
                raise _lib.NksrError("interleaved rows: depth <= 4, value or gradient rows")
            e = torch.empty((m, width // _lib.ROW_STRIDE, _lib.ROW_STRIDE, 4), dtype=torch.float32, device=dev)
            call("nksr_build_rows", svh.view(), self.feat_view(), xs, base, m, mode | 4,
                 int(self.approx_kernel_grad), e, st)
            return xs, ex, base, ranges, e
        e = torch.empty((m, svh.depth, width), dtype=torch.float32, device=dev)      # location-major
        # 'location' (default): one warp per location (any channel count); 'voxel': one warp per voxel, stencil +
        # features fetched once for all the voxel's locations (bitwise the same rows)
        # ('voxel' saves gathers, but its per-level launches and zero pass cost about as much)
        rows = self.solver_config.get("rows") or os.environ.get("NKSR_ROWS") or "location"
        if rows == "voxel" and self.z[0].shape[1] in (4, 8, 16):
            call("nksr_build_rows_voxel", svh.view(), self.feat_view(), xs, base, ranges, m, mode,
                 int(self.approx_kernel_grad), e, st)
        else:
            call("nksr_build_rows", svh.view(), self.feat_view(), xs, base, m, mode,
                 int(self.approx_kernel_grad), e, st)
        return xs, ex, base, ranges, e

    def solve(self, pos_xyz, normal_xyz=None, normal_value=None, pos_weight=1.0, normal_weight=1.0,
              reg_weight=1.0, fused_mode: bool = False):
        """Assemble A = E^T W E + reg R (CSR) and solve A alpha = E^T W t with Jacobi-PCG."""
        sysm = self.assemble(pos_xyz, normal_xyz, normal_value, pos_weight, normal_weight, reg_weight)
        dev, n = self.svh.device, sysm.n
        tm = getattr(self, "_timer", None) or _lib.StageTimer(dev, enabled=False)
        alpha = torch.empty(n, dtype=torch.float32, device=dev)
        info = (C.c_double * 8)()
        profile = int(bool(self.solver_config.get("profile")))
        # 'rows' (default): one warp per row with register loads (csrc/solve.cu); 'stream': the CSR arrays reach the SMs
        # as tiles moved by bulk async copies (TMA engine) into a shared-memory ring (csrc/spmv_stream.cuh)
        spmv = self.solver_config.get("spmv") or os.environ.get("NKSR_SPMV") or "rows"
        if spmv not in ("stream", "rows"):
            raise ValueError("solver_config['spmv'] must be 'stream' or 'rows'")
        if spmv == "stream":
            nb = call("nksr_pcg_stream_workspace_bytes", n, sysm.nnz)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            # rows of the two finest levels are streamed; the coarse rows (transposed segments of up to tens of
            # thousands of entries) go warp per row, where a long row streams well and cannot hold a tile up
            offs = self.svh.offsets
            split_row = offs[2] if self.svh.depth > 2 else n
            split_nnz = int(sysm.rowptr[split_row].item()) if split_row < n else sysm.nnz
            call("nksr_pcg_solve_stream", sysm.rowptr, sysm.col, sysm.val, sysm.diag, sysm.rhs, alpha, n, sysm.nnz,
                 split_row, split_nnz, float(self.solver_config["tol"]), int(self.solver_config["max_iter"]),
                 int(self.solver_config["check_every"]), profile, ws, nb, info, stream_ptr(dev))
        else:
            nb = call("nksr_pcg_workspace_bytes", n)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            call("nksr_pcg_solve", sysm.rowptr, sysm.col, sysm.val, sysm.diag, sysm.rhs, alpha, n,
                 float(self.solver_config["tol"]), int(self.solver_config["max_iter"]),
                 int(self.solver_config["check_every"]), profile, ws, nb, info, stream_ptr(dev))
        tm.mark("pcg")
        self.alpha = alpha
        status = int(info[4])                       # 0 converged, 1 max_iter reached, 2 NaN / breakdown
        self.solve_info = {"iterations": int(info[0]), "relative_residual": float(info[1]), "n": n, "nnz": sysm.nnz,
                           "converged": status == 0}
        if status == 2:
            raise _lib.NksrError(f"PCG broke down (non-finite residual) after {int(info[0])} iterations: the system "
                                 "is not positive definite or the inputs are not finite")
        if status == 1 and int(self.solver_config["max_iter"]) > 0:
            warnings.warn(f"nksr_b200 PCG stopped at max_iter={int(self.solver_config['max_iter'])} with relative "
                          f"residual {float(info[1]):.3e} > tol={float(self.solver_config['tol']):.1e}", RuntimeWarning)
        if profile:
            self.solve_info.update(spmv_ms=float(info[2]), spmv_launches=int(info[3]))
        if self.solver_config.get("verbose"):
            print(f"[nksr_b200] PCG: n={n} nnz={sysm.nnz} iters={int(info[0])} relres={float(info[1]):.3e}")
        if self.solver_config.get("keep_system"):
            self.system = sysm
        return self

    def _count_and_place(self, n, keep):
        """structure-only part of the assembly (row lengths, placement tables, row pointers): depends on the hierarchy
        alone, so it may run on a side stream while the kernel rows are built (solver_config['overlap_count'])"""
        svh = self.svh
        dev = svh.device
        st = stream_ptr(dev)
        cnt = torch.empty(n, dtype=torch.int32, device=dev)
        placement = self.solver_config.get("placement") or os.environ.get("NKSR_PLACEMENT") or DEFAULT_PLACEMENT
        if placement not in ("sorted", "structural"):
            raise ValueError("solver_config['placement'] must be 'sorted' or 'structural'")
        place = None
        if placement == "structural":
            # transposed entries go straight to their final slot (SPEC S6b): per (fine level, offset) pair
            # a rank table on the fine level and a 125-ancestor prefix table on the coarse level
            cnt_down = torch.zeros(n, dtype=torch.int32, device=dev)
            # row lengths with one column table per sibling group (fewer lookups than a walk per slot and row)
            count = self.solver_config.get("count") or os.environ.get("NKSR_COUNT") or "grouped"
            grouped = count == "grouped" and svh.depth <= 4 and svh.depth < _lib.MAX_DEPTH
            call("nksr_gram_count_grouped" if grouped else "nksr_gram_count_own", svh.view(), cnt, st)
            place = _lib.PlacementT()
            for l in range(svh.depth - 1):
                for k in range(1, svh.depth - l):
                    n_lo, n_up = svh.num_voxels(l), svh.num_voxels(l + k)
                    if n_lo == 0 or n_up == 0:
                        continue
                    rank8 = torch.empty((n_lo, 8), dtype=torch.int32, device=dev)
                    classes = torch.empty((n_up, 27), dtype=torch.int32, device=dev)
                    prefix = torch.empty((n_up, 125), dtype=torch.int32, device=dev)
                    call("nksr_gram_place", svh.view(), l, k, rank8, classes, prefix, cnt_down, st)
                    place.rank8[l][k], place.prefix[l][k] = rank8.data_ptr(), prefix.data_ptr()
                    keep += [rank8, prefix]
        else:
            cnt_down = torch.empty(n, dtype=torch.int32, device=dev)
            call("nksr_gram_count", svh.view(), cnt, cnt_down, st)
        # (one spare row pointer, and below 4 spare entries of col / val: the streamed SpMV moves 16-byte units)
        rowptr = torch.zeros(n + 2, dtype=torch.int64, device=dev)[:n + 1]
        nb = call("nksr_scan_workspace_bytes", n)
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        call("nksr_gram_rowptr", cnt, cnt_down, n, rowptr, ws, nb, st)
        return cnt, cnt_down, place, rowptr

    def assemble(self, pos_xyz, normal_xyz=None, normal_value=None, pos_weight=1.0, normal_weight=1.0,
                 reg_weight=1.0):
        """Kernel rows + Gram assembly: returns the CSR system (rowptr, col, val, rhs, diag, n, nnz)."""
        svh = self.svh
        dev = svh.device
        _lib.require_cuda(pos_xyz, "pos_xyz")
        st = stream_ptr(dev)
        n = svh.num_unknowns
        if n == 0:
            raise _lib.NksrError("empty hierarchy: nothing to solve")
        if n >= 2 ** 31:
            raise _lib.NksrError("more than 2^31 unknowns: shard the cloud (chunk_size)")
        pos_xyz = pos_xyz.detach().to(dev, torch.float32).contiguous()
        cs = _lib.ConstraintsT()
        keep = []
        # row lengths + placement tables need the hierarchy only: optionally on a side stream, under the row building
        overlap = self.solver_config.get("overlap_count")
        if overlap is None:
            overlap = os.environ.get("NKSR_OVERLAP", "0") == "1"
        side = None
        if overlap:
            side = _side_stream(dev)
            side.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(side):
                cnt, cnt_down, place, rowptr = self._count_and_place(n, keep)
        # row layout.  'interleaved' (depth <= 4, row fill, plain gradient rows): the four levels of a slot are one float4,
        # so the fill reads a location with 1 + 3 128-bit loads per lane instead of 4 + 12 32-bit ones (csrc/assemble.cu,
        # ILV); 'levels': one 128-byte line per (location, level, axis).  Both give bitwise the same matrix.
        layout = self.solver_config.get("row_layout") or os.environ.get("NKSR_ROW_LAYOUT") or DEFAULT_ROW_LAYOUT
        if layout not in ("interleaved", "levels"):
            raise ValueError("solver_config['row_layout'] must be 'interleaved' or 'levels'")
        compact = self.solver_config.get("compact_rows")
        if compact is None:
            compact = os.environ.get("NKSR_COMPACT_ROWS", "0") == "1"
        ilv = (layout == "interleaved" and svh.depth <= 4 and not (self.approx_kernel_grad and compact)
               and (self.solver_config.get("fill") or os.environ.get("NKSR_FILL") or DEFAULT_FILL) in ("rows", "brick")
               and (self.solver_config.get("rows") or os.environ.get("NKSR_ROWS") or "location") == "location")
        _, _, _, range_pos, e_pos = self._sorted_rows(pos_xyz, 0, interleaved=ilv)
        keep += [range_pos, e_pos]
        cs.e_pos, cs.range_pos, cs.n_pos, cs.w_pos = e_pos.data_ptr(), range_pos.data_ptr(), pos_xyz.shape[0], float(pos_weight)
        if normal_xyz is not None and normal_xyz.shape[0] > 0:
            normal_xyz = normal_xyz.detach().to(dev, torch.float32).contiguous()
            normal_value = normal_value.detach().to(dev, torch.float32).contiguous()
            # approx_kernel_grad: compact gradient rows (one 128 B line per location and level)
            # compact gradient rows (one line instead of three per location and level) save 2/3 of
            # the row memory but cost ALU in the assembly, so they are opt-in for clouds that would not fit otherwise
            nrm_mode = 2 if (self.approx_kernel_grad and compact) else 1
            _, t_nrm, _, range_nrm, e_nrm = self._sorted_rows(normal_xyz, nrm_mode, normal_value, interleaved=ilv)
            cs.nrm_compact = 2 if ilv else int(nrm_mode == 2)          # the C struct's row-layout code
            keep += [t_nrm, range_nrm, e_nrm]
            cs.e_nrm, cs.range_nrm, cs.t_nrm = e_nrm.data_ptr(), range_nrm.data_ptr(), t_nrm.data_ptr()
            cs.n_nrm, cs.w_nrm = normal_xyz.shape[0], float(normal_weight)
        else:
            cs.e_nrm = cs.range_nrm = cs.t_nrm = None
            cs.n_nrm, cs.w_nrm = 0, 0.0
            cs.nrm_compact = 2 if ilv else 0
        cs.w_reg = float(reg_weight)

        tm = getattr(self, "_timer", None) or _lib.StageTimer(dev, enabled=False)
        tm.mark("kernel_rows")
        if side is None:
            cnt, cnt_down, place, rowptr = self._count_and_place(n, keep)
        else:
            torch.cuda.current_stream(dev).wait_stream(side)
        nnz = int(rowptr[-1].item())
        tm.mark("gram_count")
        # coarse levels (>= split): a voxel owns hundreds of constraint rows, so their 27x27 products
        # are reduced once per voxel (nksr_gram_blocks) and the matrix rows only gather block lines
        cs.mblocks, cs.split_level = None, svh.depth
        split = self.solver_config.get("block_split_level", None)
        if split is None and os.environ.get("NKSR_BLOCK_SPLIT"):
            split = int(os.environ["NKSR_BLOCK_SPLIT"])
        # (allocator bookkeeping only: cudaMemGetInfo costs tens of milliseconds next to large allocations)
        free_bytes = _total_memory(dev) - torch.cuda.memory_allocated(dev)
        budget = free_bytes - 1.25 * (8.0 * nnz + 64.0 * n)          # leave room for the CSR arrays + PCG vectors
        if split is None:                                            # deepest split whose blocks fit the budget
            split = svh.depth
            # (level 1 was measured too: +45 GB of blocks for 4 % -- not worth it; `block_split_level` overrides)
            for cand in (2, 3):
                if cand < svh.depth and 4 * call("nksr_gram_block_floats", svh.view(), cand) <= min(budget, 32e9):
                    split = cand
                    break
        split = int(split)
        if split < svh.depth and cs.nrm_compact != 1:        # (compact gradient rows have no block kernel)
            nfl = call("nksr_gram_block_floats", svh.view(), split)
            if 0 < nfl * 4 <= max(budget, 0):
                off = 0
                for l in range(split, svh.depth):
                    cs.mblock_off[l] = off
                    off += svh.num_voxels(l) * (svh.depth - l)
                cs.split_level = split
                mblocks = torch.empty(nfl, dtype=torch.float32, device=dev)
                call("nksr_gram_blocks", svh.view(), cs, mblocks, st)
                cs.mblocks = mblocks.data_ptr()
                keep.append(mblocks)
                tm.mark("gram_blocks")
        col = torch.empty(nnz + 4, dtype=torch.int32, device=dev)[:nnz]
        val = torch.empty(nnz + 4, dtype=torch.float32, device=dev)[:nnz]
        rhs = torch.empty(n, dtype=torch.float32, device=dev)
        diag = torch.zeros(n, dtype=torch.float32, device=dev)
        # numeric phase.  'brick' (default): the rows of the dense levels below the block split level one brick of
        # 4^3 rows per block, every constraint line of a source voxel loaded once per brick (csrc/gram_fill_brick.cu),
        # the other rows as 'rows'; 'rows': one warp per matrix row (csrc/assemble.cu); 'grouped': one warp per
        # sibling group -- eight rows share their constraint lines, column tables and flush indices
        # (csrc/gram_fill_group.cu).  The sharing halves the loads but the per-sibling tests and flushes cost as many
        # instructions as they save, and 13.4 KB of shared memory + 128 registers per warp cut the resident warps per SM
        fill = self.solver_config.get("fill") or os.environ.get("NKSR_FILL") or DEFAULT_FILL
        if fill not in ("brick", "grouped", "rows"):
            raise ValueError("solver_config['fill'] must be 'brick', 'grouped' or 'rows'")
        if place is not None and fill == "grouped" and svh.depth <= 4 and svh.depth < _lib.MAX_DEPTH:
            call("nksr_gram_fill_grouped", svh.view(), self.feat_view(), cs, cnt, rowptr, place, col, val, rhs, diag, st)
        elif place is not None and fill == "brick":
            call("nksr_gram_fill_brick", svh.view(), self.feat_view(), cs, cnt, rowptr, place, col, val, rhs, diag,
                 float(BRICK_MIN_LOCATIONS_PER_VOXEL), st)
        elif place is not None:
            call("nksr_gram_fill_placed", svh.view(), self.feat_view(), cs, cnt, rowptr, place, col, val, rhs, diag, st)
        else:
            cursor = torch.zeros(n, dtype=torch.int32, device=dev)
            call("nksr_gram_fill", svh.view(), self.feat_view(), cs, cnt, rowptr, col, val, rhs, diag, cursor, st)
        tm.mark("gram_fill")
        # atomic-cursor variant: deterministic storage order of the transposed (finer-level) segments
        # (rows binned by segment length so that short rows do not pay for a large tile)
        offs = svh.offsets
        if place is None and svh.depth > 1 and n > offs[1]:
            seg = cnt_down[offs[1]:]
            lo_b = 1
            for cap in (32, 128, 512, 1024, 2048, 4096, 8192, 16384):
                rows = (torch.nonzero((seg > lo_b) & (seg <= cap)).reshape(-1) + offs[1]).to(torch.int32)
                lo_b = cap
                if rows.numel():
                    call("nksr_gram_sort_down", cnt, cnt_down, rowptr, rows, rows.numel(), cap, col, val, st)
        del keep
        tm.mark("gram_sort")
        return SimpleNamespace(rowptr=rowptr, col=col, val=val, rhs=rhs, diag=diag, cnt=cnt, cnt_down=cnt_down,
                               n=n, nnz=nnz)

    # the reference exposes both spellings; both run the same fused assembly here
    def solve_non_fused(self, pos_xyz, normal_xyz, normal_value, pos_weight, normal_weight, reg_weight):
        return self.solve(pos_xyz, normal_xyz, normal_value, pos_weight, normal_weight, reg_weight)

    # ------------------------------------------------------------------ evaluation
    def evaluate_f(self, xyz: torch.Tensor, grad: bool = False) -> EvaluationResult:
        if self.alpha is None:
            raise _lib.NksrError("KernelField.evaluate_f called before solve()")
        _lib.require_cuda(xyz, "xyz")
        xyz = xyz.detach().to(self.svh.device, torch.float32).contiguous()
        m = xyz.shape[0]
        f = torch.empty(m, dtype=torch.float32, device=xyz.device)
        g = torch.empty((m, 3), dtype=torch.float32, device=xyz.device) if grad else None
        call("nksr_evaluate", self.svh.view(), self.feat_view(), self.alpha, xyz, m, int(grad),
             int(self.approx_kernel_grad), f, g, stream_ptr(xyz.device))
        return EvaluationResult(value=f, gradient=g)

    def evaluate_f_bar(self, xyz: torch.Tensor) -> torch.Tensor:
        """Occupancy-style value (> 0 inside, models/loss.py:99); masked-out regions read as outside."""
        f = self.evaluate_f(xyz).value
        if self.mask_field is not None:
            f = torch.where(self.mask_field.mask(xyz), f, -f.abs())
        return f

    def mask(self, xyz):
        return self.evaluate_f(xyz).value >= self.level_set

    def to_(self, device):
        super().to_(device)
        device = torch.device(device)
        self.z = [t.to(device) for t in self.z]
        if self.alpha is not None:
            self.alpha = self.alpha.to(device)
        self._feat_view = None
        return self


class LayerField(BaseField):
    """Mask = inside an active voxel of one of the finest `adaptive_depth` levels."""

    def __init__(self, svh: SparseFeatureHierarchy, adaptive_depth: int):
        super().__init__(svh)
        self.adaptive_depth = int(adaptive_depth)
        self.level_set = 0.5

    def evaluate_f(self, xyz, grad=False):
        _lib.require_cuda(xyz, "xyz")
        xyz = xyz.detach().to(torch.float32).contiguous()
        out = torch.empty(xyz.shape[0], dtype=torch.float32, device=xyz.device)
        call("nksr_layer_mask", self.svh.view(), xyz, xyz.shape[0], self.adaptive_depth, out, stream_ptr(xyz.device))
        return EvaluationResult(value=out, gradient=None)

    def mask(self, xyz):
        return self.evaluate_f(xyz).value >= self.level_set


class NeuralField(BaseField):
    """MLP-decoded field over trilinearly interpolated voxel features (used as the UDF mask,
    models/nksr_net.py:124-130).  The decoder is a PyTorch module and stays on PyTorch
    (north_star: the network is not part of the hot path); interpolation uses the SVH tables."""

    def __init__(self, svh: SparseFeatureHierarchy, decoder, features):
        super().__init__(svh)
        self.decoder = decoder
        self.features = _as_level_list(features, svh.depth)

    def _interp(self, xyz):
        svh = self.svh
        base = svh.locate(xyz).long()
        out = None
        for l in range(svh.depth):
            f = self.features[l]
            if f is None or svh.num_voxels(l) == 0:
                continue
            w = svh.voxel_size * (2 ** l)
            b = base[l]
            ok = b >= 0
            bc = b.clamp(min=0)
            ijk = SparseFeatureHierarchyCoords.ijk(svh, l)[bc].to(torch.float32)
            tau = xyz / w - (ijk + 0.5)
            nb = svh.nbr27[l][bc].long()
            acc = torch.zeros((xyz.shape[0], f.shape[1]), device=xyz.device, dtype=torch.float32)
            d = torch.tensor([-1.0, 0.0, 1.0], device=xyz.device)
            tw = (1.0 - (tau[:, :, None] - d[None, None, :]).abs()).clamp(min=0.0)      # (M,3,3)
            w27 = (tw[:, 0, :, None, None] * tw[:, 1, None, :, None] * tw[:, 2, None, None, :]).reshape(-1, 27)
            for s in range(27):
                idx = nb[:, s]
                good = ok & (idx >= 0)
                acc += torch.where(good[:, None], f[idx.clamp(min=0)] * w27[:, s:s + 1], torch.zeros_like(acc))
            out = acc if out is None else torch.cat([out, acc], dim=1)
        return out

    def evaluate_f(self, xyz, grad=False):
        xyz = xyz.detach().to(self.svh.device, torch.float32).contiguous()
        with torch.no_grad():
            v = self.decoder(self._interp(xyz)).reshape(-1)
        return EvaluationResult(value=v, gradient=None)

    def mask(self, xyz):
        # UDF semantics: keep geometry closer than the level set to the data
        return self.evaluate_f(xyz).value <= self.level_set


class SparseFeatureHierarchyCoords:
    @staticmethod
    def ijk(svh, l):
        from .svh import SparseIndexGrid
        return SparseIndexGrid(svh, l).active_grid_coords()


class PCNNField:
    """Nearest-neighbour colour texture (examples/recons_colored_mesh.py:28-31; SURVEY section 8(f) row 3): the colour
    of a query is the colour of the nearest input point.  The cloud is hashed once (multi-level voxel hash of the
    Morton-sorted points, shared with the kNN normal estimation); queries run one warp each in
    csrc/nearest.cu (k_nearest_point) -- exact nearest neighbour, O(V log N) instead of the V x N distance matrix."""

    START_LEVEL = 2       # cells of ~0.6 mean point spacings: the first level that usually holds the answer

    def __init__(self, xyz: torch.Tensor, color: torch.Tensor):
        _lib.require_cuda(xyz, "xyz")
        from .reconstructor import _knn_hash
        xyz = xyz.detach().to(torch.float32).contiguous()
        perm, self.svh, _, self.ranges, self.origin = _knn_hash(xyz)
        self.xyz = xyz[perm].contiguous()
        self.color = color.detach().to(xyz.device)[perm].contiguous()
        self._origin_host = (C.c_float * 3)(*[float(v) for v in self.origin.tolist()])

    def nearest(self, q: torch.Tensor):
        """(index into the SORTED cloud, squared distance) of the nearest input point of every query"""
        q = q.detach().to(self.xyz.device, torch.float32).contiguous()
        m = q.shape[0]
        idx = torch.empty(m, dtype=torch.int32, device=q.device)
        d2 = torch.empty(m, dtype=torch.float32, device=q.device)
        call("nksr_nearest_point", self.svh.view(), self.xyz, self.ranges, self.xyz.shape[0], q, m,
             C.addressof(self._origin_host),
             self.START_LEVEL, idx, d2, stream_ptr(q.device))
        return idx, d2

    def evaluate_f(self, q: torch.Tensor, grad=False):
        idx, _ = self.nearest(q)
        return EvaluationResult(value=self.color[idx.long().clamp(min=0)], gradient=None)
