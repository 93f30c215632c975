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

# the layout every parity test runs on unless a test selects the other
DEFAULT_ROW_LAYOUT = "levels"
# the Gram fill (solver_config['fill'] or the NKSR_FILL environment variable override it): "brick", "rows", "grouped"
DEFAULT_FILL = "brick"
# 'brick' bricks a fine level only when it holds at least this many constraint locations per voxel (measured on H100:
# faster than the row fill at 18 per voxel, slower at 1.7, 4.9 and 8.2; DESIGN 4.1)
BRICK_MIN_LOCATIONS_PER_VOXEL = 12.0
# the matrix-free operator is the default (with approx_kernel_grad) from this many unknowns on.  Measured on H100: 15 %
# faster per bench.py step at 17.1 M unknowns (cfg4), 11 % slower at 2.0 M (cfg3, whose solve takes 16 iterations of an
# operator that costs 2.5 packed SpMVs); the crossover between the two was not measured (DESIGN 4.2.1)
MATRIX_FREE_MIN_UNKNOWNS = 8_000_000
# locations per work item of the matrix-free gather-scatter (csrc/operator.cu; DESIGN 4.2.1)
OP_ITEM_SIZE = 64


_TOTAL_MEMORY = {}


def _total_memory(dev) -> int:
    key = torch.device(dev).index or 0
    if key not in _TOTAL_MEMORY:
        _TOTAL_MEMORY[key] = int(torch.cuda.get_device_properties(dev).total_memory * 0.94)   # driver / context reserve
    return _TOTAL_MEMORY[key]


def operator_bytes_per_apply(svh, n_pos: int, n_nrm: int, nrm_lines: int, channels: int,
                             item_size: int = OP_ITEM_SIZE) -> int:
    """Byte model of one matrix-free application of A (csrc/operator.cu), from shapes: the kernel rows (128 B per
    location, level and line: nrm_lines = 1 compact, 3 full), the merged location order and its containing voxels
    (4 B per location and level, plus 4), the work items (16 B each) and their edge partials written and summed
    (2 x 108 B per item and level above the cut), nbr27 read once per voxel by each kernel, the planar partial sums
    written and gathered once (27 floats per voxel each), the features z (4 C B per voxel) and x read twice and y
    written (12 B per voxel).  Voxels without locations are counted as if they had some, and the item count is its
    bound 2 m / item_size + top voxels, so it is an upper bound of the algorithmic bytes.  bench.py's roofline_spmv
    (8 nnz + 12 n) describes the assembled matrix, not this path."""
    L, n = svh.depth, svh.num_unknowns
    m = n_pos + n_nrm
    rows = 128 * L * (n_pos + nrm_lines * n_nrm)
    items = 2 * -(-m // item_size) + svh.num_voxels(L - 1)
    edge_levels = max(L - 3, 0)                         # levels above the cut level 2
    return int(rows + 4 * (L + 1) * m + items * (16 + 2 * 2 * 108 * edge_levels) + 2 * 108 * n + 2 * 108 * n
               + 4 * channels * n + 12 * n)


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

    def evaluate_f_bar(self, xyz: torch.Tensor) -> torch.Tensor:
        """Occupancy-style value (> 0 inside, models/loss.py:99); masked-out regions read as outside."""
        f = self.evaluate_f(xyz).value
        if self.mask_field is not None:
            f = torch.where(self.mask_field.mask(xyz), f, -f.abs())
        return f

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
        with torch.no_grad():          # meshing records no graph, even of a field that is being trained
            return extract_dual_mesh(self, grid_upsample=grid_upsample, mise_iter=mise_iter, max_points=max_points,
                                     cell_filter=cell_filter)


def _as_level_list(features, depth):
    if isinstance(features, dict):
        return [features.get(d, None) for d in range(depth)]
    return [features[d] if d < len(features) else None for d in range(depth)]


def _sorted_locations(svh: SparseFeatureHierarchy, xyz: torch.Tensor, extra: Optional[torch.Tensor] = None,
                      with_keys: bool = False):
    """Morton-sort locations and locate them on every level: (perm, sorted xyz, sorted extra, base (depth, m),
    ranges (n, 2): the first / last + 1 sorted location of every voxel, levels concatenated), and with `with_keys`
    also their sorted half-voxel keys (m,) int64, the order the matrix-free operator merges by."""
    dev = xyz.device
    st = stream_ptr(dev)
    m = xyz.shape[0]
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    hk = torch.empty(m, dtype=torch.int64, device=dev)
    call("nksr_point_half_keys", xyz, m, svh.voxel_size, hk, status, st)
    if int(status.item()) & 1:
        raise _lib.NksrError("constraint locations outside the supported range (|x| < 2^19 voxels) or non-finite")
    keys, perm = _lib.sort_pairs(hk, torch.arange(m, dtype=torch.int32, device=dev))
    perm = perm.long()
    xs = xyz[perm].contiguous()
    ex = extra[perm].contiguous() if extra is not None else None
    base = svh.locate(xs)
    n_total = svh.num_unknowns
    ranges = torch.empty((n_total, 2), dtype=torch.int32, device=dev)
    offs = svh.offsets
    for l in range(svh.depth):
        call("nksr_row_ranges", base[l], m, ranges[offs[l]:], svh.num_voxels(l), st)
    return (perm, xs, ex, base, ranges, keys) if with_keys else (perm, xs, ex, base, ranges)


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
            mod = None
            if self.interpolator is not None:
                mod = self.interpolator[l] if not isinstance(self.interpolator, dict) else self.interpolator[str(l)]
            # training: keep the interpolator's graph, so that the kernel solve / evaluation backpropagate into the
            # basis features and the interpolator parameters (the same operations, so the same z)
            graph = torch.is_grad_enabled() and (f.requires_grad or (
                mod is not None and any(p.requires_grad for p in getattr(mod, "parameters", lambda: [])())))
            f = (f if graph else f.detach()).to(dev, torch.float32)
            if mod is not None:
                with torch.set_grad_enabled(graph):
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
    def _sorted_locations(self, xyz: torch.Tensor, extra: Optional[torch.Tensor] = None, with_keys: bool = False):
        return _sorted_locations(self.svh, xyz, extra, with_keys)

    def _sorted_rows(self, xyz: torch.Tensor, mode: int, extra: Optional[torch.Tensor] = None,
                     interleaved: bool = False, loc=None):
        """Morton-sort locations, locate them on every level, build their kernel rows.
        `interleaved` (depth <= 4, modes 0 / 1): rows as (m, rows, 32, 4 levels) -- the four levels of a slot are one
        float4 -- instead of (m, depth, rows * 32).  `loc`: the result of _sorted_locations, when the caller has it."""
        svh, dev = self.svh, xyz.device
        st = stream_ptr(dev)
        m = xyz.shape[0]
        _, xs, ex, base, ranges = loc if loc is not None else self._sorted_locations(xyz, extra)
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

    def _wants_grad(self, *tensors):
        return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (*self.z, *tensors))

    def solve(self, pos_xyz, normal_xyz=None, normal_value=None, pos_weight=1.0, normal_weight=1.0,
              reg_weight=1.0, fused_mode: bool = False):
        """Assemble A = E^T W E + reg R (CSR) and solve A alpha = E^T W t with Jacobi-PCG.
        When grad is enabled and the features (or normal_value) require grad, alpha carries a graph: its backward runs
        the adjoint solve and the feature-VJP kernels (_KernelSolve)."""
        if self._wants_grad(normal_value if normal_xyz is not None else None):
            nv = normal_value if normal_xyz is not None and normal_xyz.shape[0] > 0 else None
            self.alpha = _KernelSolve.apply(self, (pos_xyz, normal_xyz, pos_weight, normal_weight, reg_weight), nv,
                                            *self.z)
            return self
        if self._operator() == "matrix_free" and not self.solver_config.get("keep_system"):
            self.alpha = self._solve_matrix_free(pos_xyz, normal_xyz, normal_value, pos_weight, normal_weight,
                                                 reg_weight)
            return self
        sysm = self.assemble(pos_xyz, normal_xyz, normal_value, pos_weight, normal_weight, reg_weight)
        self.alpha = self._pcg(sysm, sysm.rhs)
        if self.solver_config.get("keep_system"):
            self.system = sysm
        return self

    def _operator(self):
        """solver_config['operator'] or NKSR_OPERATOR: 'matrix_free' (A applied from the kernel rows, csrc/operator.cu)
        or 'assembled' (the CSR Gram matrix).  Default: matrix-free with approx_kernel_grad (compact rows) on systems of
        at least MATRIX_FREE_MIN_UNKNOWNS unknowns, assembled otherwise.  A Gram fill chosen explicitly
        (solver_config['fill'] or NKSR_FILL) asks for the matrix that fill builds, so it too selects the assembled
        operator unless the operator is given as well.  keep_system always assembles.  Grad-recording solves do not
        use this rule: they take the operator from _grad_operator, which reads the explicit names only.  The global
        solve (dist_solve.reconstruct_global) takes the operator as an argument or from NKSR_OPERATOR, and assembles
        when neither names one."""
        op = self.solver_config.get("operator") or os.environ.get("NKSR_OPERATOR")
        if op is None:
            big = self.svh.num_unknowns >= MATRIX_FREE_MIN_UNKNOWNS
            fill_chosen = bool(self.solver_config.get("fill") or os.environ.get("NKSR_FILL"))
            op = "matrix_free" if self.approx_kernel_grad and big and not fill_chosen else "assembled"
        if op not in ("matrix_free", "assembled"):
            raise ValueError("solver_config['operator'] must be 'matrix_free' or 'assembled'")
        return op

    def _grad_operator(self):
        """The operator of a grad-recording solve (_KernelSolve): 'matrix_free' only when solver_config['operator'] or
        NKSR_OPERATOR names it, else 'assembled'.  The size rule of _operator was measured on inference solves and does
        not apply here.  keep_system always assembles."""
        op = self.solver_config.get("operator") or os.environ.get("NKSR_OPERATOR") or "assembled"
        if op not in ("matrix_free", "assembled"):
            raise ValueError("solver_config['operator'] must be 'matrix_free' or 'assembled'")
        return "assembled" if self.solver_config.get("keep_system") else op

    def _solve_matrix_free(self, pos_xyz, normal_xyz, normal_value, pos_weight, normal_weight, reg_weight):
        """Jacobi-PCG on A = E^T W E + reg R without assembling A (DESIGN 4.2.1): kernel rows (compact gradient lines
        with approx_kernel_grad), then rhs and diagonal (nksr_op_setup), then the PCG, whose every iteration applies A
        from the rows (nksr_pcg_solve_matrix_free).  No count, placement, blocks or fill; solve_info['nnz'] = 0."""
        op = self.matrix_free_system(pos_xyz, normal_xyz, normal_value, pos_weight, normal_weight, reg_weight)
        return self._pcg_matrix_free(op, op.rhs)

    def _pcg_matrix_free(self, op, rhs, adjoint: bool = False):
        """Jacobi-PCG on the operator of a matrix_free_system: the forward solve (A alpha = b) and the adjoint solve of
        the backward (A lambda = dL/dalpha) run on the same workspace.  Reports as _pcg does."""
        svh, dev, n = self.svh, self.svh.device, op.n
        alpha = torch.empty(n, dtype=torch.float32, device=dev)
        info = (C.c_double * 8)()
        profile = int(bool(self.solver_config.get("profile")))
        nb = call("nksr_pcg_workspace_bytes", n)
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        call("nksr_pcg_solve_matrix_free", svh.view(), self.feat_view(), op.cs, op.base_pos, op.base_nrm, op.diag,
             rhs, alpha, float(self.solver_config["tol"]), int(self.solver_config["max_iter"]),
             int(self.solver_config["check_every"]), profile, op.ws, op.ws_bytes, ws, nb, info, stream_ptr(dev))
        tm = getattr(self, "_timer", None) or _lib.StageTimer(dev, enabled=False)
        tm.mark("adjoint_pcg" if adjoint else "pcg")
        self._pcg_report(info, n, 0, adjoint, operator="matrix_free", operator_bytes_per_apply=op.bytes_per_apply)
        return alpha

    def constraint_values(self, op, x0: torch.Tensor, x1: torch.Tensor):
        """E_j x0 and E_j x1 at the sorted constraint locations of a matrix_free_system, read from its kernel rows
        (nksr_op_constraint_values): (n_pos, 2) values of the sorted positions and (n_nrm, 2, 3) gradient rows of the
        sorted normal locations, for x0 then x1.  No weights."""
        dev = self.svh.device
        vp = torch.empty((op.cs.n_pos, 2), dtype=torch.float32, device=dev)
        vn = torch.empty((op.cs.n_nrm, 2, 3), dtype=torch.float32, device=dev)
        call("nksr_op_constraint_values", self.svh.view(), op.cs, op.base_pos, op.base_nrm,
             x0.to(torch.float32).contiguous(), x1.to(torch.float32).contiguous(), vp, vn, stream_ptr(dev))
        return vp, vn

    def matrix_free_system(self, pos_xyz, normal_xyz=None, normal_value=None, pos_weight=1.0, normal_weight=1.0,
                           reg_weight=1.0, item_size: Optional[int] = None, owned: Optional[torch.Tensor] = None,
                           keep_constraints: bool = False):
        """Kernel rows of the sorted constraint locations and the operator's setup (nksr_op_setup): returns
        .rhs, .diag, .n, .locations_kept and what apply_operator needs (the rows, the constraint struct, the
        operator's workspace).  item_size: at most that many locations per work item of the gather-scatter (default
        OP_ITEM_SIZE; see operator_items).  owned (bool or uint8 per unknown, levels concatenated): the rows a rank of
        the global solve owns.  Only the locations that contribute to an owned row are kept, so rhs, diag and A x are
        those of the whole system on the owned rows and incomplete elsewhere; None keeps every location.
        keep_constraints: also `.cons`, the record assemble(keep_constraints=True) returns (what the backward needs)."""
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
        *loc_pos, key_pos = self._sorted_locations(pos_xyz, with_keys=True)
        _, _, base_pos, range_pos, e_pos = self._sorted_rows(pos_xyz, 0, loc=loc_pos)
        cs.e_pos, cs.range_pos, cs.n_pos, cs.w_pos = e_pos.data_ptr(), range_pos.data_ptr(), pos_xyz.shape[0], float(pos_weight)
        keep = [e_pos, range_pos, key_pos]
        cons = SimpleNamespace(pos=(loc_pos[1], loc_pos[3], loc_pos[4]),
                               nrm=None, perm_nrm=None, w_pos=float(pos_weight), w_nrm=float(normal_weight),
                               w_reg=float(reg_weight)) if keep_constraints else None
        base_nrm, key_nrm, lines, K = None, None, 0, 0
        if normal_xyz is not None and normal_xyz.shape[0] > 0:
            normal_xyz = normal_xyz.detach().to(dev, torch.float32).contiguous()
            normal_value = normal_value.detach().to(dev, torch.float32).contiguous()
            mode = 2 if self.approx_kernel_grad else 1          # compact lines: one 128 B line per location and level
            *loc_nrm, key_nrm = self._sorted_locations(normal_xyz, normal_value, with_keys=True)
            _, t_nrm, base_nrm, range_nrm, e_nrm = self._sorted_rows(normal_xyz, mode, normal_value, loc=loc_nrm)
            if cons is not None:
                cons.nrm, cons.t_nrm, cons.perm_nrm = (loc_nrm[1], loc_nrm[3], loc_nrm[4]), t_nrm, loc_nrm[0]
            keep += [t_nrm, range_nrm, e_nrm, key_nrm]
            cs.e_nrm, cs.range_nrm, cs.t_nrm = e_nrm.data_ptr(), range_nrm.data_ptr(), t_nrm.data_ptr()
            K, lines = normal_xyz.shape[0], (1 if mode == 2 else 3)
            cs.n_nrm, cs.w_nrm, cs.nrm_compact = K, float(normal_weight), int(mode == 2)
        else:
            cs.e_nrm = cs.range_nrm = cs.t_nrm = None
            cs.n_nrm, cs.w_nrm, cs.nrm_compact = 0, 0.0, 0
        cs.w_reg = float(reg_weight)
        cs.mblocks, cs.split_level = None, svh.depth
        tm = getattr(self, "_timer", None) or _lib.StageTimer(dev, enabled=False)
        tm.mark("kernel_rows")
        S = int(item_size or OP_ITEM_SIZE)
        if S < 1:
            raise ValueError("item_size must be at least 1")
        own8 = None
        if owned is not None:
            if owned.shape != (n,):
                raise ValueError(f"owned must hold one entry per unknown ({n}), got shape {tuple(owned.shape)}")
            own8 = owned.to(dev, torch.uint8).contiguous()
            keep.append(own8)
        nb_op = call("nksr_op_workspace_bytes", svh.view(), cs, S)
        op_ws = torch.empty(nb_op, dtype=torch.uint8, device=dev)
        rhs = torch.empty(n, dtype=torch.float32, device=dev)
        diag = torch.empty(n, dtype=torch.float32, device=dev)
        call("nksr_op_setup", svh.view(), self.feat_view(), cs, base_pos, base_nrm, key_pos, key_nrm, own8, S, rhs,
             diag, op_ws, nb_op, st)
        tm.mark("operator_setup")
        kept = cs.n_pos + cs.n_nrm                          # without a mask every location is kept
        if own8 is not None:                                # (a read-back: the kept count lives on the device)
            layout = (C.c_int64 * 5)()
            call("nksr_op_workspace_layout", svh.view(), cs, nb_op, C.addressof(layout))
            kept = int(op_ws[layout[4]:layout[4] + 4].view(torch.int32).item())
        return SimpleNamespace(cs=cs, base_pos=base_pos, base_nrm=base_nrm, rhs=rhs, diag=diag, ws=op_ws,
                               ws_bytes=nb_op, n=n, keep=keep, item_size=S, owned=own8, locations_kept=kept,
                               bytes_per_apply=operator_bytes_per_apply(svh, pos_xyz.shape[0], K, lines, self.channels,
                                                                        S), cons=cons)

    def operator_items(self, op):
        """The work of a matrix_free_system, from its workspace: (order, vox, items).  order (kept,) int32 is the
        merged order of the kept locations (r >= 0: sorted position r, ~r: sorted normal location r; every location
        without an owned mask), vox (depth, kept) their containing voxels, items (count, 4) int32 the work items:
        begin, end in order, flags (1: first, 2: last item of its top-level voxel), 0.  Reads the item count back to
        the host."""
        out = (C.c_int64 * 5)()
        call("nksr_op_workspace_layout", self.svh.view(), op.cs, op.ws_bytes, C.addressof(out))
        m = op.cs.n_pos + op.cs.n_nrm
        i32 = lambda off, cnt: op.ws[off:off + 4 * cnt].view(torch.int32)
        count, kept = int(i32(out[2], 1).item()), int(i32(out[4], 1).item())
        return i32(out[0], kept), i32(out[1], self.svh.depth * m).view(self.svh.depth, m)[:, :kept], \
            i32(out[3], 4 * count).view(count, 4)

    def apply_operator(self, op, x: torch.Tensor) -> torch.Tensor:
        """y = A x for a system of matrix_free_system (nksr_op_apply)"""
        y = torch.empty(op.n, dtype=torch.float32, device=self.svh.device)
        call("nksr_op_apply", self.svh.view(), self.feat_view(), op.cs, op.base_pos, op.base_nrm,
             x.to(torch.float32).contiguous(), y, op.ws, op.ws_bytes, stream_ptr(self.svh.device))
        return y

    def _pcg(self, sysm, rhs, adjoint: bool = False):
        """Jacobi-PCG on the assembled system: the forward solve (A alpha = b) and the adjoint solve of the backward
        (A lambda = dL/dalpha, the same symmetric matrix) share it.  A breakdown raises, max_iter warns; the forward
        fills solve_info, the adjoint adds 'adjoint_iterations' / 'adjoint_relative_residual' to it."""
        dev, n = self.svh.device, sysm.n
        tm = getattr(self, "_timer", None) or _lib.StageTimer(dev, enabled=False)
        alpha = torch.empty(n, dtype=torch.float32, device=dev)
        info = (C.c_double * 8)()
        profile = int(bool(self.solver_config.get("profile")))
        # 'stream' (default): the CSR arrays reach the SMs as tiles moved by bulk async copies (TMA engine) into a
        # shared-memory ring, with packed column tiles (csrc/spmv_stream.cuh); 'rows': one warp per row with register
        # loads (csrc/solve.cu), the reference the stream is tested against
        spmv = self.solver_config.get("spmv") or os.environ.get("NKSR_SPMV") or "stream"
        if spmv not in ("stream", "rows"):
            raise ValueError("solver_config['spmv'] must be 'stream' or 'rows'")
        packed = None
        if spmv == "stream":
            nb = call("nksr_pcg_stream_workspace_bytes", n, sysm.nnz)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            # every row is streamed: the coarse rows too (transposed segments of up to tens of thousands of
            # entries), which on the H100 stream faster as tiles than warp per row (DESIGN 4.2)
            call("nksr_pcg_solve_stream", sysm.rowptr, sysm.col, sysm.val, sysm.diag, rhs, alpha, n, sysm.nnz,
                 n, sysm.nnz, float(self.solver_config["tol"]), int(self.solver_config["max_iter"]),
                 int(self.solver_config["check_every"]), profile, ws, nb, info, stream_ptr(dev))
            packed = (C.c_int64 * 4)()
            call("nksr_spmv_plan_stats", ws[call("nksr_pcg_workspace_bytes", n):], C.addressof(packed),
                 stream_ptr(dev))
        else:
            nb = call("nksr_pcg_workspace_bytes", n)
            ws = torch.empty(nb, dtype=torch.uint8, device=dev)
            call("nksr_pcg_solve", sysm.rowptr, sysm.col, sysm.val, sysm.diag, rhs, alpha, n,
                 float(self.solver_config["tol"]), int(self.solver_config["max_iter"]),
                 int(self.solver_config["check_every"]), profile, ws, nb, info, stream_ptr(dev))
        tm.mark("adjoint_pcg" if adjoint else "pcg")
        extra = {"operator": "assembled"}
        if packed is not None:
            extra.update(spmv_packed_tiles=packed[0], spmv_packed_entries=packed[1], spmv_streamed_tiles=packed[2],
                         spmv_streamed_entries=packed[3])
        self._pcg_report(info, n, sysm.nnz, adjoint, **extra)
        return alpha

    def _pcg_report(self, info, n, nnz, adjoint, **extra):
        """solve_info from a PCG's info[] (the forward replaces it, the adjoint adds to it); a breakdown raises,
        max_iter warns"""
        status = int(info[4])                       # 0 converged, 1 max_iter reached, 2 NaN / breakdown
        if adjoint:
            self.solve_info.update(adjoint_iterations=int(info[0]), adjoint_relative_residual=float(info[1]))
        else:
            self.solve_info = {"iterations": int(info[0]), "relative_residual": float(info[1]), "n": n,
                               "nnz": nnz, "converged": status == 0, **extra}
        what = "adjoint PCG" if adjoint else "PCG"
        if status == 2:
            raise _lib.NksrError(f"{what} broke down (non-finite residual) after {int(info[0])} iterations: the system "
                                 "is not positive definite or the inputs are not finite")
        if status == 1 and int(self.solver_config["max_iter"]) > 0:
            warnings.warn(f"nksr_b200 {what} stopped at max_iter={int(self.solver_config['max_iter'])} with relative "
                          f"residual {float(info[1]):.3e} > tol={float(self.solver_config['tol']):.1e}", RuntimeWarning)
        if self.solver_config.get("profile") and not adjoint:
            self.solve_info.update(spmv_ms=float(info[2]), spmv_launches=int(info[3]))
        if self.solver_config.get("verbose"):
            print(f"[nksr_b200] {what}: n={n} nnz={nnz} iters={int(info[0])} relres={float(info[1]):.3e}")

    def _count_and_place(self, n, keep):
        """structure-only part of the assembly (row lengths, placement tables, row pointers): depends on the hierarchy
        alone, so it may run on a side stream while the kernel rows are built (solver_config['overlap_count'])"""
        svh = self.svh
        dev = svh.device
        st = stream_ptr(dev)
        cnt = torch.empty(n, dtype=torch.int32, device=dev)
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
        # (one spare row pointer, and below 4 spare entries of col / val: the streamed SpMV moves 16-byte units)
        rowptr = torch.zeros(n + 2, dtype=torch.int64, device=dev)[:n + 1]
        nb = call("nksr_scan_workspace_bytes", n)
        ws = torch.empty(nb, dtype=torch.uint8, device=dev)
        call("nksr_gram_rowptr", cnt, cnt_down, n, rowptr, ws, nb, st)
        return cnt, cnt_down, place, rowptr

    def assemble(self, pos_xyz, normal_xyz=None, normal_value=None, pos_weight=1.0, normal_weight=1.0,
                 reg_weight=1.0, keep_constraints: bool = False):
        """Kernel rows + Gram assembly: returns the CSR system (rowptr, col, val, rhs, diag, n, nnz).
        keep_constraints: also `.cons`, the sorted constraint locations, their containing voxels and ranges, the
        sorted normal targets and the weights -- what the backward needs (it rebuilds no kernel row from E)."""
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
        loc_pos = self._sorted_locations(pos_xyz)
        _, _, _, range_pos, e_pos = self._sorted_rows(pos_xyz, 0, interleaved=ilv, loc=loc_pos)
        cons = SimpleNamespace(pos=(loc_pos[1], loc_pos[3], loc_pos[4]),
                               nrm=None, perm_nrm=None, w_pos=float(pos_weight), w_nrm=float(normal_weight),
                               w_reg=float(reg_weight)) if keep_constraints else None
        keep += [range_pos, e_pos]
        cs.e_pos, cs.range_pos, cs.n_pos, cs.w_pos = e_pos.data_ptr(), range_pos.data_ptr(), pos_xyz.shape[0], float(pos_weight)
        if normal_xyz is not None and normal_xyz.shape[0] > 0:
            normal_xyz = normal_xyz.detach().to(dev, torch.float32).contiguous()
            normal_value = normal_value.detach().to(dev, torch.float32).contiguous()
            # approx_kernel_grad: compact gradient rows (one 128 B line per location and level)
            # compact gradient rows (one line instead of three per location and level) save 2/3 of
            # the row memory but cost ALU in the assembly, so they are opt-in for clouds that would not fit otherwise
            nrm_mode = 2 if (self.approx_kernel_grad and compact) else 1
            loc_nrm = self._sorted_locations(normal_xyz, normal_value)
            _, t_nrm, _, range_nrm, e_nrm = self._sorted_rows(normal_xyz, nrm_mode, normal_value, interleaved=ilv,
                                                              loc=loc_nrm)
            if cons is not None:
                cons.nrm, cons.t_nrm, cons.perm_nrm = (loc_nrm[1], loc_nrm[3], loc_nrm[4]), t_nrm, loc_nrm[0]
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
        if fill == "grouped" and svh.depth <= 4 and svh.depth < _lib.MAX_DEPTH:
            call("nksr_gram_fill_grouped", svh.view(), self.feat_view(), cs, cnt, rowptr, place, col, val, rhs, diag, st)
        elif fill == "brick":
            call("nksr_gram_fill_brick", svh.view(), self.feat_view(), cs, cnt, rowptr, place, col, val, rhs, diag,
                 float(BRICK_MIN_LOCATIONS_PER_VOXEL), st)
        else:
            call("nksr_gram_fill_placed", svh.view(), self.feat_view(), cs, cnt, rowptr, place, col, val, rhs, diag, st)
        tm.mark("gram_fill")
        del keep
        return SimpleNamespace(rowptr=rowptr, col=col, val=val, rhs=rhs, diag=diag, cnt=cnt, cnt_down=cnt_down,
                               n=n, nnz=nnz, cons=cons)

    # the reference exposes both spellings; both run the same fused assembly here
    def solve_non_fused(self, pos_xyz, normal_xyz, normal_value, pos_weight, normal_weight, reg_weight):
        return self.solve(pos_xyz, normal_xyz, normal_value, pos_weight, normal_weight, reg_weight)

    # ------------------------------------------------------------------ evaluation
    def evaluate_f(self, xyz: torch.Tensor, grad: bool = False) -> EvaluationResult:
        """f (and grad f) at xyz.  When grad is enabled and alpha or the features require grad, the result carries a
        graph into alpha and the features (_KernelEvaluate); query positions get no gradient."""
        if self.alpha is None:
            raise _lib.NksrError("KernelField.evaluate_f called before solve()")
        _lib.require_cuda(xyz, "xyz")
        xyz = xyz.detach().to(self.svh.device, torch.float32).contiguous()
        if self._wants_grad(self.alpha):
            out = _KernelEvaluate.apply(self, xyz, bool(grad), self.alpha, *self.z)
            return EvaluationResult(value=out[0], gradient=out[1] if grad else None)
        f, g = self._evaluate(self.alpha, xyz, grad)
        return EvaluationResult(value=f, gradient=g)

    def _evaluate(self, alpha, xyz, grad):
        m = xyz.shape[0]
        f = torch.empty(m, dtype=torch.float32, device=xyz.device)
        g = torch.empty((m, 3), dtype=torch.float32, device=xyz.device) if grad else None
        call("nksr_evaluate", self.svh.view(), self.feat_view(), alpha, xyz, m, int(grad),
             int(self.approx_kernel_grad), f, g, stream_ptr(xyz.device))
        return f, g

    # ------------------------------------------------------------------ backward (DESIGN 4.6)
    def _query_locations(self, xyz):
        """sorted locations of the queries the forward can evaluate (finite, inside the key range); the others
        evaluate to 0 and get no gradient.  Returns (index into xyz, sorted xyz, base, ranges)."""
        half = self.svh.voxel_size * 0.5
        ok = torch.isfinite(xyz).all(dim=1) & ((xyz / half).abs() < float(2 ** 20 - 64)).all(dim=1)
        keep = torch.nonzero(ok).reshape(-1)
        q = xyz[keep].contiguous()
        perm, xs, _, base, ranges = self._sorted_locations(q)
        return keep[perm], xs, base, ranges

    def _feature_vjp(self, loc, mode, coef, a0, a1, dz):
        """dz (n, C) += d/dz sum_q sum_s omega_{q,s} E_q[n_s] at the sorted locations `loc` = (xs, base, ranges)"""
        xs, base, ranges = loc
        m = xs.shape[0]
        if m == 0:
            return
        nb = call("nksr_field_bwd_workspace_bytes", self.svh.depth, m, self.channels, mode,
                  int(self.approx_kernel_grad), 1)
        ws = _lib._ws(nb, xs.device)
        call("nksr_feature_vjp", self.svh.view(), self.feat_view(), xs, base, ranges, m, mode,
             int(self.approx_kernel_grad), a0, a1, coef.contiguous(), dz, ws, nb, stream_ptr(xs.device))

    def _evaluate_adjoint(self, loc, mode, coef):
        """dalpha = sum_q coef_q E_q at the sorted locations `loc`"""
        xs, base, ranges = loc
        m = xs.shape[0]
        dalpha = torch.empty(self.svh.num_unknowns, dtype=torch.float32, device=self.svh.device)
        nb = call("nksr_field_bwd_workspace_bytes", self.svh.depth, m, self.channels, mode,
                  int(self.approx_kernel_grad), 0)
        ws = _lib._ws(nb, dalpha.device)
        call("nksr_evaluate_adjoint", self.svh.view(), self.feat_view(), xs, base, ranges, m, mode,
             int(self.approx_kernel_grad), coef.contiguous(), dalpha, ws, nb, stream_ptr(dalpha.device))
        return dalpha

    def _level_grads(self, dz):
        offs = self.svh.offsets
        return tuple(dz[offs[l]:offs[l] + self.svh.num_voxels(l)] for l in range(self.svh.depth))

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


class _KernelSolve(torch.autograd.Function):
    """alpha = A(z)^-1 b(z, t).  Forward: the assembly and PCG of KernelField.solve (the same alpha, bit for bit).
    Backward, with lambda = A^-1 dL/dalpha (one more PCG on the same symmetric matrix):
      dL/dz   = sum_j w_j [(t_j - E_j alpha) d(E_j lambda) - (E_j lambda) d(E_j alpha)] - reg d(lambda^T R alpha)
      dL/dt_j = w_j E_j lambda                                                     (the normal rows' targets)
    The first line is a row functional with omega = c^lambda lambda + c^alpha alpha per row (nksr_feature_vjp).  On the
    assembled operator E_j alpha, E_j lambda are field evaluations at the constraint locations and E itself is not
    kept.  On the matrix-free operator (KernelField._grad_operator) the kernel rows stay resident with the operator's
    workspace until the backward: the adjoint PCG runs on the same operator and E_j alpha, E_j lambda are read from the
    rows (nksr_op_constraint_values)."""

    @staticmethod
    def forward(ctx, field, args, normal_value, *z):
        pos_xyz, normal_xyz, pos_weight, normal_weight, reg_weight = args
        ctx.matrix_free = field._grad_operator() == "matrix_free"
        if ctx.matrix_free:
            sysm = field.matrix_free_system(pos_xyz, normal_xyz, normal_value, pos_weight, normal_weight, reg_weight,
                                            keep_constraints=True)
            alpha = field._pcg_matrix_free(sysm, sysm.rhs)
            ctx.field, ctx.sysm = field, sysm
            ctx.save_for_backward(alpha)
            return alpha
        sysm = field.assemble(pos_xyz, normal_xyz, normal_value, pos_weight, normal_weight, reg_weight,
                              keep_constraints=True)
        alpha = field._pcg(sysm, sysm.rhs)
        if field.solver_config.get("keep_system"):
            field.system = sysm
        ctx.field, ctx.sysm = field, sysm
        ctx.save_for_backward(alpha)
        return alpha

    @staticmethod
    def backward(ctx, g_alpha):
        field, sysm, mf = ctx.field, ctx.sysm, ctx.matrix_free
        (alpha,) = ctx.saved_tensors
        cons = sysm.cons
        tm = getattr(field, "_timer", None) or _lib.StageTimer(alpha.device, enabled=False)
        tm.mark("backward_start")
        g_alpha = g_alpha.detach().to(torch.float32).contiguous()
        if bool((g_alpha != 0).any()):
            lam = field._pcg_matrix_free(sysm, g_alpha, adjoint=True) if mf else field._pcg(sysm, g_alpha, adjoint=True)
        else:
            lam = torch.zeros_like(alpha)
            field.solve_info.update(adjoint_iterations=0, adjoint_relative_residual=0.0)
        n, C_ = sysm.n, field.channels
        dz = torch.zeros((n, C_), dtype=torch.float32, device=alpha.device)
        xs, base, ranges = cons.pos
        if mf:
            vp, vn = field.constraint_values(sysm, alpha, lam)
            f_a, f_l = vp[:, 0], vp[:, 1]
        else:
            f_a, _ = field._evaluate(alpha, xs, False)
            f_l, _ = field._evaluate(lam, xs, False)
        coef = torch.stack([-cons.w_pos * f_a, -cons.w_pos * f_l], dim=1)         # omega = c^lam lam + c^alpha alpha
        field._feature_vjp(cons.pos, 0, coef, lam, alpha, dz)
        d_nv = None
        if cons.nrm is not None:
            xs_n = cons.nrm[0]
            if mf:
                g_a, g_l = vn[:, 0], vn[:, 1]
            else:
                _, g_a = field._evaluate(alpha, xs_n, True)
                _, g_l = field._evaluate(lam, xs_n, True)
            coef = torch.stack([cons.w_nrm * (cons.t_nrm - g_a), -cons.w_nrm * g_l], dim=1)     # (k, 2, 3)
            field._feature_vjp(cons.nrm, 1, coef, lam, alpha, dz)
            if ctx.needs_input_grad[2]:                                             # back to the caller's order
                d_nv = torch.empty_like(g_l)
                d_nv[cons.perm_nrm] = cons.w_nrm * g_l
        if cons.w_reg != 0.0:
            call("nksr_regulariser_vjp", field.svh.view(), field.feat_view(), lam, alpha, -cons.w_reg, dz,
                 stream_ptr(alpha.device))
        tm.mark("feature_vjp")
        ctx.field = ctx.sysm = None          # (field.alpha -> this node -> field: do not keep the system alive)
        return (None, None, d_nv) + field._level_grads(dz)


class _KernelEvaluate(torch.autograd.Function):
    """(f, grad f) = E(z, xyz) alpha.  Forward: nksr_evaluate (the same values as without grad).  Backward:
    dL/dalpha = sum_q g_q E_q (nksr_evaluate_adjoint); dL/dz = the row functional with omega = g_q alpha
    (nksr_feature_vjp), for the value and the gradient rows."""

    @staticmethod
    def forward(ctx, field, xyz, grad, alpha, *z):
        f, g = field._evaluate(alpha, xyz, grad)
        ctx.field, ctx.xyz, ctx.grad = field, xyz, grad
        ctx.save_for_backward(alpha)
        return (f, g) if grad else (f,)

    @staticmethod
    def backward(ctx, g_f, g_g=None):
        field = ctx.field
        (alpha,) = ctx.saved_tensors
        tm = getattr(field, "_timer", None) or _lib.StageTimer(alpha.device, enabled=False)
        tm.mark("evaluate_backward_start")
        n = field.svh.num_unknowns
        idx, xs, base, ranges = field._query_locations(ctx.xyz)
        loc = (xs, base, ranges)
        d_alpha = torch.zeros(n, dtype=torch.float32, device=alpha.device)
        dz = torch.zeros((n, field.channels), dtype=torch.float32, device=alpha.device)
        want_z = any(ctx.needs_input_grad[4:])
        for mode, g in ((0, g_f), (1, g_g if ctx.grad else None)):
            if g is None:
                continue
            coef = g.detach().to(torch.float32)[idx].contiguous()
            if ctx.needs_input_grad[3]:
                d_alpha += field._evaluate_adjoint(loc, mode, coef)
            if want_z:
                field._feature_vjp(loc, mode, coef, alpha, None, dz)
        tm.mark("evaluate_vjp")
        ctx.field = ctx.xyz = None
        return (None, None, None, d_alpha) + field._level_grads(dz)


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
    """MLP-decoded field over trilinearly interpolated voxel features (the UDF mask, models/nksr_net.py:124-130, and the
    output field of geometry='neural', :114-119; SPEC S17): f(x) = decoder(u(x)), u(x) = the interpolated features of
    every given level (a level with features, empty or not) in ascending order, C columns each.  The interpolation and
    its VJP are CUDA (csrc/neural_field.cu); the decoder is a PyTorch module.  When grad is enabled and the features or
    the decoder's parameters require grad, the values carry a graph into both (queries get no gradient).

    position_gradient: evaluate_f(xyz, grad=True) also returns grad f = sum_k (d decoder / d u_k)(u) J_k with J = du/dx
    (SPEC S17a, nksr_neural_interp_jacobian).  The decoder's Jacobian is taken with torch.autograd.grad of the sum of its
    outputs with respect to u, which assumes that the decoder acts on every row of u on its own (as the Linear / ReLU
    MLPs here do).  When grad is enabled and the features or the decoder's parameters require grad, the gradient keeps
    its graph (create_graph), so a loss on it reaches both: torch differentiates the decoder twice, and the CUDA nodes
    (_NeuralInterp for u, _NeuralJacobian for J) only need their first-order VJPs.  Without it (the default) the field
    is value-only and `gradient` is None."""

    def __init__(self, svh: SparseFeatureHierarchy, decoder, features, position_gradient: bool = False):
        super().__init__(svh)
        self.decoder = decoder
        self.position_gradient = bool(position_gradient)
        self.features = _as_level_list(features, svh.depth)
        given = [l for l, f in enumerate(self.features) if f is not None]
        if not given:
            raise ValueError("NeuralField needs features on at least one level")
        channels = {self.features[l].shape[1] for l in given}
        if len(channels) != 1:
            raise ValueError("all given levels must share one feature width")
        self.channels = channels.pop()
        if not (1 <= self.channels <= 32):
            raise ValueError("NeuralField features must have 1..32 channels")
        for l in given:
            if self.features[l].shape[0] != svh.num_voxels(l):
                raise ValueError(f"features[{l}] has {self.features[l].shape[0]} rows but level {l} has "
                                 f"{svh.num_voxels(l)} voxels")
        self.levels = given
        self.level_mask = sum(1 << l for l in given)

    def _inputs(self, xyz):
        _lib.require_cuda(xyz, "xyz")
        xyz = xyz.detach().to(self.svh.device, torch.float32).contiguous()
        feats = [f.to(self.svh.device, torch.float32).contiguous() if f is not None else None for f in self.features]
        return xyz, feats, torch.is_grad_enabled() and any(f is not None and f.requires_grad for f in feats)

    def interpolate(self, xyz: torch.Tensor) -> torch.Tensor:
        """u(x), (M, C * len(levels)) fp32 (nksr_neural_interp); differentiable in the features when grad is enabled
        and they require grad"""
        xyz, feats, graph = self._inputs(xyz)
        if graph:
            return _NeuralInterp.apply(self, xyz, *feats)
        return self._interp_cuda(xyz, feats)

    def jacobian(self, xyz: torch.Tensor) -> torch.Tensor:
        """J = du/dx, (M, 3, C * len(levels)) fp32 (nksr_neural_interp_jacobian, SPEC S17a): J[i][a] = d u(x_i) / dx_a;
        differentiable in the features when grad is enabled and they require grad"""
        xyz, feats, graph = self._inputs(xyz)
        if graph:
            return _NeuralJacobian.apply(self, xyz, *feats)
        return self._jacobian_cuda(xyz, feats)

    def _feat_view(self, feats):
        fv = _lib.FeatT()
        fv.channels = self.channels
        for l, f in enumerate(feats):
            fv.z[l] = f.data_ptr() if f is not None and f.shape[0] > 0 else None
        return fv

    def _interp_cuda(self, xyz, feats):
        m = xyz.shape[0]
        out = torch.empty((m, self.channels * len(self.levels)), dtype=torch.float32, device=xyz.device)
        call("nksr_neural_interp", self.svh.view(), self._feat_view(feats), self.level_mask, xyz, m, out,
             stream_ptr(xyz.device))
        return out

    def _jacobian_cuda(self, xyz, feats, with_values: bool = False):
        """J, or (u, J) from the same pass with `with_values` (u bitwise what _interp_cuda gives)"""
        m, w = xyz.shape[0], self.channels * len(self.levels)
        jac = torch.empty((m, 3, w), dtype=torch.float32, device=xyz.device)
        u = torch.empty((m, w), dtype=torch.float32, device=xyz.device) if with_values else None
        call("nksr_neural_interp_jacobian", self.svh.view(), self._feat_view(feats), self.level_mask, xyz, m, u, jac,
             stream_ptr(xyz.device))
        return (u, jac) if with_values else jac

    def _interp_vjp(self, xyz, g, jacobian: bool = False):
        """dL/dF_l for every level (None where not given) from g = dL/du (nksr_neural_interp_vjp), or with `jacobian`
        from g = dL/dJ, (M, 3, C * len(levels)) (nksr_neural_interp_jacobian_vjp): the queries with a containing voxel
        are Morton sorted and gathered per voxel, in one fixed order"""
        svh, dev = self.svh, xyz.device
        dz = torch.zeros((svh.num_unknowns, self.channels), dtype=torch.float32, device=dev)
        if svh.num_unknowns > 0 and xyz.shape[0] > 0:
            keep = torch.nonzero(svh.locate(xyz)[svh.depth - 1] >= 0).reshape(-1)
            perm, xs, _, _, ranges = _sorted_locations(svh, xyz[keep].contiguous())
            gs = g.detach().to(torch.float32)[keep[perm]].contiguous()
            call("nksr_neural_interp_jacobian_vjp" if jacobian else "nksr_neural_interp_vjp", svh.view(), self.channels,
                 self.level_mask, xs, ranges, xs.shape[0], gs, dz, stream_ptr(dev))
        offs = svh.offsets
        return tuple(dz[offs[l]:offs[l] + svh.num_voxels(l)] if l in self.levels else None for l in range(svh.depth))

    def _interp(self, xyz):
        """plain-torch restatement of `interpolate` (27 masked gathers per level, SPEC S17); a given empty level
        gives C zero columns"""
        svh = self.svh
        base = svh.locate(xyz).long()
        out = None
        for l in range(svh.depth):
            f = self.features[l]
            if f is None:
                continue
            if svh.num_voxels(l) == 0:
                acc = torch.zeros((xyz.shape[0], f.shape[1]), device=xyz.device, dtype=torch.float32)
                out = acc if out is None else torch.cat([out, acc], dim=1)
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
        """f at xyz; with `grad` and position_gradient also grad f (M, 3), else `gradient` is None"""
        if not (grad and self.position_gradient):
            v = self.decoder(self.interpolate(xyz)).reshape(-1)
            return EvaluationResult(value=v, gradient=None)
        xyz, feats, feat_graph = self._inputs(xyz)
        graph = feat_graph or (torch.is_grad_enabled() and any(
            p.requires_grad for p in getattr(self.decoder, "parameters", lambda: [])()))
        if feat_graph:
            u, jac = _NeuralInterp.apply(self, xyz, *feats), _NeuralJacobian.apply(self, xyz, *feats)
        else:
            u, jac = self._jacobian_cuda(xyz, feats, with_values=True)
        with torch.enable_grad():
            if not graph or not u.requires_grad:
                u = u.detach().requires_grad_(True)
            v = self.decoder(u).reshape(-1)
            (du,) = torch.autograd.grad(v.sum(), u, create_graph=graph)
        g = torch.einsum("mk,mak->ma", du, jac)
        if not graph:
            v = v.detach()
        return EvaluationResult(value=v, gradient=g)

    def mask(self, xyz):
        # UDF semantics: keep geometry closer than the level set to the data
        with torch.no_grad():
            return self.evaluate_f(xyz).value <= self.level_set

    def to_(self, device):
        super().to_(device)
        device = torch.device(device)
        self.features = [f.to(device) if f is not None else None for f in self.features]
        return self


class _NeuralInterp(torch.autograd.Function):
    """u = interpolate(F, xyz).  Forward: nksr_neural_interp (the same values as without grad).  Backward:
    dL/dF_l = sum_q T3(q) dL/du_q,l (nksr_neural_interp_vjp); the queries get no gradient."""

    @staticmethod
    def forward(ctx, field, xyz, *feats):
        ctx.field, ctx.xyz = field, xyz
        return field._interp_cuda(xyz, feats)

    @staticmethod
    def backward(ctx, g):
        dfeat = ctx.field._interp_vjp(ctx.xyz, g)
        ctx.field = ctx.xyz = None
        return (None, None) + tuple(d if need else None for d, need in zip(dfeat, ctx.needs_input_grad[2:]))


class _NeuralJacobian(torch.autograd.Function):
    """J = du/dx (F, xyz).  Forward: nksr_neural_interp_jacobian.  Backward: dL/dF_l = sum_q sum_a dT3_a(q) / W_l
    dL/dJ_q,a,l (nksr_neural_interp_jacobian_vjp); the queries get no gradient.  J is linear in F, so this VJP is the
    whole derivative: no CUDA op needs a second derivative."""

    @staticmethod
    def forward(ctx, field, xyz, *feats):
        ctx.field, ctx.xyz = field, xyz
        return field._jacobian_cuda(xyz, feats)

    @staticmethod
    def backward(ctx, g):
        dfeat = ctx.field._interp_vjp(ctx.xyz, g, jacobian=True)
        ctx.field = ctx.xyz = None
        return (None, None) + tuple(d if need else None for d, need in zip(dfeat, ctx.needs_input_grad[2:]))


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
