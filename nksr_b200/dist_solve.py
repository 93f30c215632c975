"""One GLOBAL solve sharded over several GPUs (SURVEY.md section 8e, mapping B; north_star:
"NCCL-over-NVLink only for the CG dot-product/norm allreduce and halo exchange at chunk boundaries").

The cloud is cut into slabs along its longest axis.  Rank r keeps the points of its slab plus a
halo of `halo_voxels` coarsest voxels on either side, builds the hierarchy, features, kernel rows
and Gram rows of that region with the ordinary single-GPU kernels, and OWNS the unknowns whose
voxel centre lies inside its slab.  Because every ingredient of a Gram row is a function of the
points within a few coarsest voxels, the rows of owned unknowns are bit-for-bit the rows of the
single-GPU system; the halo unknowns only serve as columns.  Conjugate gradients then run on the
union of the owned rows:

    per iteration:  halo exchange of u = M^-1 r (pack kernel -> ONE all-to-all -> unpack kernel)
                    SpMV on the owned rows of the local CSR + the three local dot products
                    ONE fused fp64 all-reduce of {(r,u), (w,u), (r,r)}
                    one fused vector-update kernel (Chronopoulos-Gear recurrences, verdict on the device)

Everything between the two collectives is a hand-written kernel of libnksr_b200.so (csrc/solve.cu,
`nksr_dcg_*`); the host only enqueues, and reads the device-side verdict every `check_every`
iterations.  Points travel once, by an all-to-all to the ranks whose slab (+ halo) contains them, so
no rank ever holds the whole cloud.  Works with `nccl` on GPUs; the key matching / ownership /
exchange logic is plain tensor code tested on gloo (CPU tensors).
"""
from __future__ import annotations

import ctypes as C
import os
from types import SimpleNamespace
from typing import List, Optional

import torch
import torch.distributed as dist

from . import _lib
from ._lib import call, stream_ptr
from .fields import KernelField, LayerField
from .svh import SparseFeatureHierarchy, SparseIndexGrid


def _world(group=None):
    return dist.get_world_size(group) if dist.is_initialized() else 1


def _rank(group=None):
    return dist.get_rank(group) if dist.is_initialized() else 0


def all_to_all_rows(chunks: List[torch.Tensor], group=None) -> List[torch.Tensor]:
    """Variable-size all-to-all of row blocks (same trailing shape and dtype): chunks[r] goes to rank r;
    returns what every rank sent here.  NCCL: one all_to_all_single for the counts and one for the payload;
    other backends (gloo CPU tests): point-to-point."""
    world, rank = _world(group), _rank(group)
    if world == 1:
        return [chunks[0]]
    dev, dtype, tail = chunks[0].device, chunks[0].dtype, tuple(chunks[0].shape[1:])
    width = 1
    for t in tail:
        width *= t
    send_counts = torch.tensor([c.shape[0] for c in chunks], dtype=torch.int64, device=dev)
    if dist.get_backend(group) == "nccl":
        recv_counts = torch.empty_like(send_counts)
        dist.all_to_all_single(recv_counts, send_counts, group=group)
        rc = recv_counts.tolist()
        send = torch.cat([c.reshape(c.shape[0], width) for c in chunks]).contiguous()
        recv = torch.empty((sum(rc), width), dtype=dtype, device=dev)
        dist.all_to_all_single(recv, send, output_split_sizes=rc, input_split_sizes=send_counts.tolist(), group=group)
        return [t.reshape((t.shape[0],) + tail) for t in torch.split(recv, rc)]
    allc = [torch.zeros(world, dtype=torch.int64, device=dev) for _ in range(world)]
    dist.all_gather(allc, send_counts, group=group)
    out, ops = [None] * world, []
    for r in range(world):
        n_in = int(allc[r][rank])
        if r == rank:
            out[r] = chunks[r]
            continue
        out[r] = torch.empty((n_in,) + tail, dtype=dtype, device=dev)
        if chunks[r].shape[0]:
            ops.append(dist.P2POp(dist.isend, chunks[r].contiguous(), r, group))
        if n_in:
            ops.append(dist.P2POp(dist.irecv, out[r], r, group))
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()
    return out


def slab_bounds(coord: torch.Tensor, world: int, quantum: float, group=None) -> List[float]:
    """world+1 increasing bounds along one axis, interior ones at point-count quantiles snapped to
    multiples of `quantum` (the coarsest voxel size): no voxel centre of any level lies on a bound.
    `coord` is this rank's share of the coordinates: the quantiles are taken over an equal-size sample
    of every rank (identical bounds on all ranks)."""
    if world <= 1:
        return [-float("inf"), float("inf")]
    m = 1 << 17
    if coord.numel() > 0:
        pick = torch.linspace(0, coord.numel() - 1, m, device=coord.device).long()
        sample = coord.double()[pick]
    else:
        sample = torch.full((m,), float("nan"), dtype=torch.float64, device=coord.device)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        parts = [torch.empty_like(sample) for _ in range(dist.get_world_size(group))]
        dist.all_gather(parts, sample, group=group)
        sample = torch.cat(parts)
    # (quantiles on the device the sample lives on: sorting world x 131 072 doubles on the host cost ~20 ms at 4 ranks)
    sample = sample[~torch.isnan(sample)]
    qs = torch.quantile(sample, torch.linspace(0, 1, world + 1, dtype=torch.float64, device=sample.device)[1:-1])
    inner = [round(float(q) / quantum) * quantum for q in qs.tolist()]
    for i in range(1, len(inner)):                         # strictly increasing
        inner[i] = max(inner[i], inner[i - 1] + quantum)
    return [-float("inf")] + inner + [float("inf")]


def owner_of(coord: torch.Tensor, bounds: List[float]) -> torch.Tensor:
    """rank owning a coordinate: number of interior bounds <= coord."""
    inner = torch.tensor(bounds[1:-1], dtype=torch.float64, device=coord.device)
    if inner.numel() == 0:
        return torch.zeros(coord.shape[0], dtype=torch.long, device=coord.device)
    return torch.searchsorted(inner, coord.double().contiguous(), right=True)


def route_points(coord: torch.Tensor, bounds: List[float], halo: float, arrays: List[torch.Tensor], group=None):
    """Point all-to-all: every rank sends each of its points (rows of `arrays`) to every rank whose slab widened
    by `halo` contains it.  Returns the list of arrays this rank receives (its slab + halo region)."""
    world = _world(group)
    if world == 1:
        return list(arrays)
    c = coord.double()
    per_rank = []
    for r in range(world):
        sel = torch.nonzero((c >= bounds[r] - halo) & (c < bounds[r + 1] + halo)).reshape(-1)
        per_rank.append(sel)
    out = []
    for a in arrays:
        got = all_to_all_rows([a[sel].contiguous() for sel in per_rank], group)
        out.append(torch.cat(got))
    return out


class HaloPlan:
    """Who sends which unknowns to whom.  send_idx[r]: my owned unknowns rank r needs;
    recv_idx[r]: my halo unknowns owned by rank r (same order on both sides)."""

    def __init__(self, send_idx, recv_idx, group=None):
        self.send_idx, self.recv_idx, self.group = send_idx, recv_idx, group
        self.send_cat = torch.cat(send_idx) if send_idx else None
        self.recv_cat = torch.cat(recv_idx) if recv_idx else None
        self.send_counts = [int(i.numel()) for i in send_idx]
        self.recv_counts = [int(i.numel()) for i in recv_idx]
        self._bufs = None

    @property
    def bytes_per_exchange(self) -> int:
        return 4 * (sum(self.send_counts) + sum(self.recv_counts))

    def exchange(self, vec: torch.Tensor):
        """halo entries of `vec` <- the owners' values.  CUDA: pack kernel, one all-to-all, unpack kernel."""
        if _world(self.group) == 1:
            return vec
        if vec.is_cuda and dist.get_backend(self.group) == "nccl":
            st = stream_ptr(vec.device)
            if self._bufs is None:
                self._bufs = (torch.empty(max(sum(self.send_counts), 1), dtype=torch.float32, device=vec.device),
                              torch.empty(max(sum(self.recv_counts), 1), dtype=torch.float32, device=vec.device))
            sbuf, rbuf = self._bufs
            ns, nr = sum(self.send_counts), sum(self.recv_counts)
            call("nksr_gather_f32", vec, self.send_cat, ns, sbuf, st)
            dist.all_to_all_single(rbuf[:nr], sbuf[:ns], output_split_sizes=self.recv_counts,
                                   input_split_sizes=self.send_counts, group=self.group)
            call("nksr_scatter_f32", rbuf, self.recv_cat, nr, vec, st)
            return vec
        got = all_to_all_rows([vec[i] for i in self.send_idx], self.group)
        rank = _rank(self.group)
        for r, idx in enumerate(self.recv_idx):
            if r != rank and idx.numel():
                vec[idx] = got[r]
        return vec


def build_halo_plan(level_keys: List[torch.Tensor], owner: List[torch.Tensor], offsets: List[int], group=None):
    """level_keys[l]: sorted Morton keys of my local voxels; owner[l]: owning rank of each.
    Voxels are matched across ranks by (level, key) -- bit-exact keys make this an integer join."""
    world, rank = _world(group), _rank(group)
    dev = level_keys[0].device
    empty = torch.zeros(0, dtype=torch.long, device=dev)
    if world == 1:
        return HaloPlan([empty], [empty], group)
    # what I need from rank r: (level, key) of my halo voxels owned by r, as int64 rows
    want, recv_idx = [], []
    for r in range(world):
        rows, idx = [], []
        if r != rank:
            for l, (keys, own) in enumerate(zip(level_keys, owner)):
                sel = torch.nonzero(own == r).reshape(-1)
                rows.append(torch.stack([torch.full_like(keys[sel], l), keys[sel]], dim=1))
                idx.append(sel + offsets[l])
        want.append(torch.cat(rows) if rows else torch.zeros((0, 2), dtype=torch.int64, device=dev))
        recv_idx.append(torch.cat(idx) if idx else empty)
    asked = all_to_all_rows(want, group)                               # asked[s]: what rank s wants from me
    send_idx, answers = [], []
    for s in range(world):
        req = asked[s]
        if s == rank or req.shape[0] == 0:
            send_idx.append(empty)
            answers.append(torch.zeros((0, 1), dtype=torch.int64, device=dev))
            continue
        parts = torch.zeros(req.shape[0], dtype=torch.long, device=dev)
        found = torch.zeros(req.shape[0], dtype=torch.bool, device=dev)
        for l, keys in enumerate(level_keys):
            m = req[:, 0] == l
            if keys.numel() == 0 or not bool(m.any()):
                continue
            k = req[m, 1]
            pos = torch.searchsorted(keys, k).clamp(max=keys.numel() - 1)
            hit = keys[pos] == k
            parts[m] = pos + offsets[l]
            found[m] = hit
        # A halo voxel the owner does not hold: both ranks built their hierarchy from the same points EXCEPT at the
        # outer rim of the requester's halo, where a per-rank preprocess (kNN normals + grazing filter on truncated
        # neighbourhoods) may keep a point the owner dropped.  Such voxels are many coarse voxels away from any row the
        # requester owns, so they are simply left out of the exchange (their entries stay zero); a voxel missing close
        # to the slab would mean the halo is too thin, which the thickness check of reconstruct_global guards.
        send_idx.append(parts[found])
        answers.append(found.to(torch.int64).reshape(-1, 1))
    replies = all_to_all_rows(answers, group)                          # replies[r]: which of my requests rank r serves
    asked_total, dropped = 0, 0
    for r in range(world):
        if r != rank and recv_idx[r].numel():
            ok = replies[r].reshape(-1).bool()
            asked_total += int(ok.numel())
            dropped += int((~ok).sum().item())
            recv_idx[r] = recv_idx[r][ok]
    if dropped > 0.05 * max(asked_total, 1) + 64:
        import warnings
        warnings.warn(f"nksr_b200 global solve, rank {rank}: {dropped} of {asked_total} halo voxels are unknown to their "
                      "owners -- more than the rim of a per-rank preprocess explains", RuntimeWarning)
    plan = HaloPlan(send_idx, recv_idx, group)
    plan.dropped = dropped
    return plan


def _gsum(t: torch.Tensor, group) -> torch.Tensor:
    s = t.sum(dtype=torch.float64).reshape(1)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(s, group=group)
    return s


def pcg_distributed(sysm, owned: torch.Tensor, plan: HaloPlan, tol: float, max_iter: int, check_every: int = 16,
                    group=None):
    """Jacobi-PCG (Chronopoulos-Gear form: one fused all-reduce per iteration) on the rows every rank owns of its
    local system: the CSR system of KernelField.assemble, or the matrix-free operator of
    KernelField.matrix_free_system (set up with the same `owned`).  `owned`: bool per local unknown.  Returns (x with
    halo entries filled, info dict)."""
    n, dev = sysm.n, sysm.rhs.device
    st = stream_ptr(dev)
    world = _world(group)
    own8 = owned.to(torch.uint8).contiguous()
    x, r, u, w, p, s = (torch.empty(n, dtype=torch.float32, device=dev) for _ in range(6))
    nb = call("nksr_dcg_workspace_bytes")
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    red = torch.zeros(3, dtype=torch.float64, device=dev)
    info = (C.c_double * 4)()
    if hasattr(sysm, "rowptr"):
        def apply_and_dots():
            call("nksr_dcg_spmv_dots", sysm.rowptr, sysm.col, sysm.val, own8, r, u, w, n, ws, red, st)
    else:
        def apply_and_dots():
            call("nksr_dcg_op_dots", sysm.svh_view, sysm.feat_view, sysm.cs, sysm.base_pos, sysm.base_nrm, sysm.ws,
                 sysm.ws_bytes, own8, r, u, w, ws, red, st)
    call("nksr_dcg_init", sysm.diag, sysm.rhs, own8, x, r, u, p, s, n, ws, nb, red, st)
    if world > 1:
        dist.all_reduce(red, group=group)
    call("nksr_dcg_begin", ws, red, float(tol), int(max_iter), st)
    launched, allreduces, exchanges = 0, 1 if world > 1 else 0, 0
    while True:
        for _ in range(max(int(check_every), 1)):
            plan.exchange(u)
            apply_and_dots()
            if world > 1:
                dist.all_reduce(red, group=group)
                allreduces += 1
                exchanges += 1
            call("nksr_dcg_update", sysm.diag, own8, x, r, u, w, p, s, n, ws, red, st)
            launched += 1
        call("nksr_dcg_status", ws, info, st)
        if info[3] != 0 or launched > max_iter + check_every:
            break
    plan.exchange(x)                                           # halo coefficients for evaluation / meshing
    return x, {"iterations": int(info[0]), "relative_residual": float(info[1]), "converged": int(info[2]) == 0,
               "allreduces": allreduces, "halo_exchanges": exchanges + (1 if world > 1 else 0),
               "iterations_launched": launched}


def resolve_operator(operator: Optional[str] = None) -> str:
    """The global solve's operator: the argument, else NKSR_OPERATOR, else 'assembled'."""
    op = operator or os.environ.get("NKSR_OPERATOR") or "assembled"
    if op not in ("matrix_free", "assembled"):
        raise ValueError("solver_config['operator'] must be 'matrix_free' or 'assembled'")
    return op


def local_system(reconstructor, lx: torch.Tensor, ln: Optional[torch.Tensor], lsens: Optional[torch.Tensor],
                 bounds: List[float], rank: int, axis: int, voxel_size: float, approx_kernel_grad: bool = False,
                 timer=None):
    """One rank's share of the global system, from the points routed to it (its slab [bounds[rank],
    bounds[rank + 1]) plus halo): hierarchy, network features and KernelField of the region, the owner of every
    unknown by voxel centre, and the constraint locations.  Touches no process group.  Returns a namespace with
    .field, .owner (per level: owning rank of each voxel), .owned (bool per unknown), .pos_xyz, .normal_xyz,
    .normal_value, and .counts (float64 [2]: points inside the slab, owned normal locations), which summed over the
    ranks give the constraint weights (constraint_weights)."""
    dev = lx.device
    if ln is not None:
        feat = ln
    elif lsens is not None:
        view = lsens - lx
        feat = view / (torch.linalg.norm(view, dim=-1, keepdim=True) + 1e-6)
    else:
        raise ValueError("either normal or sensor (with a normal-estimating preprocess_fn) is required")
    L = reconstructor.tree_depth
    lo, hi = bounds[rank], bounds[rank + 1]
    inside = (lx[:, axis].double() >= lo) & (lx[:, axis].double() < hi)
    counts = torch.tensor([float(inside.sum().item()), 0.0], dtype=torch.float64, device=dev)

    svh = SparseFeatureHierarchy(voxel_size, L, dev).build_point_splatting(lx)
    net = reconstructor.network
    enc = net.encoder(lx, feat, svh, 0)
    feats, dec_svh, _ = net.unet(enc, svh, adaptive_depth=reconstructor.adaptive_depth)
    field = KernelField(dec_svh, net.interpolators, feats.basis_features, approx_kernel_grad)
    if timer is not None:
        timer.mark("svh_and_network")
    ad = min(reconstructor.adaptive_depth, L)
    # ownership of every unknown / normal location by voxel-centre coordinate (exact: integer ijk)
    owner, centres = [], []
    for l in range(L):
        g = SparseIndexGrid(dec_svh, l)
        ijk = g.active_grid_coords()
        cen = (ijk[:, axis].double() + 0.5) * (float(voxel_size) * (2 ** l))
        owner.append(owner_of(cen, bounds))
        centres.append(g.grid_to_world(ijk))
    owned = torch.cat([o == rank for o in owner])
    counts[1] = float(sum(int((owner[d] == rank).sum().item()) for d in range(ad)))
    normal_xyz = torch.cat([centres[d] for d in range(ad)])
    normal_value = torch.cat([feats.normal_features[d] for d in range(ad)])
    return SimpleNamespace(field=field, owner=owner, owned=owned, pos_xyz=lx, normal_xyz=normal_xyz,
                           normal_value=-normal_value, counts=counts, adaptive_depth=ad)


def constraint_weights(n_points_global: float, k_global: float, voxel_size: float):
    """(pos_weight, normal_weight, reg_weight) of the global system from the global point and normal-location counts:
    the weights the single-GPU reconstruct uses for the whole cloud"""
    from .reconstructor import NORMAL_WEIGHT, POS_WEIGHT
    return POS_WEIGHT / n_points_global, NORMAL_WEIGHT / k_global * (float(voxel_size) ** 2), 1.0


def reconstruct_global(reconstructor, xyz: torch.Tensor, normal: Optional[torch.Tensor], voxel_size: float,
                       halo_voxels: int = 8, axis: Optional[int] = None, approx_kernel_grad: bool = False,
                       solver_tol: float = 1e-5, solver_max_iter: int = 2000, group=None, sensor=None,
                       preprocess_fn=None, distributed_input: bool = False, operator: Optional[str] = None):
    """ONE global system over all ranks.  `distributed_input=False`: every rank passes the same whole cloud
    (each keeps its slab + halo); True: every rank passes ITS SHARE of the cloud and the points are routed to
    the ranks that need them by one all-to-all.  `operator`: 'assembled' (the CSR Gram matrix of every rank's region)
    or 'matrix_free' (A applied from the kernel rows of the locations that feed owned rows, csrc/operator.cu); None
    reads NKSR_OPERATOR and assembles when that is unset.  Returns a KernelField over this rank's slab+halo region
    with `.owned` (per-unknown bool), `.owned_cells` (level-0 mask for meshing) and `.solve_info`."""
    op = resolve_operator(operator)
    if getattr(reconstructor.network, "structure", "encoder") == "predicted":
        # every rank would grow its own hierarchy from its own predictions, which can disagree in the halo
        raise _lib.NksrError("the global solve needs structure='encoder': hierarchies grown from the predicted "
                             "structure are not kept consistent across ranks")
    if getattr(reconstructor.network, "geometry", "kernel") == "neural":
        # the global solve is a kernel solve; a neural output field has nothing to solve
        raise _lib.NksrError("the global solve does not support geometry='neural': build the network with "
                             "geometry='kernel'")
    if getattr(reconstructor.network, "udf_enabled", False):
        # the sharded field is masked per slab by LayerField; there is no UDF hierarchy across ranks
        raise _lib.NksrError("the global solve does not support udf.enabled: build the network with "
                             "udf=dict(enabled=False)")
    world, rank = _world(group), _rank(group)
    dev = reconstructor.device
    xyz = xyz.detach().to(dev, torch.float32).contiguous()
    normal = normal.detach().to(dev, torch.float32).contiguous() if normal is not None else None
    sensor = sensor.detach().to(dev, torch.float32).contiguous() if sensor is not None else None
    tm = _lib.StageTimer(dev)                      # CUDA-event marks (NKSR_STAGE_TIMES=1), read by bench.py
    L = reconstructor.tree_depth
    w_top = float(voxel_size) * (2 ** (L - 1))
    lo_hi = torch.stack([xyz.min(dim=0).values, -xyz.max(dim=0).values]) if xyz.shape[0] else \
        torch.full((2, 3), float("inf"), device=dev)
    if world > 1:
        dist.all_reduce(lo_hi, op=dist.ReduceOp.MIN, group=group)
    if axis is None:
        axis = int(torch.argmax(-lo_hi[1] - lo_hi[0]).item())
    bounds = slab_bounds(xyz[:, axis], world, w_top, group) if world > 1 else \
        [-float("inf"), float("inf")]
    if world > 1 and not distributed_input:                    # same cloud everywhere -> same bounds; make sure
        b = torch.tensor(bounds[1:-1], dtype=torch.float64, device=dev)
        dist.broadcast(b, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        bounds = [-float("inf")] + b.tolist() + [float("inf")]
    lo, hi = bounds[rank], bounds[rank + 1]
    H = halo_voxels * w_top
    extras = [t for t in (normal, sensor) if t is not None]
    if distributed_input:
        routed = route_points(xyz[:, axis], bounds, H, [xyz] + extras, group)
    else:
        c = xyz[:, axis]
        local = (c >= lo - H) & (c < hi + H)
        routed = [t[local].contiguous() for t in [xyz] + extras]
    lx = routed[0].contiguous()
    ln = routed[1].contiguous() if normal is not None else None
    lsens = routed[-1].contiguous() if sensor is not None else None
    tm.mark("bounds_and_point_routing")
    if preprocess_fn is not None:
        lx, ln, lsens = preprocess_fn(lx, ln, lsens)
        lx = lx.contiguous()
    tm.mark("preprocess")
    loc = local_system(reconstructor, lx, ln, lsens, bounds, rank, axis, voxel_size, approx_kernel_grad, tm)
    field, owner, owned, counts = loc.field, loc.owner, loc.owned, loc.counts
    dec_svh, ad = field.svh, loc.adaptive_depth
    if world > 1:
        dist.all_reduce(counts, group=group)
    n_points_global, k_global = float(counts[0].item()), float(counts[1].item())
    weights = constraint_weights(n_points_global, k_global, voxel_size)
    if op == "matrix_free":
        # only the locations that feed an owned row are kept: the halo's other locations cost nothing per iteration
        sysm = field.matrix_free_system(loc.pos_xyz, loc.normal_xyz, loc.normal_value, *weights, owned=owned)
        sysm.svh_view, sysm.feat_view = dec_svh.view(), field.feat_view()
        tm.mark("ownership_and_operator_setup")
        op_info = dict(operator="matrix_free", operator_bytes_per_apply=sysm.bytes_per_apply,
                       locations_kept=sysm.locations_kept, locations_total=int(sysm.cs.n_pos + sysm.cs.n_nrm), nnz=0)
    else:
        sysm = field.assemble(loc.pos_xyz, loc.normal_xyz, loc.normal_value, *weights)
        tm.mark("ownership_and_assembly")
        op_info = dict(operator="assembled", nnz=sysm.nnz)
    plan = build_halo_plan(dec_svh.keys, owner, dec_svh.offsets, group)
    tm.mark("halo_plan")
    alpha, info = pcg_distributed(sysm, owned, plan, solver_tol, solver_max_iter, 16, group)
    tm.mark("pcg")
    field._stage_timer = tm
    field.alpha = alpha
    field.owned = owned
    field.owned_cells = owner[0] == rank
    field.solve_info = dict(info, n=sysm.n, **op_info, n_owned=int(owned.sum().item()),
                            halo_recv=int(sum(plan.recv_counts)), halo_send=int(sum(plan.send_counts)),
                            halo_bytes_per_exchange=plan.bytes_per_exchange, halo_dropped=getattr(plan, "dropped", 0),
                            slab=(lo, hi), axis=axis,
                            points_local=int(lx.shape[0]), points_global=int(n_points_global))
    field.set_mask_field(LayerField(dec_svh, ad))
    return field


def extract_global_mesh(field, mise_iter: int = 0, grid_upsample: int = 1, group=None):
    """Every rank meshes the dual cells whose min-corner voxel it owns; pieces are gathered on rank 0."""
    from .dist import gather_mesh
    mesh = field.extract_dual_mesh(grid_upsample=grid_upsample, mise_iter=mise_iter, cell_filter=field.owned_cells)
    v, f = gather_mesh(mesh.v, mesh.f, 0, group)
    return None if v is None else SimpleNamespace(v=v, f=f, c=None)
