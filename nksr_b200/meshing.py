"""Dual marching cubes / MISE driver -- host mirror of field.extract_dual_mesh.

Reference contract: field.extract_dual_mesh(grid_upsample=, mise_iter=, max_points=) ->
mesh with .v (V,3) float tensor, .f (T,3) int tensor, .c colours
(models/nksr_net.py:214,284; examples/recons_simple.py:27; examples/recons_colored_mesh.py:30;
NKSR-USAGE.md:52,79).  Algorithm: DESIGN.md SPEC S8-S10; kernels: csrc/mesh.cu.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch

from . import _lib
from ._lib import call, stream_ptr

MAX_LATTICE_EXTENT = 1 << 20      # per axis, so that (morton << 2) | axis fits 62 bits
MAX_VIRTUAL_LEVEL = 6             # coarsest level whose leaves nksr_mesh_virtual_anchors expands (csrc/mesh.cu)


class DualMesh(SimpleNamespace):
    """Attribute bag like the reference's mesh result (callers overwrite fields, examples/gis_app.py:47-52)."""


def _evaluate(field, xyz, max_points):
    m = xyz.shape[0]
    if max_points is None or max_points <= 0 or m <= max_points:
        return field.evaluate_f(xyz).value
    out = torch.empty(m, dtype=torch.float32, device=xyz.device)
    for s in range(0, m, max_points):
        out[s:s + max_points] = field.evaluate_f(xyz[s:s + max_points]).value
    return out


def extract_dual_mesh(field, grid_upsample: int = 1, mise_iter: int = 0, max_points: int = -1,
                      cell_filter=None, multi_level=None) -> DualMesh:
    """`cell_filter` (optional, (n_0,) bool): only dual cells whose min-corner voxel passes are meshed --
    used by the multi-GPU path so that every rank meshes the cells it owns.
    `multi_level` (default: on for hierarchies built by build_adaptive_normal_variation, models/nksr_net.py:175-179):
    leaf voxels of the coarser levels are meshed as if subdivided down to the finest level, so pruned regions are
    covered and the surface has no cracks at level transitions."""
    svh = field.svh
    dev = svh.device
    st = stream_ptr(dev)
    W = svh.voxel_size
    g = int(grid_upsample)
    rounds = int(mise_iter)
    if g < 1 or rounds < 0:
        raise ValueError("grid_upsample >= 1 and mise_iter >= 0 required")
    R = g * (2 ** rounds)
    empty = DualMesh(v=torch.zeros((0, 3), device=dev), f=torch.zeros((0, 3), dtype=torch.int64, device=dev), c=None)
    n0 = svh.num_voxels(0)
    if n0 == 0 and not (multi_level or getattr(svh, "adaptive_depth", 0)):
        return empty
    if multi_level is None:
        multi_level = bool(getattr(svh, "adaptive_depth", 0))
    coarse = min(int(getattr(svh, "adaptive_depth", 0)) or svh.depth, svh.depth) if multi_level else 1
    if coarse <= 1:
        # ---- stage-0 cells: duals of 2x2x2 active finest voxels
        flag = torch.empty(n0, dtype=torch.int32, device=dev)
        call("nksr_mesh_cell_flags", svh.view(), flag, st)
        if cell_filter is not None:
            flag = (flag * cell_filter.to(torch.int32)).contiguous()
        scan = _lib.exclusive_scan32(flag)
        n_cells = int(scan[-1].item())
        if n_cells == 0:
            return empty
        cells = torch.empty((n_cells, 3), dtype=torch.int32, device=dev)
        call("nksr_mesh_stage0_cells", svh.view(), flag, scan, R, cells, st)
    else:
        # ---- adaptive hierarchy: leaves of the coarser levels count as subdivided ("virtual" finest voxels); a cell
        # is the cube between 2x2x2 finest voxels, real or virtual -- one lattice, no cracks at level transitions
        if cell_filter is not None:
            raise _lib.NksrError("multi-level meshing does not take a cell filter (multi-GPU meshing)")
        # leaves above MAX_VIRTUAL_LEVEL (8^7 finest voxels each) are refused before any anchor is allocated
        for l in range(MAX_VIRTUAL_LEVEL + 1, coarse):
            if svh.num_voxels(l) == 0:
                continue
            leaf = torch.empty(svh.num_voxels(l), dtype=torch.int32, device=dev)
            call("nksr_mesh_leaf_flags", svh.view(), l, leaf, st)
            n_leaf = int(leaf.sum().item())
            if n_leaf:
                raise _lib.NksrError(f"multi-level meshing expands leaves of levels 1..{MAX_VIRTUAL_LEVEL} only: level "
                                     f"{l} has {n_leaf} leaves (8^{l} finest voxels each); use adaptive_depth <= "
                                     f"{MAX_VIRTUAL_LEVEL + 1}")
        anchors = [torch.empty((n0, 3), dtype=torch.int32, device=dev)]
        if n0:
            call("nksr_decode_ijk", svh.keys[0], n0, 0, anchors[0], st)
        for l in range(1, coarse):
            n_l = svh.num_voxels(l)
            if n_l == 0:
                continue
            leaf = torch.empty(n_l, dtype=torch.int32, device=dev)
            call("nksr_mesh_leaf_flags", svh.view(), l, leaf, st)
            lscan = _lib.exclusive_scan32(leaf)
            n_leaf = int(lscan[-1].item())
            if n_leaf:
                va = torch.empty((n_leaf * 8 ** l, 3), dtype=torch.int32, device=dev)
                call("nksr_mesh_virtual_anchors", svh.view(), l, leaf, lscan, va, st)
                anchors.append(va)
        anchors = torch.cat(anchors) if len(anchors) > 1 else anchors[0]
        flag = torch.empty(anchors.shape[0], dtype=torch.int32, device=dev)
        call("nksr_mesh_anchor_flags", svh.view(), anchors, anchors.shape[0], coarse, flag, st)
        scan = _lib.exclusive_scan32(flag)
        n_cells = int(scan[-1].item())
        if n_cells == 0:
            return empty
        cells = (_lib.compact_rows(anchors, flag, scan, n_cells) * R).contiguous()
        del anchors
    lo = cells.min(dim=0).values.tolist()
    hi = cells.max(dim=0).values.tolist()
    if max(h - l for h, l in zip(hi, lo)) + R >= MAX_LATTICE_EXTENT:
        raise _lib.NksrError("mesh lattice extent exceeds 2^20 samples per axis: lower grid_upsample/mise_iter or chunk")
    ox, oy, oz = (int(v) for v in lo)
    size = R
    if g > 1:
        out = torch.empty((n_cells * g ** 3, 3), dtype=torch.int32, device=dev)
        call("nksr_mesh_split_cells", cells, n_cells, size, g, out, st)
        cells, n_cells, size = out, n_cells * g ** 3, size // g
    while True:
        # ---- evaluate f on the (deduplicated) corners of the current cells
        keys8 = torch.empty(n_cells * 8, dtype=torch.int64, device=dev)
        call("nksr_mesh_corner_keys", cells, n_cells, size, ox, oy, oz, keys8, st)
        ukeys = _lib.unique_sorted(_lib.sort_keys(keys8))
        nu = ukeys.numel()
        pos = torch.empty((nu, 3), dtype=torch.float32, device=dev)
        call("nksr_mesh_lattice_pos", ukeys, nu, ox, oy, oz, W, R, pos, st)
        uval = _evaluate(field, pos, max_points).contiguous()
        cval8 = torch.empty((n_cells, 8), dtype=torch.float32, device=dev)
        mc_case = torch.empty(n_cells, dtype=torch.int32, device=dev)
        crossing = torch.empty(n_cells, dtype=torch.int32, device=dev)
        call("nksr_mesh_classify", keys8, n_cells, ukeys, uval, nu, cval8, mc_case, crossing, st)
        del keys8, ukeys, pos, uval
        scan = _lib.exclusive_scan32(crossing)
        n_cross = int(scan[-1].item())
        if n_cross == 0:
            return empty
        cells = _lib.compact_rows(cells, crossing, scan, n_cross)
        if rounds == 0:
            cval8 = _lib.compact_rows(cval8, crossing, scan, n_cross)
            mc_case = _lib.compact_rows(mc_case, crossing, scan, n_cross)
            n_cells = n_cross
            break
        rounds -= 1
        out = torch.empty((n_cross * 8, 3), dtype=torch.int32, device=dev)
        call("nksr_mesh_split_cells", cells, n_cross, size, 2, out, st)
        cells, n_cells, size = out, n_cross * 8, size // 2
    # ---- edges -> welded vertices
    ntri = torch.empty(n_cells, dtype=torch.int32, device=dev)
    ekeys = torch.empty(n_cells * 12, dtype=torch.int64, device=dev)
    call("nksr_mesh_cell_edges", cells, mc_case, n_cells, size, ox, oy, oz, ntri, ekeys, st)
    skeys, ssrc = _lib.sort_pairs(ekeys, torch.arange(n_cells * 12, dtype=torch.int32, device=dev))
    heads = torch.empty(n_cells * 12, dtype=torch.int32, device=dev)
    call("nksr_run_heads", skeys, n_cells * 12, heads, st)
    hscan = _lib.exclusive_scan32(heads)
    n_v = int(hscan[-1].item())
    uekeys = _lib.compact_rows(skeys, heads, hscan, n_v)
    usrc = _lib.compact_rows(ssrc, heads, hscan, n_v)
    v = torch.empty((n_v, 3), dtype=torch.float32, device=dev)
    call("nksr_mesh_vertices", uekeys, usrc, n_v, cells, cval8, size, W, R, v, st)
    tscan = _lib.exclusive_scan32(ntri)
    n_t = int(tscan[-1].item())
    tri = torch.empty((n_t, 3), dtype=torch.int64, device=dev)
    call("nksr_mesh_triangles", mc_case, ekeys, tscan, n_cells, uekeys, n_v, tri, st)
    # ---- mask trimming (models/nksr_net.py:124-133): drop faces touching a masked-out vertex
    mask_field = getattr(field, "mask_field", None)
    if mask_field is not None and n_v > 0:
        keep_v = mask_field.mask(v)
        keep_f = keep_v[tri].all(dim=1)
        tri = tri[keep_f]
        used = torch.zeros(n_v, dtype=torch.bool, device=dev)
        used[tri.reshape(-1)] = True
        remap = torch.cumsum(used.long(), 0) - 1
        v, tri = v[used], remap[tri]
    mesh = DualMesh(v=v, f=tri, c=None)
    tex = getattr(field, "texture_field", None)
    if tex is not None and v.shape[0] > 0:
        mesh.c = tex.evaluate_f(v).value
    return mesh
