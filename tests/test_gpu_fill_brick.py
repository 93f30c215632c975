"""The brick fill (csrc/gram_fill_brick.cu, solver_config['fill'] = 'brick') against the row fill
(csrc/assemble.cu, 'rows', the default): the same CSR pattern and storage order bit for bit, values that differ only by the order in
which a row adds its 27 per-source partial sums (and its rhs chain), reproducible run to run, and within the oracle's
bounds like the row fill."""
import os

import numpy as np
import pytest
import torch

from oracle import nksr_oracle as O
from tests import clouds
from tests.bounds import KAPPA_GRAM, KAPPA_RHS, assert_within, level_of, level_pair_label

pytestmark = pytest.mark.gpu

# Reassociation bound: the row fill and the brick fill add the same 27 fp32 partial sums of an entry in two different
# orders, each order within 26 u of the exact sum in units of the sum of magnitudes, so the two differ by <= 52 u
# (u = 2^-24) of the oracle's magnitude scale of the entry; the rhs chain likewise.
KAPPA_REORDER = 52.0


def _np(t):
    return t.detach().cpu().numpy()


@pytest.fixture
def every_level(monkeypatch):
    """brick every level below the split level, whatever its constraint locations per voxel: the small clouds here
    would leave their sparse fine levels to the row fill"""
    from nksr_b200 import fields
    monkeypatch.setattr(fields, "BRICK_MIN_LOCATIONS_PER_VOXEL", 0.0)


def _csr(s):
    import scipy.sparse as sp
    n = s.rowptr.numel() - 1
    return sp.csr_matrix((_np(s.val).astype(np.float64), _np(s.col), _np(s.rowptr)), shape=(n, n))


def _hierarchy(cuda, xyz, W, L, prune=0.0, seed=0):
    """hierarchy from keys; `prune` drops that share of the finest level's voxels (isolated voxels, one-row bricks,
    bricks whose halo is inactive)"""
    import nksr_b200
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    keys = list(osvh.keys)
    if prune:
        keep = np.random.default_rng(seed).random(keys[0].shape[0]) >= prune
        keys[0] = keys[0][keep]
        osvh = O.OracleSVH(W, L).build_from_keys(keys)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_from_keys([t(k) for k in keys])
    return svh, osvh


def _systems(cuda, svh, osvh, xyz, W, approx, split, normals, layout, placement, compact=False,
             fills=("rows", "brick", "brick")):
    import nksr_b200
    L = osvh.depth
    rng = np.random.default_rng(5)
    feats = [(0.5 + 0.2 * rng.normal(size=(osvh.n(l), 4))).astype(np.float32) for l in range(L)]
    nxyz = np.concatenate([osvh.centers(d) for d in range(min(2, L))])
    nxyz = (nxyz + np.random.default_rng(3).uniform(-0.3, 0.3, nxyz.shape) * W).astype(np.float32)
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True)).astype(np.float32)
    pw, nw = 1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * W * W
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    out = []
    for fill in fills:
        field = nksr_b200.KernelField(svh, None, [t(f) for f in feats], approx)
        field.solver_config.update(keep_system=True, max_iter=0, fill=fill, row_layout=layout, placement=placement,
                                   compact_rows=compact)
        if split is not None:
            field.solver_config["block_split_level"] = split
        if normals:
            field.solve(t(xyz), t(nxyz), t(nval), pw, nw, 1.0)
        else:
            field.solve(t(xyz), None, None, pw, 0.0, 1.0)
        out.append(field.system)
    if not normals:
        nxyz, nval, nw = np.zeros((0, 3), np.float32), np.zeros((0, 3), np.float32), 0.0
    assert int(O.tent_branch_ambiguous(osvh, nxyz).sum()) == 0
    ref = O.build_system(osvh, feats, xyz, nxyz, nval, pw, nw, 1.0, approx, abs_terms=True)
    return out, ref


def _compare(out, ref, osvh, what):
    rows, brick, again = out
    A_ref, b_ref, _, A_abs, b_abs = ref
    offs = osvh.offsets()
    for name in ("rowptr", "col"):
        assert torch.equal(getattr(rows, name), getattr(brick, name)), f"{name} ({what})"
    for name in ("rowptr", "col", "val", "rhs", "diag"):
        assert torch.equal(getattr(brick, name), getattr(again, name)), f"{name} not reproducible ({what})"
    row = lambda i: f"row {i} level {level_of(offs, i)}"
    worst = [assert_within(_csr(brick), _csr(rows), A_abs, KAPPA_REORDER, f"brick vs rows values ({what})",
                           level_pair_label(offs)),
             assert_within(_np(brick.diag), _np(rows.diag), A_abs.diagonal(), KAPPA_REORDER,
                           f"brick vs rows diagonal ({what})", row),
             assert_within(_np(brick.rhs), _np(rows.rhs), b_abs, KAPPA_REORDER, f"brick vs rows rhs ({what})", row)]
    assert_within(_csr(brick), A_ref, A_abs, KAPPA_GRAM, f"brick vs oracle values ({what})", level_pair_label(offs))
    assert_within(_np(brick.rhs), b_ref, b_abs, KAPPA_RHS, f"brick vs oracle rhs ({what})", row)
    assert_within(_np(brick.diag), A_ref.diagonal(), A_abs.diagonal(), KAPPA_GRAM, f"brick vs oracle diagonal ({what})",
                  row)
    return worst


@pytest.mark.parametrize("L,W,prune,approx,split,normals,layout,placement,compact", [
    (4, 0.02, 0.0, False, None, True, "levels", "structural", False),      # bench settings: automatic split level
    (4, 0.02, 0.0, True, None, True, "interleaved", "structural", False),
    (4, 0.02, 0.5, True, 4, True, "levels", "structural", False),          # pruned finest level, every level bricked
    (4, 0.02, 0.0, False, 4, True, "interleaved", "structural", False),
    (4, 0.02, 0.0, False, 1, True, "levels", "structural", False),         # blocks from level 1: level 0 bricked
    (4, 0.02, 0.0, False, 0, True, "interleaved", "structural", False),    # blocks everywhere: no brick
    (4, 0.02, 0.0, False, None, True, "levels", "sorted", False),          # atomic-cursor placement: the row fill
    (4, 0.02, 0.0, True, None, True, "levels", "structural", True),        # compact gradient rows: the row fill
    (3, 0.03, 0.0, True, None, True, "interleaved", "structural", False),
    (2, 0.04, 0.0, False, None, True, "levels", "structural", False),
    (1, 0.05, 0.0, False, None, True, "interleaved", "structural", False),  # single level
    (4, 0.02, 0.0, False, None, False, "levels", "structural", False),     # position constraints only
    (5, 0.02, 0.0, False, None, True, "levels", "structural", False),      # depth > 4: the row fill
])
def test_brick_fill_is_the_row_fill(cuda, every_level, L, W, prune, approx, split, normals, layout, placement, compact):
    xyz, _ = clouds.shapenet_like(3000)
    svh, osvh = _hierarchy(cuda, xyz, W, L, prune)
    out, ref = _systems(cuda, svh, osvh, xyz, W, approx, split, normals, layout, placement, compact)
    worst = _compare(out, ref, osvh, f"L={L} W={W} prune={prune} approx={approx} split={split} normals={normals} "
                                     f"{layout} {placement} compact={compact}")
    print(f"[brick] worst reorder ratios (values, diagonal, rhs): {worst}")


def test_brick_layouts_give_the_same_system(cuda, every_level):
    """the brick fill under both row layouts: same products in the same order, bitwise the same system"""
    xyz, _ = clouds.shapenet_like(3000)
    svh, osvh = _hierarchy(cuda, xyz, 0.02, 4)
    (a,), _ = _systems(cuda, svh, osvh, xyz, 0.02, False, 4, True, "levels", "structural", fills=("brick",))
    (b,), _ = _systems(cuda, svh, osvh, xyz, 0.02, False, 4, True, "interleaved", "structural", fills=("brick",))
    for name in ("rowptr", "col", "val", "rhs", "diag"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name


def test_brick_edge_cases(cuda, every_level):
    """sparse scattered clouds around the origin (negative coordinates), with points on brick corners of every axis
    (4^3-voxel bricks: multiples of 4 W), a finest level with 85 % of its voxels removed (one-row bricks, bricks whose
    whole halo is inactive, source voxels without constraint rows) and a top level with fewer voxels than one brick"""
    W = 0.05
    rng = np.random.default_rng(11)
    corners = (np.array([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], np.float32) *
               np.float32(4 * W))
    scatter = rng.uniform(-0.3, 0.3, (300, 3)).astype(np.float32)
    xyz = np.concatenate([corners, corners + np.float32(0.001), scatter]).astype(np.float32)
    for L, prune, split in ((3, 0.85, 3), (4, 0.0, 4), (2, 0.6, None)):
        svh, osvh = _hierarchy(cuda, xyz, W, L, prune, seed=L)
        if L == 4:
            assert osvh.n(L - 1) <= 64
        out, ref = _systems(cuda, svh, osvh, xyz, W, False, split, True, "levels", "structural")
        _compare(out, ref, osvh, f"edge L={L} prune={prune} split={split}")


def test_sparse_levels_take_the_row_fill(cuda, monkeypatch):
    """a level with fewer constraint locations per voxel than fields.BRICK_MIN_LOCATIONS_PER_VOXEL runs the row fill:
    with the threshold above every level's density the 'brick' system is the row fill's, bit for bit"""
    from nksr_b200 import fields
    monkeypatch.setattr(fields, "BRICK_MIN_LOCATIONS_PER_VOXEL", 1e9)
    xyz, _ = clouds.shapenet_like(3000)
    svh, osvh = _hierarchy(cuda, xyz, 0.02, 4)
    (rows, brick), _ = _systems(cuda, svh, osvh, xyz, 0.02, False, 4, True, "levels", "structural",
                                fills=("rows", "brick"))
    for name in ("rowptr", "col", "val", "rhs", "diag"):
        assert torch.equal(getattr(rows, name), getattr(brick, name)), name


def test_brick_fill_at_bench_scale(cuda, every_level):
    """dev_outdoor_1M through reconstruct() with the bench settings, row fill against brick fill (every level below the
    split bricked): the same pattern,
    the largest |dval| per level pair relative to that pair's largest |val|, equal PCG iteration counts and field values
    within 1e-5 of max|f|"""
    import bench
    import nksr_b200
    from nksr_b200 import fields
    xyz, sensor = bench.make_cloud("dev_outdoor_1M", 4)
    xyz, sensor = xyz.to(cuda), sensor.to(cuda)
    rec = nksr_b200.Reconstructor(cuda, network=None, tree_depth=bench.TREE_DEPTH, adaptive_depth=bench.ADAPTIVE_DEPTH,
                                  kernel_dim=bench.KERNEL_DIM)
    prep = nksr_b200.get_estimate_normal_preprocess_fn(bench.KNN, bench.MAX_ANGLE)
    probe = xyz[::97].contiguous()
    systems, res = {}, {}
    orig = fields.KernelField.assemble

    def keep(self, *a, **kw):
        s = orig(self, *a, **kw)
        systems[self.solver_config.get("fill")] = (s, list(self.svh.offsets) + [self.svh.num_unknowns])
        return s
    old_env = os.environ.get("NKSR_FILL")
    try:
        fields.KernelField.assemble = keep
        for fill in ("rows", "brick"):
            os.environ["NKSR_FILL"] = fill
            orig_init = fields.KernelField.__init__

            def init(self, *a, _fill=fill, **kw):
                orig_init(self, *a, **kw)
                self.solver_config["fill"] = _fill
            fields.KernelField.__init__ = init
            try:
                f = rec.reconstruct(xyz, sensor=sensor, voxel_size=0.1, preprocess_fn=prep, **bench.SOLVER)
            finally:
                fields.KernelField.__init__ = orig_init
            res[fill] = (f.solve_info["iterations"], f.evaluate_f(probe).value.clone())
            del f
    finally:
        fields.KernelField.assemble = orig
        if old_env is None:
            os.environ.pop("NKSR_FILL", None)
        else:
            os.environ["NKSR_FILL"] = old_env
    (sr, offs), (sb, _) = systems["rows"], systems["brick"]
    assert torch.equal(sr.rowptr, sb.rowptr) and torch.equal(sr.col, sb.col)
    L = len(offs) - 1
    bounds = torch.tensor(offs[1:], device=cuda)
    report = {}
    for l in range(L):
        lo, hi = int(sr.rowptr[offs[l]]), int(sr.rowptr[offs[l + 1]])
        cl = torch.bucketize(sr.col[lo:hi].long(), bounds, right=True)
        dv = (sr.val[lo:hi] - sb.val[lo:hi]).abs()
        for m in range(L):
            sel = cl == m
            if bool(sel.any()):
                top = float(sr.val[lo:hi][sel].abs().max())
                report[(l, m)] = float(dv[sel].max()) / max(top, 1e-30)
    print(f"[brick] bench-scale max |dval| / max |val| per level pair: {report}")
    assert max(report.values()) <= 1e-5
    assert res["rows"][0] == res["brick"][0], f"PCG iterations {res['rows'][0]} vs {res['brick'][0]}"
    fr, fb = res["rows"][1], res["brick"][1]
    rel = float((fr - fb).abs().max()) / float(fr.abs().max())
    print(f"[brick] bench-scale field max |df| / max |f| = {rel:.3g}")
    assert rel <= 1e-5
