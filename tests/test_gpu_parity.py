"""GPU parity tests: every CUDA stage, called through the C-ABI (nksr_b200._lib), against the CPU
oracle on the same seeded inputs.  Integer work bit-exact; floating point entry by entry within
kappa * 2^-24 of the oracle's fp64 magnitude scale of that entry (tests/bounds.py)."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import nksr_oracle as O
from tests import clouds
from tests.bounds import (KAPPA_FIELD, KAPPA_GRAM, KAPPA_RHS, KAPPA_ROWS, KAPPA_SPMV, assert_within, level_of,
                          level_pair_label)
from tests.placement_checks import assert_structural_placement

pytestmark = pytest.mark.gpu


def _np(t):
    return t.detach().cpu().numpy()


def _build(cuda, xyz, W, L):
    import nksr_b200
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_point_splatting(torch.from_numpy(xyz).to(cuda))
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    return svh, osvh


@pytest.mark.parametrize("cloud,W,L", [("shapenet", 0.02, 4), ("blob", 0.1, 4), ("sphere", 0.05, 3), ("blob", 0.37, 2)])
def test_svh_bit_exact(cuda, cloud, W, L):
    xyz = {"shapenet": clouds.shapenet_like(3000)[0], "blob": clouds.offset_blob(20000)[0],
           "sphere": clouds.sphere(5000)[0]}[cloud]
    svh, osvh = _build(cuda, xyz, W, L)
    for l in range(L):
        assert np.array_equal(_np(svh.keys[l]), osvh.keys[l]), f"keys level {l}"
        assert np.array_equal(_np(svh.grids[l].active_grid_coords()), osvh.ijk(l))
        assert np.array_equal(_np(svh.nbr27[l]).astype(np.int64), osvh.nbr27(l)), f"nbr27 level {l}"
        cen = _np(svh.get_voxel_centers(l))
        assert np.allclose(cen, osvh.centers(l), rtol=1e-6, atol=1e-7)
    for l in range(L - 1):
        par = osvh.lookup(l + 1, osvh.ijk(l).astype(np.int64) >> 1)
        assert np.array_equal(_np(svh.parent[l]).astype(np.int64), par)
        ch = _np(svh.child8[l + 1])
        for i in np.random.default_rng(0).integers(0, osvh.n(l), 200):
            slot = int(osvh.keys[l][i] & 7)
            assert ch[par[i], slot] == i
    q = (xyz[:4000] + np.float32(0.5 * W)).astype(np.float32)
    assert np.array_equal(_np(svh.locate(torch.from_numpy(q).to(cuda))).astype(np.int64), osvh.locate(q))


def test_svh_empty_and_single_point(cuda):
    import nksr_b200
    svh = nksr_b200.SparseFeatureHierarchy(0.1, 4, cuda).build_point_splatting(torch.zeros((0, 3), device=cuda))
    assert all(g is None for g in svh.grids)
    one = np.array([[0.123, -4.5, 7.7]], np.float32)
    svh, osvh = _build(cuda, one, 0.1, 4)
    for l in range(4):
        assert svh.num_voxels(l) == 8 and np.array_equal(_np(svh.keys[l]), osvh.keys[l])
    with pytest.raises(RuntimeError):
        nksr_b200.SparseFeatureHierarchy(1e-9, 4, cuda).build_point_splatting(torch.ones((4, 3), device=cuda))


def _feats(osvh, C, seed):
    rng = np.random.default_rng(seed)
    return [(0.5 + 0.2 * rng.normal(size=(osvh.n(l), C))).astype(np.float32) for l in range(osvh.depth)]


def _field(cuda, svh, feats, approx=False):
    import nksr_b200
    return nksr_b200.KernelField(svh, None, [torch.from_numpy(f).to(cuda) for f in feats], approx)


@pytest.mark.parametrize("C,approx", [(4, False), (16, False), (4, True), (3, False)])
def test_kernel_rows_match_oracle(cuda, C, approx):
    xyz, _ = clouds.shapenet_like(3000)
    svh, osvh = _build(cuda, xyz, 0.02, 4)
    feats = _feats(osvh, C, 7)
    field = _field(cuda, svh, feats, approx)
    q = torch.from_numpy(xyz[:1500]).to(cuda)
    for mode in (0, 1):
        xs, _, base, _, e = field._sorted_rows(q, mode)
        xs_np, base_np, e_np = _np(xs), _np(base).astype(np.int64), _np(e)
        assert np.array_equal(base_np, osvh.locate(xs_np))
        assert O.tent_branch_ambiguous(osvh, xs_np).sum() == 0        # no location to leave out (see _snap_free)
        for l in range(4):
            nbr, K, dK, Ka, dKa = O.level_rows(osvh, l, xs_np, base_np[l], feats[l], mode == 1, approx, abs_terms=True)
            if mode == 0:
                got, ref, scale, shape = e_np[:, l, :27], K, Ka, (-1, 27)
            else:
                got, ref, scale, shape = e_np[:, l].reshape(-1, 3, 32)[:, :, :27], dK, dKa, (-1, 3, 27)
            assert np.abs(ref).max() > 0
            assert_within(got, ref, scale, KAPPA_ROWS, f"{'dK' if mode else 'K'} rows level {l} (C={C}, approx={approx})",
                          lambda j, sh=shape: f"location {np.unravel_index(j, got.shape)[0]} "
                                              f"entry {np.unravel_index(j, got.shape)[1:]}")
            assert np.all(e_np[:, l].reshape(-1, 32)[:, 27:] == 0)


@pytest.mark.parametrize("L,C,approx", [(4, 4, False), (4, 4, True), (3, 16, False), (1, 4, True), (2, 3, False)])
def test_interleaved_rows_are_the_level_rows(cuda, L, C, approx):
    """nksr_build_rows mode | 4: the rows with the four levels of a slot in one float4 are, value for value (bitwise),
    the rows of the plain layout; levels the hierarchy does not have are zero."""
    xyz, _ = clouds.shapenet_like(3000)
    svh, osvh = _build(cuda, xyz, 0.02, L)
    field = _field(cuda, svh, _feats(osvh, C, 7), approx)
    rng = np.random.default_rng(4)
    q = np.concatenate([xyz[:2000], osvh.centers(0)[:1500],
                        osvh.centers(0)[:1500] + rng.uniform(-0.4, 0.4, (1500, 3)).astype(np.float32) * 0.02])
    q = torch.from_numpy(np.ascontiguousarray(q.astype(np.float32))).to(cuda)
    for mode in (0, 1):
        _, _, base, _, e = field._sorted_rows(q, mode)
        _, _, base_i, _, ei = field._sorted_rows(q, mode, interleaved=True)
        rows = 3 if mode == 1 else 1
        assert torch.equal(base, base_i) and ei.shape == (q.shape[0], rows, 32, 4)
        plain = e.reshape(q.shape[0], L, rows, 32).permute(0, 2, 3, 1)             # (m, rows, 32, L)
        assert torch.equal(ei[..., :L], plain)
        assert bool((ei[..., L:] == 0).all())
        assert float(plain.abs().max()) > 0


_LAYOUT_CASES = [
    (4, 0.02, False, None, True),     # automatic split level: blocks on the two coarse levels
    (4, 0.02, True, None, True),
    (4, 0.02, False, 4, True),        # every level through the row loops
    (4, 0.02, False, 1, True),        # blocks from level 1
    (4, 0.02, False, 0, True),        # blocks everywhere
    (3, 0.03, False, None, True),     # a level the layout pads with zeros
    (1, 0.05, False, None, True),
    (4, 0.02, False, None, False),    # position constraints only
]


# (the ids keep the "structural" they had while the placement was a parameter, so every case keeps its history)
@pytest.mark.parametrize("L,W,approx,split,normals", _LAYOUT_CASES,
                         ids=["-".join(map(str, case)) + "-structural" for case in _LAYOUT_CASES])
def test_interleaved_layout_gives_the_same_system(cuda, L, W, approx, split, normals):
    """solver_config['row_layout'] = 'interleaved' (csrc/assemble.cu, ILV: 128-bit loads of all levels of a location)
    against 'levels': same products in the same order -- row pointers, columns, values, rhs and diagonal are bitwise
    equal, through the row loops and through the per-voxel blocks."""
    import nksr_b200
    xyz, _ = clouds.shapenet_like(3000)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    svh, osvh = _build(cuda, xyz, W, L)
    feats = _feats(osvh, 4, 5)
    nxyz = np.concatenate([osvh.centers(d) for d in range(min(2, L))])
    rng = np.random.default_rng(3)
    nxyz[::2] += (rng.uniform(-0.3, 0.3, nxyz[::2].shape) * W).astype(np.float32)   # half at the centres, half generic
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True)).astype(np.float32)
    pw, nw = 1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * W * W
    out = []
    for layout in ("levels", "interleaved"):
        field = _field(cuda, svh, feats, approx)
        field.solver_config.update(keep_system=True, max_iter=0, row_layout=layout)
        if split is not None:
            field.solver_config["block_split_level"] = split
        if normals:
            field.solve(t(xyz), t(nxyz), t(nval), pw, nw, 1.0)
        else:
            field.solve(t(xyz), None, None, pw, 0.0, 1.0)
        s_ = field.system
        out.append([_np(a).copy() for a in (s_.rowptr, s_.col, s_.val, s_.rhs, s_.diag)])
    assert out[0][0][-1] > 0 and np.abs(out[0][2]).max() > 0
    for a, b in zip(*out):
        assert np.array_equal(a, b)


def test_overlapped_count_is_the_same_system(cuda):
    """solver_config['overlap_count']: row lengths, placement tables and row pointers on a side stream while the kernel
    rows are built -- the system must be the serial one bit for bit (and stay so when the allocator recycles the side
    stream's blocks over several solves)."""
    import nksr_b200
    xyz, nrm = clouds.sphere(40_000, noise=0.001)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    svh = nksr_b200.SparseFeatureHierarchy(0.02, 4, cuda).build_point_splatting(t(xyz))
    osvh = O.OracleSVH(0.02, 4).build_from_keys([_np(k) for k in svh.keys])
    feats = _feats(osvh, 4, 5)
    nxyz = _np(torch.cat([svh.get_voxel_centers(d) for d in range(2)]))
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True)).astype(np.float32)
    pw, nw = 1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * 0.02 * 0.02
    out = []
    for overlap in (False, True, True, False, True):
        field = _field(cuda, svh, feats, True)
        field.solver_config.update(keep_system=True, max_iter=3, overlap_count=overlap)
        field.solve(t(xyz), t(nxyz), t(nval), pw, nw, 1.0)
        s_ = field.system
        out.append([_np(a).copy() for a in (s_.rowptr, s_.col, s_.val, s_.rhs, s_.diag, field.alpha)])
        del field
    for other in out[1:]:
        for a, b in zip(out[0], other):
            assert np.array_equal(a, b)


@pytest.mark.parametrize("C,approx,mode", [(4, False, 0), (4, False, 1), (4, True, 1), (4, True, 2), (16, False, 1),
                                           (8, True, 2), (16, False, 0)])
def test_voxel_rows_are_the_location_rows(cuda, C, approx, mode):
    """csrc/field.cu: the warp-per-voxel row builder (solver_config['rows'] = 'voxel') writes
    bitwise the rows of the warp-per-location builder -- including the zero lines of locations whose containing
    voxel is inactive on some level (here: constraint locations at the centres of childless level-1 voxels)."""
    xyz, _ = clouds.shapenet_like(3000)
    svh, osvh = _build(cuda, xyz, 0.02, 4)
    feats = _feats(osvh, C, 7)
    rng = np.random.default_rng(4)
    q = np.concatenate([xyz[:2000], osvh.centers(1), osvh.centers(0)[:3000] + rng.uniform(-0.4, 0.4, (3000, 3)).astype(np.float32) * 0.02])
    q = torch.from_numpy(np.ascontiguousarray(q.astype(np.float32))).to(cuda)
    out = {}
    for rows in ("location", "voxel"):
        field = _field(cuda, svh, feats, approx)
        field.solver_config["rows"] = rows
        _, _, base, _, e = field._sorted_rows(q, mode)
        out[rows] = _np(e).copy()
    assert (_np(base) < 0).any()                                      # the zero-line case is exercised
    assert np.array_equal(out["location"], out["voxel"])


def _solve_setup(cuda, C=4, approx=False, n_pts=3000, W=0.02, L=4, cloud="shapenet"):
    xyz, nrm = clouds.shapenet_like(n_pts) if cloud == "shapenet" else clouds.sphere(n_pts)
    svh, osvh = _build(cuda, xyz, W, L)
    feats = _feats(osvh, C, 11)
    field = _field(cuda, svh, feats, approx)
    nxyz = np.concatenate([osvh.centers(0), osvh.centers(1)])
    rng = np.random.default_rng(3)
    nval = rng.normal(size=nxyz.shape).astype(np.float32)
    nval /= np.linalg.norm(nval, axis=1, keepdims=True)
    pw, nw, rw = 1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * W * W, 1.0
    return field, svh, osvh, feats, xyz, nxyz, nval, (pw, nw, rw)


def _gpu_csr(field):
    s = field.system
    n = s.rowptr.numel() - 1
    return sp.csr_matrix((_np(s.val).astype(np.float64), _np(s.col), _np(s.rowptr)), shape=(n, n))


@pytest.mark.parametrize("C,approx,compact,split", [(4, False, False, None), (16, True, False, 1), (4, True, True, None),
                                                    (4, False, False, 4), (4, True, False, 3)])
def test_gram_assembly_matches_oracle(cuda, C, approx, compact, split):
    """split = level from which per-voxel Gram blocks are used (None: automatic, 4: never)."""
    field, svh, osvh, feats, xyz, nxyz, nval, (pw, nw, rw) = _solve_setup(cuda, C, approx)
    field.solver_config.update(keep_system=True, max_iter=0, compact_rows=compact, block_split_level=split)
    t = lambda a: torch.from_numpy(a).to(cuda)
    field.solve(t(xyz), t(nxyz), t(nval), pw, nw, rw)
    _snap_free(osvh, nxyz)
    A_ref, b_ref, _, A_abs, b_abs = O.build_system(osvh, feats, xyz, nxyz, nval, pw, nw, rw, approx, abs_terms=True)
    A = _gpu_csr(field)
    # structure: exactly the structural pattern of SPEC S6, no duplicates, sorted transposed segments
    P = O.structural_pattern(osvh)
    Ab = A.copy(); Ab.data[:] = 1
    assert A.nnz == P.nnz
    Ab.sum_duplicates()
    assert Ab.nnz == P.nnz and (Ab - P).count_nonzero() == 0
    # values
    assert abs(A - A.T).max() <= 1e-6 * abs(A_ref).max()          # transposed copies are bitwise copies
    _check_system(field, osvh, A_ref, b_ref, A_abs, b_abs, f"C={C} approx={approx} compact={compact} split={split}")


@pytest.mark.parametrize("L,W,prune", [(4, 0.02, False), (2, 0.04, False), (5, 0.02, False), (3, 0.03, True)])
def test_structural_placement_is_the_same_matrix(cuda, monkeypatch, L, W, prune):
    """SPEC S6b, with the row fill and with the default brick fill (every level below the split bricked): the transposed
    entries, placed from prefix tables (no atomics, no sort), give row lengths that split the structural pattern at the
    level offsets, fill every slot once, stand in every row's finer-level segment in the order of the host reference
    (placement_proto.transposed_order), each hold bitwise the entry they copy, and are stored identically run to run."""
    import nksr_b200
    from nksr_b200 import fields
    monkeypatch.setattr(fields, "BRICK_MIN_LOCATIONS_PER_VOXEL", 0.0)
    xyz, _ = clouds.shapenet_like(3000)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    keys = list(osvh.keys)
    if prune:                                               # a pruned finest level: childless level-1 voxels
        keys[0] = keys[0][O.key_to_ijk(keys[0], 0)[:, 0] >= 0]
        osvh = O.OracleSVH(W, L).build_from_keys(keys)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_from_keys([t(k) for k in keys])
    feats = _feats(osvh, 4, 5)
    nxyz = np.concatenate([osvh.centers(d) for d in range(min(2, L))])
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True)).astype(np.float32)
    pw, nw = 1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * W * W
    for fill in ("rows", "brick"):
        out = []
        for _ in range(2):
            field = _field(cuda, svh, feats, False)
            field.solver_config.update(keep_system=True, max_iter=0, fill=fill)
            field.solve(t(xyz), t(nxyz), t(nval), pw, nw, 1.0)
            s = field.system
            out.append([_np(a).copy() for a in (s.rowptr, s.col, s.val, s.cnt, s.cnt_down)])
        assert_structural_placement(osvh, *out[0], fill)
        again = out[1]
        for a, b in zip(out[0][:3], again[:3]):
            assert np.array_equal(a, b), fill


@pytest.mark.parametrize("L,W,prune,approx,compact,split,normals", [
    (4, 0.02, False, False, False, None, True),     # bench settings: automatic block split level
    (4, 0.02, True, True, False, 4, True),          # pruned finest level, no blocks at all
    (4, 0.02, False, True, True, None, True),       # compact gradient rows (approx_kernel_grad)
    (4, 0.02, False, False, False, 1, True),        # blocks from level 1 upwards
    (3, 0.03, False, True, False, 0, True),         # every level through blocks
    (2, 0.04, False, False, False, None, True),
    (1, 0.05, False, False, False, None, True),     # single level: rows of the top level only
    (4, 0.02, False, False, False, None, False),    # position constraints only
])
def test_grouped_fill_is_the_row_fill(cuda, L, W, prune, approx, compact, split, normals):
    """The sibling-group fill (csrc/gram_fill_group.cu, solver_config['fill'] = 'grouped') stores the matrix of the
    row-per-warp fill (the default):
    identical row pointers and columns (same structural order, same placement of the transposed entries), values /
    rhs / diagonal equal up to fp32 summation order, and it is run-to-run bitwise reproducible."""
    import nksr_b200
    xyz, _ = clouds.shapenet_like(3000)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    keys = list(osvh.keys)
    if prune:
        keys[0] = keys[0][O.key_to_ijk(keys[0], 0)[:, 0] >= 0]
        osvh = O.OracleSVH(W, L).build_from_keys(keys)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_from_keys([t(k) for k in keys])
    feats = _feats(osvh, 4, 5)
    nxyz = np.concatenate([osvh.centers(d) for d in range(min(2, L))])
    rng = np.random.default_rng(3)
    nxyz = (nxyz + rng.uniform(-0.3, 0.3, nxyz.shape) * W).astype(np.float32)     # off-centre: generic tau
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True)).astype(np.float32)
    pw, nw = 1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * W * W
    out = []
    for fill in ("rows", "grouped", "grouped"):
        field = _field(cuda, svh, feats, approx)
        field.solver_config.update(keep_system=True, max_iter=0, fill=fill, compact_rows=compact)
        if split is not None:
            field.solver_config["block_split_level"] = split
        if normals:
            field.solve(t(xyz), t(nxyz), t(nval), pw, nw, 1.0)
        else:
            field.solve(t(xyz), None, None, pw, 0.0, 1.0)
        s = field.system
        out.append([_np(a).copy() for a in (s.rowptr, s.col, s.val, s.rhs, s.diag)])
    (rp_r, col_r, val_r, rhs_r, dg_r), (rp_g, col_g, val_g, rhs_g, dg_g), second = out
    assert np.array_equal(rp_r, rp_g) and np.array_equal(col_r, col_g)
    scale = np.abs(val_r).max()
    assert np.abs(val_r - val_g).max() <= 5e-6 * scale
    assert np.abs(rhs_r - rhs_g).max() <= 1e-5 * max(np.abs(rhs_r).max(), 1e-30)
    assert np.abs(dg_r - dg_g).max() <= 5e-6 * scale
    for a, b in zip(out[1], second):
        assert np.array_equal(a, b)


def _snap_free(osvh, xyz):
    """The tent derivative switches formula at |tau| = 2^-12 (the snap zone); an fp32 tau within a few ulps of that
    edge may take the other formula than the fp64 oracle, which is no rounding error.  The fixtures here have no
    such location: none is left out, and this assertion says so should a fixture change."""
    assert int(O.tent_branch_ambiguous(osvh, xyz).sum()) == 0


def _check_system(field, osvh, A_ref, b_ref, A_abs, b_abs, what):
    """values, rhs and diagonal of the assembled system entry by entry against the oracle's magnitude scales"""
    offs = osvh.offsets()
    assert_within(_gpu_csr(field), A_ref, A_abs, KAPPA_GRAM, f"Gram values ({what})", level_pair_label(offs))
    row = lambda i: f"row {i} level {level_of(offs, i)}"
    assert_within(_np(field.system.rhs), b_ref, b_abs, KAPPA_RHS, f"rhs ({what})", row)
    assert_within(_np(field.system.diag), A_ref.diagonal(), A_abs.diagonal(), KAPPA_GRAM, f"diagonal ({what})", row)


def test_gram_position_only_and_determinism(cuda):
    field, svh, osvh, feats, xyz, nxyz, nval, (pw, nw, rw) = _solve_setup(cuda, 4, False, 2000, 0.05, 3, "sphere")
    field.solver_config.update(keep_system=True, max_iter=0)
    t = lambda a: torch.from_numpy(a).to(cuda)
    field.solve(t(xyz), None, None, pw, 0.0, rw)
    A1 = (_np(field.system.val).copy(), _np(field.system.col).copy())
    A_ref, b_ref, _, A_abs, b_abs = O.build_system(osvh, feats, xyz, np.zeros((0, 3), np.float32), np.zeros((0, 3)),
                                                   pw, 0.0, rw, abs_terms=True)
    assert_within(_gpu_csr(field), A_ref, A_abs, KAPPA_GRAM, "Gram values (positions only)",
                  level_pair_label(osvh.offsets()))
    assert_within(_np(field.system.diag), A_ref.diagonal(), A_abs.diagonal(), KAPPA_GRAM, "diagonal (positions only)")
    field.solve(t(xyz), None, None, pw, 0.0, rw)
    assert np.array_equal(A1[0], _np(field.system.val)) and np.array_equal(A1[1], _np(field.system.col))


def test_spmv_and_pcg_match_oracle(cuda):
    import nksr_b200._lib as L
    field, svh, osvh, feats, xyz, nxyz, nval, (pw, nw, rw) = _solve_setup(cuda)
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True)).astype(np.float32)
    field.solver_config.update(keep_system=True, tol=1e-6, max_iter=3000, check_every=1)
    t = lambda a: torch.from_numpy(a).to(cuda)
    field.solve(t(xyz), t(nxyz), t(nval), pw, nw, rw)
    A = _gpu_csr(field)
    s = field.system
    x = torch.randn(A.shape[0], device=cuda)
    y = torch.empty_like(x)
    L.call("nksr_spmv", s.rowptr, s.col, s.val, x, y, A.shape[0], L.stream_ptr(cuda))
    yr = A @ _np(x).astype(np.float64)
    assert_within(_np(y), yr, abs(A) @ np.abs(_np(x)).astype(np.float64), KAPPA_SPMV, "row SpMV (assembled)")
    # PCG: converged, and the solution solves the oracle's system
    assert field.solve_info["relative_residual"] <= 1e-6
    A_ref, b_ref, _ = O.build_system(osvh, feats, xyz, nxyz, nval, pw, nw, rw)
    xo, it, res = O.pcg(A_ref, b_ref, 1e-9, 5000)
    alpha = _np(field.alpha).astype(np.float64)
    assert np.linalg.norm(A_ref @ alpha - b_ref) <= 1e-4 * np.linalg.norm(b_ref)
    # same field: compare f at the points rather than alpha (ill-conditioned directions)
    fo = O.evaluate_f(osvh, feats, xo, xyz[:500])
    fg = _np(field.evaluate_f(t(xyz[:500])).value)
    assert np.abs(fo - fg).max() <= 2e-3 * max(np.abs(fo).max(), 1e-3) + 2e-4
    assert abs(field.solve_info["iterations"] - O.pcg(A_ref, b_ref, 1e-6, 5000, dtype=np.float32)[1]) <= \
        0.25 * field.solve_info["iterations"] + 5


def _random_csr(n, lengths, seed, cuda):
    """CSR with the given row lengths (columns random with repeats allowed: SpMV does not care), fp32 values"""
    rng = np.random.default_rng(seed)
    rowptr = np.zeros(n + 2, np.int64)
    rowptr[1:n + 1] = np.cumsum(lengths)
    nnz = int(rowptr[n])
    col = rng.integers(0, n, nnz + 4).astype(np.int32)
    val = rng.normal(size=nnz + 4).astype(np.float32)
    t = lambda a: torch.from_numpy(a).to(cuda)
    return t(rowptr)[:n + 1], t(col)[:nnz], t(val)[:nnz], nnz


@pytest.mark.parametrize("kind", ["assembled", "ragged", "long_rows", "tiny_rows", "one_tile"])
def test_streamed_spmv_matches_row_spmv(cuda, kind):
    """The TMA-streamed SpMV (bulk async copies of 4096-entry tiles, csrc/spmv_stream.cuh) against the warp-per-row
    kernel and a float64 product: rows cut by tile boundaries (heads added in tile order), rows longer than several
    tiles, tiles holding more rows than the staged row-pointer slice, a matrix smaller than one tile; and the
    result is bitwise reproducible."""
    import nksr_b200._lib as L
    rng = np.random.default_rng(11)
    if kind == "assembled":
        field, *_rest = _solve_setup(cuda)
        xyz, nxyz, nval, (pw, nw, rw) = _rest[3], _rest[4], _rest[5], _rest[6]
        field.solver_config.update(keep_system=True, max_iter=0)
        t = lambda a: torch.from_numpy(a).to(cuda)
        field.solve(t(xyz), t(nxyz), t(nval), pw, nw, rw)
        s = field.system
        rowptr, col, val, nnz = s.rowptr, s.col, s.val, s.nnz
        n = rowptr.numel() - 1
    else:
        n = {"ragged": 30_000, "long_rows": 4_000, "tiny_rows": 200_000, "one_tile": 37}[kind]
        if kind == "ragged":
            lengths = rng.choice([1, 7, 120, 213, 317, 900, 5000], n, p=[.05, .1, .3, .3, .2, .04, .01])
        elif kind == "long_rows":
            lengths = rng.choice([3, 200, 4096, 9000, 40_000], n, p=[.3, .5, .1, .07, .03])
        elif kind == "tiny_rows":
            lengths = rng.choice([1, 2, 3], n)                  # > 512 rows per tile: row pointers read from HBM
        else:
            lengths = rng.integers(1, 60, n)
        rowptr, col, val, nnz = _random_csr(n, lengths, 5, cuda)
    x = torch.randn(n, device=cuda)
    y_rows = torch.empty_like(x)
    L.call("nksr_spmv", rowptr, col, val, x, y_rows, n, L.stream_ptr(cuda))
    nb = L.call("nksr_spmv_plan_bytes", nnz)
    plan = torch.empty(nb, dtype=torch.uint8, device=cuda)
    ys = []
    for _ in range(2):
        y = torch.full_like(x, float("nan"))
        # everything streamed, and (second pass) the last third of the rows handed to the warp-per-row kernel
        split = n if len(ys) == 0 else (2 * n) // 3
        L.call("nksr_spmv_stream", rowptr, col, val, x, y, n, nnz, split, int(rowptr[split].item()), plan, nb,
               L.stream_ptr(cuda))
        ys.append(_np(y).copy())
    y2 = torch.full_like(x, float("nan"))
    L.call("nksr_spmv_stream", rowptr, col, val, x, y2, n, nnz, n, nnz, plan, nb, L.stream_ptr(cuda))
    assert np.array_equal(ys[0], _np(y2))                         # bitwise reproducible
    A = sp.csr_matrix((_np(val).astype(np.float64), _np(col), _np(rowptr)), shape=(n, n))
    ref = A @ _np(x).astype(np.float64)
    absA = abs(A) @ np.abs(_np(x)).astype(np.float64)           # scale of the terms of each row sum
    assert_within(ys[0], ref, absA, KAPPA_SPMV, f"streamed SpMV ({kind})")
    assert_within(ys[1], ref, absA, KAPPA_SPMV, f"streamed SpMV, last third by rows ({kind})")
    assert_within(_np(y_rows), ref, absA, KAPPA_SPMV, f"row SpMV ({kind})")


def test_streamed_pcg_is_the_row_pcg(cuda):
    """Same system, PCG with the streamed SpMV against PCG with the row SpMV: both converge to the tolerance and to
    the same solution (fp32 summation order is the only difference)."""
    out = {}
    for spmv in ("rows", "stream"):
        field, svh, osvh, feats, xyz, nxyz, nval, (pw, nw, rw) = _solve_setup(cuda)
        field.solver_config.update(tol=1e-6, max_iter=3000, spmv=spmv)
        t = lambda a: torch.from_numpy(a).to(cuda)
        field.solve(t(xyz), t(nxyz), t(nval), pw, nw, rw)
        assert field.solve_info["converged"] and field.solve_info["relative_residual"] <= 1e-6
        out[spmv] = (_np(field.alpha).astype(np.float64), field.solve_info["iterations"])
    (a_r, it_r), (a_s, it_s) = out["rows"], out["stream"]
    assert abs(it_r - it_s) <= 0.1 * it_r + 3
    assert np.linalg.norm(a_r - a_s) <= 1e-3 * np.linalg.norm(a_r)


@pytest.mark.parametrize("C,approx", [(4, False), (16, True)])
def test_evaluate_matches_oracle(cuda, C, approx):
    xyz, _ = clouds.shapenet_like(3000)
    svh, osvh = _build(cuda, xyz, 0.02, 4)
    feats = _feats(osvh, C, 5)
    field = _field(cuda, svh, feats, approx)
    rng = np.random.default_rng(1)
    alpha = rng.normal(size=osvh.offsets()[-1]).astype(np.float32)
    field.alpha = torch.from_numpy(alpha).to(cuda)
    q = np.concatenate([xyz[:1000] + rng.normal(size=(1000, 3)).astype(np.float32) * 0.01,
                        rng.uniform(-0.7, 0.7, size=(500, 3)).astype(np.float32),       # mostly outside the band
                        osvh.centers(0)[:300], osvh.centers(2)[:100]]).astype(np.float32)
    _snap_free(osvh, q)
    r = field.evaluate_f(torch.from_numpy(q).to(cuda), grad=True)
    fo, go, fa, ga = O.evaluate_f(osvh, feats, alpha.astype(np.float64), q, grad=True, approx_kernel_grad=approx,
                                  abs_terms=True)
    assert_within(_np(r.value), fo, fa, KAPPA_FIELD, f"f (C={C}, approx={approx})", lambda j: f"query {j}")
    assert_within(_np(r.gradient), go, ga, KAPPA_FIELD, f"grad f (C={C}, approx={approx})",
                  lambda j: f"query {j // 3} axis {j % 3}")
    r2 = field.evaluate_f(torch.from_numpy(q).to(cuda))
    assert np.array_equal(_np(r2.value), _np(r.value))


@pytest.mark.parametrize("g,mise", [(1, 0), (2, 0), (1, 1), (1, 2), (2, 1)])
def test_dual_mesh_matches_oracle(cuda, g, mise):
    """Same field values on both sides (the oracle's MC driver calls the GPU evaluator), so the
    topology must agree exactly and the vertices to float tolerance."""
    field, svh, osvh, feats, xyz, nxyz, nval, (pw, nw, rw) = _solve_setup(cuda, 4, False, 4000, 0.05, 3, "sphere")
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True)).astype(np.float32)
    t = lambda a: torch.from_numpy(a).to(cuda)
    field.solve(t(xyz), t(nxyz), t(nval), pw, nw, rw)
    mesh = field.extract_dual_mesh(grid_upsample=g, mise_iter=mise)
    vo, fo = O.extract_dual_mesh(osvh, lambda q: _np(field.evaluate_f(t(q.astype(np.float32))).value), g, mise)
    assert mesh.f.shape[0] == fo.shape[0] and mesh.v.shape[0] == vo.shape[0] and fo.shape[0] > 100
    assert np.array_equal(_np(mesh.f), fo)
    assert np.abs(_np(mesh.v) - vo).max() <= 1e-5
    # closed where sampled, outward oriented
    v, f = _np(mesh.v).astype(np.float64), _np(mesh.f)
    nrm = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    assert (np.sum(nrm * v[f].mean(1), axis=1) > 0).mean() > 0.99
    # max_points batching does not change the result
    mesh2 = field.extract_dual_mesh(grid_upsample=g, mise_iter=mise, max_points=1000)
    assert torch.equal(mesh2.f, mesh.f) and torch.equal(mesh2.v, mesh.v)


def test_mask_trimming_matches_oracle(cuda):
    import nksr_b200
    field, svh, osvh, feats, xyz, nxyz, nval, (pw, nw, rw) = _solve_setup(cuda, 4, False, 4000, 0.05, 3, "sphere")
    t = lambda a: torch.from_numpy(a).to(cuda)
    field.solve(t(xyz), t(nxyz), t(nval), pw, nw, rw)        # random normals: spurious sheets exist
    field.set_mask_field(nksr_b200.LayerField(svh, 1))
    mesh = field.extract_dual_mesh(mise_iter=1)

    def mask(v):
        return osvh.locate(v.astype(np.float32))[0] >= 0
    vo, fo = O.extract_dual_mesh(osvh, lambda q: _np(field.evaluate_f(t(q.astype(np.float32))).value), 1, 1, mask)
    assert np.array_equal(_np(mesh.f), fo) and np.abs(_np(mesh.v) - vo).max() <= 1e-5


def test_reconstructor_end_to_end_sphere(cuda):
    import nksr_b200
    xyz, nrm = clouds.sphere(40000, noise=0.001)
    rec = nksr_b200.Reconstructor(cuda)
    field = rec.reconstruct(torch.from_numpy(xyz).to(cuda), torch.from_numpy(nrm).to(cuda), voxel_size=0.02)
    mesh = field.extract_dual_mesh(mise_iter=1)
    r = np.linalg.norm(_np(mesh.v), axis=1)
    assert mesh.f.shape[0] > 1000
    assert abs(np.median(r) - 0.35) < 0.004 and np.percentile(np.abs(r - 0.35), 99) < 0.02
    res = field.evaluate_f(torch.from_numpy(xyz[:1000]).to(cuda), grad=True)
    assert res.value.abs().mean().item() < 5e-3
    g = _np(res.gradient)
    assert np.mean(np.sum(-g / (np.linalg.norm(g, axis=1, keepdims=True) + 1e-9) * nrm[:1000], axis=1)) > 0.9
    # detail_level path and chunked path run
    f2 = rec.reconstruct(torch.from_numpy(xyz).to(cuda), torch.from_numpy(nrm).to(cuda), detail_level=0.5)
    assert f2.extract_dual_mesh().f.shape[0] > 100
    f3 = rec.reconstruct(torch.from_numpy(xyz * 10).to(cuda), torch.from_numpy(nrm).to(cuda), detail_level=None,
                         chunk_size=4.0)
    m3 = f3.extract_dual_mesh()
    r3 = np.linalg.norm(_np(m3.v), axis=1)
    assert m3.f.shape[0] > 500 and abs(np.median(r3) - 3.5) < 0.05


def test_normal_estimation_preprocess(cuda):
    """get_estimate_normal_preprocess_fn (examples/recons_waymo.py:36; CPU twin recons_waymo_cpu.py:21-41):
    PCA normals on a sphere point outward after the sensor-side flip; grazing points are dropped."""
    import nksr_b200
    xyz, nrm = clouds.sphere(60000, radius=1.0, noise=0.001)
    sensor = (xyz * 3.0).astype(np.float32)                      # sensors outside, along the radius
    fn = nksr_b200.get_estimate_normal_preprocess_fn(64, 85.0)
    x2, n2, s2 = fn(torch.from_numpy(xyz).to(cuda), None, torch.from_numpy(sensor).to(cuda))
    assert s2 is None and x2.shape == n2.shape and x2.shape[0] > 0.95 * xyz.shape[0]
    x2, n2 = _np(x2), _np(n2)
    radial = x2 / np.linalg.norm(x2, axis=1, keepdims=True)
    cos = np.sum(radial * n2, axis=1)
    assert np.median(cos) > 0.995 and (cos > 0.9).mean() > 0.98
    assert np.allclose(np.linalg.norm(n2, axis=1), 1.0, atol=1e-4)
    # grazing filter: a sensor in the tangent plane sees the surface edge-on
    sensor_g = (xyz + np.cross(radial_full(xyz), np.array([0.0, 0.0, 1.0]))).astype(np.float32)
    x3, n3, _ = fn(torch.from_numpy(xyz).to(cuda), None, torch.from_numpy(sensor_g).to(cuda))
    assert x3.shape[0] < 0.2 * xyz.shape[0]


def radial_full(xyz):
    return xyz / np.linalg.norm(xyz, axis=1, keepdims=True)


def test_neural_field_mask_and_texture(cuda):
    """NeuralField(svh, decoder, features).set_level_set + PCNNField texture (models/nksr_net.py:114-130,
    examples/recons_colored_mesh.py:28-31): interpolation weights are checked against the oracle's tent
    weights through a linear decoder; colours follow the nearest input point."""
    import nksr_b200
    field, svh, osvh, feats, xyz, nxyz, nval, (pw, nw, rw) = _solve_setup(cuda, 4, False, 4000, 0.05, 3, "sphere")
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True)).astype(np.float32)
    t = lambda a: torch.from_numpy(a).to(cuda)
    field.solve(t(xyz), t(nxyz), t(nval), pw, nw, rw)
    # features = voxel centre x-coordinate on level 0 only -> trilinear interpolation reproduces x
    f0 = svh.get_voxel_centers(0)[:, :1].contiguous()
    dec = torch.nn.Linear(1, 1, bias=False).to(cuda)
    with torch.no_grad():
        dec.weight.fill_(1.0)
    nf = nksr_b200.NeuralField(svh, dec, {0: f0})
    q = t(xyz[:500])            # the input points themselves: their 8 trilinear voxels are active by construction
    got = nf.evaluate_f(q).value
    assert torch.allclose(got, q[:, 0], atol=2e-5)
    nf.set_level_set(0.0)                       # keep x <= 0 only
    field.set_mask_field(nf)
    mesh = field.extract_dual_mesh(mise_iter=1)
    assert mesh.v.shape[0] > 100 and float(mesh.v[:, 0].max()) <= 1e-4
    # texture: colour = nearest input point's colour
    col = torch.rand(xyz.shape[0], 3, device=cuda)
    field.set_texture_field(nksr_b200.PCNNField(t(xyz), col))
    mesh = field.extract_dual_mesh()
    d = (mesh.v[:200, None, :].double() - t(xyz)[None].double()).norm(dim=2)
    picked = (mesh.c[:200, None, :] == col[None]).all(dim=2).double().argmax(dim=1)      # which point's colour
    assert ((d[torch.arange(200), picked] - d.min(dim=1).values).abs() < 1e-5).all()
    # evaluate_f_bar: masked-out side reads as outside
    fb = field.evaluate_f_bar(t(np.array([[0.33, 0.0, 0.0], [-0.33, 0.0, 0.0]], np.float32)))
    assert fb[0] <= 0 and fb[1] > 0, fb


def test_reconstruct_distributed_single_rank(cuda):
    """dist.reconstruct_distributed without an initialised process group = all chunks on this rank."""
    import nksr_b200
    from nksr_b200 import dist as nd
    xyz, nrm = clouds.sphere(40000, radius=3.5, noise=0.01)
    rec = nksr_b200.Reconstructor(cuda)
    field, mesh = nd.reconstruct_distributed(rec, torch.from_numpy(xyz).to(cuda), torch.from_numpy(nrm).to(cuda),
                                              chunk_size=4.0, mise_iter=0)
    r = np.linalg.norm(_np(mesh.v), axis=1)
    assert mesh.f.shape[0] > 500 and abs(np.median(r) - 3.5) < 0.05
    assert len(field.fields) == 8            # 2 x 2 x 2 chunks of edge 4 around the origin
