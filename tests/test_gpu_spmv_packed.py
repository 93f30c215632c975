"""Packed column tiles of the streamed SpMV (csrc/spmv_stream.cuh): a tile whose columns lie in at most 8 aligned windows
of 8192 columns streams a uint16 (window, offset) per entry instead of the int32 column.  The decoded columns are the
raw ones, so y must be bitwise what the raw tiles give.  Relabelling the columns by a random permutation (and x to
match) keeps every product and its order but spreads each tile over many windows: the same CSR then streams raw."""
import warnings

import numpy as np
import pytest
import torch

from tests import clouds

pytestmark = pytest.mark.gpu

TILE, WIN, MAX_WINDOWS = 4096, 8192, 8


def _np(t):
    return t.detach().cpu().numpy()


def _expected_stats(rowptr, col, split):
    """packed tiles and their entries by the packing rule, restated on the host"""
    nnz = int(rowptr[split])
    tiles, entries = 0, 0
    for e0 in range(0, nnz, TILE):
        c = col[e0:min(e0 + TILE, nnz)]
        if np.unique(c // WIN).size <= MAX_WINDOWS:
            tiles += 1
            entries += c.size
    return tiles, entries


def _stream(L, cuda, rowptr, col, val, x, split):
    """y of the first SpMV over a new plan (nksr_spmv_stream: every tile read raw, the packable ones packed on the way),
    y of the next SpMV over the same plan (nksr_spmv_stream_planned: packed tiles decoded from their slots), and the
    plan's packing counts"""
    n, nnz = x.numel(), col.size
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    pad = lambda a: t(np.concatenate([a, np.zeros(4, a.dtype)]))[:a.size]   # bulk copies read whole 16-byte units
    rowptr_d, col_d, val_d = pad(rowptr), pad(col), pad(val)
    nb = L.call("nksr_spmv_plan_bytes", nnz)
    plan = torch.empty(nb, dtype=torch.uint8, device=cuda)
    y_first = torch.full_like(x, float("nan"))
    L.call("nksr_spmv_stream", rowptr_d, col_d, val_d, x, y_first, n, nnz, split, int(rowptr[split]), plan, nb,
           L.stream_ptr(cuda))
    y = torch.full_like(x, float("nan"))
    L.call("nksr_spmv_stream_planned", rowptr_d, col_d, val_d, x, y, n, nnz, split, int(rowptr[split]), plan,
           L.stream_ptr(cuda))
    stats = (np.ctypeslib.ctypes.c_int64 * 4)()
    L.call("nksr_spmv_plan_stats", plan, np.ctypeslib.ctypes.addressof(stats), L.stream_ptr(cuda))
    return _np(y_first), _np(y), list(stats)


def _check_against_permuted(cuda, rowptr, col, val, seed, split=None):
    """y of the CSR (second SpMV over its plan: packed tiles decoded) and of its column-permuted copy (tiles raw),
    bitwise (the raw stream itself is held to fp64 in test_gpu_parity.py); the plans' counts against the packing rule.
    Returns the two plans' counts."""
    import nksr_b200._lib as L
    n = rowptr.size - 1
    split = n if split is None else split
    rng = np.random.default_rng(seed)
    x = rng.normal(size=n).astype(np.float32)
    perm = rng.permutation(n).astype(np.int32)             # column j becomes perm[j]
    xp = np.empty_like(x)
    xp[perm] = x
    y_first, y, st = _stream(L, cuda, rowptr, col, val, torch.from_numpy(x).to(cuda), split)
    yp_first, yp, stp = _stream(L, cuda, rowptr, perm[col], val, torch.from_numpy(xp).to(cuda), split)
    assert not np.isnan(y_first).any(), "a row was not written"
    bits = lambda a: a.view(np.uint32)
    # the packed tiles decoded (y) against the same tiles read raw (y_first) and against the permuted copy, raw
    assert np.array_equal(bits(y), bits(y_first)), "packed tiles give other bits than the packing launch"
    assert np.array_equal(bits(y), bits(yp)), "packed and raw tiles give different bits"
    assert np.array_equal(bits(yp_first), bits(yp))
    nnz = int(rowptr[split])
    assert st[2:] == stp[2:] == [-(-nnz // TILE), nnz]
    assert st[:2] == list(_expected_stats(rowptr, col, split))
    assert stp[:2] == list(_expected_stats(rowptr, perm[col], split))
    return st, stp


def _local_csr(n, lengths, reach, rng):
    rowptr = np.zeros(n + 1, np.int64)
    rowptr[1:] = np.cumsum(lengths)
    rows = np.repeat(np.arange(n), lengths)
    col = np.clip(rows + rng.integers(-reach, reach + 1, rows.size), 0, n - 1).astype(np.int32)
    return rowptr, col, rng.normal(size=rows.size).astype(np.float32)


@pytest.mark.parametrize("kind", ["short_rows", "long_rows", "tiny_rows"])
def test_packed_tiles_are_bitwise_the_raw_tiles(cuda, kind):
    """local columns (most tiles pack) against the permuted copy (every tile raw): cut rows, rows longer than several
    tiles, tiles of more than 512 rows; everything streamed and the last third of the rows by the row kernel"""
    rng = np.random.default_rng(3)
    n = {"short_rows": 120_000, "long_rows": 100_000, "tiny_rows": 300_000}[kind]
    if kind == "short_rows":
        lengths = rng.integers(1, 80, n)
    elif kind == "long_rows":
        lengths = rng.choice([3, 60, 5000, 20_000], n, p=[.3, .6985, .001, .0005])
    else:
        lengths = rng.choice([1, 2, 3], n)
    rowptr, col, val = _local_csr(n, lengths, 3000, rng)
    for split in (n, (2 * n) // 3):
        st, stp = _check_against_permuted(cuda, rowptr, col, val, 5, split)
        assert st[1] >= 0.9 * st[3], f"local columns should mostly pack: {st}"
        assert stp[0] <= 1, f"permuted columns should stay raw: {stp}"


def test_window_limits(cuda):
    """tile 0: exactly 8 windows, with offsets 0 and 8191 (packed); tile 1: 9 windows (raw); tile 2: the last column
    of the matrix; then local rows and a short last tile"""
    rng = np.random.default_rng(7)
    n = 11 * WIN + 77
    lengths = np.full(n, 4)                                # 1024 rows per tile
    rowptr = np.zeros(n + 1, np.int64)
    rowptr[1:] = np.cumsum(lengths)
    nnz = int(rowptr[-1])
    rows = np.repeat(np.arange(n), lengths)
    col = np.clip(rows + rng.integers(-100, 101, nnz), 0, n - 1).astype(np.int32)
    w8 = np.array([0, 1, 2, 3, 5, 6, 8, 10])
    col[:TILE] = w8[rng.integers(0, 8, TILE)] * WIN + rng.integers(0, WIN, TILE)
    col[:16] = w8[:, None].repeat(2, 1).ravel() * WIN + np.tile([0, WIN - 1], 8)
    w9 = np.arange(9)
    col[TILE:2 * TILE] = w9[rng.integers(0, 9, TILE)] * WIN + rng.integers(0, WIN, TILE)
    col[TILE:TILE + 9] = w9 * WIN + WIN - 1
    col[2 * TILE:3 * TILE] = n - 1 - rng.integers(0, 50, TILE)
    val = rng.normal(size=nnz).astype(np.float32)
    st, _ = _check_against_permuted(cuda, rowptr, col, val, 9)
    assert _expected_stats(rowptr[:2048 + 1], col, 2048) == (1, TILE)       # tile 0 packs, tile 1 does not
    assert st[0] == st[2] - 1


def test_packed_stream_on_a_deep_hierarchy(cuda):
    """the Gram system of a 6-level hierarchy, streamed with packed tiles against its permuted copy; and the PCG
    reports its plan's counts"""
    import nksr_b200
    xyz, _ = clouds.sphere(6000, seed=6)
    nrm_xyz = xyz[::4].copy()
    nrm_val = -(nrm_xyz / np.linalg.norm(nrm_xyz, axis=1, keepdims=True)).astype(np.float32)
    W, L = 0.01, 6
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_point_splatting(t(xyz))
    rng = np.random.default_rng(6)
    feats = [t((0.5 + 0.2 * rng.normal(size=(int(svh.num_voxels(l)), 4))).astype(np.float32)) for l in range(L)]
    field = nksr_b200.KernelField(svh, None, feats)
    field.solver_config.update(keep_system=True, max_iter=2)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)                 # stopped at max_iter
        field.solve(t(xyz), t(nrm_xyz), t(nrm_val), 1e4 / xyz.shape[0], 1e4 / nrm_xyz.shape[0] * W * W, 1.0)
    s = field.system
    rowptr, col, val = _np(s.rowptr).astype(np.int64), _np(s.col)[:s.nnz], _np(s.val)[:s.nnz]
    st, _ = _check_against_permuted(cuda, rowptr, col, val, 4)        # KernelField streams every row
    info = field.solve_info
    assert [info["spmv_packed_tiles"], info["spmv_packed_entries"], info["spmv_streamed_tiles"],
            info["spmv_streamed_entries"]] == st
    assert st[0] > 0
