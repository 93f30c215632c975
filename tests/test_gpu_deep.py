"""Hierarchy depths 6, 7 and 8 against the fp64 oracle.  Depth 8 (= NKSR_MAX_DEPTH) has no room for the virtual level
above the coarsest one in the C view: the top level owns an explicit 5^3 neighbour table (nbr125_top), and every
same-level look-up on it goes through that table (gram_common.cuh lookup_near).  Cross-level slots reach up to 7
levels, the placement tables rank8 / prefix every (l, k) pair, the per-voxel Gram blocks split levels up to 8.

Inputs: (a) shapenet_like at W = 0.02, depths 6, 7, 8 (top levels of 8 - 32 voxels); (b) a sphere at W = 0.005, depth 8
(every level populated); (c) scattered small clusters with negative coordinates over more than 6 coarsest voxels per
axis (top level with neighbours at offset +-2 and holes in its 5^3 table), splatted and with a pruned finest level.
Integer tables bit-exact, floating point entry by entry within the tests/bounds.py constants."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import nksr_oracle as O
from tests import clouds
from tests import grad_oracle as G
from tests.bounds import (KAPPA_FIELD, KAPPA_GRAM, KAPPA_RHS, KAPPA_ROWS, KAPPA_SPMV, assert_within, level_of,
                          level_pair_label, ratios)
from tests.test_gpu_kernel_grad import KAPPA_VJP

pytestmark = pytest.mark.gpu

_OFF125 = np.array([[a, b, c] for a in range(-2, 3) for b in range(-2, 3) for c in range(-2, 3)], np.int64)


def _np(t):
    return t.detach().cpu().numpy()


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _scattered(n_clusters=30, per=40, seed=3):
    """small point clusters (radius ~1.5 finest voxels at W = 0.02) spread over [-12, 6]^3: about 7 coarsest voxels
    (2.56) per axis at depth 8, negative coordinates"""
    rng = np.random.default_rng(seed)
    centres = rng.uniform(-12.0, 6.0, (n_clusters, 3))
    pts = centres[:, None, :] + rng.normal(size=(n_clusters, per, 3)) * 0.03
    return pts.reshape(-1, 3).astype(np.float32)


# name: (cloud, W, depth, prune the finest level)
_CASES = {
    "a6": ("shapenet", 0.02, 6, False),
    "a7": ("shapenet", 0.02, 7, False),
    "a8": ("shapenet", 0.02, 8, False),
    "b8": ("sphere", 0.005, 8, False),
    "c8": ("scattered", 0.02, 8, False),
    "c8pruned": ("scattered", 0.02, 8, True),
}


class _Case:
    """one hierarchy on both sides, its features and constraints; oracle systems built on first use"""

    def __init__(self, name, cuda):
        import nksr_b200
        cloud, W, L, prune = _CASES[name]
        xyz = {"shapenet": lambda: clouds.shapenet_like(3000)[0], "sphere": lambda: clouds.sphere(3000)[0],
               "scattered": _scattered}[cloud]()
        self.name, self.W, self.L, self.cuda = name, W, L, cuda
        full = O.OracleSVH(W, L + 1).build_point_splatting(xyz)          # (its level L: the splatted virtual level)
        keys = list(full.keys[:L])
        if prune:                                                         # childless voxels on level 1
            keys[0] = keys[0][O.key_to_ijk(keys[0], 0)[:, 0] >= int(np.median(O.key_to_ijk(keys[0], 0)[:, 0]))]
            self.top = np.unique(keys[L - 1] >> 3)
            self.svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_from_keys([_t(k, cuda) for k in keys])
        else:
            self.top = full.keys[L]
            self.svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_point_splatting(_t(xyz, cuda))
        self.osvh = O.OracleSVH(W, L).build_from_keys(keys)
        self.otop = O.OracleSVH(W, L + 1).build_from_keys(keys + [self.top])
        rng = np.random.default_rng(L)
        self.feats = [(0.5 + 0.2 * rng.normal(size=(self.osvh.n(l), 4))).astype(np.float32) for l in range(L)]
        nxyz = np.concatenate([self.osvh.centers(d) for d in range(2)])
        nxyz[::2] += (rng.uniform(-0.3, 0.3, nxyz[::2].shape) * W).astype(np.float32)   # half at centres, half generic
        nval = rng.normal(size=nxyz.shape)
        self.nval = (nval / np.linalg.norm(nval, axis=1, keepdims=True)).astype(np.float32)
        # (no location within a few ulps of the tent derivative's snap-zone edge: see test_gpu_parity._snap_free)
        keep = ~O.tent_branch_ambiguous(self.osvh, nxyz)
        self.nxyz, self.nval = nxyz[keep], self.nval[keep]
        self.xyz = xyz[~O.tent_branch_ambiguous(self.osvh, xyz)]
        self.pw, self.nw = 1e4 / self.xyz.shape[0], 1e4 / self.nxyz.shape[0] * W * W
        self._systems = {}

    def field(self, approx=False, feats=None):
        import nksr_b200
        return nksr_b200.KernelField(self.svh, None, [_t(f, self.cuda) for f in (feats or self.feats)], approx)

    def solve(self, field, normals=True):
        t = lambda a: _t(a, self.cuda)
        if normals:
            field.solve(t(self.xyz), t(self.nxyz), t(self.nval), self.pw, self.nw, 1.0)
        else:
            field.solve(t(self.xyz), None, None, self.pw, 0.0, 1.0)
        return field

    def oracle_system(self, normals=True, approx=False):
        """(A, b, A_abs, b_abs, E) of O.build_system (E: the constraint rows)"""
        key = (normals, approx)
        if key not in self._systems:
            nx = self.nxyz if normals else np.zeros((0, 3), np.float32)
            nv = self.nval if normals else np.zeros((0, 3), np.float32)
            A, b, E, Aa, ba = O.build_system(self.osvh, self.feats, self.xyz, nx, nv, self.pw,
                                             self.nw if normals else 0.0, 1.0, approx, abs_terms=True)
            self._systems[key] = (A, b, Aa, ba, E)
        return self._systems[key]


_cache = {}


@pytest.fixture(scope="module")
def case(request, cuda):
    if request.param not in _cache:
        _cache[request.param] = _Case(request.param, cuda)
    yield _cache[request.param]


def teardown_module(module):
    _cache.clear()


def _gpu_csr(s):
    return sp.csr_matrix((_np(s.val).astype(np.float64), _np(s.col), _np(s.rowptr)), shape=(s.n, s.n))


# ------------------------------------------------------------------------------------------------------ 1. tables
@pytest.mark.parametrize("case", list(_CASES), indirect=True)
def test_tables_bit_exact(case):
    svh, osvh, otop, L = case.svh, case.osvh, case.otop, case.L
    assert np.array_equal(_np(svh.top_keys), case.top), "top_keys"
    for l in range(L):
        assert osvh.n(l) > 0
        assert np.array_equal(_np(svh.keys[l]), osvh.keys[l]), f"keys level {l}"
        assert np.array_equal(_np(svh.nbr27[l]).astype(np.int64), osvh.nbr27(l)), f"nbr27 level {l}"
        par = otop.lookup(l + 1, osvh.ijk(l).astype(np.int64) >> 1)
        assert (par >= 0).all() and np.array_equal(_np(svh.parent[l]).astype(np.int64), par), f"parent level {l}"
        ch = np.full((otop.n(l + 1), 8), -1, np.int64)
        ch[par, osvh.keys[l] & 7] = np.arange(osvh.n(l))
        assert np.array_equal(_np(svh.child8[l + 1]).astype(np.int64), ch), f"child8 level {l + 1}"
    assert np.array_equal(_np(svh.nbr27[L]).astype(np.int64), otop.nbr27(L)), f"nbr27 virtual level {L}"
    if L == 8:
        ref = osvh.lookup(L - 1, osvh.ijk(L - 1).astype(np.int64)[:, None, :] + _OFF125[None])
        got = _np(svh.nbr125_top).astype(np.int64)
        assert np.array_equal(got, ref), f"nbr125_top (level {L - 1})"
        assert svh.view().parent[L - 1] is None          # every top-level look-up goes through the 5^3 table
        if case.name.startswith("c"):                    # neighbours at offset +-2 and holes in the 5^3 table
            outer = np.abs(_OFF125).max(axis=1) == 2
            assert (ref[:, outer] >= 0).any() and (ref < 0).any() and osvh.n(L - 1) > 100
    else:
        assert svh.nbr125_top is None
    # locate: data points, jittered points, points beyond the top level
    rng = np.random.default_rng(1)
    x = case.xyz
    top_w = osvh.level_w(L - 1)
    q = np.concatenate([x, x + rng.uniform(-1.5, 1.5, x.shape) * case.W, x[:300] + rng.uniform(-2, 2, (300, 3)) * top_w,
                        x[:100] + np.float32(3.5 * top_w)]).astype(np.float32)
    got = _np(svh.locate(_t(q, case.cuda))).astype(np.int64)
    ref = osvh.locate(q)
    assert (ref[L - 1] < 0).any() and (ref[0] >= 0).any()
    for l in range(L):
        assert np.array_equal(got[l], ref[l]), f"locate level {l}"


# ------------------------------------------------------------------------------------------------------ 2. rows
@pytest.mark.parametrize("approx", [False, True])
@pytest.mark.parametrize("case", ["a6", "a7", "a8", "c8"], indirect=True)
def test_kernel_rows_match_oracle(case, approx):
    osvh, L = case.osvh, case.L
    field = case.field(approx)
    rng = np.random.default_rng(4)
    q = np.concatenate([case.xyz[:1500], case.xyz[:1000] + rng.uniform(-0.5, 0.5, (1000, 3)).astype(np.float32) * case.W])
    q = q[~O.tent_branch_ambiguous(osvh, q)].astype(np.float32)
    for mode in ((0, 1, 2) if approx else (0, 1)):
        xs, _, base, _, e = field._sorted_rows(_t(q, case.cuda), mode)
        xs_np, base_np, e_np = _np(xs), _np(base).astype(np.int64), _np(e)
        assert np.array_equal(base_np, osvh.locate(xs_np))
        for l in range(L):
            what = f"{['K', 'dK', 'compact dK'][mode]} rows level {l} (L={L}, {case.name}, approx={approx})"
            if mode == 2:       # <phi, z_s> in slots 0..26 and tau in 27..29 (gram_common.cuh CompactSpline)
                one = lambda tau: (np.ones(tau.shape + (3,)), np.zeros(tau.shape + (3,)))
                nbr, dots, _ = O._level_rows(osvh, l, xs_np, base_np[l], case.feats[l], False, True, one, O._tent)
                _, dabs, _ = O._level_rows(osvh, l, xs_np, base_np[l], np.abs(case.feats[l]), False, True, one,
                                           O._tent_abs)
                _, tau = O._level_tau(osvh, l, xs_np, base_np[l])
                ok = base_np[l] >= 0
                assert_within(e_np[:, l, :27], dots, dabs, KAPPA_ROWS, what)
                ijk = osvh.ijk(l)[np.where(ok, base_np[l], 0)]
                tscale = np.abs(xs_np.astype(np.float64) / osvh.level_w(l)) + np.abs(ijk + 0.5)
                assert_within(e_np[ok, l, 27:30], tau[ok], tscale[ok], KAPPA_ROWS, f"tau level {l} ({case.name})")
                continue
            nbr, K, dK, Ka, dKa = O.level_rows(osvh, l, xs_np, base_np[l], case.feats[l], mode == 1, approx,
                                               abs_terms=True)
            if mode == 0:
                got, ref, scale = e_np[:, l, :27], K, Ka
            else:
                got, ref, scale = e_np[:, l].reshape(-1, 3, 32)[:, :, :27], dK, dKa
            assert np.abs(ref).max() > 0
            assert_within(got, ref, scale, KAPPA_ROWS, what,
                          lambda j, g=got: f"location {np.unravel_index(j, g.shape)[0]} "
                                           f"entry {np.unravel_index(j, g.shape)[1:]}")
            assert np.all(e_np[:, l].reshape(-1, 32)[:, 27:] == 0)


# ------------------------------------------------------------------------------------------------------ 3. Gram
def _assemble(case, approx=False, normals=True, **config):
    field = case.field(approx)
    field.solver_config.update(keep_system=True, max_iter=0, **config)
    return case.solve(field, normals).system


def _outside_top(M, t0):
    """M without the coarsest level's block (rows and columns >= t0)"""
    c = sp.coo_matrix(M)
    k = (c.row < t0) | (c.col < t0)
    return sp.csr_matrix((c.data[k], (c.row[k], c.col[k])), shape=M.shape)


def _top_kappas(case, normals, approx):
    """Per-entry bounds of the coarsest level's block, derived from the number of terms each entry sums.  Entry (i, j)
    of A sums the products w e_ri e_rj of the n_ij constraint rows r whose supports hold both voxels, plus one
    regulariser term.  Each product carries the rows' error (<= KAPPA_ROWS u of its abs-term scale each) and one
    rounding; a sum of n terms in fp32, in any order, adds at most (n - 1) u times the sum of their magnitudes.  So
    |got - ref| <= (n_ij + 2 KAPPA_ROWS) u scale_ij.  The rhs: n_i target-weighted products w e_ri t_r,
    (n_i + KAPPA_ROWS + 1) u scale_i.  The bounds are never below KAPPA_GRAM / KAPPA_RHS.  A level-(L-1) entry at depth
    8 sums up to ~10^5 terms (every location within two coarsest voxels), so the fixed constants, measured on levels
    that sum far fewer, do not describe it."""
    A_ref, b_ref, A_abs, b_abs, E = case.oracle_system(normals, approx)
    t0 = int(case.osvh.offsets()[-2])
    B = (sp.csc_matrix(E)[:, t0:] != 0).astype(np.float64)
    n_terms = (B.T @ B).toarray() + 1
    kap = np.maximum(KAPPA_GRAM, n_terms + 2 * KAPPA_ROWS)
    targets = np.concatenate([np.zeros(case.xyz.shape[0], bool)] + ([case.nval.reshape(-1) != 0] if normals else []))
    n_rhs = np.asarray(B[targets].sum(axis=0)).ravel()
    return t0, kap, np.maximum(KAPPA_RHS, n_rhs + KAPPA_ROWS + 1), n_terms


def _check_values(case, s, normals, approx, what):
    """values, rhs and diagonal entry by entry: KAPPA_GRAM / KAPPA_RHS outside the coarsest level's block, the
    term-count bounds of _top_kappas inside it (whose worst ratio in units of KAPPA_GRAM is printed too)"""
    A_ref, b_ref, A_abs, b_abs, _ = case.oracle_system(normals, approx)
    offs = case.osvh.offsets()
    t0, kap, kap_rhs, n_terms = _top_kappas(case, normals, approx)
    lab = level_pair_label(offs)
    A = _gpu_csr(s)
    assert_within(_outside_top(A, t0), _outside_top(A_ref, t0), _outside_top(A_abs, t0), KAPPA_GRAM,
                  f"Gram values outside level ({case.L - 1},{case.L - 1}) ({what})", lab)
    top = [M[t0:, t0:].toarray() for M in (A, A_ref, A_abs)]
    q = ratios(*top)[0]
    i = int(np.argmax(q))
    print(f"[bounds] Gram values level ({case.L - 1},{case.L - 1}) ({what}): worst ratio {q[i]:.4g} in units of "
          f"u scale, at an entry summing {int(n_terms.reshape(-1)[i])} terms (KAPPA_GRAM {KAPPA_GRAM:g})")
    assert_within(top[0], top[1], top[2] * kap, 1.0, f"Gram values level ({case.L - 1},{case.L - 1}) against "
                  f"(n + 2 KAPPA_ROWS) u scale ({what})",
                  lambda j: f"({t0 + j // kap.shape[0]},{t0 + j % kap.shape[0]}) terms {int(n_terms.reshape(-1)[j])}")
    row = lambda i: f"row {i} level {level_of(offs, i)}"
    for name, got, ref, scale, kappa, k_top in (
            ("rhs", _np(s.rhs), b_ref, b_abs, KAPPA_RHS, kap_rhs),
            ("diagonal", _np(s.diag), A_ref.diagonal(), A_abs.diagonal(), KAPPA_GRAM, np.diagonal(kap))):
        assert_within(got[:t0], ref[:t0], scale[:t0], kappa, f"{name} below level {case.L - 1} ({what})", row)
        assert_within(got[t0:], ref[t0:], scale[t0:] * k_top, 1.0, f"{name} level {case.L - 1} against its "
                      f"term-count bound ({what})", lambda i: row(t0 + i))


def _record_split(monkeypatch):
    """the block split level each Gram fill ran with (fields.assemble skips the blocks that do not fit memory)"""
    from nksr_b200 import fields
    seen, real = [], fields.call

    def record(name, *args):
        if name.startswith("nksr_gram_fill"):
            seen.append(int(args[2].split_level))
        return real(name, *args)
    monkeypatch.setattr(fields, "call", record)
    return seen


@pytest.mark.parametrize("case", ["a6", "a7", "a8", "b8", "c8", "c8pruned"], indirect=True)
def test_gram_system_matches_oracle(case, monkeypatch):
    from tests.placement_checks import assert_structural_placement
    L = case.L
    seen = _record_split(monkeypatch)
    ref = None
    # (b: the largest oracle, 19 M entries -- the position-only and approx systems are checked on the others)
    for normals in ((True,) if case.name == "b8" else (True, False)):
        for split in (None, 2, L - 2, L):
            s = _assemble(case, normals=normals, block_split_level=split, fill="rows")
            what = f"{case.name} L={L} split={split}" + ("" if normals else " positions only")
            assert seen[-1] == split if split is not None else seen[-1] < L, (what, seen[-1])    # the blocks ran
            if ref is None:
                # (row lengths first: a wrong one is reported with its row and level)
                assert_structural_placement(case.osvh, *(_np(a) for a in (s.rowptr, s.col, s.val, s.cnt,
                                                                           s.cnt_down)), what)
                assert s.nnz == O.structural_pattern(case.osvh).nnz, what
                ref = [_np(a).copy() for a in (s.rowptr, s.col)]
            else:                                       # the placement does not depend on split level or constraints
                assert np.array_equal(_np(s.rowptr), ref[0]) and np.array_equal(_np(s.col), ref[1]), what
            _check_values(case, s, normals, False, what)
    if case.name == "b8":
        return
    for compact in (False, True):
        s = _assemble(case, approx=True, compact_rows=compact, fill="rows")
        assert seen[-1] == L if compact else seen[-1] < L           # compact gradient rows have no block kernel
        _check_values(case, s, True, True, f"{case.name} L={L} approx compact={compact}")


@pytest.mark.parametrize("case", ["a6", "a8", "c8pruned"], indirect=True)
def test_brick_and_grouped_fills_fall_back_to_the_row_fill(case):
    """At depth > 4 'brick' and 'grouped' run the placed row fill: bitwise the 'rows' system"""
    out = {}
    for fill in ("rows", "brick", "grouped"):
        s = _assemble(case, fill=fill)
        out[fill] = [_np(a).copy() for a in (s.rowptr, s.col, s.val, s.rhs, s.diag)]
    for fill in ("brick", "grouped"):
        for a, b in zip(out["rows"], out[fill]):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), fill


# ------------------------------------------------------------------------------------------------------ 4. solve
@pytest.mark.parametrize("spmv", ["rows", "stream"])
@pytest.mark.parametrize("case", ["a8", "b8", "c8"], indirect=True)
def test_spmv_and_solve_at_depth_8(case, spmv):
    import nksr_b200._lib as LB
    field = case.field()
    field.solver_config.update(keep_system=True, tol=1e-6, max_iter=4000, check_every=1, spmv=spmv)
    case.solve(field)
    s = field.system
    assert field.solve_info["converged"], field.solve_info
    A = _gpu_csr(s)
    x = _t(np.random.default_rng(3).normal(size=s.n).astype(np.float32), case.cuda)
    y = torch.empty_like(x)
    if spmv == "rows":
        LB.call("nksr_spmv", s.rowptr, s.col, s.val, x, y, s.n, LB.stream_ptr(case.cuda))
    else:
        nb = LB.call("nksr_spmv_plan_bytes", s.nnz)
        plan = torch.empty(nb, dtype=torch.uint8, device=case.cuda)
        LB.call("nksr_spmv_stream", s.rowptr, s.col, s.val, x, y, s.n, s.nnz, s.n, s.nnz, plan, nb,
                LB.stream_ptr(case.cuda))
    xd = _np(x).astype(np.float64)
    offs = case.osvh.offsets()
    assert_within(_np(y), A @ xd, abs(A) @ np.abs(xd), KAPPA_SPMV, f"{spmv} SpMV ({case.name})",
                  lambda i: f"row {i} level {level_of(offs, i)}")
    A_ref, b_ref = case.oracle_system(True, False)[:2]
    alpha = _np(field.alpha).astype(np.float64)
    res = np.linalg.norm(A_ref @ alpha - b_ref) / np.linalg.norm(b_ref)
    print(f"[bounds] fp64 residual ({spmv}, {case.name}): {res:.3g} of ||b|| (bound 2e-4)")
    assert res <= 2e-4


# ------------------------------------------------------------------------------------------------------ 5. field
@pytest.mark.parametrize("approx", [False, True])
@pytest.mark.parametrize("case", ["a6", "a7", "a8", "b8", "c8pruned"], indirect=True)
def test_field_matches_oracle(case, approx):
    osvh, W = case.osvh, case.W
    field = case.field(approx)
    rng = np.random.default_rng(1)
    alpha = rng.normal(size=osvh.offsets()[-1]).astype(np.float32)
    field.alpha = _t(alpha, case.cuda)
    cen = np.concatenate([osvh.centers(0)[:1500], osvh.centers(1)[:1000]])
    x = case.xyz
    q = np.concatenate([x[:1500], cen, x[:1000] + rng.uniform(-0.5, 0.5, (1000, 3)).astype(np.float32) * W])
    q = q[~O.tent_branch_ambiguous(osvh, q)].astype(np.float32)
    r = field.evaluate_f(_t(q, case.cuda), grad=True)
    fo, go, fa, ga = O.evaluate_f(osvh, case.feats, alpha.astype(np.float64), q, grad=True, approx_kernel_grad=approx,
                                  abs_terms=True)
    what = f"{case.name} L={case.L} approx={approx}"
    assert_within(_np(r.value), fo, fa, KAPPA_FIELD, f"f ({what})", lambda j: f"query {j}")
    assert_within(_np(r.gradient), go, ga, KAPPA_FIELD, f"grad f ({what})", lambda j: f"query {j // 3} axis {j % 3}")


# ------------------------------------------------------------------------------------------------------ 6. backward
@pytest.mark.parametrize("case", ["a8", "c8"], indirect=True)
def test_backward_kernels_match_oracle(case):
    from nksr_b200._lib import call, stream_ptr
    osvh, L, feats, cuda = case.osvh, case.L, case.feats, case.cuda
    field = case.field()
    rng = np.random.default_rng(5)
    cen = np.concatenate([osvh.centers(0), osvh.centers(1)])[:1500]
    q = np.concatenate([case.xyz[:1500], cen,
                        case.xyz[:1000] + rng.uniform(-0.5, 0.5, (1000, 3)).astype(np.float32) * case.W])
    q = q[~O.tent_branch_ambiguous(osvh, q)].astype(np.float32)
    _, xs, _, base, ranges = field._sorted_locations(_t(q, cuda))
    xs_np, loc = _np(xs), (xs, base, ranges)
    n, m, offs = case.svh.num_unknowns, xs.shape[0], osvh.offsets()
    a0, a1 = rng.normal(size=n).astype(np.float32), rng.normal(size=n).astype(np.float32)
    t = lambda a: _t(a, cuda)
    for mode in (0, 1):
        coef = rng.normal(size=(m,) if mode == 0 else (m, 3)).astype(np.float32)
        got = _np(field._evaluate_adjoint(loc, mode, t(coef)))
        ref, scale = G.evaluate_adjoint(osvh, feats, xs_np, mode, False, coef.astype(np.float64), abs_terms=True)
        for l in range(L):
            assert_within(got[offs[l]:offs[l + 1]], ref[offs[l]:offs[l + 1]], scale[offs[l]:offs[l + 1]], KAPPA_VJP,
                          f"evaluate_adjoint mode {mode} level {l} ({case.name})")
        for two in (False, True):
            cf = rng.normal(size=(m, 2 if two else 1) + ((3,) if mode == 1 else ())).astype(np.float32)
            dz = torch.zeros((n, 4), dtype=torch.float32, device=cuda)
            field._feature_vjp(loc, mode, t(cf), t(a0), t(a1) if two else None, dz)
            vecs = [a0.astype(np.float64)] + ([a1.astype(np.float64)] if two else [])
            ref, scale = G.feature_vjp(osvh, feats, xs_np, mode, False, cf.astype(np.float64), vecs, abs_terms=True)
            for l in range(L):
                assert_within(_np(dz)[offs[l]:offs[l + 1]], ref[l], scale[l], KAPPA_VJP,
                              f"feature_vjp mode {mode} two={two} level {l} ({case.name})")
    dz = torch.zeros((n, 4), dtype=torch.float32, device=cuda)
    call("nksr_regulariser_vjp", case.svh.view(), field.feat_view(), t(a0), t(a1), 1.0, dz, stream_ptr(cuda))
    ref, scale = G.regulariser_vjp(osvh, feats, a0.astype(np.float64), a1.astype(np.float64), abs_terms=True)
    for l in range(L):
        assert_within(_np(dz)[offs[l]:offs[l + 1]], ref[l], scale[l], KAPPA_VJP, f"regulariser_vjp level {l} "
                                                                                  f"({case.name})")


# ------------------------------------------------------------------------------------------------------ 7. growth
def _chain_svh(cuda, depth):
    """one voxel per level, below a single coarsest voxel"""
    import nksr_b200
    from nksr_b200.structure import morton_encode
    c = 1 << 19
    key = morton_encode(torch.tensor([c - 5]), torch.tensor([c + 9]), torch.tensor([c - 2]))
    return nksr_b200.SparseFeatureHierarchy(0.02, depth, cuda).build_from_keys([(key >> (3 * l)).to(cuda)
                                                                                 for l in range(depth)])


@pytest.mark.parametrize("D", [8, 6])
@pytest.mark.parametrize("case", ["a8"], indirect=True)
def test_growth_on_a_depth_8_encoder_hierarchy(case, D):
    """D = 8: the grown hierarchy takes the encoder's nbr125_top; D = 6: the encoder's level 6 is its virtual level"""
    from tests.test_gpu_structure import _check_closed_sorted, _grow_pair
    E = case.svh
    # (full subdivision of the 8 - 32 top voxels of E would give 8^7 times as many finest voxels: a one-voxel chain)
    for mode, enc in (("random", E), ("leaf", E), ("subdivide", _chain_svh(case.cuda, 8) if D == 8 else E)):
        a = D - 2
        gc, gt = _grow_pair(enc, D, a, mode, seed=D)
        _check_closed_sorted(gc, D)
        for g in (gc, gt):
            if D == 8:
                assert g.T.nbr125_top is enc.nbr125_top and g.T.top_keys is enc.top_keys
                assert g.T.view().nbr125_top == enc.nbr125_top.data_ptr()
            else:
                assert g.T.nbr125_top is None and torch.equal(g.T.top_keys, enc.keys[D])
        if mode == "subdivide":
            assert gc.T.num_voxels(0) == enc.num_voxels(D - 1) * 8 ** (D - 1)
        elif mode == "leaf":                    # leaves below a stop the growth, above it they subdivide
            for l in range(D - 1):
                assert gc.T.num_voxels(l) == (8 * gc.T.num_voxels(l + 1) if l + 1 >= a else 0), l
        else:
            assert gc.T.num_voxels(0) > 0


# ------------------------------------------------------------------------------------------------------ 8. mesh
@pytest.mark.parametrize("case", ["a8"], indirect=True)
def test_dual_mesh_matches_oracle_at_depth_8(case):
    field = case.field()
    field.solver_config.update(tol=1e-5, max_iter=4000)
    case.solve(field)
    t = lambda a: _t(a, case.cuda)
    mesh = field.extract_dual_mesh(mise_iter=1)
    vo, fo = O.extract_dual_mesh(case.osvh, lambda q: _np(field.evaluate_f(t(q.astype(np.float32))).value), 1, 1)
    assert mesh.f.shape[0] == fo.shape[0] and mesh.v.shape[0] == vo.shape[0] and fo.shape[0] > 100
    assert np.array_equal(_np(mesh.f), fo)
    assert np.abs(_np(mesh.v) - vo).max() <= 1e-5


def _analytic(svh):
    import nksr_b200

    class Analytic(nksr_b200.fields.BaseField):                      # f = r0 - |x|: the mesher alone is under test
        def evaluate_f(self, q, grad=False):
            return nksr_b200.fields.EvaluationResult(value=0.35 - q.norm(dim=1), gradient=None)
    return Analytic(svh)


def _drop_below(keys, level, leaf_keys):
    """keys without the descendants of the level-`level` voxels `leaf_keys` (which become leaves)"""
    out = list(keys)
    gone = leaf_keys
    for l in range(level - 1, -1, -1):
        out[l] = out[l][~np.isin(out[l] >> 3, gone)]
        gone = keys[l][np.isin(keys[l] >> 3, gone)]
    return out


def test_multi_level_mesh_with_level_6_leaves(cuda):
    """depth 7, adaptive_depth 7: one level-6 leaf (the +++ octant of a sphere, 8^6 virtual finest voxels) and
    level-1 leaves where x < 0 -- the CUDA mesher against the oracle's coarse_levels = 7, cell for cell"""
    import nksr_b200
    from nksr_b200.meshing import extract_dual_mesh
    xyz, _ = clouds.sphere(60_000, noise=0.0005)
    W, L = 0.01, 7
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    k6 = O.voxel_key(np.zeros((1, 3), np.int64), 6)
    assert np.isin(k6, osvh.keys[6]).all()
    keys = _drop_below(osvh.keys, 6, k6)
    keys[0] = keys[0][O.key_to_ijk(keys[0], 0)[:, 0] >= 0]
    osvh = O.OracleSVH(W, L).build_from_keys(keys)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_from_keys([_t(k, cuda) for k in keys])
    svh.adaptive_depth = L
    field = _analytic(svh)
    # (both sides read the same field values: a corner value within rounding of 0 moves a vertex by up to a cell)
    ev = lambda q: _np(field.evaluate_f(_t(q.astype(np.float32), cuda)).value)
    m = extract_dual_mesh(field, 1, 1)
    vo, fo = O.extract_dual_mesh(osvh, ev, 1, 1, coarse_levels=L)
    v, f = _np(m.v), _np(m.f)
    assert v.shape == vo.shape and f.shape == fo.shape and f.shape[0] > 1000
    assert np.abs(v - vo).max() <= 1e-5 and np.array_equal(f, fo)
    assert (np.all(v > 0.05, axis=1)).any()                      # surface inside the level-6 leaf
    assert np.abs(np.linalg.norm(v, axis=1) - 0.35).max() <= 0.02 * W


@pytest.mark.parametrize("case", ["a8"], indirect=True)
def test_multi_level_mesh_refuses_level_7_leaves(case):
    """a leaf on level 7 would expand to 8^7 virtual finest voxels: NksrError naming the level, before any anchor"""
    import nksr_b200
    from nksr_b200._lib import NksrError
    from nksr_b200.meshing import extract_dual_mesh
    keys = _drop_below(case.osvh.keys, 7, case.osvh.keys[7][:1])
    svh = nksr_b200.SparseFeatureHierarchy(case.W, 8, case.cuda).build_from_keys([_t(k, case.cuda) for k in keys])
    svh.adaptive_depth = 8
    with pytest.raises(NksrError, match="level 7 has 1 leaves"):
        extract_dual_mesh(_analytic(svh), 1, 0)


# ------------------------------------------------------------------------------------------------------ 9. end to end
def test_reconstructor_depth_8_sphere(cuda, monkeypatch):
    import nksr_b200
    from nksr_b200 import fields
    captured = {}
    solve = fields.KernelField.solve

    def keep(self, *args, **kw):                                   # the system the Reconstructor solves
        self.solver_config["keep_system"] = True
        captured.update(field=self, args=args)
        return solve(self, *args, **kw)
    monkeypatch.setattr(fields.KernelField, "solve", keep)
    xyz, nrm = clouds.sphere(10_000, noise=0.001)
    rec = nksr_b200.Reconstructor(cuda, tree_depth=8)
    field = rec.reconstruct(_t(xyz, cuda), _t(nrm, cuda), voxel_size=0.02)
    assert field is captured["field"] and field.solve_info["converged"], field.solve_info
    pos, nxyz, nval, pw, nw, rw = captured["args"][:6]
    svh = field.svh
    assert svh.depth == 8
    osvh = O.OracleSVH(svh.voxel_size, 8).build_from_keys([_np(k) for k in svh.keys])
    feats = [_np(z) for z in field.z]
    nxyz, nval = _np(nxyz), _np(nval)
    A_ref, b_ref, _ = O.build_system(osvh, feats, _np(pos), nxyz, nval, pw, nw, rw)
    alpha = _np(field.alpha).astype(np.float64)
    res = np.linalg.norm(A_ref @ alpha - b_ref) / np.linalg.norm(b_ref)
    print(f"[bounds] fp64 residual (Reconstructor, depth 8): {res:.3g} of ||b||")
    assert res <= 2e-4
    mesh = field.extract_dual_mesh(mise_iter=1)
    r = np.linalg.norm(_np(mesh.v), axis=1)
    assert mesh.f.shape[0] > 1000 and abs(np.median(r) - 0.35) < 0.02
