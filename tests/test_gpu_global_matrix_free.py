"""The global solve on the matrix-free operator (dist_solve.reconstruct_global(..., operator='matrix_free')): the
owned-location filter of nksr_op_setup and the Chronopoulos-Gear step nksr_dcg_op_dots.  Ranks are simulated in
lockstep in one process through dist_solve.local_system, as tests/test_gpu_solver.py does for the CSR step: the dots
are summed over the ranks, and u is exchanged by copying the owner's value, joined on (level, key).  Every rank's
owned rows are compared with the whole-cloud single-GPU operator at the same (level, key)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests import clouds
from tests.bounds import assert_within

# the per-entry bound of tests/test_gpu_matrix_free.py, in units of 2^-24 of the entry's magnitude scale
KAPPA_OP = 64.0
W = 0.05
HALO = 8


def _capsule(n=50_000, length=12.0, radius=0.5, seed=0):
    rng = np.random.default_rng(seed)
    x = rng.uniform(-length / 2, length / 2, n)
    th = rng.uniform(0, 2 * np.pi, n)
    nrm = np.stack([np.zeros(n), np.cos(th), np.sin(th)], 1)
    xyz = np.stack([x, radius * np.cos(th), radius * np.sin(th)], 1) + rng.normal(size=(n, 3)) * 0.002
    return xyz.astype(np.float32), nrm.astype(np.float32)


def _lib():
    from nksr_b200 import _lib as L
    return L


class Rank:
    """one rank's share: local_system, the filtered operator and the Chronopoulos-Gear vectors"""

    def __init__(self, rec, xyz, nrm, bounds, rank, L, approx, owned=None):
        from nksr_b200 import dist_solve as ds
        H = HALO * W * 2 ** (L - 1)
        c = xyz[:, 0]
        sel = (c >= bounds[rank] - H) & (c < bounds[rank + 1] + H)
        self.loc = ds.local_system(rec, xyz[sel].contiguous(), nrm[sel].contiguous(), None, bounds, rank, 0, W, approx)
        self.field = self.loc.field
        self.owned = self.loc.owned if owned is None else owned
        self.n = self.field.svh.num_unknowns
        self.level = torch.cat([torch.full((self.field.svh.num_voxels(l),), l, dtype=torch.int64,
                                           device=xyz.device) for l in range(L)])
        self.key = torch.cat(self.field.svh.keys)

    def system(self, weights, owned=True):
        op = self.field.matrix_free_system(self.loc.pos_xyz, self.loc.normal_xyz, self.loc.normal_value, *weights,
                                           owned=self.owned if owned else None)
        op.svh_view, op.feat_view = self.field.svh.view(), self.field.feat_view()
        return op


def _join(a, b):
    """index into b of every (level, key) of a, -1 where b does not hold it"""
    wa = a.level * (1 << 58) + a.key
    wb = b.level * (1 << 58) + b.key
    order = torch.argsort(wb)
    sb = wb[order]
    pos = torch.searchsorted(sb, wa).clamp(max=sb.numel() - 1)
    hit = sb[pos] == wa
    return torch.where(hit, order[pos], torch.full_like(pos, -1))


def _op_dots(rk, op, r, u, w, ws, red):
    L = _lib()
    L.call("nksr_dcg_op_dots", op.svh_view, op.feat_view, op.cs, op.base_pos, op.base_nrm, op.ws, op.ws_bytes,
           rk.owned.to(torch.uint8).contiguous(), r, u, w, ws, red, L.stream_ptr(u.device))


_SCENES = {}


def _scene(cuda, L, approx, R):
    """(the R ranks with their filtered operators, the constraint weights); R = 1 is the whole cloud"""
    import nksr_b200
    from nksr_b200 import dist_solve as ds
    k = (L, approx)
    if k not in _SCENES:
        xyz, nrm = _capsule()
        rec = nksr_b200.Reconstructor(cuda, tree_depth=L)
        _SCENES[k] = (rec, torch.from_numpy(xyz).to(cuda), torch.from_numpy(nrm).to(cuda), {})
    rec, xyz, nrm, cache = _SCENES[k]
    if R not in cache:
        with torch.no_grad():
            bounds = ds.slab_bounds(xyz[:, 0], R, W * 2 ** (L - 1)) if R > 1 else [-math.inf, math.inf]
            ranks = [Rank(rec, xyz, nrm, bounds, r, L, approx) for r in range(R)]
            counts = sum(rk.loc.counts for rk in ranks)
            weights = ds.constraint_weights(float(counts[0]), float(counts[1]), W)
            for rk in ranks:
                rk.op = rk.system(weights)
        cache[R] = (ranks, weights)
    return cache[R]


CASES = [(L, approx) for L in (3, 4) for approx in (True, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("L,approx", CASES)
def test_one_rank_keeps_everything_and_matches_apply(cuda, L, approx):
    """bounds +-inf: the filter keeps every location, w is nksr_op_apply's y bit for bit, the dots are fp64 dots"""
    ranks, weights = _scene(cuda, L, approx, 1)
    rk = ranks[0]
    plain = rk.system(weights, owned=False)
    m = int(plain.cs.n_pos + plain.cs.n_nrm)
    assert rk.op.locations_kept == m and plain.locations_kept == m
    assert torch.equal(rk.op.rhs, plain.rhs) and torch.equal(rk.op.diag, plain.diag)
    g = torch.Generator(device=cuda).manual_seed(5)
    u = torch.randn(rk.n, device=cuda, generator=g)
    r = torch.randn(rk.n, device=cuda, generator=g)
    w = torch.full_like(u, float("nan"))
    ws = torch.zeros(_lib().call("nksr_dcg_workspace_bytes"), dtype=torch.uint8, device=cuda)
    red = torch.zeros(3, dtype=torch.float64, device=cuda)
    _op_dots(rk, rk.op, r, u, w, ws, red)
    y = rk.field.apply_operator(plain, u)
    assert torch.equal(w, y)
    ref = [float((r.double() * u.double()).sum()), float((w.double() * u.double()).sum()),
           float((r.double() * r.double()).sum())]
    for got, want in zip(red.tolist(), ref):
        assert abs(got - want) <= 1e-12 * abs(want), (got, want)


def _global(cuda, L, approx):
    ranks, _ = _scene(cuda, L, approx, 1)
    return ranks[0]


@pytest.mark.gpu
@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("L,approx", CASES)
def test_owned_rows_match_the_whole_cloud_operator(cuda, L, approx, R):
    """rhs, diag and w = A u on each rank's owned rows against the whole-cloud operator at the same (level, key); the
    kept set against a torch restatement of the criterion"""
    G = _global(cuda, L, approx)
    ranks, _ = _scene(cuda, L, approx, R)
    g = torch.Generator(device=cuda).manual_seed(9)
    u_glob = torch.randn(G.n, device=cuda, generator=g)
    # the whole-cloud scale of A u: |A| |u| with the assembled matrix of the same field, no larger than the oracle's
    # abs-term scale, so the bound is at least as strict as tests/test_gpu_matrix_free.py's
    Gw = G.field
    Gw.solver_config.update(operator="assembled", keep_system=True, max_iter=0, compact_rows=approx)
    Gw.solve(G.loc.pos_xyz, G.loc.normal_xyz, G.loc.normal_value, *_scene(cuda, L, approx, 1)[1])
    S = Gw.system
    Gw.solver_config.update(keep_system=False)
    Gw.system = None
    import scipy.sparse as sp
    A_abs = sp.csr_matrix((np.abs(S.val.cpu().numpy()).astype(np.float64), S.col.cpu().numpy(),
                           S.rowptr.cpu().numpy()), shape=(G.n, G.n))
    scale_w = A_abs @ np.abs(u_glob.cpu().numpy()).astype(np.float64)
    y_glob = G.field.apply_operator(G.op, u_glob)
    lv_g = G.level.cpu().numpy()
    for rk in ranks:
        idx = _join(rk, G)
        own = rk.owned
        assert bool((idx[own] >= 0).all())
        u = torch.where(idx >= 0, u_glob[idx.clamp(min=0)], torch.zeros_like(u_glob[:1]))
        r = torch.zeros_like(u)
        w = torch.full_like(u, float("nan"))
        ws = torch.zeros(_lib().call("nksr_dcg_workspace_bytes"), dtype=torch.uint8, device=cuda)
        red = torch.zeros(3, dtype=torch.float64, device=cuda)
        _op_dots(rk, rk.op, r, u, w, ws, red)
        assert bool((w[~own] == 0).all())
        gi = idx[own].cpu().numpy()
        assert_within(w[own].cpu().numpy(), y_glob[idx[own]].cpu().numpy(), scale_w[gi], KAPPA_OP,
                      f"A u on owned rows (L={L} approx={approx} R={R})")
        assert_within(rk.op.diag[own].cpu().numpy(), G.op.diag[idx[own]].cpu().numpy(),
                      np.abs(G.op.diag[idx[own]].cpu().numpy()), KAPPA_OP, "diagonal on owned rows")
        # rhs: scaled by the largest |rhs| of its level (no per-entry abs-term of E^T W t is at hand)
        rhs_g = G.op.rhs.cpu().numpy().astype(np.float64)
        lvl_max = np.array([np.abs(rhs_g[lv_g == l]).max(initial=0.0) for l in range(L)])
        assert_within(rk.op.rhs[own].cpu().numpy(), rhs_g[gi], lvl_max[lv_g[gi]], KAPPA_OP, "rhs on owned rows")
        # the kept set: a location is kept iff on some level an owned unknown neighbours its containing voxel
        svh = rk.field.svh
        order, vox, _ = rk.field.operator_items(rk.op)
        plain = rk.system(_scene(cuda, L, approx, R)[1], owned=False)
        all_order, all_vox, _ = rk.field.operator_items(plain)
        keep = torch.zeros(all_order.numel(), dtype=torch.bool, device=cuda)
        for l in range(L):
            v = all_vox[l].long()
            nb = svh.nbr27[l][v.clamp(min=0)].long()
            hit = (nb >= 0) & rk.owned[(svh.offsets[l] + nb).clamp(min=0, max=rk.n - 1)]
            keep |= (v >= 0) & hit.any(dim=1)
        assert torch.equal(order, all_order[keep]) and torch.equal(vox, all_vox[:, keep])
        assert rk.op.locations_kept == int(keep.sum())
        halo = bool((~own).any())
        if halo:
            assert rk.op.locations_kept < plain.locations_kept, (rk.op.locations_kept, plain.locations_kept)


def _exchange_plan(ranks):
    """for every rank: (source rank, my halo indices, the owner's indices) joined on (level, key)"""
    for rk in ranks:
        rk.recv = []
        owner = torch.cat(rk.loc.owner)
        for src, other in enumerate(ranks):
            if other is rk:
                continue
            mine = torch.nonzero((~rk.owned) & (owner == src)).reshape(-1)
            idx = _join(SimpleKeys(rk, mine), other)
            ok = idx >= 0
            rk.recv.append((src, mine[ok], idx[ok]))


class SimpleKeys:
    def __init__(self, rk, sel):
        self.level, self.key = rk.level[sel], rk.key[sel]


def _lockstep(ranks, tol, max_iter, extra=0):
    """the host loop of dist_solve.pcg_distributed over the simulated ranks; `extra` steps more after the verdict.
    Returns per rank x, the last w, the status and the steps launched"""
    L = _lib()
    dev = ranks[0].op.rhs.device
    st = L.stream_ptr(dev)
    nb = L.call("nksr_dcg_workspace_bytes")
    for rk in ranks:
        rk.v = {k: torch.full((rk.n,), float("nan"), device=dev) for k in "xruwps"}
        rk.ws = torch.full((nb,), 255, dtype=torch.uint8, device=dev)
        rk.red = torch.zeros(3, dtype=torch.float64, device=dev)
        rk.own8 = rk.owned.to(torch.uint8).contiguous()
        v = rk.v
        L.call("nksr_dcg_init", rk.op.diag, rk.op.rhs, rk.own8, v["x"], v["r"], v["u"], v["p"], v["s"], rk.n, rk.ws,
               nb, rk.red, st)

    def allreduce():
        s = sum(rk.red for rk in ranks)
        for rk in ranks:
            rk.red.copy_(s)

    allreduce()
    for rk in ranks:
        L.call("nksr_dcg_begin", rk.ws, rk.red, float(tol), int(max_iter), st)
    steps, after, snap = 0, 0, None
    while True:
        info = (C.c_double * 4)()
        L.call("nksr_dcg_status", ranks[0].ws, info, st)
        if info[3] != 0:
            if snap is None:
                snap = [(rk.v["x"].clone(), rk.v["w"].clone()) for rk in ranks]
            if after >= extra:
                break
            after += 1
        elif steps > max_iter + 2:
            break
        for rk in ranks:
            for src, dst, srci in rk.recv:
                rk.v["u"][dst] = ranks[src].v["u"][srci]
        for rk in ranks:
            v = rk.v
            _op_dots(rk, rk.op, v["r"], v["u"], v["w"], rk.ws, rk.red)
        allreduce()
        for rk in ranks:
            v = rk.v
            L.call("nksr_dcg_update", rk.op.diag, rk.own8, v["x"], v["r"], v["u"], v["w"], v["p"], v["s"], rk.n,
                   rk.ws, rk.red, st)
        steps += 1
    return [float(t) for t in info], steps, snap


@pytest.mark.gpu
@pytest.mark.parametrize("R", [2, 3])
@pytest.mark.parametrize("L,approx", CASES)
def test_lockstep_solve_matches_single_gpu(cuda, L, approx, R):
    """owned alpha gathered over R ranks against the single-GPU matrix-free solve (the tolerance of
    tests/test_gpu_global.py); launches after the verdict change nothing; two runs agree bit for bit"""
    G = _global(cuda, L, approx)
    ranks, weights = _scene(cuda, L, approx, R)
    G.field.solver_config.update(operator="matrix_free", tol=1e-6, max_iter=2000, keep_system=False)
    ref = G.field.solve(G.loc.pos_xyz, G.loc.normal_xyz, G.loc.normal_value, *weights).alpha
    _exchange_plan(ranks)
    info, steps, snap = _lockstep(ranks, 1e-6, 2000, extra=3)
    assert info[2] == 0 and steps == info[0] + 1 + 3, (info, steps)   # the verdict's step, then 3 more
    scale = float(ref.abs().max())
    worst = 0.0
    for rk, (x0, w0) in zip(ranks, snap):
        assert torch.equal(rk.v["x"], x0) and torch.equal(rk.v["w"], w0)      # no-ops after the verdict
        idx = _join(rk, G)
        own = rk.owned
        worst = max(worst, float((rk.v["x"][own] - ref[idx[own]]).abs().max()))
    print(f"[bounds] lockstep matrix-free global solve L={L} approx={approx} R={R}: iterations {info[0]:.0f} vs "
          f"{G.field.solve_info['iterations']}, max |alpha - ref| / max |ref| = {worst / scale:.3g}")
    assert worst <= 2e-3 * scale
    first = [(rk.v["x"].clone(), rk.v["w"].clone()) for rk in ranks]
    _lockstep(ranks, 1e-6, 2000)
    for rk, (x1, w1) in zip(ranks, first):
        assert torch.equal(rk.v["x"], x1) and torch.equal(rk.v["w"], w1)


@pytest.mark.gpu
def test_rank_that_owns_nothing(cuda):
    """no owned unknown: no location kept, w = 0, zero dots, no NaN"""
    G = _global(cuda, 3, True)
    _, weights = _scene(cuda, 3, True, 1)
    none = Rank.__new__(Rank)
    none.__dict__.update(G.__dict__)
    none.owned = torch.zeros(G.n, dtype=torch.bool, device=cuda)
    op = none.system(weights)
    assert op.locations_kept == 0
    assert bool(torch.isfinite(op.rhs).all()) and bool(torch.isfinite(op.diag).all())
    order, _, items = none.field.operator_items(op)
    assert order.numel() == 0 and items.shape[0] == 0
    u = torch.randn(G.n, device=cuda)
    w = torch.full_like(u, float("nan"))
    ws = torch.zeros(_lib().call("nksr_dcg_workspace_bytes"), dtype=torch.uint8, device=cuda)
    red = torch.full((3,), float("nan"), dtype=torch.float64, device=cuda)
    _op_dots(none, op, u, u, w, ws, red)
    assert bool((w == 0).all()) and red.tolist() == [0.0, 0.0, 0.0]


@pytest.mark.gpu
def test_driver_world1_matches_single_gpu_matrix_free(cuda, monkeypatch):
    """reconstruct_global(..., operator='matrix_free') at world 1 against reconstruct() with NKSR_OPERATOR=matrix_free:
    the checks of tests/test_gpu_global.py"""
    import nksr_b200
    from nksr_b200 import dist_solve as ds
    xyz, nrm = clouds.sphere(30000, noise=0.001)
    t = lambda a: torch.from_numpy(a).to(cuda)
    rec = nksr_b200.Reconstructor(cuda, tree_depth=3)
    monkeypatch.setenv("NKSR_OPERATOR", "matrix_free")
    ref = rec.reconstruct(t(xyz), t(nrm), voxel_size=0.03, solver_tol=1e-6)
    monkeypatch.delenv("NKSR_OPERATOR")
    assert ref.solve_info["operator"] == "matrix_free"
    glob = ds.reconstruct_global(rec, t(xyz), t(nrm), 0.03, solver_tol=1e-6, operator="matrix_free")
    info = glob.solve_info
    assert info["operator"] == "matrix_free" and info["nnz"] == 0
    assert info["locations_kept"] == info["locations_total"] and info["operator_bytes_per_apply"] > 0
    assert info["converged"] and info["iterations_launched"] > info["iterations"]
    assert glob.owned.all() and info["halo_recv"] == 0
    for l in range(3):
        assert torch.equal(ref.svh.keys[l], glob.svh.keys[l])
    a, b = ref.alpha.double(), glob.alpha.double()
    assert float((a - b).abs().max()) <= 2e-3 * float(a.abs().max())
    q = t(xyz[:2000])
    assert float((ref.evaluate_f(q).value - glob.evaluate_f(q).value).abs().max()) < 1e-3
    mesh = ds.extract_global_mesh(glob, mise_iter=1)
    r = np.linalg.norm(mesh.v.cpu().numpy(), axis=1)
    assert mesh.f.shape[0] > 1000 and abs(np.median(r) - 0.35) < 0.004
    # the default still assembles
    dflt = ds.reconstruct_global(rec, t(xyz), t(nrm), 0.03, solver_tol=1e-6)
    assert dflt.solve_info["operator"] == "assembled" and dflt.solve_info["nnz"] > 0


def test_unknown_operator_is_refused(monkeypatch):
    from nksr_b200 import dist_solve as ds
    with pytest.raises(ValueError):
        ds.reconstruct_global(None, torch.zeros(1, 3), None, 0.1, operator="csr")
    monkeypatch.setenv("NKSR_OPERATOR", "csr")
    with pytest.raises(ValueError):
        ds.reconstruct_global(None, torch.zeros(1, 3), None, 0.1)
    monkeypatch.setenv("NKSR_OPERATOR", "matrix_free")
    assert ds.resolve_operator() == "matrix_free" and ds.resolve_operator("assembled") == "assembled"
    monkeypatch.delenv("NKSR_OPERATOR")
    assert ds.resolve_operator() == "assembled"
