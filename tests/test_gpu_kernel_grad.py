"""Backward of the kernel field on the GPU (csrc/field_bwd.cu, fields._KernelSolve / _KernelEvaluate): every kernel
entry by entry against the fp64 VJPs of tests/grad_oracle.py given the same fp32 inputs, the end-to-end gradient of a
solve + evaluation loss against the oracle's fp64 gradient, bitwise repeatability, and that grad mode leaves the
forward's alpha and f unchanged."""
import numpy as np
import pytest
import torch

from oracle import nksr_oracle as O
from tests import clouds
from tests import grad_oracle as G
from tests.bounds import assert_blockwise, assert_within

pytestmark = pytest.mark.gpu

# per-entry bound of the backward kernels, in units of 2^-24 of the abs-term scale (measured on H100 worst 5.7, the
# regulariser VJP; the feature VJP 4.4, the evaluation adjoint 1.6)
KAPPA_VJP = 32.0
# end to end: the gradient through an fp32 PCG solve (tol 1e-6) against the fp64 sparse solve, per level block
# (measured on H100: 9.3e-5 of the block's largest entry)
RTOL_E2E = 5e-4
# brick against row fill: the reassociation of the Gram entries carried through two solves (measured 2.8e-5)
RTOL_FILL = 2e-4


def _np(t):
    return t.detach().cpu().numpy()


def _setup(cuda, L, C, W=0.05, n=3000, seed=1):
    import nksr_b200
    xyz, _ = clouds.sphere(n)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_point_splatting(torch.from_numpy(xyz).to(cuda))
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    rng = np.random.default_rng(seed)
    feats = [(0.5 + 0.2 * rng.normal(size=(osvh.n(l), C))).astype(np.float32) for l in range(L)]
    return svh, osvh, feats, xyz, rng


def _locations(osvh, xyz, W, rng):
    """data points, voxel centres of the two finest levels (the tent snap zone) and jittered points"""
    cen = np.concatenate([osvh.centers(l) for l in range(min(2, osvh.depth))])[:1500]
    jit = xyz[:1000] + rng.uniform(-0.5, 0.5, (1000, 3)).astype(np.float32) * W
    q = np.concatenate([xyz[:1500], cen, jit]).astype(np.float32)
    return q[~O.tent_branch_ambiguous(osvh, q)]


def _field(cuda, svh, feats, approx):
    import nksr_b200
    return nksr_b200.KernelField(svh, None, [torch.from_numpy(f).to(cuda) for f in feats], approx)


@pytest.mark.parametrize("L,C,approx", [(1, 1, False), (2, 3, False), (3, 4, True), (3, 8, False), (4, 16, False),
                                        (5, 32, False), (4, 4, True), (5, 3, True)])
def test_kernels_match_oracle(cuda, L, C, approx):
    svh, osvh, feats, xyz, rng = _setup(cuda, L, C)
    field = _field(cuda, svh, feats, approx)
    q = _locations(osvh, xyz, 0.05, rng)
    _, xs, _, base, ranges = field._sorted_locations(torch.from_numpy(q).to(cuda))
    xs_np = _np(xs)
    loc = (xs, base, ranges)
    n, m = svh.num_unknowns, xs.shape[0]
    a0, a1 = rng.normal(size=n).astype(np.float32), rng.normal(size=n).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    offs = osvh.offsets()
    for mode in (0, 1):
        shape = (m,) if mode == 0 else (m, 3)
        coef = rng.normal(size=shape).astype(np.float32)
        got = _np(field._evaluate_adjoint(loc, mode, t(coef)))
        ref, scale = G.evaluate_adjoint(osvh, feats, xs_np, mode, approx, coef.astype(np.float64), abs_terms=True)
        assert np.abs(ref).max() > 0
        assert_within(got, ref, scale, KAPPA_VJP, f"evaluate_adjoint mode {mode} L={L} C={C} approx={approx}")
        for two in (False, True):
            cshape = (m, 2 if two else 1) + ((3,) if mode == 1 else ())
            cf = rng.normal(size=cshape).astype(np.float32)
            dz = torch.zeros((n, C), dtype=torch.float32, device=cuda)
            field._feature_vjp(loc, mode, t(cf), t(a0), t(a1) if two else None, dz)
            vecs = [a0.astype(np.float64)] + ([a1.astype(np.float64)] if two else [])
            ref, scale = G.feature_vjp(osvh, feats, xs_np, mode, approx, cf.astype(np.float64), vecs, abs_terms=True)
            got = _np(dz)
            for l in range(L):
                assert_within(got[offs[l]:offs[l + 1]], ref[l], scale[l], KAPPA_VJP,
                              f"feature_vjp mode {mode} two={two} level {l} L={L} C={C} approx={approx}")
    dz = torch.zeros((n, C), dtype=torch.float32, device=cuda)
    from nksr_b200._lib import call, stream_ptr
    call("nksr_regulariser_vjp", svh.view(), field.feat_view(), t(a0), t(a1), 1.0, dz, stream_ptr(cuda))
    ref, scale = G.regulariser_vjp(osvh, feats, a0.astype(np.float64), a1.astype(np.float64), abs_terms=True)
    for l in range(L):
        assert_within(_np(dz)[offs[l]:offs[l + 1]], ref[l], scale[l], KAPPA_VJP, f"regulariser_vjp level {l}")


def test_kernels_on_an_adaptive_hierarchy(cuda):
    """a pruned hierarchy (build_adaptive_normal_variation: fine levels only near detail), where many locations have no
    containing voxel on the fine levels"""
    import nksr_b200
    xyz, nrm = clouds.sphere(20000, noise=0.001)
    W, L, C = 0.02, 4, 4
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_adaptive_normal_variation(t(xyz), t(nrm), adaptive_depth=2)
    osvh = O.OracleSVH(W, L).build_from_keys([_np(svh.keys[l]) for l in range(L)])
    rng = np.random.default_rng(2)
    feats = [(0.5 + 0.2 * rng.normal(size=(osvh.n(l), C))).astype(np.float32) for l in range(L)]
    field = _field(cuda, svh, feats, False)
    # locations on the surface and 3 voxels off it along the normal (outside the finest levels, inside coarse ones)
    off = (xyz[::8] + 3.0 * W * nrm[::8]).astype(np.float32)
    q = _locations(osvh, np.concatenate([xyz[::8], off]).astype(np.float32), W, rng)
    _, xs, _, base, ranges = field._sorted_locations(t(q))
    assert bool((base < 0).any()) and bool((base >= 0).any())
    xs_np, n, m, offs = _np(xs), svh.num_unknowns, xs.shape[0], osvh.offsets()
    a0 = rng.normal(size=n).astype(np.float32)
    for mode in (0, 1):
        coef = rng.normal(size=(m,) if mode == 0 else (m, 3)).astype(np.float32)
        ref, scale = G.evaluate_adjoint(osvh, feats, xs_np, mode, False, coef.astype(np.float64), abs_terms=True)
        assert_within(_np(field._evaluate_adjoint((xs, base, ranges), mode, t(coef))), ref, scale, KAPPA_VJP,
                      f"adaptive evaluate_adjoint mode {mode}")
        cf = coef.reshape((m, 1) + coef.shape[1:])
        dz = torch.zeros((n, C), dtype=torch.float32, device=cuda)
        field._feature_vjp((xs, base, ranges), mode, t(cf), t(a0), None, dz)
        ref, scale = G.feature_vjp(osvh, feats, xs_np, mode, False, cf.astype(np.float64), [a0.astype(np.float64)],
                                   abs_terms=True)
        for l in range(L):
            assert_within(_np(dz)[offs[l]:offs[l + 1]], ref[l], scale[l], KAPPA_VJP, f"adaptive feature_vjp {mode} {l}")


def _train_field(cuda, svh, feats, approx, fill=None):
    import nksr_b200
    z = [torch.from_numpy(f).to(cuda).requires_grad_(True) for f in feats]
    field = nksr_b200.KernelField(svh, None, z, approx)
    field.solver_config.update(tol=1e-6, check_every=1)
    if fill:
        field.solver_config["fill"] = fill
    return field, z


def _problem(osvh, xyz, rng, W):
    nxyz = np.concatenate([osvh.centers(0), osvh.centers(1)]).astype(np.float32)
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True)).astype(np.float32)
    pw, nw = 1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * W * W
    qx = np.concatenate([xyz[::3] + np.float32(0.3 * W), osvh.centers(0)[::5] * np.float32(1.05)]).astype(np.float32)
    qx = qx[~O.tent_branch_ambiguous(osvh, qx)]
    hv = rng.normal(size=qx.shape[0])
    hg = rng.normal(size=(qx.shape[0], 3))
    return nxyz, nval, pw, nw, qx, hv, hg


def _run(cuda, field, z, xyz, nxyz, nval, pw, nw, qx, hv, hg):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(cuda)
    nv = t(nval).requires_grad_(True)
    field.solve(t(xyz), t(nxyz), nv, pw, nw, 1.0)
    out = field.evaluate_f(t(qx), grad=True)
    loss = (out.value * t(hv)).sum() + (out.gradient * t(hg)).sum()
    loss.backward()
    return field.alpha.detach().clone(), out, [g.grad.clone() for g in z], nv.grad.clone()


@pytest.mark.parametrize("L,C,approx", [(3, 4, False), (2, 8, False), (3, 4, True)])
def test_end_to_end_gradient_matches_fp64(cuda, L, C, approx):
    W = 0.05
    svh, osvh, feats, xyz, rng = _setup(cuda, L, C, W=W, n=2000)
    nxyz, nval, pw, nw, qx, hv, hg = _problem(osvh, xyz, rng, W)
    field, z = _train_field(cuda, svh, feats, approx)
    alpha, _, dz, dnv = _run(cuda, field, z, xyz, nxyz, nval, pw, nw, qx, hv, hg)
    assert field.solve_info["adjoint_iterations"] > 0
    # fp64 reference: the solve's VJP plus the evaluation's, at the fp64 sparse solution
    g_alpha = (G.evaluate_adjoint(osvh, feats, qx, 0, approx, hv) + G.evaluate_adjoint(osvh, feats, qx, 1, approx, hg))
    ref = G.solve_vjp(osvh, feats, xyz, nxyz, nval, pw, nw, 1.0, approx, g_alpha)
    ev = G.feature_vjp(osvh, feats, qx, 0, approx, hv[:, None], [ref["alpha"]])
    eg = G.feature_vjp(osvh, feats, qx, 1, approx, hg[:, None, :], [ref["alpha"]])
    offs = osvh.offsets()
    got = np.concatenate([_np(g) for g in dz]).reshape(-1)
    want = np.concatenate([a + b + c for a, b, c in zip(ref["dz"], ev, eg)]).reshape(-1)
    offs_c = [int(o) * C for o in offs]
    assert_blockwise(got, want, offs_c, RTOL_E2E, f"dL/dz L={L} C={C} approx={approx}")
    assert_blockwise(_np(dnv).reshape(-1), ref["dt"].reshape(-1), [0, ref["dt"].size], RTOL_E2E, "dL/dnormal_value")


def test_repeatable_and_forward_unchanged(cuda):
    W = 0.05
    svh, osvh, feats, xyz, rng = _setup(cuda, 4, 4, W=W, n=3000)
    nxyz, nval, pw, nw, qx, hv, hg = _problem(osvh, xyz, rng, W)
    runs = []
    for _ in range(2):
        field, z = _train_field(cuda, svh, feats, False)
        runs.append(_run(cuda, field, z, xyz, nxyz, nval, pw, nw, qx, hv, hg))
    (a1, o1, dz1, n1), (a2, o2, dz2, n2) = runs
    assert torch.equal(a1, a2) and torch.equal(n1, n2)
    assert all(torch.equal(x, y) for x, y in zip(dz1, dz2))
    # no_grad forward: bitwise the same alpha, f and grad f
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(cuda)
    with torch.no_grad():
        field = _field(cuda, svh, feats, False)
        field.solver_config.update(tol=1e-6, check_every=1)
        field.solve(t(xyz), t(nxyz), t(nval), pw, nw, 1.0)
        out = field.evaluate_f(t(qx), grad=True)
    assert field.alpha.grad_fn is None and torch.equal(field.alpha, a1)
    assert torch.equal(out.value, o1.value.detach()) and torch.equal(out.gradient, o1.gradient.detach())


def test_fill_choice_does_not_change_the_gradient(cuda):
    W = 0.05
    svh, osvh, feats, xyz, rng = _setup(cuda, 3, 4, W=W, n=3000)
    nxyz, nval, pw, nw, qx, hv, hg = _problem(osvh, xyz, rng, W)
    res = {}
    for fill in ("rows", "brick"):
        field, z = _train_field(cuda, svh, feats, False, fill)
        res[fill] = _run(cuda, field, z, xyz, nxyz, nval, pw, nw, qx, hv, hg)
    offs = [int(o) * 4 for o in osvh.offsets()]
    a = np.concatenate([_np(g) for g in res["rows"][2]]).reshape(-1)
    b = np.concatenate([_np(g) for g in res["brick"][2]]).reshape(-1)
    assert_blockwise(b, a, offs, RTOL_FILL, "dL/dz brick vs rows")


def test_outside_queries_and_zero_upstream(cuda):
    svh, osvh, feats, xyz, rng = _setup(cuda, 3, 4)
    field, z = _train_field(cuda, svh, feats, False)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(cuda)
    field.solve(t(xyz), None, None, 1.0, 1.0, 1.0)           # no normal constraints
    far = np.array([[50.0, 50.0, 50.0], [1e9, 0.0, 0.0], [np.nan, 0.0, 0.0]], np.float32)
    out = field.evaluate_f(t(far), grad=True)
    assert torch.all(out.value[:2] == 0)
    (out.value[:2].sum() + out.gradient[:2].sum()).backward()
    assert all(g.grad is not None and bool((g.grad == 0).all()) for g in z)
    # zero upstream gradient: the adjoint solve is skipped, the gradient is exactly zero
    field, z = _train_field(cuda, svh, feats, False)
    field.solve(t(xyz), None, None, 1.0, 1.0, 1.0)
    (field.evaluate_f(t(xyz[:100])).value * 0.0).sum().backward()
    assert field.solve_info["adjoint_iterations"] == 0
    assert all(bool((g.grad == 0).all()) for g in z)


def test_interpolator_gets_gradient_and_mesh_records_no_graph(cuda):
    svh, osvh, feats, xyz, rng = _setup(cuda, 3, 4)
    import nksr_b200
    interp = torch.nn.ModuleList([torch.nn.Linear(4, 4) for _ in range(3)]).to(cuda)
    basis = [torch.from_numpy(f).to(cuda).requires_grad_(True) for f in feats]
    field = nksr_b200.KernelField(svh, interp, basis)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(cuda)
    nxyz = osvh.centers(0).astype(np.float32)
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True)).astype(np.float32)
    field.solve(t(xyz), t(nxyz), t(nval), 1.0, 0.01, 1.0)
    field.evaluate_f(t(xyz[:500] * 1.02)).value.abs().sum().backward()
    for l in range(3):
        assert interp[l].weight.grad is not None and bool(torch.isfinite(interp[l].weight.grad).all())
        assert float(interp[l].weight.grad.abs().sum()) > 0 and float(basis[l].grad.abs().sum()) > 0
    mesh = field.extract_dual_mesh()
    assert mesh.v.grad_fn is None
