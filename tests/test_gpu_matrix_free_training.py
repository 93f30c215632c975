"""Training through the matrix-free kernel solve (fields._KernelSolve with solver_config['operator'] = 'matrix_free'):
the constraint values kernel (csrc/operator.cu, nksr_op_constraint_values) entry by entry against the fp64 oracle and
against nksr_evaluate, the end-to-end gradient against the fp64 VJPs and against the assembled operator, the forward
alpha against the no-grad matrix-free solve, repeatability, the edge cases of the backward, and seeded training."""
import numpy as np
import pytest
import torch

from oracle import nksr_oracle as O
from tests import clouds
from tests import grad_oracle as G
from tests.bounds import assert_blockwise, assert_within
from tests.test_gpu_kernel_grad import RTOL_E2E, _problem, _run, _setup, _train_field

pytestmark = pytest.mark.gpu

# Measured on an NVIDIA H100 80GB HBM3 (power limit 700 W).
# Constraint values against the fp64 field values / gradients at the same locations, per entry in units of 2^-24 of
# the abs-term scale.  Worst 3.24 (3-line gradient rows, L = 2, C = 4).
KAPPA_VALUES = 16.0
# Against nksr_evaluate at the same locations, same scale.  Worst 1.28.
KAPPA_VS_EVALUATE = 8.0
# Matrix-free against assembled gradient, both solved to tol 1e-6, per level block (each is within RTOL_E2E of fp64).
# Worst 1.7e-4 of the block's largest entry (L = 4, C = 4, approx_kernel_grad).
RTOL_OPERATORS = 1e-3
# The first training step's kernel losses, matrix-free against assembled (PCG tol 1e-5 on both).  Worst 1.0e-7.
RTOL_FIRST_STEP = 1e-6


def _np(t):
    return t.detach().cpu().numpy()


def _t(cuda, a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).to(cuda)


def _values_case(cuda, field, osvh, feats, pos, nrm, label, seed=0):
    """constraint values of the matrix-free system at pos / nrm against the fp64 oracle, nksr_evaluate and themselves"""
    rng = np.random.default_rng(seed)
    nval = rng.normal(size=nrm.shape).astype(np.float32)
    op = field.matrix_free_system(_t(cuda, pos), _t(cuda, nrm), _t(cuda, nval), 1.0, 0.5, 1.0, keep_constraints=True)
    n = op.n
    x = [rng.normal(size=n).astype(np.float32) for _ in range(2)]
    vp, vn = field.constraint_values(op, _t(cuda, x[0]), _t(cuda, x[1]))
    xs, xn = op.cons.pos[0], op.cons.nrm[0]
    approx = field.approx_kernel_grad
    for k in range(2):
        f, fa = O.evaluate_f(osvh, feats, x[k].astype(np.float64), _np(xs), False, approx, abs_terms=True)
        _, g, _, ga = O.evaluate_f(osvh, feats, x[k].astype(np.float64), _np(xn), True, approx, abs_terms=True)
        assert np.abs(f).max() > 0 and np.abs(g).max() > 0
        assert_within(_np(vp[:, k]), f, fa, KAPPA_VALUES, f"E x{k} positions ({label})")
        assert_within(_np(vn[:, k]), g, ga, KAPPA_VALUES, f"gradient rows x{k} normals ({label})")
        ef, _ = field._evaluate(_t(cuda, x[k]), xs, False)
        _, eg = field._evaluate(_t(cuda, x[k]), xn, True)
        assert_within(_np(vp[:, k]), _np(ef), fa, KAPPA_VS_EVALUATE, f"positions vs nksr_evaluate ({label})")
        assert_within(_np(vn[:, k]), _np(eg), ga, KAPPA_VS_EVALUATE, f"normals vs nksr_evaluate ({label})")
    vp2, vn2 = field.constraint_values(op, _t(cuda, x[0]), _t(cuda, x[1]))
    assert torch.equal(vp, vp2) and torch.equal(vn, vn2)
    return op


@pytest.mark.parametrize("L,C,approx", [(2, 4, False), (3, 8, True), (4, 4, False), (4, 16, True), (5, 3, False),
                                        (6, 4, True), (8, 4, False), (8, 32, True)])
def test_constraint_values_match_oracle(cuda, L, C, approx):
    """value rows (positions), compact lines (approx_kernel_grad) and 3-line gradient rows, depths 2 to 8"""
    import nksr_b200
    W = 0.05 if L <= 4 else 0.03
    xyz, _ = clouds.sphere(2000)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_point_splatting(_t(cuda, xyz))
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    rng = np.random.default_rng(L * 100 + C)
    feats = [(0.5 + 0.2 * rng.normal(size=(osvh.n(l), C))).astype(np.float32) for l in range(L)]
    field = nksr_b200.KernelField(svh, None, [_t(cuda, f) for f in feats], approx)
    jit = (xyz[:800] + rng.uniform(-0.5, 0.5, (800, 3)) * W).astype(np.float32)
    pos = np.concatenate([xyz, jit]).astype(np.float32)
    nrm = np.concatenate([osvh.centers(0), osvh.centers(1), jit[::2] * np.float32(1.01)]).astype(np.float32)
    pos, nrm = pos[~O.tent_branch_ambiguous(osvh, pos)], nrm[~O.tent_branch_ambiguous(osvh, nrm)]
    op = _values_case(cuda, field, osvh, feats, pos, nrm, f"L={L} C={C} approx={approx}")
    assert op.cs.nrm_compact == int(approx)


@pytest.mark.parametrize("approx", [False, True])
def test_constraint_values_on_an_adaptive_hierarchy(cuda, approx):
    """a pruned hierarchy, where many locations have no containing voxel on the fine levels"""
    import nksr_b200
    xyz, nrm = clouds.sphere(20000, noise=0.001)
    W, L, C = 0.02, 4, 4
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_adaptive_normal_variation(
        _t(cuda, xyz), _t(cuda, nrm), adaptive_depth=2)
    osvh = O.OracleSVH(W, L).build_from_keys([_np(svh.keys[l]) for l in range(L)])
    rng = np.random.default_rng(2)
    feats = [(0.5 + 0.2 * rng.normal(size=(osvh.n(l), C))).astype(np.float32) for l in range(L)]
    field = nksr_b200.KernelField(svh, None, [_t(cuda, f) for f in feats], approx)
    off = (xyz[::8] + 3.0 * W * nrm[::8]).astype(np.float32)
    q = np.concatenate([xyz[::8], off]).astype(np.float32)
    q = q[~O.tent_branch_ambiguous(osvh, q)]
    op = _values_case(cuda, field, osvh, feats, q[::2], q[1::2], f"adaptive approx={approx}")
    assert bool((op.base_pos < 0).any()) and bool((op.base_nrm < 0).any()) and bool((op.base_pos >= 0).any())


def _mf_field(cuda, svh, feats, approx):
    field, z = _train_field(cuda, svh, feats, approx)
    field.solver_config["operator"] = "matrix_free"
    return field, z


@pytest.mark.parametrize("L,C,approx", [(3, 4, False), (2, 8, False), (3, 4, True), (4, 4, True)])
def test_end_to_end_gradient_matches_fp64_and_assembled(cuda, L, C, approx):
    W = 0.05
    svh, osvh, feats, xyz, rng = _setup(cuda, L, C, W=W, n=2000)
    prob = _problem(osvh, xyz, rng, W)
    nxyz, nval, pw, nw, qx, hv, hg = prob
    field, z = _mf_field(cuda, svh, feats, approx)
    _, _, dz, dnv = _run(cuda, field, z, xyz, *prob)
    info = field.solve_info
    assert info["operator"] == "matrix_free" and info["nnz"] == 0 and info["operator_bytes_per_apply"] > 0
    assert info["adjoint_iterations"] > 0 and info["adjoint_relative_residual"] <= 1e-6
    g_alpha = (G.evaluate_adjoint(osvh, feats, qx, 0, approx, hv) + G.evaluate_adjoint(osvh, feats, qx, 1, approx, hg))
    ref = G.solve_vjp(osvh, feats, xyz, nxyz, nval, pw, nw, 1.0, approx, g_alpha)
    ev = G.feature_vjp(osvh, feats, qx, 0, approx, hv[:, None], [ref["alpha"]])
    eg = G.feature_vjp(osvh, feats, qx, 1, approx, hg[:, None, :], [ref["alpha"]])
    offs_c = [int(o) * C for o in osvh.offsets()]
    got = np.concatenate([_np(g) for g in dz]).reshape(-1)
    want = np.concatenate([a + b + c for a, b, c in zip(ref["dz"], ev, eg)]).reshape(-1)
    assert_blockwise(got, want, offs_c, RTOL_E2E, f"dL/dz matrix-free L={L} C={C} approx={approx}")
    assert_blockwise(_np(dnv).reshape(-1), ref["dt"].reshape(-1), [0, ref["dt"].size], RTOL_E2E,
                     "dL/dnormal_value matrix-free")
    fa, za = _train_field(cuda, svh, feats, approx)
    _, _, dz_a, dnv_a = _run(cuda, fa, za, xyz, *prob)
    assert fa.solve_info["operator"] == "assembled"
    asm = np.concatenate([_np(g) for g in dz_a]).reshape(-1)
    assert_blockwise(got, asm, offs_c, RTOL_OPERATORS, f"dL/dz matrix-free vs assembled L={L} C={C} approx={approx}")
    assert_blockwise(_np(dnv).reshape(-1), _np(dnv_a).reshape(-1), [0, dnv.numel()], RTOL_OPERATORS,
                     "dL/dnormal_value matrix-free vs assembled")


def test_forward_is_the_no_grad_solve_and_backward_is_repeatable(cuda):
    W = 0.05
    svh, osvh, feats, xyz, rng = _setup(cuda, 4, 4, W=W, n=3000)
    prob = _problem(osvh, xyz, rng, W)
    nxyz, nval, pw, nw = prob[:4]
    runs = []
    for _ in range(2):
        field, z = _mf_field(cuda, svh, feats, True)
        runs.append(_run(cuda, field, z, xyz, *prob))
    (a1, o1, dz1, n1), (a2, o2, dz2, n2) = runs
    assert torch.equal(a1, a2) and torch.equal(n1, n2)
    assert all(torch.equal(x, y) for x, y in zip(dz1, dz2))
    import nksr_b200
    with torch.no_grad():
        field = nksr_b200.KernelField(svh, None, [_t(cuda, f) for f in feats], True)
        field.solver_config.update(tol=1e-6, check_every=1, operator="matrix_free")
        field.solve(_t(cuda, xyz), _t(cuda, nxyz), _t(cuda, nval), pw, nw, 1.0)
    assert field.alpha.grad_fn is None and field.solve_info["operator"] == "matrix_free"
    assert torch.equal(field.alpha, a1)
    # a second solve on one operator workspace sees the same A: A x before the forward solve and after the adjoint
    op = field.matrix_free_system(_t(cuda, xyz), _t(cuda, nxyz), _t(cuda, nval), pw, nw, 1.0, keep_constraints=True)
    x = torch.randn(op.n, device=cuda, generator=torch.Generator(device=cuda).manual_seed(0))
    y0 = field.apply_operator(op, x)
    alpha = field._pcg_matrix_free(op, op.rhs)
    assert torch.equal(alpha, a1)
    field._pcg_matrix_free(op, torch.randn(op.n, device=cuda), adjoint=True)
    assert field.solve_info["adjoint_iterations"] > 0
    assert torch.equal(field.apply_operator(op, x), y0)


def test_zero_upstream_and_no_normal_constraints(cuda):
    svh, osvh, feats, xyz, rng = _setup(cuda, 3, 4)
    field, z = _mf_field(cuda, svh, feats, False)
    field.solve(_t(cuda, xyz), None, None, 1.0, 1.0, 1.0)
    (field.evaluate_f(_t(cuda, xyz[:100])).value * 0.0).sum().backward()
    assert field.solve_info["operator"] == "matrix_free" and field.solve_info["adjoint_iterations"] == 0
    assert all(bool((g.grad == 0).all()) for g in z)
    # no normal constraints: every target is 0, so alpha = 0 and, with a nonzero upstream gradient, the adjoint PCG
    # runs and every term of dL/dz holds a factor alpha or a target -- exactly zero, as on the assembled operator
    q = _t(cuda, xyz[::4] * 1.03)
    grads = {}
    for op in ("matrix_free", "assembled"):
        field, z = _train_field(cuda, svh, feats, False)
        field.solver_config["operator"] = op
        field.solve(_t(cuda, xyz), None, None, 1.0, 1.0, 1.0)
        assert not bool(field.alpha.any())
        field.evaluate_f(q).value.sum().backward()
        assert field.solve_info["operator"] == op and field.solve_info["adjoint_iterations"] > 0
        grads[op] = np.concatenate([_np(g.grad) for g in z]).reshape(-1)
    assert not grads["matrix_free"].any() and not grads["assembled"].any()


def test_interpolators_get_gradient(cuda):
    import nksr_b200
    svh, osvh, feats, xyz, rng = _setup(cuda, 3, 4)
    interp = torch.nn.ModuleList([torch.nn.Linear(4, 4) for _ in range(3)]).to(cuda)
    basis = [_t(cuda, f).requires_grad_(True) for f in feats]
    field = nksr_b200.KernelField(svh, interp, basis)
    field.solver_config["operator"] = "matrix_free"
    nxyz = osvh.centers(0).astype(np.float32)
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True)).astype(np.float32)
    field.solve(_t(cuda, xyz), _t(cuda, nxyz), _t(cuda, nval), 1.0, 0.01, 1.0)
    field.evaluate_f(_t(cuda, xyz[:500] * 1.02)).value.abs().sum().backward()
    assert field.solve_info["operator"] == "matrix_free"
    for l in range(3):
        assert interp[l].weight.grad is not None and bool(torch.isfinite(interp[l].weight.grad).all())
        assert float(interp[l].weight.grad.abs().sum()) > 0 and float(basis[l].grad.abs().sum()) > 0


def test_which_operator_a_grad_solve_uses(cuda, monkeypatch):
    monkeypatch.delenv("NKSR_OPERATOR", raising=False)
    svh, osvh, feats, xyz, rng = _setup(cuda, 3, 4)
    t = _t(cuda, xyz)
    field, z = _train_field(cuda, svh, feats, True)          # no operator named: assembled
    field.solve(t, None, None, 1.0, 1.0, 1.0)
    assert field.solve_info["operator"] == "assembled" and field.solve_info["nnz"] > 0
    field, z = _train_field(cuda, svh, feats, True)
    field.solver_config.update(operator="matrix_free", keep_system=True)
    field.solve(t, None, None, 1.0, 1.0, 1.0)
    assert field.solve_info["operator"] == "assembled" and field.system is not None
    monkeypatch.setenv("NKSR_OPERATOR", "matrix_free")
    field, z = _train_field(cuda, svh, feats, True)
    field.solve(t, None, None, 1.0, 1.0, 1.0)
    assert field.solve_info["operator"] == "matrix_free" and field.solve_info["nnz"] == 0


STEPS = 30


def _train(cuda, operator, steps=STEPS, seed=3):
    from nksr_b200 import training as T
    from nksr_b200.network import NKSRNetwork
    xyz, nrm = clouds.sphere(30_000, noise=0.001)
    scene = T.TrainingScene(_t(cuda, xyz), _t(cuda, nrm), 0.02, 4)
    net = NKSRNetwork(dict(backbone="unet", tree_depth=4, kernel_dim=4, trainable=True, seed=seed)).to(cuda)
    opt = T.make_optimizer(net)
    gen = torch.Generator(device=cuda).manual_seed(seed)
    curve, grads = [], None
    for step in range(steps):
        _, _, k = T.train_step(net, opt, scene, gen, kernel=True, operator=operator)
        curve.append({key: float(v) for key, v in k.items()})
        if step == 0:
            grads = {name: p.grad.detach().clone() for name, p in net.named_parameters() if p.grad is not None}
    return net, scene, curve, grads


def test_matrix_free_training_reaches_the_heads_lowers_the_losses_and_is_repeatable(cuda):
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        net, scene, curve, grads = _train(cuda, "matrix_free")
        net2, _, curve2, grads2 = _train(cuda, "matrix_free")
        _, _, curve_a, _ = _train(cuda, "assembled", steps=1)
    finally:
        torch.use_deterministic_algorithms(False)
    C, ad = net.kernel_dim, scene.adaptive_depth
    for l in range(net.tree_depth):
        w = grads[f"backbone_net.heads.{l}.weight"]
        basis = w[6:6 + C]
        assert bool(torch.isfinite(basis).all()) and bool((basis.abs().sum(dim=1) > 0).all()), f"basis head {l}"
        if l < ad:
            assert float(w[3:6].abs().sum()) > 0, f"normal head {l}"
        names = [n for n in grads if n.startswith(f"interpolators.{l}.")]
        assert names and all(bool(torch.isfinite(grads[n]).all()) and float(grads[n].abs().sum()) > 0 for n in names)
    first = np.mean([c["total"] for c in curve[:3]])
    last = np.mean([c["total"] for c in curve[-3:]])
    print(f"[train] matrix-free kernel losses: first {curve[0]} last {curve[-1]}; total {first:.5g} -> {last:.5g}")
    assert last < first
    assert curve == curve2
    assert all(torch.equal(a, b) for a, b in zip(net.state_dict().values(), net2.state_dict().values()))
    assert grads.keys() == grads2.keys() and all(torch.equal(grads[k], grads2[k]) for k in grads)
    worst = max(abs(curve[0][k] - curve_a[0][k]) / abs(curve_a[0][k]) for k in curve_a[0])
    print(f"[train] first step, matrix-free vs assembled: worst relative difference {worst:.3g} "
          f"({curve[0]} vs {curve_a[0]})")
    assert worst <= RTOL_FIRST_STEP
