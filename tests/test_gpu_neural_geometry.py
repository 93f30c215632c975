"""The neural output field (geometry='neural', models/nksr_net.py:114-119): the position Jacobian of the interpolation
(DESIGN.md SPEC S17a, csrc/neural_field.cu) and its VJP against the fp64 restatement of tests/jacobian_oracle.py, entry by
entry within kappa * 2^-24 * scale (tests/bounds.py's convention); NeuralField's position gradient and the second-order
training gradients against torch autograd through NeuralField._interp; the Reconstructor and train_step with
geometry='neural'."""
import numpy as np
import pytest
import torch

from nksr_b200._lib import NksrError
from oracle import nksr_oracle as O
from tests import clouds
from tests.bounds import assert_within
from tests.jacobian_oracle import jacobian64, jacobian_vjp64

pytestmark = pytest.mark.gpu

# kappa in units of 2^-24 (tests/bounds.py), each at most 8x the worst ratio measured on an NVIDIA H100 80GB HBM3
# (power limit 700 W) over this file.
# nksr_neural_interp_jacobian against fp64: the fp32 local coordinate, the tent factors of every slot and the fma chain
# over up to 20 slots, times the fp32 1 / W_l.  Worst 6.18.
KAPPA_JAC = 32.0
# nksr_neural_interp_jacobian_vjp against fp64: an fp32 fma chain over three axes and the queries of 27 ranges.
# Worst 6.00.
KAPPA_JAC_VJP = 32.0

np_ = lambda a: a.detach().double().cpu().numpy()


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


_HIER = {}


def _hierarchy(cuda, depth):
    """a sphere splatted at W = 0.05 (depth <= 4) or 0.02, with the oracle's hierarchy of the same points"""
    if depth not in _HIER:
        from nksr_b200.svh import SparseFeatureHierarchy
        W = 0.05 if depth <= 4 else 0.02
        xyz, _ = clouds.sphere(3000, noise=0.001)
        svh = SparseFeatureHierarchy(W, depth, cuda).build_point_splatting(_t(xyz, cuda))
        osvh = O.OracleSVH(W, depth).build_point_splatting(xyz)
        for l in range(depth):
            assert np.array_equal(svh.keys[l].cpu().numpy(), osvh.keys[l]), l
        _HIER[depth] = (svh, osvh, xyz)
    return _HIER[depth]


def _features(svh, C, seed):
    g = torch.Generator().manual_seed(seed)
    return {l: torch.randn((svh.num_voxels(l), C), generator=g).to(svh.device) for l in range(svh.depth)}


def _queries(osvh, xyz, n, seed):
    """random queries (the input points, points near them, points uniform over a box larger than the cloud), exact
    voxel centres of every level, and queries inside the snap zone |tau| < 2^-12 of one level on some axes; the ones
    whose fp32 tau may fall on the other side of the snap zone's edge are dropped (a different formula there)"""
    rng = np.random.default_rng(seed)
    near = xyz[rng.integers(0, xyz.shape[0], n)] + rng.normal(0.0, 0.03, (n, 3))
    box = rng.uniform(-1.4, 1.4, (n, 3))
    cen = np.concatenate([osvh.centers(l)[rng.integers(0, osvh.n(l), n // 4)] for l in range(osvh.depth)
                          if osvh.n(l)])
    lv = rng.integers(0, osvh.depth, cen.shape[0])
    w = np.array([osvh.level_w(l) for l in range(osvh.depth)])[lv]
    snap = cen + (rng.uniform(-1e-4, 1e-4, cen.shape) * (rng.random(cen.shape) < 0.6)) * w[:, None]
    q = np.concatenate([xyz[:n], near, box, cen, snap]).astype(np.float32)
    return q[~O.tent_branch_ambiguous(osvh, q)]


_BAD = [[5.0, 5.0, 5.0], [-3.0, 0.2, 0.1], [float("nan"), 0.0, 0.0], [0.0, float("inf"), 0.0],
        [0.0, 0.0, -float("inf")], [1.0e7, 0.0, 0.0], [0.0, -3.0e5, 0.0]]

_GIVEN = {"0": lambda D: [0], "02": lambda D: [0, 2], "all": lambda D: list(range(D)), "top": lambda D: [D - 1]}
_SWEEP = [(d, c, g) for d in (1, 3, 4, 6, 8) for c in (1, 3, 4, 16, 32) for g in sorted(_GIVEN)
          if not (d == 1 and g != "all") and not (d > 1 and g == "top" and c not in (4, 16))]


def _field(svh, feats, levels, decoder=None, position_gradient=False):
    import nksr_b200
    return nksr_b200.NeuralField(svh, decoder if decoder is not None else torch.nn.Identity(),
                                 {l: feats[l] for l in levels}, position_gradient=position_gradient)


@pytest.mark.parametrize("depth,C,given", _SWEEP)
def test_jacobian_against_fp64(cuda, depth, C, given):
    svh, osvh, xyz = _hierarchy(cuda, depth)
    levels = _GIVEN[given](depth)
    feats = _features(svh, C, seed=depth * 100 + C)
    nf = _field(svh, feats, levels)
    q = _queries(osvh, xyz, 600, seed=C)
    qt = _t(q, cuda)
    jac = nf.jacobian(qt)
    assert jac.shape == (q.shape[0], 3, C * len(levels))
    ref, scale = jacobian64(osvh, {l: f.cpu().numpy() for l, f in feats.items()}, levels, q)
    assert_within(np_(jac), ref, scale, KAPPA_JAC, f"jacobian depth {depth} C {C} G {levels}")
    # the values of the same pass: bitwise those of nksr_neural_interp; the Jacobian the same without them
    u, jac2 = nf._jacobian_cuda(qt, nf.features, with_values=True)
    assert torch.equal(u, nf.interpolate(qt)) and torch.equal(jac2, jac)
    # outside the hierarchy, non-finite, outside the key range: exactly-zero rows
    bad = torch.tensor(_BAD, device=cuda)
    assert torch.equal(nf.jacobian(bad), torch.zeros((len(_BAD), 3, C * len(levels)), device=cuda))


@pytest.mark.parametrize("depth,C,given", _SWEEP)
def test_jacobian_vjp_against_fp64_and_repeatable(cuda, depth, C, given):
    svh, osvh, xyz = _hierarchy(cuda, depth)
    levels = _GIVEN[given](depth)
    feats = _features(svh, C, seed=7)
    nf = _field(svh, feats, levels)
    q = _queries(osvh, xyz, 600, seed=depth)
    q = np.concatenate([q, q[:200]])                           # repeated queries
    qt = _t(q, cuda)
    g = torch.randn((q.shape[0], 3, C * len(levels)), generator=torch.Generator().manual_seed(3)).to(cuda)
    d1 = nf._interp_vjp(qt, g, jacobian=True)
    d2 = nf._interp_vjp(qt, g, jacobian=True)
    ref = jacobian_vjp64(osvh, levels, C, q, g.cpu().double().numpy())
    for l in range(depth):
        if l not in levels:
            assert d1[l] is None
            continue
        assert torch.equal(d1[l], d2[l]), l
        assert_within(np_(d1[l]), ref[l][0], ref[l][1], KAPPA_JAC_VJP, f"jacobian vjp depth {depth} C {C} level {l}")
    # no queries: zero gradients
    z = nf._interp_vjp(qt[:0], g[:0], jacobian=True)
    for l in levels:
        assert torch.equal(z[l], torch.zeros_like(feats[l]))


def test_empty_given_level(cuda):
    import nksr_b200
    from nksr_b200.svh import SparseFeatureHierarchy
    svh, osvh, xyz = _hierarchy(cuda, 4)
    C, D = 3, 4
    keys = [torch.zeros(0, dtype=torch.int64, device=cuda)] + [svh.keys[l] for l in range(1, D)]
    part = SparseFeatureHierarchy(svh.voxel_size, D, cuda).build_from_keys(keys)
    feats = _features(part, C, seed=1)
    nf = nksr_b200.NeuralField(part, torch.nn.Identity(), feats)
    q = _t(xyz[:300], cuda)
    jac = nf.jacobian(q)
    assert jac.shape == (300, 3, C * D)
    assert torch.equal(jac[:, :, :C], torch.zeros_like(jac[:, :, :C])) and (jac[:, :, C:] != 0).any()
    d = nf._interp_vjp(q, torch.ones_like(jac), jacobian=True)
    assert d[0].shape == (0, C) and (d[1] != 0).any()


def _away_from_centres(svh, q, margin=0.01):
    """queries whose local coordinate is at least `margin` from a voxel centre on every level that contains them: there
    the one-sided tent derivative is the derivative torch autograd takes through NeuralField._interp"""
    from nksr_b200.fields import SparseFeatureHierarchyCoords
    base = svh.locate(q).long()
    keep = torch.ones(q.shape[0], dtype=torch.bool, device=q.device)
    for l in range(svh.depth):
        if svh.num_voxels(l) == 0:
            continue
        b = base[l]
        ijk = SparseFeatureHierarchyCoords.ijk(svh, l)[b.clamp(min=0)].double()
        tau = q.double() / (svh.voxel_size * 2 ** l) - (ijk + 0.5)
        keep &= (b < 0) | (tau.abs() > margin).all(dim=1)
    return q[keep].contiguous()


def _smooth_decoder(cuda, width, seed=0):
    # a smooth decoder: ReLU kinks would make the comparison depend on the last bits of u
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(width, 32), torch.nn.Tanh(), torch.nn.Linear(32, 32), torch.nn.Tanh(),
                               torch.nn.Linear(32, 1)).to(cuda)


def _torch_gradient(nf, dec, q, create_graph):
    qq = q.clone().requires_grad_(True)
    v = dec(nf._interp(qq)).reshape(-1)
    (g,) = torch.autograd.grad(v.sum(), qq, create_graph=create_graph)
    return v, g


def test_position_gradient_agrees_with_torch_autograd(cuda):
    svh, osvh, xyz = _hierarchy(cuda, 4)
    C = 4
    dec = _smooth_decoder(cuda, C * 4)
    feats = {l: f.requires_grad_(True) for l, f in _features(svh, C, seed=9).items()}
    nf = _field(svh, feats, list(range(4)), dec, position_gradient=True)
    q = _away_from_centres(svh, _t(_queries(osvh, xyz, 1000, seed=2), cuda))
    assert q.shape[0] > 2000
    v_ref, g_ref = _torch_gradient(nf, dec, q, False)
    tol = 1e-4 * float(g_ref.abs().max())
    with torch.no_grad():
        ev = nf.evaluate_f(q, grad=True)
    assert ev.gradient.shape == (q.shape[0], 3) and ev.value.grad_fn is None and ev.gradient.grad_fn is None
    assert torch.allclose(ev.gradient, g_ref, rtol=1e-4, atol=tol)
    ev = nf.evaluate_f(q, grad=True)
    assert ev.value.grad_fn is not None and ev.gradient.grad_fn is not None
    assert torch.allclose(ev.gradient, g_ref, rtol=1e-4, atol=tol)
    assert torch.allclose(ev.value, v_ref, rtol=1e-4, atol=1e-4 * float(v_ref.abs().max()))
    # the value-only field is unchanged: no gradient
    assert _field(svh, feats, list(range(4)), dec).evaluate_f(q, grad=True).gradient is None


def test_second_order_training_gradients_agree_with_torch(cuda):
    from types import SimpleNamespace
    from nksr_b200 import training as T
    svh, osvh, xyz = _hierarchy(cuda, 4)
    C = 4
    dec = _smooth_decoder(cuda, C * 4, seed=1)
    feats = {l: f.requires_grad_(True) for l, f in _features(svh, C, seed=11).items()}
    nf = _field(svh, feats, list(range(4)), dec, position_gradient=True)
    pts = _away_from_centres(svh, _t(xyz, cuda))
    nrm = torch.nn.functional.normalize(pts, dim=1)
    params = list(feats.values()) + list(dec.parameters())

    def grads(field):
        l_val, l_nrm = T.gt_surface_loss(field, pts, nrm, subsample=0)
        return torch.autograd.grad(l_val + l_nrm, params), (float(l_val), float(l_nrm))

    got, lg = grads(nf)

    def torch_eval(q, grad=False):
        v, g = _torch_gradient(nf, dec, q, True)
        return SimpleNamespace(value=v, gradient=g)

    want, lw = grads(SimpleNamespace(evaluate_f=torch_eval))
    print(f"[second order] losses cuda {lg} torch {lw}")
    assert np.allclose(lg, lw, rtol=1e-4)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape
        err = float((a - b).abs().max())
        top = float(b.abs().max())
        print(f"[second order] parameter {i}: max |d| {err:.3g}, max |ref| {top:.3g}")
        assert top > 0 and torch.allclose(a, b, rtol=1e-3, atol=1e-3 * top), i


def _net(cuda, depth, structure="encoder", udf=False, trainable=False, seed=0):
    from nksr_b200.network import NKSRNetwork
    return NKSRNetwork(dict(backbone="unet", tree_depth=depth, kernel_dim=4, udf=dict(enabled=udf),
                            structure=structure, structure_max_ratio=float("inf"), trainable=trainable,
                            seed=seed, geometry="neural")).to(cuda)


@pytest.mark.parametrize("structure", ["encoder", "predicted"])
@pytest.mark.parametrize("udf", [False, True])
def test_reconstructor_neural_geometry(cuda, monkeypatch, structure, udf):
    import nksr_b200
    from nksr_b200.dist_solve import reconstruct_global
    from nksr_b200.fields import KernelField, LayerField, NeuralField
    D, W = 4, 0.02
    xyz, nrm = clouds.sphere(20_000, noise=0.001)
    net = _net(cuda, D, structure, udf)
    rec = nksr_b200.Reconstructor(cuda, network=net, tree_depth=D, adaptive_depth=2)

    def no_solve(*a, **k):
        raise AssertionError("geometry='neural' ran a kernel solve")

    monkeypatch.setattr(KernelField, "solve", no_solve)
    monkeypatch.setattr(KernelField, "_pcg", no_solve)
    field = rec.reconstruct(_t(xyz, cuda), _t(nrm, cuda), voxel_size=W)
    assert isinstance(field, NeuralField) and field.position_gradient
    assert field.decoder is net.sdf_decoder and field.levels == list(range(D))
    assert rec.last_stats == dict(voxel_size=W, points=xyz.shape[0], geometry="neural")
    mf = field.mask_field
    if udf:
        assert isinstance(mf, NeuralField) and mf.decoder is net.udf_decoder and mf.level_set == 2 * W
        assert not mf.position_gradient
    else:
        assert isinstance(mf, LayerField) and mf.svh is field.svh and mf.adaptive_depth == 2
    q = _t(xyz[:2000], cuda)
    ev = field.evaluate_f(q, grad=True)
    assert ev.gradient.shape == (2000, 3) and bool(torch.isfinite(ev.gradient).all())
    assert torch.equal(field.evaluate_f_bar(q), torch.where(mf.mask(q), ev.value, -ev.value.abs()))
    # a random decoder need not cross 0 near the points: shift its last bias by the median value there
    with torch.no_grad():
        net.sdf_decoder[-1].bias -= ev.value.median()
    field.set_mask_field(None)
    full = field.extract_dual_mesh(mise_iter=1)
    field.set_mask_field(mf)
    mesh = field.extract_dual_mesh(mise_iter=1)
    assert full.f.shape[0] > 0 and bool(torch.isfinite(full.v).all())
    assert mesh.v.shape[1] == 3 and 0 <= mesh.f.shape[0] <= full.f.shape[0]
    print(f"[neural reconstruct] {structure} udf={udf}: T={full.f.shape[0]} unmasked, {mesh.f.shape[0]} masked")
    if structure == "encoder":
        with pytest.raises(NksrError, match="geometry='neural'"):
            rec.reconstruct(_t(xyz, cuda), _t(nrm, cuda), chunk_size=0.5)
        with pytest.raises(NksrError, match="geometry='neural'"):
            reconstruct_global(rec, _t(xyz, cuda), _t(nrm, cuda), W)


STEPS = 30


def _train(cuda, seed=3):
    from nksr_b200 import training as T
    xyz, nrm = clouds.sphere(30_000, noise=0.001)
    scene = T.TrainingScene(_t(xyz, cuda), _t(nrm, cuda), 0.02, 4)
    net = _net(cuda, 4, trainable=True, seed=seed)
    opt = T.make_optimizer(net)
    gen = torch.Generator(device=cuda).manual_seed(seed)
    curve, grads = [], None
    for step in range(STEPS):
        _, _, k = T.train_step(net, opt, scene, gen, kernel=True)
        curve.append({key: float(v) for key, v in k.items()})
        if step == 0:
            grads = {name: p.grad.detach().clone() for name, p in net.named_parameters() if p.grad is not None}
    return net, scene, curve, grads


def test_neural_training(cuda):
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        net, scene, curve, grads = _train(cuda)
        net2, _, curve2, grads2 = _train(cuda)
    finally:
        torch.use_deterministic_algorithms(False)
    C = net.kernel_dim
    for l in range(net.tree_depth):
        assert scene.enc_svh.num_voxels(l) > 0
        basis = grads[f"backbone_net.heads.{l}.weight"][6:6 + C]
        assert bool(torch.isfinite(basis).all()) and bool((basis.abs().sum(dim=1) > 0).all()), f"basis head {l}"
    # the neural field does not use the interpolators: they get no gradient from these losses
    assert not any(n.startswith("interpolators.") for n in grads)
    for name, p in net.sdf_decoder.named_parameters():
        g = grads[f"sdf_decoder.{name}"]
        assert bool(torch.isfinite(g).all()) and float(g.abs().sum()) > 0, name
    first = np.mean([c["total"] for c in curve[:3]])
    last = np.mean([c["total"] for c in curve[-3:]])
    print(f"[train neural] first {curve[0]} last {curve[-1]}; total mean of 3 {first:.5g} -> {last:.5g}")
    assert last < first
    assert curve == curve2
    assert all(torch.equal(a, b) for a, b in zip(net.state_dict().values(), net2.state_dict().values()))
    assert grads.keys() == grads2.keys() and all(torch.equal(grads[k], grads2[k]) for k in grads)
