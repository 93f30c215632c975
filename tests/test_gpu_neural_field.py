"""The neural field's interpolation (DESIGN.md SPEC S17, csrc/neural_field.cu) and its use as the UDF mask and loss.

Forward against an fp64 restatement built from the oracle (locate, _tent, centers), entry by entry within
kappa * 2^-24 * sum_s T_s |F_s| (tests/bounds.py's convention); exact zeros where the SPEC says 0; the VJP against fp64
T^T g and bitwise repeatable; NeuralField's gradients against torch autograd through decoder(_interp(x)); the
Reconstructor's UDF mask; the entries that refuse it; and training with udf.enabled.
"""
import numpy as np
import pytest
import torch

from nksr_b200._lib import NksrError
from oracle import nksr_oracle as O
from tests import clouds
from tests.bounds import U32, assert_within

pytestmark = pytest.mark.gpu

# kappa in units of 2^-24 (tests/bounds.py), each at most 8x the worst ratio measured on an NVIDIA H100 80GB HBM3
# (power limit 700 W) over this file.
# nksr_neural_interp against fp64: the fp32 local coordinate, three fp32 tent factors per corner and eight corners
# summed with fma.  Worst 6.15.
KAPPA_INTERP = 32.0
# NeuralField._interp against fp64: its local coordinate is an fp32 difference x / W_l - (ijk + 1/2), which cancels up
# to |x| / W_l units of rounding (up to 64 here) and moves that much weight onto neighbours the scale may not weigh.
# Worst 506 (depth 6, level 0).
KAPPA_INTERP_TORCH = 4000.0
# nksr_neural_interp_vjp against fp64 T^T g: an fp32 fma chain over the queries of 27 ranges.  Worst 8.94.
KAPPA_VJP = 64.0
# UDF loss over 30 training steps with udf.enabled (depth 3, 40 k sphere points), measured on the same GPU: 0.420 at
# step 1, 0.340 for the mean of the last three.
UDF_FIELD_LOSS_AFTER_30 = 0.37

np_ = lambda a: a.detach().double().cpu().numpy()


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


_HIER = {}


def _hierarchy(cuda, depth):
    """a sphere splatted at depth 3, 4 (W = 0.05) or 6 (W = 0.02), with the oracle's hierarchy of the same points"""
    if depth not in _HIER:
        from nksr_b200.svh import SparseFeatureHierarchy
        W = 0.05 if depth < 6 else 0.02
        xyz, _ = clouds.sphere(3000, noise=0.001)
        svh = SparseFeatureHierarchy(W, depth, cuda).build_point_splatting(_t(xyz, cuda))
        osvh = O.OracleSVH(W, depth).build_point_splatting(xyz)
        for l in range(depth):
            assert np.array_equal(svh.keys[l].cpu().numpy(), osvh.keys[l]), l
        _HIER[depth] = (svh, osvh, xyz)
    return _HIER[depth]


def _queries(xyz, n, seed):
    """the input points, points near them, and points uniform over a box larger than the cloud"""
    rng = np.random.default_rng(seed)
    near = xyz[rng.integers(0, xyz.shape[0], n)] + rng.normal(0.0, 0.03, (n, 3))
    box = rng.uniform(-1.4, 1.4, (n, 3))
    return np.concatenate([xyz[:n], near, box]).astype(np.float32)


def _weights64(osvh, l, q):
    """per query: the level-l neighbour rows (M, 27) and fp64 tent weights T_s (M, 27), 0 where absent"""
    base = osvh.locate(q)[l]
    nbr, tau = O._level_tau(osvh, l, q, base)
    tx, ty, tz = (O._tent(tau[:, a])[0] for a in range(3))
    w = O._prod3(tx, ty, tz)
    return nbr, np.where(nbr >= 0, w, 0.0)


def _interp64(osvh, feats, levels, q):
    """u(x) in fp64 and its error scale sum_s T_s |F_s|, (M, C |G|)"""
    cols, scale = [], []
    for l in levels:
        F = feats[l].astype(np.float64)
        if osvh.n(l) == 0:
            cols.append(np.zeros((q.shape[0], F.shape[1])))
            scale.append(np.zeros((q.shape[0], F.shape[1])))
            continue
        nbr, w = _weights64(osvh, l, q)
        g = F[np.where(nbr >= 0, nbr, 0)]                       # (M, 27, C)
        cols.append(np.einsum("ms,msc->mc", w, g))
        scale.append(np.einsum("ms,msc->mc", w, np.abs(g)))
    return np.concatenate(cols, 1), np.concatenate(scale, 1)


def _features(svh, C, seed, positive=False):
    g = torch.Generator().manual_seed(seed)
    out = {}
    for l in range(svh.depth):
        f = torch.rand((svh.num_voxels(l), C), generator=g) if positive else torch.randn((svh.num_voxels(l), C),
                                                                                         generator=g)
        out[l] = f.to(svh.device)
    return out


def _field(svh, feats, levels, decoder=None):
    import nksr_b200
    return nksr_b200.NeuralField(svh, decoder if decoder is not None else torch.nn.Identity(),
                                 {l: feats[l] for l in levels})


_GIVEN = {"0": lambda D: [0], "02": lambda D: [0, 2], "all": lambda D: list(range(D))}


@pytest.mark.parametrize("depth", [3, 4, 6])
@pytest.mark.parametrize("C", [1, 3, 4, 16, 32])
@pytest.mark.parametrize("given", sorted(_GIVEN))
def test_forward_against_fp64(cuda, depth, C, given):
    svh, osvh, xyz = _hierarchy(cuda, depth)
    levels = _GIVEN[given](depth)
    feats = _features(svh, C, seed=depth * 100 + C)
    nf = _field(svh, feats, levels)
    q = _queries(xyz, 700, seed=C)
    u = nf.interpolate(_t(q, cuda))
    assert u.shape == (q.shape[0], C * len(levels))
    ref, scale = _interp64(osvh, {l: f.cpu().numpy() for l, f in feats.items()}, levels, q)
    assert_within(np_(u), ref, scale, KAPPA_INTERP, f"interp depth {depth} C {C} G {levels}")
    ut = nf._interp(_t(q, cuda))
    assert_within(np_(ut), ref, scale, KAPPA_INTERP_TORCH, f"_interp depth {depth} C {C} G {levels}")


def test_exact_zeros_and_exact_weights(cuda):
    import nksr_b200
    from nksr_b200.svh import SparseFeatureHierarchy
    W, D, C = 2.0 ** -5, 4, 3                    # power-of-two voxel size: centres and faces are exact in fp32
    xyz, _ = clouds.sphere(3000, noise=0.001)
    svh = SparseFeatureHierarchy(W, D, cuda).build_point_splatting(_t(xyz, cuda))
    feats = _features(svh, C, seed=5, positive=True)
    nf = _field(svh, feats, list(range(D)))
    # outside every voxel; NaN, inf and out-of-range coordinates
    bad = torch.tensor([[5.0, 5.0, 5.0], [float("nan"), 0.0, 0.0], [0.0, float("inf"), 0.0],
                        [0.0, 0.0, -float("inf")], [1.0e7, 0.0, 0.0], [0.0, -3.0e5, 0.0]], device=cuda)
    assert torch.equal(nf.interpolate(bad), torch.zeros((bad.shape[0], C * D), device=cuda))
    assert torch.equal(nf._interp(bad), torch.zeros((bad.shape[0], C * D), device=cuda))
    # an absent fine voxel under a present coarse one: the fine columns are 0, the coarse ones are not
    rng = np.random.default_rng(1)
    cand = _t(rng.uniform(-1.1, 1.1, (200_000, 3)).astype(np.float32), cuda)
    base = svh.locate(cand)
    hole = cand[(base[0] < 0) & (base[1] >= 0)][:500]
    assert hole.shape[0] > 10
    u = nf.interpolate(hole)
    assert torch.equal(u[:, :C], torch.zeros_like(u[:, :C])) and (u[:, C:2 * C] > 0).all()
    # a voxel centre takes weight 1 on its own voxel; a point on the face x = centre + W/2 weight 1/2 on both sides
    for l in range(D):
        Wl = W * 2 ** l
        cen = svh.get_voxel_centers(l)
        got = nf.interpolate(cen)[:, l * C:(l + 1) * C]
        assert torch.equal(got, feats[l]), l
        face = cen + torch.tensor([Wl / 2, 0.0, 0.0], device=cuda)
        nb = svh.nbr27[l][:, 22].long()                          # slot of d = (+1, 0, 0)
        has = nb >= 0
        want = ((feats[l].double() + feats[l][nb.clamp(min=0)].double()) / 2).float()
        assert torch.equal(nf.interpolate(face)[:, l * C:(l + 1) * C][has], want[has]), l
    # a given level without voxels: C zero columns, in the kernel and in _interp
    keys = [None] + [svh.keys[l] for l in range(1, D)]
    keys[0] = torch.zeros(0, dtype=torch.int64, device=cuda)
    part = SparseFeatureHierarchy(W, D, cuda).build_from_keys(keys)
    assert part.num_voxels(0) == 0 and part.num_voxels(1) > 0
    pf = {0: torch.zeros((0, C), device=cuda), **{l: feats[l] for l in range(1, D)}}
    pn = nksr_b200.NeuralField(part, torch.nn.Identity(), pf)
    q = _t(xyz[:300], cuda)
    u, ut = pn.interpolate(q), pn._interp(q)
    assert u.shape == (300, C * D) and ut.shape == (300, C * D)
    assert torch.equal(u[:, :C], torch.zeros_like(u[:, :C])) and torch.equal(ut[:, :C], torch.zeros_like(ut[:, :C]))
    assert (u[:, C:] != 0).any()


@pytest.mark.parametrize("depth,C,given", [(3, 4, "all"), (4, 1, "02"), (4, 16, "all"), (6, 32, "0"), (6, 3, "all")])
def test_vjp_against_fp64_and_repeatable(cuda, depth, C, given):
    svh, osvh, xyz = _hierarchy(cuda, depth)
    levels = _GIVEN[given](depth)
    feats = _features(svh, C, seed=7)
    nf = _field(svh, feats, levels)
    q = _queries(xyz, 1500, seed=depth)
    q = np.concatenate([q, q[:200]])                           # repeated queries
    qt = _t(q, cuda)
    g = torch.randn((q.shape[0], C * len(levels)), generator=torch.Generator().manual_seed(3)).to(cuda)
    d1 = nf._interp_vjp(qt, g)
    d2 = nf._interp_vjp(qt, g)
    gn = g.cpu().double().numpy()
    for j, l in enumerate(levels):
        assert torch.equal(d1[l], d2[l]), l
        nbr, w = _weights64(osvh, l, q)
        ref = np.zeros((osvh.n(l), C))
        sc = np.zeros((osvh.n(l), C))
        gl = gn[:, j * C:(j + 1) * C]
        for s in range(27):
            ok = nbr[:, s] >= 0
            np.add.at(ref, nbr[ok, s], w[ok, s, None] * gl[ok])
            np.add.at(sc, nbr[ok, s], w[ok, s, None] * np.abs(gl[ok]))
        assert_within(np_(d1[l]), ref, sc, KAPPA_VJP, f"vjp depth {depth} C {C} level {l}")
    for l in range(depth):
        if l not in levels:
            assert d1[l] is None


def test_gradients_agree_with_torch_autograd(cuda):
    svh, _, xyz = _hierarchy(cuda, 4)
    C = 4
    torch.manual_seed(0)
    dec = torch.nn.Sequential(torch.nn.Linear(C * 4, 32), torch.nn.ReLU(), torch.nn.Linear(32, 1)).to(cuda)
    feats = {l: f.requires_grad_(True) for l, f in _features(svh, C, seed=9).items()}
    nf = _field(svh, feats, list(range(4)), dec)
    q = _t(_queries(xyz, 1000, seed=2), cuda)
    v = nf.evaluate_f(q, grad=True)
    assert v.gradient is None and v.value.grad_fn is not None
    (v.value ** 2).sum().backward()
    got = [feats[l].grad.clone() for l in range(4)] + [p.grad.clone() for p in dec.parameters()]
    for t_ in list(feats.values()) + list(dec.parameters()):
        t_.grad = None
    (dec(nf._interp(q)).reshape(-1) ** 2).sum().backward()
    want = [feats[l].grad for l in range(4)] + [p.grad for p in dec.parameters()]
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.shape == b.shape
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-4 * float(b.abs().max()) + 1e-12), i
    # no grad, or nothing that requires grad: no graph
    with torch.no_grad():
        assert nf.evaluate_f(q).value.grad_fn is None
    frozen = _field(svh, {l: f.detach() for l, f in feats.items()}, list(range(4)),
                    dec.requires_grad_(False))
    assert frozen.evaluate_f(q).value.grad_fn is None
    dec.requires_grad_(True)
    # features frozen, decoder trainable: the graph reaches the decoder only
    only_dec = _field(svh, {l: f.detach() for l, f in feats.items()}, list(range(4)), dec)
    assert only_dec.evaluate_f(q).value.grad_fn is not None


def _udf_net(cuda, depth, structure="encoder", trainable=False, seed=0):
    from nksr_b200.network import NKSRNetwork
    return NKSRNetwork(dict(backbone="unet", tree_depth=depth, kernel_dim=4, udf=dict(enabled=True),
                            structure=structure, structure_max_ratio=float("inf"), trainable=trainable,
                            seed=seed)).to(cuda)


def _decoder_bound(dec, feats, levels):
    """|decoder(u1) - decoder(u2)| for two u within (KAPPA_INTERP + KAPPA_INTERP_TORCH) u sum T |F| of fp64: the
    product of the layers' spectral norms times the 2-norm of the per-column bound, max |F| per column"""
    lip = 1.0
    for m in dec:
        if isinstance(m, torch.nn.Linear):
            lip *= float(torch.linalg.matrix_norm(m.weight.detach().double(), ord=2))
    col = torch.cat([feats[l].detach().abs().amax(dim=0) if feats[l].shape[0] else
                     torch.zeros(feats[l].shape[1], device=feats[l].device) for l in levels]).double()
    return lip * (KAPPA_INTERP + KAPPA_INTERP_TORCH) * U32 * float(col.norm())


def test_reconstructor_udf_mask(cuda):
    import nksr_b200
    from nksr_b200.fields import LayerField, NeuralField
    from nksr_b200.reconstructor import mask_field
    D, W = 4, 0.02
    xyz, nrm = clouds.sphere(20_000, noise=0.001)
    net = _udf_net(cuda, D)
    rec = nksr_b200.Reconstructor(cuda, network=net, tree_depth=D, adaptive_depth=2)
    field = rec.reconstruct(_t(xyz, cuda), _t(nrm, cuda), voxel_size=W, solver_tol=1e-4)
    mf = field.mask_field
    assert isinstance(mf, NeuralField) and mf.svh is field.svh and mf.level_set == 2 * W
    assert mf.levels == list(range(D)) and mf.decoder is net.udf_decoder
    field.set_mask_field(None)
    full = field.extract_dual_mesh(mise_iter=1)
    field.set_mask_field(mf)
    with torch.no_grad():
        f_ref = net.udf_decoder(mf._interp(full.v)).reshape(-1)
        f_ker = mf.evaluate_f(full.v).value
    margin = _decoder_bound(net.udf_decoder, mf.features, mf.levels) + 64 * U32 * float(f_ref.abs().max())
    assert float((f_ker - f_ref).abs().max()) <= margin
    # the level set of the reconstruction, and the median value (a random decoder may keep all or nothing at 2W)
    for ls in (2 * W, float(f_ref.median())):
        mf.set_level_set(ls)
        masked = field.extract_dual_mesh(mise_iter=1)
        keep_ref = (f_ref <= ls)[full.f].all(dim=1)
        keep_ker = (f_ker <= ls)[full.f].all(dim=1)
        far = ((f_ref - ls).abs() > margin)[full.f].all(dim=1)
        print(f"[udf mask] level set {ls:.4g}: faces {full.f.shape[0]}, kept {int(keep_ker.sum())}, near the level "
              f"set {int((~far).sum())}, margin {margin:.3g}")
        assert torch.equal(keep_ref[far], keep_ker[far])
        # the masked mesh is the unmasked one with exactly the kernel's faces kept
        used = torch.zeros(full.v.shape[0], dtype=torch.bool, device=cuda)
        used[full.f[keep_ker].reshape(-1)] = True
        idx = torch.nonzero(used).reshape(-1)
        assert torch.equal(masked.v, full.v[used]) and torch.equal(idx[masked.f], full.f[keep_ker])
    # the compared faces are most of the mesh (88 % at the median level set on the H100), and both sides occur
    assert far.float().mean() > 0.75 and 0 < int(keep_ker.sum()) < full.f.shape[0]
    # structure='predicted', teacher-forced: the helper puts the NeuralField on the grown hierarchy
    from nksr_b200.training import TrainingScene
    sc = TrainingScene(_t(xyz, cuda), _t(nrm, cuda), W, D)
    pnet = _udf_net(cuda, D, "predicted")
    with torch.no_grad():
        enc = pnet.encoder(sc.xyz, sc.normal, sc.enc_svh, 0)
        feats, dec_svh, udf_svh = pnet.unet(enc, sc.enc_svh, adaptive_depth=2, gt_decoder_svh=sc.gt_svh)
        pm = mask_field(pnet, feats, dec_svh, udf_svh, 2, W)
        assert isinstance(pm, NeuralField) and pm.svh is udf_svh and pm.level_set == 2 * W
        assert pm.levels == list(range(D))
        q = full.v[:5000]
        a, b = pm.evaluate_f(q).value, pnet.udf_decoder(pm._interp(q)).reshape(-1)
        assert float((a - b).abs().max()) <= _decoder_bound(pnet.udf_decoder, pm.features, pm.levels) + \
            64 * U32 * float(b.abs().max())
    # UDF disabled: LayerField, as before
    plain = nksr_b200.Reconstructor(cuda, tree_depth=D, adaptive_depth=2)
    f2 = plain.reconstruct(_t(xyz, cuda), _t(nrm, cuda), voxel_size=W)
    assert isinstance(f2.mask_field, LayerField)


def test_entries_that_refuse_udf(cuda):
    import nksr_b200
    from nksr_b200.dist_solve import reconstruct_global
    xyz, nrm = clouds.sphere(5_000, noise=0.001)
    rec = nksr_b200.Reconstructor(cuda, network=_udf_net(cuda, 3), tree_depth=3)
    with pytest.raises(NksrError, match="chunk mode does not support udf.enabled"):
        rec.reconstruct(_t(xyz, cuda), _t(nrm, cuda), chunk_size=0.5)
    with pytest.raises(NksrError, match="chunk mode does not support udf.enabled"):
        rec._reconstruct_chunks(_t(xyz, cuda), _t(nrm, cuda), None, 0.02, 0.5, None, False, 1e-5, True, 2000)
    with pytest.raises(NksrError, match="global solve does not support udf.enabled"):
        reconstruct_global(rec, _t(xyz, cuda), _t(nrm, cuda), 0.02)


def _train(cuda, steps, seed=0, depth=3):
    from nksr_b200 import training as T
    sc = _scene(cuda, depth)
    net = _udf_net(cuda, depth, trainable=True, seed=seed)
    opt = T.make_optimizer(net)
    gen = torch.Generator(device=cuda).manual_seed(seed)
    curve = [tuple(float(v) for v in T.train_step(net, opt, sc, gen)) for _ in range(steps)]
    return net, curve


def _scene(cuda, depth):
    from nksr_b200.training import TrainingScene
    xyz, nrm = clouds.sphere(40_000, noise=0.001)
    return TrainingScene(_t(xyz, cuda), _t(nrm, cuda), 0.02, depth)


def test_training_with_udf(cuda):
    from nksr_b200 import training as T
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        # step 1: the UDF loss reaches the UDF features of every level
        sc = _scene(cuda, 3)
        net = _udf_net(cuda, 3, trainable=True)
        enc = net.encoder(sc.xyz, sc.normal, sc.enc_svh, 0)
        feat, _, udf_svh = net.unet(enc, sc.enc_svh, adaptive_depth=sc.adaptive_depth)
        for f in feat.udf_features.values():
            f.retain_grad()
        l_udf = T.udf_field_loss(net.udf_decoder, feat.udf_features, udf_svh, sc.xyz, sc.normal, sc.voxel_size,
                                 generator=torch.Generator(device=cuda).manual_seed(0))
        l_udf.backward()
        for l in range(3):
            gl = feat.udf_features[l].grad
            assert gl is not None and bool((gl != 0).any()), l
        assert net.udf_decoder[0].weight.grad is not None
        # 30 steps, twice: bitwise the same curve and parameters; the UDF loss falls
        net1, c1 = _train(cuda, 30)
        net2, c2 = _train(cuda, 30)
        print("[train udf] udf", [round(c[1], 4) for c in c1])
        assert all(np.isfinite(c).all() for c in c1)
        assert c1 == c2
        for (n, a), b in zip(net1.named_parameters(), net2.parameters()):
            assert torch.equal(a, b), f"{n}: two runs from one seed differ"
        last = sum(c[1] for c in c1[-3:]) / 3
        assert last < UDF_FIELD_LOSS_AFTER_30, (c1[0][1], last)
    finally:
        torch.use_deterministic_algorithms(False)
