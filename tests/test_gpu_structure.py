"""The structure-grown decoder hierarchy (DESIGN.md SPEC S16): the growth kernels of csrc/structure.cu against the torch
restatement (nksr_b200/structure.py, impl='torch') bit for bit, teacher forcing against the ground-truth hierarchy, the
U-Net decoder on the grown hierarchy against impl='torch' (forward and gradients), per-part gather tables, the
Reconstructor and training with structure='predicted', and the entries that refuse it."""
import numpy as np
import pytest
import torch

from nksr_b200._lib import NksrError
from tests import clouds, scenes

pytestmark = pytest.mark.gpu

_TABLES = ("keys", "parent", "child8", "nbr27")


def _t(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def _crop_svh(cuda, depth, n=20_000, voxel_size=0.1):
    from nksr_b200.svh import SparseFeatureHierarchy
    xyz, _ = scenes.crop("cfg4_outdoor", n)
    return SparseFeatureHierarchy(voxel_size, depth, cuda).build_point_splatting(_t(xyz, cuda))


def _sphere_svh(cuda, depth, n=20_000, voxel_size=0.02):
    from nksr_b200.svh import SparseFeatureHierarchy
    xyz, _ = clouds.sphere(n, noise=0.001)
    return SparseFeatureHierarchy(voxel_size, depth, cuda).build_point_splatting(_t(xyz, cuda))


def _single_svh(cuda, depth):
    """one voxel per level: a chain down from a single coarsest voxel"""
    from nksr_b200.structure import morton_encode
    from nksr_b200.svh import SparseFeatureHierarchy
    c = 1 << 19
    key = morton_encode(torch.tensor([c + 5]), torch.tensor([c + 9]), torch.tensor([c + 2]))
    keys = [(key >> (3 * l)).to(cuda) for l in range(depth)]
    return SparseFeatureHierarchy(0.1, depth, cuda).build_from_keys(keys)


def _logits(mode, l, n, seed, dev):
    g = torch.Generator().manual_seed(seed * 100 + l)
    x = torch.randn((n, 3), generator=g)
    if mode == "random":
        x = x + torch.tensor([-0.4, 0.2, 0.5])
    elif mode == "empty":
        x = x.abs() * torch.tensor([1.0, -1.0, -1.0])
    elif mode == "subdivide":
        x = x.abs() * torch.tensor([-1.0, -1.0, 1.0])
    elif mode == "leaf":                       # class 1 everywhere: subdivided at l >= a, a leaf below
        x = x.abs() * torch.tensor([-1.0, 1.0, -1.0]) + torch.tensor([0.0, 0.1, 0.0])
    elif mode == "ties":                       # exact ties between every pair, and some strict rows
        r = torch.randint(0, 4, (n,), generator=g)
        v = torch.round(x * 2) / 2
        x = torch.where((r == 0)[:, None], v[:, :1].expand(n, 3), v)
        x[r == 1, 2] = x[r == 1, 1]
        x[r == 2, 1] = x[r == 2, 0]
    elif mode == "nan":
        r = torch.randint(0, 5, (n,), generator=g)
        x[r == 0, 0] = float("nan")
        x[r == 1, 1] = float("nan")
        x[r == 2, 2] = float("nan")
        x[r == 3] = float("nan")
        x = x + torch.tensor([-0.4, 0.2, 0.5])
    return x.to(dev)


def _grow_pair(E, D, a, mode, seed, strided=True):
    """the CUDA and the torch growth fed the same logits, compared after every step"""
    from nksr_b200.structure import StructureGrowth
    gc = StructureGrowth(E, D, a, max_ratio=None, impl="cuda")
    gt = StructureGrowth(E, D, a, max_ratio=None, impl="torch")
    for l in range(D - 1, -1, -1):
        n = gc.T.num_voxels(l)
        assert gt.T.num_voxels(l) == n
        x = _logits(mode, l, n, seed, E.device)
        if strided:                            # a head-output slice: row stride 3 + 2 * 4 + 3
            wide = torch.zeros((n, 14), device=E.device)
            wide[:, :3] = x
            xc = wide[:, :3]
        else:
            xc = x
        gc.step(l, logits=xc)
        gt.step(l, logits=x)
        assert torch.equal(gc.classes[l].cpu(), gt.classes[l].cpu()), (mode, l)
        assert torch.equal(gc.kept[l].cpu(), gt.kept[l].cpu()), (mode, l)
        if l >= 1:
            for name in _TABLES:
                a_, b_ = getattr(gc.T, name), getattr(gt.T, name)
                i = l if name == "child8" else l - 1
                assert torch.equal(a_[i].cpu(), b_[i].cpu()), (mode, name, l)
            assert torch.equal(gc.join[l - 1].cpu(), gt.join[l - 1].cpu()), (mode, l)
    for l in range(D):
        assert torch.equal(gc.skip27(l).cpu(), gt.skip27(l).cpu()), (mode, l)
    return gc, gt


def _check_closed_sorted(g, D):
    T = g.T
    for l in range(D):
        k = T.keys[l]
        assert bool((k[1:] > k[:-1]).all())
        if l < D - 1 and k.numel():
            assert torch.equal(k >> 3, T.keys[l + 1][T.parent[l].long()])


@pytest.mark.parametrize("D,a", [(3, 1), (4, 2), (5, 3)])
@pytest.mark.parametrize("mode", ["random", "empty", "subdivide", "leaf", "ties", "nan"])
def test_growth_kernels_match_torch_bitwise(cuda, D, a, mode):
    E = _crop_svh(cuda, D, n=8_000 if mode == "subdivide" else 20_000)
    gc, _ = _grow_pair(E, D, a, mode, seed=D)
    _check_closed_sorted(gc, D)
    if mode == "empty":
        assert all(gc.T.num_voxels(l) == 0 for l in range(D - 1))
    if mode == "subdivide":
        assert gc.T.num_voxels(0) == E.num_voxels(D - 1) * 8 ** (D - 1)
    if mode == "leaf":                         # leaves below a stop the growth, above it they subdivide
        for l in range(D - 1):
            assert gc.T.num_voxels(l) == (8 * gc.T.num_voxels(l + 1) if l + 1 >= a else 0)
    # a second run stores identical arrays
    again, _ = _grow_pair(E, D, a, mode, seed=D)
    for name in _TABLES:
        for x, y in zip(getattr(gc.T, name), getattr(again.T, name)):
            assert (x is None and y is None) or torch.equal(x, y)


@pytest.mark.parametrize("D,a", [(4, 2), (5, 1)])
def test_growth_kernels_on_sphere_and_a_single_voxel(cuda, D, a):
    for E in (_sphere_svh(cuda, D), _single_svh(cuda, D)):
        for mode in ("random", "subdivide", "leaf"):
            gc, _ = _grow_pair(E, D, a, mode, seed=7, strided=False)
            _check_closed_sorted(gc, D)
    assert _single_svh(cuda, D).num_voxels(D - 1) == 1


def _scene(cuda, n=60_000, depth=4):
    """a sphere whose normals are randomly flipped on one side: the ground-truth hierarchy subdivides there (mixed
    normals) and stops at leaves elsewhere, so every structure class occurs"""
    from nksr_b200.training import TrainingScene
    xyz, nrm = clouds.sphere(n, noise=0.001)
    sign = np.where((xyz[:, 0] > 0) & (np.random.default_rng(0).random(n) < 0.5), -1.0, 1.0).astype(np.float32)
    return TrainingScene(_t(xyz, cuda), _t(nrm * sign[:, None], cuda), 0.02, depth)


def _assert_same_hierarchy(a, b):
    assert a.depth == b.depth
    for l in range(a.depth):
        assert torch.equal(a.keys[l], b.keys[l]), l
        assert torch.equal(a.parent[l], b.parent[l]), l
        assert torch.equal(a.nbr27[l], b.nbr27[l]), l
    for l in range(1, a.depth + 1):
        assert torch.equal(a.child8[l], b.child8[l]), l
    assert torch.equal(a.top_keys, b.top_keys) and torch.equal(a.nbr27[a.depth], b.nbr27[b.depth])


def test_teacher_forcing_reproduces_the_ground_truth(cuda):
    from nksr_b200.structure import grow_from_classes, teacher_classes
    from nksr_b200.svh import SparseFeatureHierarchy
    sc = _scene(cuda)
    D, G, E = 4, sc.gt_svh, sc.enc_svh
    for impl in ("cuda", "torch"):
        dec, g = grow_from_classes(E, [teacher_classes(G)] * D, sc.adaptive_depth, impl=impl)
        _assert_same_hierarchy(dec, G)
        assert dec.adaptive_depth == sc.adaptive_depth
    dec2 = SparseFeatureHierarchy(E.voxel_size, D, cuda).build_from_structure(E, [teacher_classes(G)] * D,
                                                                              sc.adaptive_depth)
    _assert_same_hierarchy(dec2, G)
    # G's coarsest level beyond E's: E from the points of one half of the sphere only
    half = sc.xyz[:, 0] > 0.1
    E2 = SparseFeatureHierarchy(E.voxel_size, D, cuda).build_point_splatting(sc.xyz[half].contiguous())
    dec, _ = grow_from_classes(E2, [teacher_classes(G)] * D, sc.adaptive_depth)
    top = E2.keys[D - 1]
    want = [G.keys[l][torch.isin(G.keys[l] >> (3 * (D - 1 - l)), top)] for l in range(D)]
    assert G.num_voxels(0) > 0 and sum(w.numel() for w in want) < G.num_unknowns
    ref = SparseFeatureHierarchy(E.voxel_size, D, cuda).build_from_keys(want, top_keys=E2.top_keys)
    _assert_same_hierarchy(dec, ref)


def _close(a, b, rel):
    scale = float(b.abs().max().item()) + 1e-30
    return float((a - b).abs().max().item()) <= rel * scale


def test_grown_backbone_matches_torch_reference(cuda):
    """forward of the whole backbone on a grown hierarchy against impl='torch': teacher-forced, and replaying the classes
    the CUDA run chose from its own logits (never two independent argmaxes); then TF32 and tc against fp32"""
    from nksr_b200.network import NKSRNetwork
    from nksr_b200.structure import teacher_classes
    sc = _scene(cuda, n=30_000, depth=3)
    net = NKSRNetwork(dict(backbone="unet", tree_depth=3, kernel_dim=4)).to(cuda)
    bb = net.backbone_net
    with torch.no_grad():
        enc = net.encoder(sc.xyz, sc.normal, sc.enc_svh, 0)
        x0 = enc.x0
        own = bb(x0, sc.enc_svh, grow=dict(adaptive_depth=2, max_ratio=float("inf")))
        replay = lambda T, l: own.classes[l]
        for forced, out in ((teacher_classes(sc.gt_svh), None), (replay, own)):
            if out is None:
                out = bb(x0, sc.enc_svh, grow=dict(adaptive_depth=2, forced=forced))
            ref = bb(x0, sc.enc_svh, impl="torch", grow=dict(adaptive_depth=2, forced=forced, max_ratio=float("inf")))
            fast = bb(x0, sc.enc_svh, tf32=True, grow=dict(adaptive_depth=2, forced=forced, max_ratio=float("inf")))
            tc = bb(x0, sc.enc_svh, tf32=3, grow=dict(adaptive_depth=2, forced=forced, max_ratio=float("inf")))
            for l in range(3):
                assert torch.equal(out.udf_svh.keys[l], ref.udf_svh.keys[l])
                assert torch.equal(out.dec_svh.keys[l], ref.dec_svh.keys[l])
                for name in ("structure", "normal", "basis", "udf", "decoder"):
                    a, b = getattr(out, name)[l], getattr(ref, name)[l]
                    assert a.shape == b.shape and torch.isfinite(a).all()
                    if b.numel() == 0:
                        continue
                    assert _close(a, b, 1e-4), (name, l, float((a - b).abs().max()), float(b.abs().max()))
                    assert _close(getattr(fast, name)[l], b, 2e-2), (name, l)
                    assert _close(getattr(tc, name)[l], b, 2e-2), (name, l)
        # through the network: features on dec_svh are the kept rows of those on udf_svh, bitwise
        net.structure = "predicted"
        feats, dec_svh, udf_svh = net.unet(enc, sc.enc_svh, adaptive_depth=2, gt_decoder_svh=sc.gt_svh)
    _assert_same_hierarchy(dec_svh, sc.gt_svh)
    teach = bb(x0, sc.enc_svh, grow=dict(adaptive_depth=2, forced=teacher_classes(sc.gt_svh)))
    for l in range(3):
        kept = teach.kept[l]
        assert torch.equal(feats.basis_features[l], teach.basis[l][kept])
        assert torch.equal(feats.normal_features[l], teach.normal[l][kept])
        assert torch.equal(feats.structure_features[l], teach.structure[l])
        assert torch.equal(feats.udf_features[l], teach.udf[l])
        assert feats.basis_features[l].shape[0] == dec_svh.num_voxels(l)
        assert feats.udf_features[l].shape[0] == udf_svh.num_voxels(l)


def _rel(a, b):
    return float((a - b).abs().max()) / (float(b.abs().max()) + 1e-30)


def test_grown_backbone_gradients_match_torch_autograd(cuda):
    """a random cotangent on every head of the grown decoder: every parameter's gradient and x0's (which reaches the
    skip inputs through the transposed skip27) against torch autograd of impl='torch'; two passes give the same bits"""
    from nksr_b200.structure import teacher_classes
    from nksr_b200.unet import SparseUNet
    sc = _scene(cuda, n=30_000, depth=3)
    torch.manual_seed(1)
    net = SparseUNet(3, 32, 4).to(cuda)
    g_ = torch.Generator(device="cpu").manual_seed(22)
    x0 = torch.randn((sc.enc_svh.num_voxels(0), 32), generator=g_).to(cuda).requires_grad_(True)
    grow = dict(adaptive_depth=2, forced=teacher_classes(sc.gt_svh))
    with torch.no_grad():
        plain = net(x0, sc.enc_svh, grow=grow)
    cot = {(name, l): torch.randn(getattr(plain, name)[l].shape, generator=g_).to(cuda)
           for name in ("structure", "normal", "basis", "udf") for l in range(3)}

    def grads(**kw):
        net.zero_grad(set_to_none=True)
        x0.grad = None
        out = net(x0, sc.enc_svh, grow=grow, **kw)
        loss = sum((getattr(out, name)[l] * cot[(name, l)]).sum() for (name, l) in cot)
        loss.backward()
        return out, [x0.grad.clone()] + [p.grad.clone() if p.grad is not None else torch.zeros_like(p)
                                          for p in net.parameters()]

    _, ref = grads(impl="torch")
    out, got = grads()
    _, again = grads()
    for l in range(3):
        assert torch.equal(out.decoder[l], plain.decoder[l])
    names = ["x0"] + [n for n, _ in net.named_parameters()]
    for name, a, b, c in zip(names, got, ref, again):
        assert torch.equal(a, c), f"{name}: two backward passes differ"
        assert _rel(a, b) <= 1e-5, (name, _rel(a, b))


def test_per_part_tables(cuda):
    """a 2-part convolution with a different table per part against the dense torch path (forward and input /
    weight gradients); with the same table tensor twice it is bitwise the single-table call"""
    from nksr_b200.unet import SparseConv
    E = _crop_svh(cuda, 2)
    nbr = E.nbr27[0]
    n = nbr.shape[0]
    g = torch.Generator(device="cpu").manual_seed(4)
    n2 = n + 333
    remap = torch.randperm(n2, generator=g)[:n].to(torch.int32).to(cuda)
    idx2 = torch.where(nbr >= 0, remap[nbr.long().clamp(min=0)], torch.full_like(nbr, -1))
    torch.manual_seed(3)
    conv = SparseConv(27, 64, 32).to(cuda)
    a = torch.randn((n, 32), generator=g).to(cuda).requires_grad_(True)
    b = torch.randn((n2, 32), generator=g).to(cuda).requires_grad_(True)
    cot = torch.randn((n, 32), generator=g).to(cuda)

    def run(**kw):
        conv.zero_grad(set_to_none=True)
        a.grad = b.grad = None
        y = conv((a, b), (nbr, idx2), **kw)
        (y * cot).sum().backward()
        return y.detach(), a.grad.clone(), b.grad.clone(), conv.weight.grad.clone(), conv.bias.grad.clone()

    got, ref = run(), run(impl="torch")
    for x, y in zip(got, ref):
        assert _rel(x, y) <= 1e-5
    # the same table twice == the single-table call, forward and backward, bit for bit
    b1 = torch.randn((n, 32), generator=g).to(cuda).requires_grad_(True)
    outs = []
    for idx in (nbr, (nbr, nbr)):
        conv.zero_grad(set_to_none=True)
        a.grad = b1.grad = None
        y = conv((a, b1), idx)
        (y * cot).sum().backward()
        outs.append((y.detach(), a.grad.clone(), b1.grad.clone(), conv.weight.grad.clone()))
        with torch.no_grad():
            outs[-1] += (conv((a, b1), idx),)
    for x, y in zip(*outs):
        assert torch.equal(x, y)


def _forced_net(cuda, depth, top_class, inner_class, fine_class, ratio=float("inf")):
    """a U-Net network whose structure head says `top_class` on the coarsest level, `inner_class` on the levels
    between, `fine_class` on level 0 (zero weights, the class in the bias)"""
    from nksr_b200.network import NKSRNetwork
    net = NKSRNetwork(dict(backbone="unet", tree_depth=depth, kernel_dim=4, structure="predicted",
                           structure_max_ratio=ratio))
    with torch.no_grad():
        for l, head in enumerate(net.backbone_net.heads):
            c = top_class if l == depth - 1 else (fine_class if l == 0 else inner_class)
            head.weight[:3] = 0.0
            head.bias[:3] = torch.nn.functional.one_hot(torch.tensor(c), 3).float()
    return net


def test_reconstructor_on_the_predicted_structure(cuda):
    import nksr_b200
    from nksr_b200.meshing import extract_dual_mesh
    from nksr_b200.svh import SparseFeatureHierarchy
    xyz, nrm = clouds.sphere(30_000, noise=0.001)
    D, W = 4, 0.02
    rec = nksr_b200.Reconstructor(cuda, network=_forced_net(cuda, D, 2, 2, 1), tree_depth=D, adaptive_depth=2)
    field = rec.reconstruct(_t(xyz, cuda), _t(nrm, cuda), voxel_size=W, solver_tol=1e-4, solver_max_iter=2000)
    dec = field.svh
    E = SparseFeatureHierarchy(W, D, cuda).build_point_splatting(_t(xyz, cuda))
    o = torch.arange(8, device=cuda)
    want = [E.keys[D - 1]]
    for _ in range(D - 1):
        want.insert(0, ((want[0][:, None] << 3) | o).reshape(-1))
    for l in range(D):                                   # the full 8-child closure of E's coarsest level
        assert torch.equal(dec.keys[l], want[l]), l
    assert dec.adaptive_depth == 2
    assert torch.isfinite(field.alpha).all() and field.solve_info["converged"], field.solve_info
    mesh = extract_dual_mesh(field)
    assert mesh.v.shape[1] == 3 and torch.isfinite(mesh.v).all()
    # explicit classes with empty coarse voxels: the closure of the others
    keep_top = torch.arange(E.num_voxels(D - 1), device=cuda) % 3 != 0
    cls = [None] * D
    cls[D - 1] = torch.where(keep_top, 2, 0)
    for l in range(1, D - 1):
        cls[l] = lambda T, l: torch.full((T.num_voxels(l),), 2, device=cuda)
    cls[0] = lambda T, l: torch.ones(T.num_voxels(0), dtype=torch.long, device=cuda)
    part = SparseFeatureHierarchy(W, D, cuda).build_from_structure(E, cls, 2)
    top = E.keys[D - 1][keep_top]
    for l in range(D):
        assert torch.equal(part.keys[l], want[l][torch.isin(want[l] >> (3 * (D - 1 - l)), top)])
    # nothing kept: the reconstruction refuses
    rec0 = nksr_b200.Reconstructor(cuda, network=_forced_net(cuda, D, 0, 2, 1), tree_depth=D)
    with pytest.raises(NksrError, match="predicted structure is empty"):
        rec0.reconstruct(_t(xyz, cuda), _t(nrm, cuda), voxel_size=W)
    # the size guard refuses the first grown level, before anything of it is allocated
    rec1 = nksr_b200.Reconstructor(cuda, network=_forced_net(cuda, D, 2, 2, 1, ratio=1.0), tree_depth=D)
    with pytest.raises(NksrError, match=f"structure: level {D - 2} would hold {want[D - 2].numel()} voxels"):
        rec1.reconstruct(_t(xyz, cuda), _t(nrm, cuda), voxel_size=W)


def _train(cuda, steps, pd, seed=0, depth=3):
    from nksr_b200 import training as T
    from nksr_b200.network import NKSRNetwork
    sc = _scene(cuda, n=40_000, depth=depth)
    net = NKSRNetwork(dict(backbone="unet", tree_depth=depth, kernel_dim=4, trainable=True, seed=seed,
                           structure="predicted", structure_max_ratio=float("inf"))).to(cuda)
    opt = T.make_optimizer(net)
    gen = torch.Generator(device=cuda).manual_seed(seed)
    curve = [tuple(float(v) for v in T.train_step(net, opt, sc, gen, pd_structure_prob=pd)) for _ in range(steps)]
    return net, curve


def test_training_on_the_predicted_structure(cuda):
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        for pd in (0.0, 1.0):
            net, curve = _train(cuda, 8, pd)
            net2, curve2 = _train(cuda, 8, pd)
            print(f"[train predicted pd={pd}] structure", [round(c[0], 4) for c in curve])
            assert all(np.isfinite(c).all() for c in curve)
            assert curve == curve2
            for (n, a), b in zip(net.named_parameters(), net2.parameters()):
                assert torch.equal(a, b), f"{n}: two runs from one seed differ"
            if pd == 0.0:
                assert sum(c[0] for c in curve[-2:]) / 2 < curve[0][0], curve
    finally:
        torch.use_deterministic_algorithms(False)


def test_entries_that_refuse_the_predicted_structure(cuda):
    import nksr_b200
    from nksr_b200.dist_solve import reconstruct_global
    xyz, nrm = clouds.sphere(5_000, noise=0.001)
    rec = nksr_b200.Reconstructor(cuda, network=_forced_net(cuda, 3, 2, 2, 1), tree_depth=3)
    with pytest.raises(NksrError, match="chunk mode"):
        rec.reconstruct(_t(xyz, cuda), _t(nrm, cuda), chunk_size=0.5)
    with pytest.raises(NksrError, match="global solve"):
        reconstruct_global(rec, _t(xyz, cuda), _t(nrm, cuda), 0.02)
