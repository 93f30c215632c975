"""Host logic of the U-Net backbone (nksr_b200/unet.py) that needs no GPU: the torch reference convolution against
explicit loops, the octant table, the key-matched restriction, the parameter layout."""
from types import SimpleNamespace

import numpy as np
import torch

from nksr_b200.unet import SparseUNet, gather_gemm, octant_of_children, restrict_to


def test_torch_gather_gemm_is_the_definition():
    g = torch.Generator().manual_seed(0)
    n_in, n_out, K, ci, co = 11, 9, 5, 4, 3
    x = torch.randn((n_in, ci), generator=g)
    w = torch.randn((K, ci, co), generator=g)
    b = torch.randn(co, generator=g)
    res = torch.randn((n_out, co), generator=g)
    idx = torch.randint(-1, n_in, (n_out, K), generator=g, dtype=torch.int32)
    ref = np.zeros((n_out, co))
    for i in range(n_out):
        acc = b.numpy().astype(np.float64) + res[i].numpy()
        for k in range(K):
            j = int(idx[i, k])
            if j >= 0:
                acc = acc + x[j].numpy().astype(np.float64) @ w[k].numpy().astype(np.float64)
        ref[i] = np.maximum(acc, 0.0)
    out = gather_gemm(x, idx, w, b, res, relu=True, impl="torch")
    assert np.allclose(out.numpy(), ref, atol=1e-5)


def test_octants_and_restriction():
    child8 = torch.tensor([[0, -1, 2, -1, -1, -1, -1, 1], [-1, 3, -1, -1, 4, -1, -1, -1]], dtype=torch.int32)
    assert octant_of_children(child8, 6).tolist() == [0, 7, 2, 1, 4, -1]
    src = SimpleNamespace(keys=[torch.tensor([2, 5, 9, 11])])
    dst = SimpleNamespace(keys=[torch.tensor([5, 6, 11, 40])])
    f = {0: torch.arange(8.0).reshape(4, 2)}
    out = restrict_to(f, src, dst)[0]
    assert out.tolist() == [[2.0, 3.0], [0.0, 0.0], [6.0, 7.0], [0.0, 0.0]]
    assert restrict_to(f, src, src) is f


def test_unet_parameter_layout_follows_the_hparams():
    """configs/default/train.yaml:9-18: kernel_dim 4, tree_depth 4, unet.f_maps 32"""
    from nksr_b200.network import NKSRNetwork
    net = NKSRNetwork(dict(backbone="unet", tree_depth=4, kernel_dim=4, unet=dict(f_maps=32)))
    u = net.backbone_net
    assert isinstance(u, SparseUNet) and u.channels == [32, 64, 128, 256]
    assert tuple(u.enc_a[0].weight.shape) == (27, 32, 32) and tuple(u.down[0].weight.shape) == (8, 32, 64)
    assert tuple(u.dec[1].weight.shape) == (27, 128, 64) and u.heads[2].out_features == 6 + 2 * 4
    # seeded: two instances carry the same weights; the stand-in's parameters do not depend on the backbone
    net2 = NKSRNetwork(dict(backbone="unet", tree_depth=4, kernel_dim=4))
    assert all(torch.equal(a, b) for a, b in zip(net.state_dict().values(), net2.state_dict().values()))
    pool = NKSRNetwork(dict(tree_depth=4, kernel_dim=4))
    for k, v in pool.state_dict().items():
        assert torch.equal(v, net.state_dict()[k])
    net2.load_state_dict(net.state_dict())


def _toy_hierarchy(depth=3, seed=0):
    """a random parent-closed voxel hierarchy with the tables the U-Net reads (nbr27, child8, parent), built on the CPU
    by brute force: level l voxels = unique (ijk >> l) of random finest voxels"""
    rng = np.random.default_rng(seed)
    ijk0 = np.unique(rng.integers(0, 12, (140, 3)), axis=0)
    levels = [np.unique(ijk0 >> l, axis=0) for l in range(depth)]
    look = [{tuple(v): i for i, v in enumerate(lv)} for lv in levels]
    offs = [(a, b, c) for a in (-1, 0, 1) for b in (-1, 0, 1) for c in (-1, 0, 1)]
    nbr27, child8, parent = [], [None], []
    for l, lv in enumerate(levels):
        nbr27.append(torch.tensor([[look[l].get((v[0] + a, v[1] + b, v[2] + c), -1) for a, b, c in offs] for v in lv],
                                  dtype=torch.int32))
        parent.append(torch.tensor([look[l + 1][tuple(v >> 1)] for v in lv], dtype=torch.int32) if l + 1 < depth
                      else torch.full((len(lv),), -1, dtype=torch.int32))
        if l >= 1:
            child8.append(torch.tensor([[look[l - 1].get((2 * v[0] + a, 2 * v[1] + b, 2 * v[2] + c), -1)
                                         for a in (0, 1) for b in (0, 1) for c in (0, 1)] for v in lv], dtype=torch.int32))
    return SimpleNamespace(depth=depth, nbr27=nbr27, child8=child8, parent=parent,
                           num_voxels=lambda l: len(levels[l]))


def test_fused_unet_glue_is_the_plain_unet(monkeypatch):
    """The GPU path of SparseUNet.forward never concatenates the skip connection (the decoder convolution runs over its
    two inputs in turn) and runs the up-projection as an 8-tap gather-GEMM over `up_table`; with the kernel call replaced
    by the torch definition of the same arguments (weights un-transposed for the wgmma layout) it must give the plain
    formulation (torch.cat + per-octant loop), for every kernel flag's weight layout."""
    import nksr_b200.unet as U
    svh = _toy_hierarchy()
    net = SparseUNet(3, 32, 4)
    g = torch.Generator().manual_seed(1)
    for q in net.parameters():
        if q.dim() == 1:
            q.data = torch.randn(q.shape, generator=g) * 0.1
    x0 = torch.randn((svh.num_voxels(0), 32), generator=g)
    t = U.up_table(svh, 0)
    assert t.shape == (svh.num_voxels(0), 8) and bool(((t >= 0).sum(dim=1) == 1).all())
    assert torch.equal(t.max(dim=1).values, svh.parent[0]) and U.up_table(svh, 0) is t           # cached
    calls = []

    def fake_kernel(x, idx, weight, bias=None, res=None, relu=False, tf32=False, impl="cuda"):
        calls.append(int(tf32))
        w = weight.transpose(1, 2) if int(tf32) == 3 else weight
        return gather_gemm(x, idx, w, bias, res, relu, impl="torch")
    with torch.no_grad():
        ref = net(x0, svh, impl="torch")
        monkeypatch.setattr(U, "gather_gemm", fake_kernel)
        for mode, flag, tol in ((False, 0, 1e-5), (True, 2, 2e-2), (3, 3, 2e-2)):
            calls.clear()
            out = net(x0, svh, tf32=mode)
            assert set(calls) == {flag} and len(calls) == 3 * 2 + 2 + 2 * 2 + 2      # enc, down, dec (2 parts), up
            for l in range(3):
                for name in ("structure", "normal", "basis", "udf", "decoder"):
                    a, b = getattr(out, name)[l], getattr(ref, name)[l]
                    assert float((a - b).abs().max()) <= tol * float(b.abs().max()), (mode, name, l)


def test_kernel_weights_follow_in_place_writes(monkeypatch):
    """The weights in kernel form (TF32-rounded, transposed for wgmma, split along c_in for the decoder's two inputs)
    follow the parameter, also after a write through `.data` (EMA updates, weight surgery), which bumps no version
    counter: the next forward of every kernel flag uses the new weights."""
    import nksr_b200.unet as U
    svh = _toy_hierarchy()
    net = SparseUNet(3, 32, 4)
    g = torch.Generator().manual_seed(2)
    x0 = torch.randn((svh.num_voxels(0), 32), generator=g)
    w1 = U.kernel_weights(net.dec[0].weight, 3, (32, 32))
    assert tuple(w1[0].shape) == (27, 32, 32) and w1[0].is_contiguous()
    assert torch.equal(w1[1], U.round_tf32(net.dec[0].weight.detach()[:, 32:]).transpose(1, 2))

    def fake_kernel(x, idx, weight, bias=None, res=None, relu=False, tf32=False, impl="cuda"):
        w = weight.transpose(1, 2) if int(tf32) == 3 else weight
        return gather_gemm(x, idx, w, bias, res, relu, impl="torch")
    monkeypatch.setattr(U, "gather_gemm", fake_kernel)
    for mode, tol in ((False, 1e-5), (True, 2e-2), (3, 2e-2)):
        with torch.no_grad():
            net(x0, svh, tf32=mode)                                      # a forward with the old weights first
            for q in net.parameters():
                q.data.copy_(torch.randn(q.shape, generator=g) * 0.2)
            out = net(x0, svh, tf32=mode)
            ref = net(x0, svh, impl="torch")
        for l in range(3):
            a, b = out.decoder[l], ref.decoder[l]
            assert float((a - b).abs().max()) <= tol * float(b.abs().max()), (mode, l)
    new = torch.randn_like(net.dec[0].weight)
    net.dec[0].weight.data.copy_(new)
    for mode in (0, 1, 2, 3):
        ws = U.kernel_weights(net.dec[0].weight, mode, (32, 32))
        for w, part in zip(ws, (new[:, :32], new[:, 32:])):
            part = U.round_tf32(part) if mode else part
            assert torch.equal(w, part.transpose(1, 2) if mode == 3 else part)
