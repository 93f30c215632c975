"""Autograd of the sparse convolution (nksr_b200/unet.py: GatherConv) without a GPU: the weight-gradient kernel, the
table transpose and the forward kernel are replaced by their torch definitions, so what is checked here is the glue --
the backward formulas, the per-part weight slices, the transposed weight layouts and the transposed tables -- in fp64
against finite differences (torch.autograd.gradcheck), and the trainable / frozen network switch."""
from types import SimpleNamespace

import pytest
import torch

import nksr_b200.unet as U
from tests.test_cpu_network import _toy_hierarchy


def _gemm_def(x, idx, weight, bias=None, res=None, relu=False, tf32=False, impl="cuda"):
    """the gather-GEMM in the dtype of x (weights un-transposed for the wgmma layout)"""
    w = weight.transpose(1, 2) if int(tf32) == 3 else weight
    n_out, K = idx.shape
    y = x.new_zeros((n_out, w.shape[2]))
    if bias is not None:
        y = y + bias
    if res is not None:
        y = y + res
    xp = torch.cat([x, x.new_zeros((1, x.shape[1]))])
    for k in range(K):
        y = y + xp[idx[:, k].long()] @ w[k]
    return torch.relu(y) if relu else y


@pytest.fixture
def torch_kernels(monkeypatch):
    wgrad, transpose, calls = U.gather_gemm_wgrad, U.transpose_taps, []

    def fake_wgrad(x, idx, g, tf32=False, bias=True, impl="cuda"):
        calls.append("wgrad")
        return wgrad(x, idx, g, tf32, bias, impl="torch")

    def fake_transpose(idx, n_src, impl="cuda"):
        calls.append("transpose")
        return transpose(idx, n_src, impl="torch")

    monkeypatch.setattr(U, "gather_gemm", _gemm_def)
    monkeypatch.setattr(U, "gather_gemm_wgrad", fake_wgrad)
    monkeypatch.setattr(U, "transpose_taps", fake_transpose)
    return calls


def _nbr_like(n, K, n_src, g, holes=0.3):
    """(n, K) table injective per tap: every tap a random partial permutation into n_src rows"""
    cols = []
    for _ in range(K):
        c = torch.randperm(n_src, generator=g)[:n].to(torch.int32)
        c[torch.rand(n, generator=g) < holes] = -1
        cols.append(c)
    return torch.stack(cols, dim=1)


def test_gradcheck_conv_with_residual_and_relu(torch_kernels):
    g = torch.Generator().manual_seed(0)
    n, K, ci, co = 13, 5, 4, 3
    idx = _nbr_like(n, K, n, g)
    x = torch.randn((n, ci), generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn((K, ci, co), generator=g, dtype=torch.float64, requires_grad=True)
    b = torch.randn(co, generator=g, dtype=torch.float64, requires_grad=True)
    res = torch.randn((n, co), generator=g, dtype=torch.float64, requires_grad=True)
    f = lambda x, w, b, res: U.GatherConv.apply(idx, None, 0, True, w, b, res, x)
    assert torch.autograd.gradcheck(f, (x, w, b, res))
    assert "wgrad" in torch_kernels and "transpose" in torch_kernels
    y = f(x, w, b, res)
    assert bool((y == 0).any()) and bool((y > 0).any())              # both sides of the ReLU are exercised


def test_gradcheck_two_part_decoder_conv(torch_kernels):
    """the decoder convolution over [skip ; up] without the concatenation: dW concatenated along c_in, one input
    gradient per part from its slice of W"""
    g = torch.Generator().manual_seed(1)
    n, K, c1, c2, co = 11, 4, 3, 5, 2
    idx = _nbr_like(n, K, n, g)
    x1 = torch.randn((n, c1), generator=g, dtype=torch.float64, requires_grad=True)
    x2 = torch.randn((n, c2), generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn((K, c1 + c2, co), generator=g, dtype=torch.float64, requires_grad=True)
    b = torch.randn(co, generator=g, dtype=torch.float64, requires_grad=True)
    f = lambda x1, x2, w, b: U.GatherConv.apply(idx, None, 0, True, w, b, None, x1, x2)
    assert torch.autograd.gradcheck(f, (x1, x2, w, b))
    ref = _gemm_def(torch.cat([x1, x2], dim=1), idx, w, b, None, True)
    assert torch.allclose(f(x1, x2, w, b), ref, rtol=1e-12, atol=1e-12)


def test_gradcheck_up_projection(torch_kernels):
    """8 taps, one source per row (the parent, in the column of the row's octant), no bias, no activation; the input
    gradient runs over the transposed table, which is the child table"""
    g = torch.Generator().manual_seed(2)
    n_par, co, ci = 4, 3, 2
    parent = torch.arange(n_par).repeat_interleave(3)[torch.randperm(3 * n_par, generator=g)]
    n = parent.numel()
    idx = torch.full((n, 8), -1, dtype=torch.int32)
    for p in range(n_par):
        rows = (parent == p).nonzero().squeeze(1)
        octs = torch.randperm(8, generator=g)[:rows.numel()]
        idx[rows, octs] = p
    y = torch.randn((n_par, co), generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn((8, co, ci), generator=g, dtype=torch.float64, requires_grad=True)
    f = lambda y, w: U.GatherConv.apply(idx, lambda: U.transpose_taps(idx, n_par), 0, False, w, None, None, y)
    assert torch.autograd.gradcheck(f, (y, w))


def test_transposed_weight_layouts():
    """the per-tap transposes W_k^T the input gradient runs the forward kernel with: (K, c_out, c_in) for modes 0-2
    (rounded for 1 / 2), rounded (K, c_in, c_out) for mode 3 (the wgmma kernel's K-major operand of W^T)"""
    w = torch.randn((27, 64, 32))
    for mode in (0, 1, 2, 3):
        ws = U.kernel_weights(w, mode, (32, 32), transposed=True)
        for q, part in zip(ws, (w[:, :32], w[:, 32:])):
            part = U.round_tf32(part) if mode else part
            assert q.is_contiguous() and torch.equal(q, part if mode == 3 else part.transpose(1, 2))


def test_transpose_taps_definition(torch_kernels):
    svh = _toy_hierarchy()
    for l in range(3):
        nbr = svh.nbr27[l]
        assert torch.equal(U.transpose_taps(nbr, nbr.shape[0], impl="torch"), nbr.flip(1))
    assert torch.equal(U.transpose_taps(svh.child8[1], svh.num_voxels(0), impl="torch"), U.up_table(svh, 0))
    bad = svh.nbr27[0].clone()
    bad[1, 3] = bad[0, 3] = 0
    with pytest.raises(U.NksrError):
        U.transpose_taps(bad, bad.shape[0], impl="torch")
    # the transpose is cached on the hierarchy while the table lives
    t1 = U.transposed_table(svh, svh.nbr27[1], svh.num_voxels(1))
    assert U.transposed_table(svh, svh.nbr27[1], svh.num_voxels(1)) is t1


def test_unet_backward_is_torch_autograd_of_the_reference(torch_kernels):
    """the whole backbone's gradients (every parameter and x0) through GatherConv equal torch autograd of the
    impl='torch' modules; the transposed tables are built once per table and cached on the hierarchy"""
    svh = _toy_hierarchy()
    torch.manual_seed(3)
    net = U.SparseUNet(3, 32, 4)
    g = torch.Generator().manual_seed(4)
    for q in net.parameters():
        if q.dim() == 1:
            q.data = torch.randn(q.shape, generator=g) * 0.1
    x0 = torch.randn((svh.num_voxels(0), 32), generator=g, requires_grad=True)
    cot = {}

    def loss(out):
        tot = 0.0
        for name in ("structure", "normal", "basis", "udf"):
            for l, t in getattr(out, name).items():
                c = cot.setdefault((name, l), torch.randn(t.shape, generator=g))
                tot = tot + (t * c).sum()
        return tot

    grads = []
    for impl in ("torch", "cuda"):
        net.zero_grad()
        x0.grad = None
        loss(net(x0, svh, impl=impl)).backward()
        grads.append([x0.grad.clone()] + [p.grad.clone() for p in net.parameters()])
    for a, b in zip(*grads):
        assert torch.allclose(a, b, rtol=1e-4, atol=1e-5 * float(b.abs().max()))
    n_transpose = torch_kernels.count("transpose")
    assert n_transpose == 3 + 2 + 2                    # nbr27 per level, child8, up tables: each transposed once
    net.zero_grad()
    loss(net(x0, svh)).backward()
    assert torch_kernels.count("transpose") == n_transpose


def test_default_network_is_frozen_and_trainable_one_is_not(torch_kernels):
    from nksr_b200.network import NKSRNetwork
    svh = _toy_hierarchy()
    svh.keys = [None] * 3
    x0 = torch.randn((svh.num_voxels(0), 32), requires_grad=True)
    frozen = NKSRNetwork(dict(backbone="unet", tree_depth=3))
    assert not frozen.trainable and not any(p.requires_grad for p in frozen.parameters())
    out, s0, _ = frozen.unet(SimpleNamespace(x0=x0), svh)
    assert s0 is svh and all(t.grad_fn is None for t in out.structure_features.values())
    assert all(t.grad_fn is None for t in out.basis_features.values())
    net = NKSRNetwork(dict(backbone="unet", tree_depth=3, trainable=True))
    assert all(p.requires_grad for p in net.parameters())
    out, _, _ = net.unet(SimpleNamespace(x0=x0), svh)
    assert all(t.grad_fn is not None for t in out.structure_features.values())
    with torch.no_grad():                                         # a trainable network follows the caller's grad mode
        out, _, _ = net.unet(SimpleNamespace(x0=x0), svh)
    assert all(t.grad_fn is None for t in out.udf_features.values())
    # same seeded weights as the frozen network
    assert all(torch.equal(a, b) for a, b in zip(net.state_dict().values(), frozen.state_dict().values()))
    with pytest.raises(ValueError):
        NKSRNetwork(dict(backbone="pool", trainable=True))
