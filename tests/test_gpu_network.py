"""SURVEY 8(f) row 2: the sparse-conv encoder / U-Net backbone of NKSRNetwork (nksr_b200/unet.py) and its kernel
(csrc/sparse_conv.cu: nksr_gather_gemm) against the same arithmetic in plain torch fp32 (dense gathers + matmul,
`impl='torch'`) -- a floating-point kernel, so the torch fp32 reference is the checker here.

Tolerances: the fp32 kernel sums the same products in another order: |diff| <= 2e-5 max|y|; the TF32 kernel rounds its
operands to 10-bit mantissas (cvt.rna): |diff| <= 4e-3 max|y| over 27 x 32..128 terms.
"""
import numpy as np
import pytest
import torch

from tests import clouds, scenes

pytestmark = pytest.mark.gpu


def _svh(cuda, n=30_000, depth=3, voxel_size=0.1):
    from nksr_b200.svh import SparseFeatureHierarchy
    xyz, _, _ = scenes.crop("cfg4_outdoor", n, with_sensor=True)
    t = torch.from_numpy(np.ascontiguousarray(xyz)).to(cuda)
    return SparseFeatureHierarchy(voxel_size, depth, cuda).build_point_splatting(t), t


def _close(a, b, rel):
    scale = float(b.abs().max().item()) + 1e-30
    return float((a - b).abs().max().item()) <= rel * scale


@pytest.mark.parametrize("tf32", [False, True])
@pytest.mark.parametrize("taps,c_in,c_out", [(27, 32, 32), (27, 64, 32), (27, 32, 64), (27, 128, 64), (8, 32, 64),
                                             (27, 32, 96)])
def test_gather_gemm_matches_torch(cuda, tf32, taps, c_in, c_out):
    from nksr_b200.unet import gather_gemm
    svh, _ = _svh(cuda)
    g = torch.Generator(device="cpu").manual_seed(taps * 1000 + c_in + c_out)
    if taps == 27:
        idx, n_in = svh.nbr27[0], svh.num_voxels(0)
    else:
        idx, n_in = svh.child8[1], svh.num_voxels(0)
    n_out = idx.shape[0]
    assert n_out % 128 != 0 and n_out > 1000
    x = torch.randn((n_in, c_in), generator=g).to(cuda)
    w = (torch.randn((taps, c_in, c_out), generator=g) / (taps * c_in) ** 0.5).to(cuda)
    b = torch.randn(c_out, generator=g).to(cuda)
    res = torch.randn((n_out, c_out), generator=g).to(cuda)
    rel = 4e-3 if tf32 else 2e-5
    for bias, r, relu in [(b, res, True), (None, None, False), (b, None, False)]:
        ref = gather_gemm(x, idx, w, bias, r, relu, impl="torch")
        out = gather_gemm(x, idx, w, bias, r, relu, tf32=tf32)
        assert out.shape == ref.shape and torch.isfinite(out).all()
        assert _close(out, ref, rel), float((out - ref).abs().max())
    if not tf32:                                      # the fp32 kernel is deterministic
        assert torch.equal(gather_gemm(x, idx, w, b, res, True), gather_gemm(x, idx, w, b, res, True))


@pytest.mark.parametrize("tf32", [False, True])
def test_gather_gemm_edge_cases(cuda, tf32):
    from nksr_b200 import _lib
    from nksr_b200.unet import gather_gemm
    g = torch.Generator(device="cpu").manual_seed(3)
    x = torch.randn((50, 32), generator=g).to(cuda)
    w = torch.randn((27, 32, 32), generator=g).to(cuda)
    b = torch.randn(32, generator=g).to(cuda)
    # no source at all: y = act(bias + res)
    idx = torch.full((300, 27), -1, dtype=torch.int32, device=cuda)
    res = torch.randn((300, 32), generator=g).to(cuda)
    assert torch.equal(gather_gemm(x, idx, w, b, res, True, tf32=tf32), torch.relu(b + res))
    # one row, one source; an empty output
    idx1 = torch.full((1, 27), -1, dtype=torch.int32, device=cuda)
    idx1[0, 13] = 7
    rel = 4e-3 if tf32 else 2e-5
    assert _close(gather_gemm(x, idx1, w, None, None, False, tf32=tf32), x[7:8] @ w[13], rel)
    assert gather_gemm(x, idx[:0], w, b, None, True, tf32=tf32).shape == (0, 32)
    # channel counts the kernel does not take are refused, not mis-computed
    with pytest.raises(_lib.NksrError):
        gather_gemm(x[:, :16].contiguous(), idx, w[:, :16].contiguous(), None, None, False, tf32=tf32)


@pytest.mark.parametrize("taps,c_in,c_out", [(27, 32, 32), (27, 64, 32), (27, 32, 64), (27, 128, 64), (8, 32, 64),
                                             (27, 32, 96), (27, 256, 256)])
def test_gather_gemm_tcgen05_matches_torch(cuda, taps, c_in, c_out):
    """the tensor-core kernel (tf32 = 3, written with wgmma on sm_90a; the name is from its first, tcgen05, version:
    operands read as TF32 by the tensor core, fp32 accumulation in registers) against
    dense torch fp32, the same bound as the mma.sync TF32 kernel; also bitwise repeatable (one accumulation order)"""
    from nksr_b200.unet import gather_gemm, round_tf32
    svh, _ = _svh(cuda)
    g = torch.Generator(device="cpu").manual_seed(taps * 1000 + c_in + c_out)
    idx, n_in = (svh.nbr27[0], svh.num_voxels(0)) if taps == 27 else (svh.child8[1], svh.num_voxels(0))
    n_out = idx.shape[0]
    x = torch.randn((n_in, c_in), generator=g).to(cuda)
    w = (torch.randn((taps, c_in, c_out), generator=g) / (taps * c_in) ** 0.5).to(cuda)
    wt = round_tf32(w).transpose(1, 2).contiguous()
    b = torch.randn(c_out, generator=g).to(cuda)
    res = torch.randn((n_out, c_out), generator=g).to(cuda)
    for bias, r, relu in [(b, res, True), (None, None, False), (b, None, False)]:
        ref = gather_gemm(x, idx, w, bias, r, relu, impl="torch")
        out = gather_gemm(x, idx, wt, bias, r, relu, tf32=3)
        assert out.shape == ref.shape and torch.isfinite(out).all()
        assert _close(out, ref, 4e-3), float((out - ref).abs().max())
    assert torch.equal(gather_gemm(x, idx, wt, b, res, True, tf32=3), gather_gemm(x, idx, wt, b, res, True, tf32=3))
    # edge cases: no source at all, one row with one source, an empty output
    none = torch.full((300, taps), -1, dtype=torch.int32, device=cuda)
    assert torch.equal(gather_gemm(x, none, wt, b, res[:300], True, tf32=3), torch.relu(b + res[:300]))
    one = torch.full((1, taps), -1, dtype=torch.int32, device=cuda)
    one[0, taps // 2] = 7
    assert _close(gather_gemm(x, one, wt, None, None, False, tf32=3), x[7:8] @ w[taps // 2], 4e-3)
    assert gather_gemm(x, none[:0], wt, b, None, True, tf32=3).shape == (0, c_out)


def test_unet_forward_matches_torch_reference(cuda):
    """the whole backbone (point encoder -> residual sparse-conv U-Net -> heads) with the CUDA convolution against the
    same modules with the dense-gather torch convolution; then TF32 against fp32"""
    from nksr_b200.network import NKSRNetwork
    svh, xyz = _svh(cuda, n=20_000, depth=3)
    net = NKSRNetwork(dict(backbone="unet", tree_depth=3, kernel_dim=4)).to(cuda)
    g = torch.Generator(device="cpu").manual_seed(5)
    feat = torch.nn.functional.normalize(torch.randn((xyz.shape[0], 3), generator=g), dim=1).to(cuda)
    with torch.no_grad():
        enc = net.encoder(xyz, feat, svh, 0)
        assert enc.x0.shape == (svh.num_voxels(0), 32) and torch.isfinite(enc.x0).all()
        out = net.backbone_net(enc.x0, svh)
        ref = net.backbone_net(enc.x0, svh, impl="torch")
        fast = net.backbone_net(enc.x0, svh, tf32=True)
    for l in range(3):
        n_l = svh.num_voxels(l)
        assert out.structure[l].shape == (n_l, 3) and out.normal[l].shape == (n_l, 3)
        assert out.basis[l].shape == (n_l, 4) and out.udf[l].shape == (n_l, 4)
        for name in ("structure", "normal", "basis", "udf", "decoder"):
            a, b, c = getattr(out, name)[l], getattr(ref, name)[l], getattr(fast, name)[l]
            assert torch.isfinite(a).all() and float(b.abs().max()) > 0
            assert _close(a, b, 1e-4), (name, l, float((a - b).abs().max()), float(b.abs().max()))
            assert _close(c, b, 2e-2), (name, l, float((c - b).abs().max()), float(b.abs().max()))


def test_unet_forward_tcgen05_matches_torch_reference(cuda):
    """the whole backbone with every convolution on the tensor-core kernel (precision='tc', wgmma on sm_90a; the name is
    from its first, tcgen05, version) against the torch fp32 modules"""
    from nksr_b200.network import NKSRNetwork
    svh, xyz = _svh(cuda, n=20_000, depth=3)
    net = NKSRNetwork(dict(backbone="unet", tree_depth=3, kernel_dim=4, precision="tc")).to(cuda)
    assert net.tf32 == 3
    g = torch.Generator(device="cpu").manual_seed(5)
    feat = torch.nn.functional.normalize(torch.randn((xyz.shape[0], 3), generator=g), dim=1).to(cuda)
    with torch.no_grad():
        enc = net.encoder(xyz, feat, svh, 0)
        ref = net.backbone_net(enc.x0, svh, impl="torch")
        tc = net.backbone_net(enc.x0, svh, tf32=3)
    for l in range(3):
        for name in ("structure", "normal", "basis", "udf", "decoder"):
            a, b = getattr(tc, name)[l], getattr(ref, name)[l]
            assert torch.isfinite(a).all() and _close(a, b, 2e-2), (name, l, float((a - b).abs().max()))


def test_unet_backbone_through_the_reconstructor(cuda):
    """contract of models/nksr_net.py:73-101 with the U-Net backbone: encoder / unet calls, per-level feature tables on
    the decoder hierarchy (also a pruned one), and a reconstruction that runs end to end on them (random weights: the
    surface is meaningless, the solve must still be a finite SPD solve)"""
    import nksr_b200
    from nksr_b200.network import NKSRNetwork
    from nksr_b200.svh import SparseFeatureHierarchy
    xyz, nrm = clouds.sphere(30_000, noise=0.001)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    net = NKSRNetwork(dict(backbone="unet", tree_depth=4, kernel_dim=4))
    rec = nksr_b200.Reconstructor(cuda, network=net)
    field = rec.reconstruct(t(xyz), t(nrm), voxel_size=0.02, solver_tol=1e-4, solver_max_iter=400)
    alpha = field.alpha
    assert torch.isfinite(alpha).all()
    f = field.evaluate_f(t(xyz[:1000])).value
    assert torch.isfinite(f).all()
    # a pruned decoder hierarchy receives the features of the voxels it shares with the encoder hierarchy
    enc_svh = SparseFeatureHierarchy(0.02, 4, cuda).build_point_splatting(t(xyz))
    dec_svh = SparseFeatureHierarchy(0.02, 4, cuda).build_adaptive_normal_variation(t(xyz), t(nrm), tau=0.2,
                                                                                     adaptive_depth=2)
    with torch.no_grad():
        enc = rec.network.encoder(t(xyz), t(nrm), enc_svh, 0)
        full, s0, _ = rec.network.unet(enc, enc_svh, adaptive_depth=2)
        part, s1, _ = rec.network.unet(enc, enc_svh, adaptive_depth=2, gt_decoder_svh=dec_svh)
    assert s0 is enc_svh and s1 is dec_svh
    for l in range(4):
        assert part.basis_features[l].shape == (dec_svh.num_voxels(l), 4)
        if dec_svh.num_voxels(l) == 0:
            continue
        pos = torch.searchsorted(enc_svh.keys[l], dec_svh.keys[l]).clamp(max=enc_svh.num_voxels(l) - 1)
        hit = enc_svh.keys[l][pos] == dec_svh.keys[l]
        assert bool(hit.all())                                     # pruning only removes voxels
        assert torch.equal(part.basis_features[l], full.basis_features[l][pos])
        assert torch.equal(part.normal_features[l], full.normal_features[l][pos])
