"""SURVEY 8(f) row 2: the sparse-conv encoder / U-Net backbone of NKSRNetwork (nksr_b200/unet.py) and its kernel
(csrc/sparse_conv.cu: nksr_gather_gemm).

The kernels are checked element by element against an fp64 reference of the same gather-GEMM, within
kappa * 2^-24 * scale, scale = sum_k |x[idx[i, k]]| . |W_k| + |bias| + |res| (tests/bounds.py):
  * fp32 FFMA kernel (tf32 = 0): against the exact operands, KAPPA_GEMM.
  * mma.sync TF32 (tf32 = 1: W rounded per fragment, 2: W rounded on the host): the kernel rounds both operands with
    cvt.rna, so the tight reference (KAPPA_GEMM_TF32) takes round_tf32(x) and round_tf32(W); a loose bound
    (KAPPA_GEMM_TF32_OPERANDS) checks the exact product.
  * wgmma (tf32 = 3): the tensor core reads the fp32 A operand in shared memory as TF32.  The whole output lies within
    the tight bound of the reference with TRUNCATED x (the upper 19 bits) and rounded W, and outside the tight bound of
    the one with rna-rounded x (WGMMA_A_OPERAND).  On an H100 the worst ratio is 147 against the truncated-x
    reference and at least 355 against the rna-x one.
The whole backbone is compared with the same modules on the dense-gather torch path (`impl='torch'`).
"""
import itertools

import numpy as np
import pytest
import torch

from tests import clouds, scenes
from tests.bounds import KAPPA_GEMM, KAPPA_GEMM_TF32, KAPPA_GEMM_TF32_OPERANDS, assert_within, ratios

pytestmark = pytest.mark.gpu

WGMMA_A_OPERAND = "truncate"


def _svh(cuda, n=30_000, depth=3, voxel_size=0.1):
    from nksr_b200.svh import SparseFeatureHierarchy
    xyz, _, _ = scenes.crop("cfg4_outdoor", n, with_sensor=True)
    t = torch.from_numpy(np.ascontiguousarray(xyz)).to(cuda)
    return SparseFeatureHierarchy(voxel_size, depth, cuda).build_point_splatting(t), t


def _close(a, b, rel):
    scale = float(b.abs().max().item()) + 1e-30
    return float((a - b).abs().max().item()) <= rel * scale


def _truncate_tf32(v):
    return (v.contiguous().view(torch.int32) & -0x2000).view(torch.float32)


def _ref64(x, idx, w, x_form=None, w_form=None):
    """fp64 sum_k x'[idx[:, k]] @ W'_k and its magnitude sum_k |x'[idx[:, k]]| @ |W'_k| (absent sources add nothing),
    x' = x_form(x), W' = w_form(W) (operand roundings); w is (K, c_in, c_out).  Gathers before widening: x may be big."""
    n_out, K = idx.shape
    acc = torch.zeros((n_out, w.shape[2]), dtype=torch.float64, device=x.device)
    mag = torch.zeros_like(acc)
    for k in range(K):
        src = idx[:, k].long()
        ok = (src >= 0)[:, None]
        g = x[src.clamp(min=0)]
        g = (x_form(g) if x_form else g).double() * ok
        wk = (w_form(w[k]) if w_form else w[k]).double()
        acc += g @ wk
        mag += g.abs() @ wk.abs()
    return acc, mag


def _epilogue(acc, mag, bias, res, relu):
    pre, scale = acc.clone(), mag.clone()
    if bias is not None:
        pre += bias.double()
        scale += bias.double().abs()
    if res is not None:
        pre += res.double()
        scale += res.double().abs()
    return (torch.relu(pre) if relu else pre), pre, scale


def _kernel_weight(w, flag):
    from nksr_b200.unet import round_tf32
    return {0: w, 1: w, 2: round_tf32(w), 3: round_tf32(w).transpose(1, 2).contiguous()}[flag]


class _Refs:
    """the fp64 references of one (x, idx, W): exact operands, rna-rounded x and W, truncated x and rounded W"""

    def __init__(self, x, idx, w):
        from nksr_b200.unet import round_tf32
        self.forms = {"exact": _ref64(x, idx, w), "rna": _ref64(x, idx, w, round_tf32, round_tf32),
                      "truncate": _ref64(x, idx, w, _truncate_tf32, round_tf32)}

    def check(self, out, flag, bias, res, relu, what):
        """out of kernel `flag` element by element; returns the worst tight ratio"""
        np_ = lambda a: a.detach().cpu().numpy()
        exact, exact_pre, exact_scale = _epilogue(*self.forms["exact"], bias, res, relu)
        tight = {0: "exact", 1: "rna", 2: "rna", 3: WGMMA_A_OPERAND}[flag]
        ref, pre, scale = _epilogue(*self.forms[tight], bias, res, relu)
        got = np_(out)
        kappa = KAPPA_GEMM_TF32 if flag else KAPPA_GEMM
        worst = assert_within(got, np_(ref), np_(scale), kappa, f"{what} tf32={flag} vs {tight} operands",
                              lambda j: f"row {j // out.shape[1]} col {j % out.shape[1]}")
        if flag:
            assert_within(got, np_(exact), np_(exact_scale), KAPPA_GEMM_TF32_OPERANDS, f"{what} tf32={flag} vs exact")
        if flag == 3:
            other = "rna" if WGMMA_A_OPERAND == "truncate" else "truncate"
            oref, _, oscale = _epilogue(*self.forms[other], bias, res, relu)
            q, _, _ = ratios(got, np_(oref), np_(oscale))
            print(f"[bounds] {what} tf32=3 vs {other} operands: worst ratio {q.max():.4g}")
            differ = bool((self.forms["rna"][0] != self.forms["truncate"][0]).any())
            assert not differ or q.max() > kappa, f"{what}: the wgmma output also fits the {other} operands"
        if relu:
            assert bool((out >= 0).all())
            assert bool((out[pre < -kappa * 2.0 ** -24 * scale] == 0).all())         # exact zeros
        return worst


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
    refs = _Refs(x, idx, w)
    for bias, r, relu in [(b, res, True), (None, None, False), (b, None, False)]:
        ref = gather_gemm(x, idx, w, bias, r, relu, impl="torch")
        out = gather_gemm(x, idx, w, bias, r, relu, tf32=tf32)
        assert out.shape == ref.shape and torch.isfinite(out).all()
        refs.check(out, int(tf32), bias, r, relu, f"{taps}x{c_in}x{c_out}")
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
    operands read as TF32 by the tensor core, fp32 accumulation in registers) against its fp64 reference (module
    docstring); also bitwise repeatable (one accumulation order)"""
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
    refs = _Refs(x, idx, w)
    for bias, r, relu in [(b, res, True), (None, None, False), (b, None, False)]:
        ref = gather_gemm(x, idx, w, bias, r, relu, impl="torch")
        out = gather_gemm(x, idx, wt, bias, r, relu, tf32=3)
        assert out.shape == ref.shape and torch.isfinite(out).all()
        refs.check(out, 3, bias, r, relu, f"{taps}x{c_in}x{c_out}")
    assert torch.equal(gather_gemm(x, idx, wt, b, res, True, tf32=3), gather_gemm(x, idx, wt, b, res, True, tf32=3))
    # edge cases: no source at all, one row with one source, an empty output
    none = torch.full((300, taps), -1, dtype=torch.int32, device=cuda)
    assert torch.equal(gather_gemm(x, none, wt, b, res[:300], True, tf32=3), torch.relu(b + res[:300]))
    one = torch.full((1, taps), -1, dtype=torch.int32, device=cuda)
    one[0, taps // 2] = 7
    assert _close(gather_gemm(x, one, wt, None, None, False, tf32=3), x[7:8] @ w[taps // 2], 4e-3)
    assert gather_gemm(x, none[:0], wt, b, None, True, tf32=3).shape == (0, c_out)


# Tile edges of the three kernels (128-row tiles; wgmma: two warpgroups of 64 rows, TN = 32 / 64 / 128 columns per CTA
# and one to three column blocks, a ring that prefetches 2 steps of (tap, 32-channel chunk)).  Each value of every
# parameter occurs at least once; every case runs on all kernels with all 8 epilogues.
#   n_out:  1, 63, 64, 65 (second warpgroup empty / one row), 127, 128, 129, a few thousand not a multiple of 128
#   c_in:   32 (one chunk per tap: "one_tap" tiles have a single step, fewer than the prefetch distance), 64, 96, 256
#   c_out:  32 .. 384;  K: 1, 8, 27, 32, and 33 (refused by the TF32 kernels, whose tile tap mask is one 32-bit word)
GEMM_CASES = [
    # n_out, c_in, c_out, K, idx pattern
    (1, 32, 32, 1, "full"),
    (63, 64, 64, 8, "absent30"),
    (64, 32, 128, 27, "full"),
    (65, 96, 192, 27, "one_tap"),
    (127, 256, 384, 8, "tile_taps"),
    (128, 32, 96, 32, "shared"),
    (129, 64, 256, 27, "absent30"),
    (64, 64, 32, 27, "tile_taps"),
    (65, 32, 384, 1, "one_tap"),
    (1000, 256, 192, 27, "shared"),
    (2777, 96, 128, 8, "full"),
    (3001, 32, 64, 27, "tile_taps"),
    (4095, 32, 32, 32, "one_tap"),
    (300, 32, 64, 33, "absent30"),
]


def _gemm_idx(pattern, n_out, K, n_in, g):
    """(n_out, K) int32 source table.  full: every entry a source; absent30: ~30 % absent; one_tap: every 128-row tile
    has its sources in one tap (a different one per tile); tile_taps: every tile its own random tap subset, rows with
    holes; shared: many rows reading the same few sources.  Every table holds the source n_in - 1."""
    rnd = lambda: torch.randint(0, n_in, (n_out, K), generator=g, dtype=torch.int32)
    tile = torch.arange(n_out) // 128
    if pattern == "full":
        idx = rnd()
    elif pattern == "absent30":
        idx = torch.where(torch.rand((n_out, K), generator=g) < 0.3, -1, rnd())
    elif pattern == "one_tap":
        idx = torch.full((n_out, K), -1, dtype=torch.int32)
        idx[torch.arange(n_out), (tile * 7 + 3) % K] = rnd()[:, 0]
    elif pattern == "tile_taps":
        taps = torch.rand((int(tile.max()) + 1, K), generator=g) < 0.4
        taps[torch.arange(taps.shape[0]), torch.randint(0, K, (taps.shape[0],), generator=g)] = True
        keep = taps[tile] & (torch.rand((n_out, K), generator=g) < 0.8)
        idx = torch.where(keep, rnd(), -1)
    elif pattern == "shared":
        idx = torch.where(torch.rand((n_out, K), generator=g) < 0.2, -1, rnd() % 3)
    r, c = (idx >= 0).nonzero()[-1].tolist()
    idx[r, c] = n_in - 1
    return idx


@pytest.mark.parametrize("n_out,c_in,c_out,K,pattern", GEMM_CASES)
def test_gather_gemm_tile_edges_fp64(cuda, n_out, c_in, c_out, K, pattern):
    """every kernel, element by element against fp64, at the tile edges; rows of x spread over six decades
    (10^U(-3, 3)), so that a bound relative to the largest output would not see most rows; bitwise repeatable"""
    from nksr_b200 import _lib
    from nksr_b200.unet import gather_gemm
    g = torch.Generator(device="cpu").manual_seed(n_out * 7919 + c_in * 31 + c_out + K)
    n_in = 2 * n_out + 50
    rows = 10.0 ** (torch.rand((n_in, 1), generator=g) * 6 - 3)
    x = (torch.randn((n_in, c_in), generator=g) * rows).to(cuda)
    w = (torch.randn((K, c_in, c_out), generator=g) / (K * c_in) ** 0.5).to(cuda)
    b = torch.randn(c_out, generator=g).to(cuda)
    res = (torch.randn((n_out, c_out), generator=g) * 10.0 ** (torch.rand((n_out, 1), generator=g) * 6 - 3)).to(cuda)
    idx = _gemm_idx(pattern, n_out, K, n_in, g).to(cuda)
    refs = _Refs(x, idx, w)
    for flag in (0, 1, 2, 3):
        wk = _kernel_weight(w, flag)
        if K > 32 and flag:
            with pytest.raises(_lib.NksrError):
                gather_gemm(x, idx, wk, b, res, True, tf32=flag)
            continue
        for bias, r, relu in itertools.product((None, b), (None, res), (False, True)):
            out = gather_gemm(x, idx, wk, bias, r, relu, tf32=flag)
            assert out.shape == (n_out, c_out)
            refs.check(out, flag, bias, r, relu,
                       f"{n_out}x{c_in}x{c_out} K={K} {pattern} bias={bias is not None} res={r is not None} relu={relu}")
        assert torch.equal(gather_gemm(x, idx, wk, b, res, True, tf32=flag), gather_gemm(x, idx, wk, b, res, True, tf32=flag))


def test_gather_gemm_large_source_index(cuda):
    """sources beyond 2^31 / c_in rows: the gather addresses exceed 2^31 floats (x is ~8.7 GB), which the kernels form
    in 64 bits"""
    from nksr_b200.unet import gather_gemm
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 16 * 2 ** 30:
        pytest.skip(f"needs ~16 GB of free device memory, {free / 2 ** 30:.1f} GB free")
    c_in, c_out, K, n_out = 32, 64, 8, 256
    n_in = 2 ** 31 // c_in + 2 ** 20
    g = torch.Generator(device="cpu").manual_seed(9)
    idx = torch.randint(n_in - 2 ** 20, n_in, (n_out, K), generator=g, dtype=torch.int32)
    idx[torch.rand((n_out, K), generator=g) < 0.3] = -1
    idx[::17, 0] = torch.randint(0, 1000, (idx[::17].shape[0],), generator=g, dtype=torch.int32)
    idx[-1, -1] = n_in - 1
    idx = idx.to(cuda)
    x = torch.empty((n_in, c_in), dtype=torch.float32, device=cuda)          # only the rows idx reads are written
    used = idx[idx >= 0].long().unique()
    x[used] = torch.randn((used.numel(), c_in), generator=g).to(cuda)
    w = (torch.randn((K, c_in, c_out), generator=g) / (K * c_in) ** 0.5).to(cuda)
    b = torch.randn(c_out, generator=g).to(cuda)
    refs = _Refs(x, idx, w)
    for flag in (0, 1, 2, 3):
        out = gather_gemm(x, idx, _kernel_weight(w, flag), b, None, False, tf32=flag)
        refs.check(out, flag, b, None, False, "large index")
    del x
    torch.cuda.empty_cache()


@pytest.mark.parametrize("tf32", [False, True, 3])
def test_weights_written_through_data_are_used(cuda, tf32):
    """An in-place write through `.data` (EMA updates, weight surgery) bumps no version counter; the next CUDA forward
    must still use the new weights: a convolution over a channel concatenation (the decoder's split weights) and the
    U-Net's up-projection, after one forward with the old weights, against impl='torch' with the new ones."""
    from nksr_b200.unet import SparseUNet, up_table
    svh, _ = _svh(cuda, n=20_000, depth=2)
    net = SparseUNet(2, 32, 4).to(cuda)
    g = torch.Generator(device="cpu").manual_seed(12)
    n0, n1 = svh.num_voxels(0), svh.num_voxels(1)
    parts = (torch.randn((n0, 32), generator=g).to(cuda), torch.randn((n0, 32), generator=g).to(cuda))
    y1 = torch.randn((n1, 64), generator=g).to(cuda)
    conv, nbr = net.dec[0], svh.nbr27[0]
    flag = {False: 0, True: 2, 3: 3}[tf32]
    with torch.no_grad():
        conv(parts, nbr, tf32=tf32)
        net.up_project(y1, svh, 0, tf32=tf32)
        for p in net.parameters():
            p.data.copy_(torch.randn(p.shape, generator=g).to(cuda) * 0.1)
        got_conv = conv(parts, nbr, tf32=tf32)
        got_up = net.up_project(y1, svh, 0, tf32=tf32)
        ref_conv = conv(parts, nbr, impl="torch")
        ref_up = net.up_project(y1, svh, 0, impl="torch")
    x = torch.cat(parts, dim=1)
    kappa = KAPPA_GEMM_TF32_OPERANDS if flag else KAPPA_GEMM
    for got, ref, refs, bias, what in ((got_conv, ref_conv, _Refs(x, nbr, conv.weight.detach()), conv.bias.detach(),
                                        "decoder conv"),
                                       (got_up, ref_up, _Refs(y1, up_table(svh, 0), net.up[0].detach()), None,
                                        "up-projection")):
        relu = what == "decoder conv"
        refs.check(got, flag, bias, None, relu, f"{what} after .data write")
        _, _, scale = _epilogue(*refs.forms["exact"], bias, None, relu)
        assert_within(got.cpu().numpy(), ref.cpu().numpy(), scale.cpu().numpy(), kappa,
                      f"{what} after .data write vs impl='torch' (tf32={tf32})")


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
