"""Backward of the sparse convolution (csrc/sparse_conv_bwd.cu, nksr_b200/unet.py: GatherConv) and training of the U-Net
backbone (nksr_b200/training.py).

Weight gradient, entry by entry against fp64 within kappa * 2^-24 * scale, scale = sum_i |x[idx[i, k]]|^T |g[i]|
(tests/bounds.py; the constants are below): the fp32 kernel against the exact operands (KAPPA_WGRAD); the TF32 kernel (both operands rounded
with cvt.rna) against the rounded operands (KAPPA_WGRAD_TF32) and, loosely, the exact ones (KAPPA_WGRAD_TF32_OPERANDS).
The input gradient is the forward kernel over the transposed table, held to the forward's constants.
"""
import numpy as np
import pytest
import torch

from tests.bounds import KAPPA_GEMM, KAPPA_GEMM_TF32_OPERANDS, assert_within
from tests.test_gpu_network import GEMM_CASES, _gemm_idx, _svh

pytestmark = pytest.mark.gpu

# kappa of the weight gradient in units of 2^-24 (the convention of tests/bounds.py), each at most 8x the worst ratio
# measured on an NVIDIA H100 80GB HBM3 (power limit 700 W) over this file.
# fp32 kernel (fp32 over <= 256 rows, fp64 across) against the exact operands, and db (an fp32 sum of the unrounded g
# in every precision).  Worst 13.7 (n_out 300, c_in 32, c_out 64, K 33); db 3.7.
KAPPA_WGRAD = 96.0
# TF32 mma.sync against the rna-rounded x and g.  Worst 18.9 (n_out 129, c_in 64, c_out 256, K 27).
KAPPA_WGRAD_TF32 = 128.0
# TF32 against the unrounded operands (both rounded: 2 x 2^13 u, plus the accumulation).  Worst 13900.
KAPPA_WGRAD_TF32_OPERANDS = 2.0 ** 15

np_ = lambda a: a.detach().double().cpu().numpy()


def _wgrad64(x, idx, g, form=None):
    """fp64 dW (K, c_in, c_out), its magnitude sum_i |x[idx]|^T |g|, db and sum |g|; form rounds both operands"""
    K = idx.shape[1]
    gg = (form(g) if form else g).double()
    dw = torch.zeros((K, x.shape[1], g.shape[1]), dtype=torch.float64, device=x.device)
    mag = torch.zeros_like(dw)
    for k in range(K):
        src = idx[:, k].long()
        ok = (src >= 0)[:, None]
        gx = x[src.clamp(min=0)]
        gx = (form(gx) if form else gx).double() * ok
        dw[k] = gx.T @ gg
        mag[k] = gx.abs().T @ gg.abs()
    return dw, mag, gg.sum(0), gg.abs().sum(0)


def _check_wgrad(x, idx, g, flag, what):
    from nksr_b200.unet import gather_gemm_wgrad, round_tf32
    dw, db = gather_gemm_wgrad(x, idx, g, flag)
    exact = _wgrad64(x, idx, g)
    worst = 0.0
    if flag:
        rna = _wgrad64(x, idx, g, round_tf32)
        worst = assert_within(np_(dw), np_(rna[0]), np_(rna[1]), KAPPA_WGRAD_TF32, f"{what} dW tf32={flag} vs rna")
        assert_within(np_(dw), np_(exact[0]), np_(exact[1]), KAPPA_WGRAD_TF32_OPERANDS, f"{what} dW tf32={flag} exact")
    else:
        worst = assert_within(np_(dw), np_(exact[0]), np_(exact[1]), KAPPA_WGRAD, f"{what} dW fp32")
    # db sums the unrounded g in fp32 in every precision
    assert_within(np_(db), np_(exact[2]), np_(exact[3]), KAPPA_WGRAD, f"{what} db tf32={flag}")
    absent = (idx < 0).all(dim=0)
    assert bool((dw[absent] == 0).all())                        # a tap without sources: exactly zero
    dw2, db2 = gather_gemm_wgrad(x, idx, g, flag)
    assert torch.equal(dw, dw2) and torch.equal(db, db2)        # bitwise repeatable
    return worst


@pytest.mark.parametrize("n_out,c_in,c_out,K,pattern", GEMM_CASES)
def test_wgrad_tile_edges_fp64(cuda, n_out, c_in, c_out, K, pattern):
    """every precision at the forward's tile edges; rows of x and g spread over six decades; tap 0 without sources"""
    from nksr_b200 import _lib
    from nksr_b200.unet import gather_gemm_wgrad
    g_ = torch.Generator(device="cpu").manual_seed(n_out * 31 + c_in * 7 + c_out + K)
    n_in = 2 * n_out + 50
    x = (torch.randn((n_in, c_in), generator=g_) * 10.0 ** (torch.rand((n_in, 1), generator=g_) * 6 - 3)).to(cuda)
    g = (torch.randn((n_out, c_out), generator=g_) * 10.0 ** (torch.rand((n_out, 1), generator=g_) * 6 - 3)).to(cuda)
    idx = _gemm_idx(pattern, n_out, K, n_in, g_)
    if K > 1:
        idx[:, 0] = -1
    idx = idx.to(cuda)
    for flag in (0, 1, 2, 3):
        if K > 32 and flag:
            with pytest.raises(_lib.NksrError):
                gather_gemm_wgrad(x, idx, g, flag)
            continue
        _check_wgrad(x, idx, g, flag, f"{n_out}x{c_in}x{c_out} K={K} {pattern}")


def test_wgrad_many_spans_and_empty(cuda):
    """n_out >= 10^6: many spans reduced in order; the fp32 error stays that of a 256-row sum.  n_out = 0: zeros."""
    from nksr_b200.unet import gather_gemm_wgrad
    g_ = torch.Generator(device="cpu").manual_seed(17)
    n_out, n_in, K, c_in, c_out = 1_200_000, 1_300_000, 8, 32, 64
    idx = torch.randint(0, n_in, (n_out, K), generator=g_, dtype=torch.int32)
    idx[torch.rand((n_out, K), generator=g_) < 0.3] = -1
    idx[:, 5] = -1
    x = (torch.randn((n_in, c_in), generator=g_) * 10.0 ** (torch.rand((n_in, 1), generator=g_) * 6 - 3)).to(cuda)
    g = torch.randn((n_out, c_out), generator=g_).to(cuda)
    idx = idx.to(cuda)
    for flag in (0, 1):
        _check_wgrad(x, idx, g, flag, "1.2M rows")
    dw, db = gather_gemm_wgrad(x, idx[:0], g[:0], 0)
    assert dw.shape == (K, c_in, c_out) and bool((dw == 0).all()) and bool((db == 0).all())


def test_wgrad_large_source_index(cuda):
    """sources beyond 2^31 / c_in rows: gather addresses beyond 2^31 floats (x is ~8.7 GB)"""
    free, _ = torch.cuda.mem_get_info(cuda)
    if free < 16 * 2 ** 30:
        pytest.skip(f"needs ~16 GB of free device memory, {free / 2 ** 30:.1f} GB free")
    c_in, c_out, K, n_out = 32, 64, 8, 256
    n_in = 2 ** 31 // c_in + 2 ** 20
    g_ = torch.Generator(device="cpu").manual_seed(9)
    idx = torch.randint(n_in - 2 ** 20, n_in, (n_out, K), generator=g_, dtype=torch.int32)
    idx[torch.rand((n_out, K), generator=g_) < 0.3] = -1
    idx[-1, -1] = n_in - 1
    idx = idx.to(cuda)
    x = torch.empty((n_in, c_in), dtype=torch.float32, device=cuda)
    used = idx[idx >= 0].long().unique()
    x[used] = torch.randn((used.numel(), c_in), generator=g_).to(cuda)
    g = torch.randn((n_out, c_out), generator=g_).to(cuda)
    for flag in (0, 1):
        _check_wgrad(x, idx, g, flag, "large index")
    del x
    torch.cuda.empty_cache()


def test_table_transposes(cuda):
    from nksr_b200 import _lib
    from nksr_b200.unet import transpose_taps, up_table
    svh, _ = _svh(cuda, n=30_000, depth=3)
    for l in range(3):
        assert torch.equal(transpose_taps(svh.nbr27[l], svh.num_voxels(l)), svh.nbr27[l].flip(1))
    for l in range(2):
        up = up_table(svh, l)
        assert torch.equal(transpose_taps(svh.child8[l + 1], svh.num_voxels(l)), up)
        assert torch.equal(transpose_taps(up, svh.num_voxels(l + 1)), svh.child8[l + 1])
    bad = svh.nbr27[0].clone()
    bad[5, 3] = bad[9, 3] = 0
    with pytest.raises(_lib.NksrError):
        transpose_taps(bad, svh.num_voxels(0))
    with pytest.raises(_lib.NksrError):
        transpose_taps(svh.nbr27[0], svh.num_voxels(0) - 1)


def _layer_grads(fn, inputs, params, dy):
    for t in list(inputs) + list(params):
        t.grad = None
    y = fn(*inputs)
    y.backward(dy)
    return y, [t.grad.clone() if t.grad is not None else None for t in list(inputs) + list(params)]


@pytest.mark.parametrize("tf32", [False, True, 3])
@pytest.mark.parametrize("layer", ["res_relu", "decoder", "down", "up"])
def test_layer_gradients_match_fp64_autograd(cuda, layer, tf32):
    """dx, dW, db and d_res of one layer against torch autograd of impl='torch' in fp64, entry by entry; the
    cotangent is zero where the fp64 pre-activation is within 1 % of its largest value of 0 (both sides then agree on
    the ReLU mask)"""
    from nksr_b200.unet import SparseUNet, up_table
    svh, _ = _svh(cuda, n=20_000, depth=2)
    torch.manual_seed(0)
    net = SparseUNet(2, 32, 4).to(cuda)
    g_ = torch.Generator(device="cpu").manual_seed(21)
    for p in net.parameters():
        p.data.copy_(torch.randn(p.shape, generator=g_).to(cuda) * (0.1 if p.dim() == 1 else 1.0 / p.shape[0] ** 0.5))
    n0, n1 = svh.num_voxels(0), svh.num_voxels(1)
    rnd = lambda *s: torch.randn(s, generator=g_).to(cuda)
    if layer == "res_relu":
        conv, idx, xs, res, relu = net.enc_b[0], svh.nbr27[0], [rnd(n0, 32)], rnd(n0, 32), True
    elif layer == "decoder":
        conv, idx, xs, res, relu = net.dec[0], svh.nbr27[0], [rnd(n0, 32), rnd(n0, 32)], None, True
    elif layer == "down":
        conv, idx, xs, res, relu = net.down[0], svh.child8[1], [rnd(n0, 32)], None, True
    else:
        conv, idx, xs, res, relu = None, up_table(svh, 0), [rnd(n1, 64)], None, False
    for t in xs + ([res] if res is not None else []):
        t.requires_grad_(True)
    params = [net.up[0]] if conv is None else [conv.weight, conv.bias]

    def run(impl, xs_, res_, params_):
        if conv is None:
            return net.up_project(xs_[0], svh, 0, tf32=tf32, impl=impl)
        return conv(tuple(xs_) if len(xs_) > 1 else xs_[0], idx, res=res_, relu=relu, tf32=tf32, impl=impl)

    # fp64 reference: the same module in double, impl='torch'
    net64 = SparseUNet(2, 32, 4).to(cuda).double()
    net64.load_state_dict({k: v.double() for k, v in net.state_dict().items()})
    xs64 = [x.detach().double().requires_grad_(True) for x in xs]
    res64 = res.detach().double().requires_grad_(True) if res is not None else None
    if conv is None:
        params64 = [net64.up[0]]
        f64 = lambda *a: net64.up_project(a[0], svh, 0, impl="torch")
    else:
        m64 = dict(net64.named_modules())[next(n for n, m in net.named_modules() if m is conv)]
        params64 = [m64.weight, m64.bias]
        f64 = lambda *a: m64(tuple(a[:len(xs)]) if len(xs) > 1 else a[0], idx, res=a[len(xs)] if res is not None
                             else None, relu=False, impl="torch")
    ins64 = xs64 + ([res64] if res is not None else [])
    with torch.no_grad():
        pre = f64(*ins64)
    dy = rnd(*pre.shape)
    if relu:
        dy[pre.abs() < 1e-2 * float(pre.abs().max())] = 0
    relu_f64 = (lambda *a: torch.relu(f64(*a))) if relu else f64
    _, ref = _layer_grads(relu_f64, ins64, params64, dy.double())
    ins = xs + ([res] if res is not None else [])
    y, got = _layer_grads(lambda *a: run("cuda", list(a[:len(xs)]), a[len(xs)] if res is not None else None, params),
                          ins, params, dy)
    with torch.no_grad():                                       # a forward in grad mode is the no_grad forward
        y0 = run("cuda", xs, res, params)
    assert torch.equal(y, y0) and y.grad_fn is not None
    g64 = dy.double() * (pre > 0) if relu else dy.double()
    flag = {False: 0, True: 1, 3: 3}[tf32]
    k_dx = KAPPA_GEMM_TF32_OPERANDS if flag else KAPPA_GEMM
    k_dw = KAPPA_WGRAD_TF32_OPERANDS if flag else KAPPA_WGRAD
    # scales: dx_p = sum_k g[idx_t] W_k^T, dW = sum_i x[idx]^T g, db = sum g
    from nksr_b200.unet import transpose_taps
    W = params64[0].detach()
    n_src = xs[0].shape[0]
    idx_t = transpose_taps(idx, n_src)
    gp = torch.cat([g64.abs(), g64.new_zeros((1, g64.shape[1]))])
    off = 0
    for p, x in enumerate(xs):
        c = x.shape[1]
        Wp = W[:, off:off + c]
        sx = sum(gp[idx_t[:, k].long()] @ Wp[k].abs().T for k in range(idx.shape[1]))
        assert_within(np_(got[p]), np_(ref[p]), np_(sx), k_dx, f"{layer} tf32={tf32} dx[{p}]")
        xp = torch.cat([x.detach().double().abs(), x.new_zeros((1, c)).double()])
        sw = torch.stack([xp[idx[:, k].long()].T @ g64.abs() for k in range(idx.shape[1])])
        dwp = got[len(ins)][:, off:off + c]
        assert_within(np_(dwp), np_(ref[len(ins)][:, off:off + c]), np_(sw), k_dw, f"{layer} tf32={tf32} dW[{p}]")
        off += c
    if conv is not None:
        assert_within(np_(got[len(ins) + 1]), np_(ref[len(ins) + 1]), np_(g64.abs().sum(0)), KAPPA_WGRAD,
                      f"{layer} tf32={tf32} db")
    if res is not None:
        assert torch.equal(got[len(xs)], ref[len(xs)].float())


def _backbone_grads(net, x0, svh, cot, **kw):
    net.zero_grad(set_to_none=True)
    x0.grad = None
    out = net(x0, svh, **kw)
    loss = sum((getattr(out, name)[l] * cot[(name, l)]).sum() for (name, l) in cot)
    loss.backward()
    return out, [x0.grad.clone()] + [p.grad.clone() for p in net.parameters()]


def _rel(a, b):
    return float((a - b).abs().max()) / (float(b.abs().max()) + 1e-30)


# whole-backbone gradient tolerances, max |diff| / max |ref| per tensor against the fp32 impl='torch' autograd, measured
# on an H100 80GB HBM3 (700 W): fp32 worst 1.3e-6; TF32 / tc worst 0.46 / 0.54.  The TF32 numbers are not a kernel error
# (the per-layer test above holds every TF32 gradient entry to its own bound): the bias and up-path gradients sum
# ~10^4 rows of a random-signed cotangent, which cancel, while the TF32 forward's perturbation of the activations and
# ReLU masks (2e-2 of the output, the forward test's tolerance) does not.
BACKBONE_GRAD_REL = {False: 1e-5, True: 1.0, 3: 1.0}


@pytest.mark.parametrize("tf32", [False, True, 3])
def test_backbone_gradients_match_torch_autograd(cuda, tf32):
    """a random cotangent on every head: the gradient of every parameter and of x0 against torch autograd of the
    impl='torch' modules (fp32), per tensor; two backward passes give the same bits; the grad-mode forward is the
    no_grad forward"""
    from nksr_b200.unet import SparseUNet
    svh, _ = _svh(cuda, n=20_000, depth=3)
    torch.manual_seed(1)
    net = SparseUNet(3, 32, 4).to(cuda)
    g_ = torch.Generator(device="cpu").manual_seed(22)
    x0 = torch.randn((svh.num_voxels(0), 32), generator=g_).to(cuda).requires_grad_(True)
    with torch.no_grad():
        plain = net(x0, svh, tf32=tf32)
    cot = {(name, l): torch.randn(getattr(plain, name)[l].shape, generator=g_).to(cuda)
           for name in ("structure", "normal", "basis", "udf") for l in range(3)}
    _, ref = _backbone_grads(net, x0, svh, cot, impl="torch")
    out, got = _backbone_grads(net, x0, svh, cot, tf32=tf32)
    _, again = _backbone_grads(net, x0, svh, cot, tf32=tf32)
    for l in range(3):
        assert torch.equal(out.decoder[l], plain.decoder[l]) and torch.equal(out.udf[l], plain.udf[l])
    names = ["x0"] + [n for n, _ in net.named_parameters()]
    rel = sorted((_rel(a, b), n) for n, a, b in zip(names, got, ref))
    print(f"[bounds] backbone gradients tf32={tf32}: per-tensor max|diff|/max|ref| worst {rel[-1][0]:.3g} "
          f"({rel[-1][1]}), median {rel[len(rel) // 2][0]:.3g}")
    for name, a, b, c in zip(names, got, ref, again):
        assert torch.equal(a, c), f"{name}: two backward passes differ"
        assert _rel(a, b) <= BACKBONE_GRAD_REL[tf32], (name, _rel(a, b))


def _train(cuda, steps, precision="fp32", seed=0):
    from nksr_b200 import training as T
    from nksr_b200.network import NKSRNetwork
    from tests import clouds
    xyz, nrm = clouds.sphere(60_000, noise=0.001)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    scene = T.TrainingScene(t(xyz), t(nrm), 0.02, 4)
    net = NKSRNetwork(dict(backbone="unet", tree_depth=4, kernel_dim=4, precision=precision, trainable=True,
                           seed=seed)).to(cuda)
    opt = T.make_optimizer(net)
    gen = torch.Generator(device=cuda).manual_seed(seed)
    curve = [tuple(float(v) for v in T.train_step(net, opt, scene, gen)) for _ in range(steps)]
    return net, scene, curve


# mean of the last three of 30 steps, measured on an H100 80GB HBM3 (700 W): structure 4.48 -> 2.09, UDF 0.433 -> 0.184
STRUCTURE_LOSS_AFTER_30 = 2.5
UDF_LOSS_AFTER_30 = 0.25


def test_training_lowers_the_losses_and_is_repeatable(cuda, tmp_path):
    from nksr_b200.network import NKSRNetwork, load_checkpoint_from_url
    torch.use_deterministic_algorithms(True, warn_only=True)      # the point encoder's index_add_ and gathers
    try:
        _training_checks(cuda, tmp_path, NKSRNetwork, load_checkpoint_from_url)
    finally:
        torch.use_deterministic_algorithms(False)


def _training_checks(cuda, tmp_path, NKSRNetwork, load_checkpoint_from_url):
    net, scene, curve = _train(cuda, 30)
    net2, _, curve2 = _train(cuda, 30)
    print("[train] structure", [round(c[0], 4) for c in curve])
    print("[train] udf", [round(c[1], 4) for c in curve])
    s_first, u_first = curve[0]
    s_last = sum(c[0] for c in curve[-3:]) / 3
    u_last = sum(c[1] for c in curve[-3:]) / 3
    assert s_last < STRUCTURE_LOSS_AFTER_30, (s_first, s_last)
    assert u_last < UDF_LOSS_AFTER_30, (u_first, u_last)
    assert curve == curve2
    for (n, a), b in zip(net.named_parameters(), net2.parameters()):
        assert torch.equal(a, b), f"{n}: two runs from one seed differ"
    # a checkpoint reloads into an identical forward
    path = str(tmp_path / "unet.pt")
    torch.save({"state_dict": net.state_dict()}, path)
    fresh = NKSRNetwork(dict(backbone="unet", tree_depth=4, kernel_dim=4, trainable=True, seed=7)).to(cuda)
    fresh.load_state_dict(load_checkpoint_from_url(path)["state_dict"])
    with torch.no_grad():
        a = net.backbone_net(net.encoder(scene.xyz, scene.normal, scene.enc_svh, 0).x0, scene.enc_svh)
        b = fresh.backbone_net(fresh.encoder(scene.xyz, scene.normal, scene.enc_svh, 0).x0, scene.enc_svh)
    for l in range(4):
        assert torch.equal(a.decoder[l], b.decoder[l]) and torch.equal(a.structure[l], b.structure[l])
