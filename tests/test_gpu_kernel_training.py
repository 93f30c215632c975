"""Training through the kernel solve (nksr_b200/training.py, train_step(kernel=True)): 30 seeded Adam steps of the
sparse-conv U-Net with the structure, UDF and kernel-field losses.  Every basis-head row and interpolator parameter of a
non-empty level gets a finite, nonzero gradient, the kernel losses go down, and two runs from one seed match bitwise."""
import numpy as np
import pytest
import torch

from tests import clouds

pytestmark = pytest.mark.gpu

STEPS = 30


def _train(cuda, seed=3):
    from nksr_b200 import training as T
    from nksr_b200.network import NKSRNetwork
    xyz, nrm = clouds.sphere(30_000, noise=0.001)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    scene = T.TrainingScene(t(xyz), t(nrm), 0.02, 4)
    net = NKSRNetwork(dict(backbone="unet", tree_depth=4, kernel_dim=4, trainable=True, seed=seed)).to(cuda)
    opt = T.make_optimizer(net)
    gen = torch.Generator(device=cuda).manual_seed(seed)
    curve, grads = [], None
    for step in range(STEPS):
        _, _, k = T.train_step(net, opt, scene, gen, kernel=True)
        curve.append({key: float(v) for key, v in k.items()})
        if step == 0:
            grads = {name: p.grad.detach().clone() for name, p in net.named_parameters() if p.grad is not None}
    return net, scene, curve, grads


def test_kernel_training_reaches_the_heads_lowers_the_losses_and_is_repeatable(cuda):
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        net, scene, curve, grads = _train(cuda)
        net2, _, curve2, grads2 = _train(cuda)
    finally:
        torch.use_deterministic_algorithms(False)
    C, ad = net.kernel_dim, scene.adaptive_depth
    for l in range(net.tree_depth):
        assert scene.enc_svh.num_voxels(l) > 0
        w = grads[f"backbone_net.heads.{l}.weight"]
        basis = w[6:6 + C]
        assert bool(torch.isfinite(basis).all()) and bool((basis.abs().sum(dim=1) > 0).all()), f"basis head {l}"
        if l < ad:                                      # normal constraints on the adaptive_depth finest levels
            assert float(w[3:6].abs().sum()) > 0, f"normal head {l}"
        for name, g in grads.items():
            if name.startswith(f"interpolators.{l}."):
                assert bool(torch.isfinite(g).all()) and float(g.abs().sum()) > 0, name
        assert any(n.startswith(f"interpolators.{l}.") for n in grads)
    first = np.mean([c["total"] for c in curve[:3]])
    last = np.mean([c["total"] for c in curve[-3:]])
    print(f"[train] kernel losses: first {curve[0]} last {curve[-1]}; total mean of 3 {first:.5g} -> {last:.5g}")
    assert last < first
    assert curve == curve2
    assert all(torch.equal(a, b) for a, b in zip(net.state_dict().values(), net2.state_dict().values()))
    assert grads.keys() == grads2.keys() and all(torch.equal(grads[k], grads2[k]) for k in grads)
