"""Time the neural output field (geometry='neural'): the position Jacobian kernels of the interpolation
(csrc/neural_field.cu) against the plain-torch restatement, a training step and a reconstruction, with CUDA events.

    python tools/neural_geometry_bench.py [--points 1000000] [--reps 5]

Prints one JSON line per measurement and a last line with the GPU's name and power limit:
  jacobian   at 50 k, 100 k and 1 M queries uniform over the voxels of the cfg4 1 M-point crop of tools/train_unet.py
             (4 levels, C = 4, the U-Net's basis features): the Jacobian kernel alone and with its VJP; and the position
             gradient of a decoder with its graph (evaluate_f(grad=True) with position_gradient) and then the backward of
             a loss on it, against torch autograd through NeuralField._interp with create_graph, then backward;
  train      one train_step(kernel=True) with geometry='neural' against 'kernel' on the 30 k-point sphere of
             tests/test_gpu_kernel_training.py (depth 4, W = 0.02);
  reconstruct  reconstruct + extract_dual_mesh(mise_iter=1) of the cfg4 crop with geometry='neural' (random decoder).
The compared runs alternate within each measurement; medians are reported.  Every result stays on the device.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

from tools.udf_mask_bench import alternate, timed  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--depth", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="50000,100000,1000000")
    args = ap.parse_args(argv)
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("neural_geometry_bench.py needs a CUDA device")
    import nksr_b200
    from bench import gpu_info
    from nksr_b200 import training as T
    from nksr_b200.fields import NeuralField, SparseFeatureHierarchyCoords
    from nksr_b200.network import NKSRNetwork
    from tests import clouds
    from tools.train_unet import make_scene
    dev = torch.device("cuda:0")
    torch.use_deterministic_algorithms(True, warn_only=True)
    scene = make_scene("cfg4", args.points, args.depth, dev)
    W = scene.voxel_size
    net = NKSRNetwork(dict(backbone="unet", tree_depth=args.depth, kernel_dim=4, trainable=True,
                           geometry="neural")).to(dev)
    with torch.no_grad():
        feat, dec_svh, _ = net.unet(net.encoder(scene.xyz, scene.normal, scene.enc_svh, 0), scene.enc_svh,
                                    adaptive_depth=scene.adaptive_depth)
    feats = {l: f.detach().clone().requires_grad_(True) for l, f in feat.basis_features.items()}
    nf = NeuralField(dec_svh, net.sdf_decoder, feats, position_gradient=True)
    params = list(feats.values()) + list(net.sdf_decoder.parameters())
    gen = torch.Generator(device=dev).manual_seed(0)
    for m in (int(s) for s in args.sizes.split(",")):
        q = T.svh_samples(dec_svh, m, 1, 3, gen).contiguous()
        r = torch.randn((m, 3), device=dev, generator=gen)
        gj = torch.randn((m, 3, nf.channels * len(nf.levels)), device=dev, generator=gen)

        def jac_fwd():
            with torch.no_grad():
                return nf.jacobian(q)

        def jac_fwd_vjp():
            return torch.autograd.grad(nf.jacobian(q), list(feats.values()), gj)

        def torch_grad():
            qq = q.clone().requires_grad_(True)
            v = net.sdf_decoder(nf._interp(qq)).reshape(-1)
            return torch.autograd.grad(v.sum(), qq, create_graph=True)[0]

        def cuda_grad():
            return nf.evaluate_f(q, grad=True).gradient

        def backward(grad_fn):
            def run():
                # (the last layer's bias does not reach the gradient)
                return torch.autograd.grad((grad_fn() * r).sum(), params, allow_unused=True)
            return run
        ms_j = alternate({"fwd": jac_fwd, "fwd_vjp": jac_fwd_vjp}, args.reps)
        ms_g = alternate({"cuda": cuda_grad, "torch": torch_grad}, args.reps)
        ms_b = alternate({"cuda": backward(cuda_grad), "torch": backward(torch_grad)}, args.reps)
        gk, gt = cuda_grad(), torch_grad()
        # the torch restatement takes the one-sided tent derivative also in the snap zone |tau| < 2^-12 around voxel
        # centres, where the kernel takes the symmetric one (SPEC S4): compare the gradients outside it
        far = torch.ones(m, dtype=torch.bool, device=dev)
        base = dec_svh.locate(q).long()
        for l in range(dec_svh.depth):
            ijk = SparseFeatureHierarchyCoords.ijk(dec_svh, l)[base[l].clamp(min=0)].double()
            tau = q.double() / (dec_svh.voxel_size * 2 ** l) - (ijk + 0.5)
            far &= (base[l] < 0) | (tau.abs() > 2.0 ** -11).all(dim=1)
        dk, dt = backward(cuda_grad)(), backward(torch_grad)()
        rel = max(float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30) for a, b in zip(dk, dt)
                  if b is not None)
        print(json.dumps(dict(measure="jacobian", queries=m, columns=nf.channels * len(nf.levels),
                              voxels=[dec_svh.num_voxels(l) for l in range(dec_svh.depth)],
                              jacobian_kernel_ms=ms_j["fwd"], jacobian_plus_vjp_kernel_ms=ms_j["fwd_vjp"],
                              gradient_cuda_ms=ms_g["cuda"], gradient_torch_ms=ms_g["torch"],
                              gradient_plus_backward_cuda_ms=ms_b["cuda"],
                              gradient_plus_backward_torch_ms=ms_b["torch"],
                              speedup=round(ms_b["torch"] / ms_b["cuda"], 2),
                              snap_zone_queries=int((~far).sum()),
                              gradient_max_abs_diff_outside_snap=float((gk - gt)[far].abs().max()),
                              gradient_max_abs=float(gt.abs().max()), backward_max_rel_diff=rel)), flush=True)
        del q, r, gj, gk, gt, dk, dt
    del feats, nf, params, feat
    torch.cuda.empty_cache()
    # train: one step of the field losses, neural against kernel, on the sphere scene of the kernel training test
    xyz, nrm = clouds.sphere(30_000, noise=0.001)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    sphere = T.TrainingScene(t(xyz), t(nrm), 0.02, 4)
    runs = {}
    for geometry in ("neural", "kernel"):
        n2 = NKSRNetwork(dict(backbone="unet", tree_depth=4, kernel_dim=4, trainable=True, seed=3,
                              geometry=geometry)).to(dev)
        opt = T.make_optimizer(n2)
        g2 = torch.Generator(device=dev).manual_seed(3)
        runs[geometry] = (lambda n2=n2, opt=opt, g2=g2: T.train_step(n2, opt, sphere, g2, kernel=True))
    for fn in runs.values():
        fn()
    ms = alternate(runs, args.reps)
    print(json.dumps(dict(measure="train", points=int(sphere.xyz.shape[0]), train_step_neural_ms=ms["neural"],
                          train_step_kernel_ms=ms["kernel"])), flush=True)
    torch.use_deterministic_algorithms(False)
    # reconstruct + mesh with geometry='neural'
    rnet = NKSRNetwork(dict(backbone="unet", tree_depth=args.depth, kernel_dim=4, geometry="neural")).to(dev)
    rec = nksr_b200.Reconstructor(dev, network=rnet, tree_depth=args.depth)

    def recon():
        with torch.no_grad():
            return rec.reconstruct(scene.xyz, scene.normal, voxel_size=W).extract_dual_mesh(mise_iter=1)
    ms = alternate({"neural": recon}, args.reps)
    mesh = recon()
    print(json.dumps(dict(measure="reconstruct", points=int(scene.xyz.shape[0]), reconstruct_mesh_neural_ms=ms["neural"],
                          vertices=int(mesh.v.shape[0]), faces=int(mesh.f.shape[0]))), flush=True)
    print(json.dumps(dict(gpu_info(0), points=int(scene.xyz.shape[0]), voxel_size=W, depth=args.depth)), flush=True)


if __name__ == "__main__":
    main()
