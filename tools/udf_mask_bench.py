"""Time the UDF neural field's interpolation kernels (csrc/neural_field.cu) against the plain-torch restatement
(NeuralField._interp) on the cfg4 1 M-point crop of tools/train_unet.py, with CUDA events.

    python tools/udf_mask_bench.py [--points 1000000] [--reps 5]

Prints one JSON line per measurement and a last line with the GPU's name and power limit:
  mask       the UDF mask's interpolation at the vertices of extract_dual_mesh(mise_iter=1) of the scene's
             reconstruction, kernel against torch (and the whole mask, decoder included, through the kernel);
  loss       forward and VJP of the interpolation at the 100 k UDF loss samples (deterministic algorithms, as in
             training), kernel against torch autograd;
  train      one train_step of the U-Net with udf.enabled (median of --reps after two warm-up steps).
Kernel and torch runs alternate within each measurement; medians are reported.  Every result stays on the device.
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


def timed(fn):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def alternate(fns, reps):
    """median ms of every function, the runs of the functions interleaved; one untimed warm-up of each"""
    for fn in fns.values():
        timed(fn)
    ms = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            ms[k].append(timed(fn)[0])
    return {k: round(statistics.median(v), 3) for k, v in ms.items()}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--depth", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("udf_mask_bench.py needs a CUDA device")
    import nksr_b200
    from bench import gpu_info
    from nksr_b200 import training as T
    from nksr_b200.fields import NeuralField
    from nksr_b200.network import NKSRNetwork
    from tools.train_unet import make_scene
    dev = torch.device("cuda:0")
    scene = make_scene("cfg4", args.points, args.depth, dev)
    W = scene.voxel_size
    net = NKSRNetwork(dict(backbone="unet", tree_depth=args.depth, kernel_dim=4, trainable=True,
                           udf=dict(enabled=True))).to(dev)
    # mask: the UDF field of the network on the scene, at the vertices of the scene's (pool-backbone) reconstruction
    with torch.no_grad():
        rec = nksr_b200.Reconstructor(dev, tree_depth=args.depth)
        field = rec.reconstruct(scene.xyz, scene.normal, voxel_size=W)
        field.set_mask_field(None)
        v = field.extract_dual_mesh(mise_iter=1).v.contiguous()
        del field
        feat, _, udf_svh = net.unet(net.encoder(scene.xyz, scene.normal, scene.enc_svh, 0), scene.enc_svh,
                                    adaptive_depth=scene.adaptive_depth)
        nf = NeuralField(udf_svh, net.udf_decoder, feat.udf_features)
        nf.set_level_set(2 * W)
        u_k, u_t = nf.interpolate(v), nf._interp(v)
        diff = float((u_k - u_t).abs().max())
        ms = alternate({"kernel": lambda: nf.interpolate(v), "torch": lambda: nf._interp(v),
                        "mask_kernel": lambda: nf.mask(v)}, args.reps)
    print(json.dumps(dict(measure="mask", vertices=int(v.shape[0]), columns=int(u_k.shape[1]),
                          voxels=[udf_svh.num_voxels(l) for l in range(udf_svh.depth)], max_abs_diff=diff,
                          interp_kernel_ms=ms["kernel"], interp_torch_ms=ms["torch"],
                          mask_kernel_ms=ms["mask_kernel"], speedup=round(ms["torch"] / ms["kernel"], 2))), flush=True)
    del v, u_k, u_t
    # loss: forward and VJP at the UDF samples, under deterministic algorithms as in training
    torch.use_deterministic_algorithms(True, warn_only=True)
    gen = torch.Generator(device=dev).manual_seed(0)
    q = T.udf_samples(udf_svh, scene.xyz, scene.normal, W, generator=gen).contiguous()
    feats = {l: f.detach().clone().requires_grad_(True) for l, f in feat.udf_features.items()}
    nfg = NeuralField(udf_svh, net.udf_decoder, feats)
    g = torch.randn((q.shape[0], nfg.channels * len(nfg.levels)), device=dev, generator=gen)

    def bwd(interp):
        def run():
            for f in feats.values():
                f.grad = None
            interp(q).backward(g)
            return [feats[l].grad for l in nfg.levels]
        return run
    ms_f = alternate({"kernel": lambda: nfg.interpolate(q), "torch": lambda: nfg._interp(q)}, args.reps)
    ms_b = alternate({"kernel": bwd(nfg.interpolate), "torch": bwd(nfg._interp)}, args.reps)
    dk, dt = bwd(nfg.interpolate)(), bwd(nfg._interp)()
    rel = max(float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30) for a, b in zip(dk, dt))
    print(json.dumps(dict(measure="loss", samples=int(q.shape[0]), forward_kernel_ms=ms_f["kernel"],
                          forward_torch_ms=ms_f["torch"], forward_plus_vjp_kernel_ms=ms_b["kernel"],
                          forward_plus_vjp_torch_ms=ms_b["torch"], vjp_max_rel_diff=rel)), flush=True)
    # train: one step with udf.enabled
    opt = T.make_optimizer(net)
    tgen = torch.Generator(device=dev).manual_seed(0)
    steps = []
    for i in range(2 + args.reps):
        t, out = timed(lambda: T.train_step(net, opt, scene, tgen))
        if i >= 2:
            steps.append(t)
    print(json.dumps(dict(measure="train", train_step_ms=round(statistics.median(steps), 3),
                          udf_loss=round(float(out[1]), 6))), flush=True)
    torch.use_deterministic_algorithms(False)
    print(json.dumps(dict(gpu_info(0), points=int(scene.xyz.shape[0]), voxel_size=W, depth=args.depth)), flush=True)


if __name__ == "__main__":
    main()
