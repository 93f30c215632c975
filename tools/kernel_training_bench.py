"""Kernel-loss training step on the assembled against the matrix-free operator (train_step(kernel=True, operator=...)).

    python tools/kernel_training_bench.py --points 1000000 --large 5000000 --steps 3 --warmup 1

The scene is the cfg4 crop of tools/train_unet.py --scene cfg4 with the U-Net backbone (depth 4, kernel_dim 4, fp32),
trained with the structure, UDF and kernel-field losses, once with approx_kernel_grad False (the reference's training
setting) and once with True.  Each case builds one network per operator from the same seed, and the two take their
steps alternately, so that both see the same machine state.  One JSON line per step gives the forward, backward and
optimizer-step times (CUDA events), the kernel solve's stages (StageTimer), the peak allocated memory of the step and
the forward / adjoint PCG iteration counts.  The per-case summary gives:
  - the medians over the steps after the warm-up;
  - the relative difference of the parameter gradients between the operators at step 0 (the same weights and samples,
    the gradients as the optimizer saw them, after clipping);
  - the constraint values the matrix-free backward needs (E_j alpha, E_j lambda at every constraint location) read from
    the kernel rows by nksr_op_constraint_values, against the four nksr_evaluate calls of the assembled backward, each
    timed with CUDA events over --reps repetitions on the step's system, with the largest difference between the two.
With --large N, one matrix-free training step (approx_kernel_grad False) on an N-point crop follows; the assembled
operator is not run there.  If it does not fit on the card, the allocator's message is reported.  The first line names
the GPU with its power limit and SM clocks, read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

SOLVE_STAGES = ("kernel_rows", "gram_count", "gram_blocks", "gram_fill", "operator_setup", "pcg")


def gpu_clocks():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        sm, sm_max = (t.strip() for t in q.split(",")[:2])
        return {"sm_clock": sm, "sm_clock_max": sm_max}
    except (OSError, ValueError, subprocess.TimeoutExpired):
        return {"sm_clock": None, "sm_clock_max": None}


class Recorder:
    """keeps the KernelField of the last kernel_field() call (its solve_info holds the iteration counts), and builds
    every training KernelField with the case's approx_kernel_grad"""

    def __init__(self, T, approx):
        from nksr_b200.fields import KernelField
        self.T, self.last = T, None
        self._orig_field, self._orig_cls = T.kernel_field, T.KernelField

        class Field(KernelField):
            def __init__(self, *a, **k):
                super().__init__(*a, approx_kernel_grad=approx, **k)

        def kernel_field(*a, **k):
            self.last = self._orig_field(*a, **k)
            return self.last
        T.kernel_field, T.KernelField = kernel_field, Field

    def close(self):
        self.T.kernel_field, self.T.KernelField = self._orig_field, self._orig_cls


def timed_step(T, net, opt, scene, gen, operator, rec):
    import torch
    from nksr_b200._lib import StageTimer
    dev = scene.xyz.device
    ev = {"start": torch.cuda.Event(enable_timing=True)}

    def marks(name):
        ev[name] = torch.cuda.Event(enable_timing=True)
        ev[name].record()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    stages = StageTimer(dev, enabled=True)
    ev["start"].record()
    _, _, k = T.train_step(net, opt, scene, gen, marks, kernel=True, timer=stages, operator=operator)
    torch.cuda.synchronize()
    st = stages.report()
    info = rec.last.solve_info
    rec.last = None
    row = dict(operator=operator,
               forward_ms=round(ev["start"].elapsed_time(ev["forward"]), 3),
               backward_ms=round(ev["forward"].elapsed_time(ev["backward"]), 3),
               step_ms=round(ev["backward"].elapsed_time(ev["step"]), 3),
               solve_ms=round(sum(st.get(s, 0.0) for s in SOLVE_STAGES), 3),
               stages_ms={s: round(float(v), 3) for s, v in st.items() if s != "start"},
               peak_gb=round(torch.cuda.max_memory_allocated(dev) / 1e9, 3),
               pcg_iterations=info.get("iterations"), adjoint_iterations=info.get("adjoint_iterations"),
               nnz=info.get("nnz"), unknowns=info.get("n"),
               losses={key: round(float(v), 6) for key, v in k.items()})
    return row


def constraint_values_ab(T, net, scene, approx, reps):
    """the step's system at the current weights, without grad: nksr_op_constraint_values against four nksr_evaluate
    calls at the same sorted locations, for alpha and a second vector"""
    import torch
    from nksr_b200.fields import KernelField
    with torch.no_grad():
        enc = net.encoder(scene.xyz, scene.normal, scene.enc_svh, 0)
        feat, dec_svh, _ = net.unet(enc, scene.enc_svh, adaptive_depth=scene.adaptive_depth)
        field = KernelField(dec_svh, net.interpolators, feat.basis_features, approx)
        ad = min(scene.adaptive_depth, dec_svh.depth)
        nxyz = torch.cat([dec_svh.get_voxel_centers(d) for d in range(ad)])
        nval = -torch.cat([feat.normal_features[d] for d in range(ad)])
        nw = T.NORMAL_WEIGHT / nxyz.shape[0] * (scene.voxel_size ** 2)
        op = field.matrix_free_system(scene.xyz, nxyz, nval, T.POS_WEIGHT / scene.xyz.shape[0], nw, 1.0,
                                      keep_constraints=True)
        alpha = field._pcg_matrix_free(op, op.rhs)
        lam = torch.randn(op.n, device=alpha.device, generator=torch.Generator(device=alpha.device).manual_seed(0))
        xs, xn = op.cons.pos[0], op.cons.nrm[0]

        def rows():
            return field.constraint_values(op, alpha, lam)

        def evaluate():
            fa, _ = field._evaluate(alpha, xs, False)
            fl, _ = field._evaluate(lam, xs, False)
            _, ga = field._evaluate(alpha, xn, True)
            _, gl = field._evaluate(lam, xn, True)
            return torch.stack([fa, fl], 1), torch.stack([ga, gl], 1)

        out = {}
        for name, fn in (("rows", rows), ("evaluate", evaluate)) * 2:        # the first round warms up
            fn()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            out[name] = e0.elapsed_time(e1) / reps
        (vp, vn), (ep, en) = rows(), evaluate()
        rel = lambda a, b: float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))
        return dict(constraint_values_ms=round(out["rows"], 4), four_evaluate_ms=round(out["evaluate"], 4),
                    positions=int(xs.shape[0]), normal_locations=int(xn.shape[0]),
                    max_rel_diff_positions=rel(vp, ep), max_rel_diff_normals=rel(vn, en))


def grad_diff(ga, gb):
    """relative difference of two parameter-gradient dicts: over all parameters, and the worst single parameter"""
    import torch
    num = torch.sqrt(sum(((ga[k] - gb[k]) ** 2).sum() for k in gb))
    den = torch.sqrt(sum((gb[k] ** 2).sum() for k in gb))
    worst = max(float((ga[k] - gb[k]).norm() / gb[k].norm().clamp_min(1e-30)) for k in gb)
    return dict(all=float(num / den), worst_parameter=worst)


def run_case(args, T, approx, scene, dev):
    import torch
    from nksr_b200.network import NKSRNetwork
    rec = Recorder(T, approx)
    try:
        ops = ("assembled", "matrix_free")
        nets, opts, gens = {}, {}, {}
        for op in ops:
            nets[op] = NKSRNetwork(dict(backbone="unet", tree_depth=args.depth, kernel_dim=4, precision="fp32",
                                        trainable=True, seed=args.seed)).to(dev)
            opts[op] = T.make_optimizer(nets[op])
            gens[op] = torch.Generator(device=dev).manual_seed(args.seed)
        rows, grads0 = {op: [] for op in ops}, {}
        for step in range(args.warmup + args.steps):
            for op in (ops if step % 2 == 0 else ops[::-1]):
                row = timed_step(T, nets[op], opts[op], scene, gens[op], op, rec)
                row.update(step=step, approx_kernel_grad=approx)
                print(json.dumps(row), flush=True)
                rows[op].append(row)
                if step == 0:
                    grads0[op] = {n: p.grad.detach().clone() for n, p in nets[op].named_parameters()
                                  if p.grad is not None}
        summary = dict(approx_kernel_grad=approx, points=int(scene.xyz.shape[0]))
        for op in ops:
            timed = rows[op][args.warmup:]
            med = lambda key: round(statistics.median(r[key] for r in timed), 3)
            stage_names = sorted({s for r in timed for s in r["stages_ms"]})
            summary[op] = dict({k: med(k) for k in ("forward_ms", "backward_ms", "step_ms", "solve_ms", "peak_gb")},
                               stages_ms={s: round(statistics.median(r["stages_ms"].get(s, 0.0) for r in timed), 3)
                                          for s in stage_names},
                               pcg_iterations=[r["pcg_iterations"] for r in timed],
                               adjoint_iterations=[r["adjoint_iterations"] for r in timed])
        summary["grad_rel_diff_step0"] = grad_diff(grads0["matrix_free"], grads0["assembled"])
        summary["constraint_values"] = constraint_values_ab(T, nets["matrix_free"], scene, approx, args.reps)
        print(json.dumps(dict(summary=summary)), flush=True)
        del nets, opts
    finally:
        rec.close()
    torch.cuda.empty_cache()


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=int, default=1_000_000)
    ap.add_argument("--large", type=int, default=0, help="points of the one matrix-free step (0: none)")
    ap.add_argument("--depth", type=int, default=4)
    ap.add_argument("--steps", type=int, default=3, help="timed steps per operator after the warm-up")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=20, help="repetitions of the constraint-value timings")
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--approx", choices=("both", "false", "true"), default="both")
    args = ap.parse_args(argv)
    if args.steps < 1 or args.warmup < 0:
        ap.error("--steps >= 1 and --warmup >= 0")
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("kernel_training_bench.py needs a CUDA device")
    from bench import gpu_info
    from nksr_b200 import training as T
    from tools.train_unet import make_scene
    torch.use_deterministic_algorithms(True, warn_only=True)
    dev = torch.device("cuda:0")
    print(json.dumps(dict(gpu=dict(gpu_info(0), **gpu_clocks()))), flush=True)
    scene, _ = make_scene("cfg4", args.points, args.depth, dev)
    print(json.dumps(dict(setup=dict(points=int(scene.xyz.shape[0]), voxel_size=scene.voxel_size, depth=args.depth,
                                     voxels=[scene.enc_svh.num_voxels(l) for l in range(args.depth)]))), flush=True)
    for approx in {"both": (False, True), "false": (False,), "true": (True,)}[args.approx]:
        run_case(args, T, approx, scene, dev)
    del scene
    torch.cuda.empty_cache()
    if args.large:
        from nksr_b200.network import NKSRNetwork
        scene, _ = make_scene("cfg4", args.large, args.depth, dev)
        rec = Recorder(T, False)
        try:
            net = NKSRNetwork(dict(backbone="unet", tree_depth=args.depth, kernel_dim=4, precision="fp32",
                                   trainable=True, seed=args.seed)).to(dev)
            opt = T.make_optimizer(net)
            gen = torch.Generator(device=dev).manual_seed(args.seed)
            row = timed_step(T, net, opt, scene, gen, "matrix_free", rec)
            row.update(points=int(scene.xyz.shape[0]), approx_kernel_grad=False,
                       voxels=[scene.enc_svh.num_voxels(l) for l in range(args.depth)])
            print(json.dumps(dict(large=row)), flush=True)
        except torch.cuda.OutOfMemoryError as e:
            print(json.dumps(dict(large=dict(points=int(scene.xyz.shape[0]), operator="matrix_free",
                                             out_of_memory=str(e).splitlines()[0]))), flush=True)
        finally:
            rec.close()
    print(json.dumps(dict(gpu_after=gpu_clocks())), flush=True)


if __name__ == "__main__":
    main()
