"""Memory and time of the global solve's two operators on one GPU (world 1 of dist_solve.reconstruct_global), on the
benchmark's cfg4 scene (bench.make_cloud, the bench's network, preprocess and solver settings):

    python tools/global_operator_bench.py [--points 5000000] [--big-points 10000000] [--runs 3] [--out out.json]

After one warm-up step of each, 'assembled' and 'matrix_free' alternate, `--runs` steps each.  Every step reports the
host time of the whole driver call (ending in a device synchronise), its stage marks (CUDA events), the PCG's
iterations and relative residual, and torch.cuda.max_memory_allocated over the step.  The last steps of the two
operators are compared on owned alpha and on query_f at points near the cloud.  With --big-points, matrix-free then
runs alone on a cloud of that size (its assembled system is not attempted).  The card's name, power limit and SM clock
are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import nksr_b200  # noqa: E402
from nksr_b200 import dist_solve  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        out = []
    return out[0] if out else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg4_outdoor_5M")
    ap.add_argument("--points", type=int, default=5_000_000)
    ap.add_argument("--big-points", type=int, default=0)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    os.environ["NKSR_STAGE_TIMES"] = "1"
    from nksr_b200.network import NKSRNetwork
    net = NKSRNetwork(dict(kernel_dim=bench.KERNEL_DIM, tree_depth=bench.TREE_DEPTH,
                           adaptive_depth=bench.ADAPTIVE_DEPTH, backbone="unet"))
    rec = nksr_b200.Reconstructor(dev, network=net, tree_depth=bench.TREE_DEPTH, adaptive_depth=bench.ADAPTIVE_DEPTH,
                                  kernel_dim=bench.KERNEL_DIM)
    prep = nksr_b200.get_estimate_normal_preprocess_fn(bench.KNN, bench.MAX_ANGLE)
    W = bench.WORKLOADS[args.workload]["voxel_size"]

    def step(xyz, sensor, op, q=None):
        """one driver call; returns its row and, for query points q, (alpha, f(q)) of the field, which is freed"""
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        t0 = time.perf_counter()
        f = dist_solve.reconstruct_global(rec, xyz, None, W, sensor=sensor, preprocess_fn=prep,
                                          approx_kernel_grad=bench.SOLVER["approx_kernel_grad"],
                                          solver_tol=bench.SOLVER["solver_tol"], operator=op)
        torch.cuda.synchronize()
        ms = 1e3 * (time.perf_counter() - t0)
        info = f.solve_info
        row = dict(operator=op, points=int(xyz.shape[0]), ms=round(ms, 2),
                   peak_gb=round(torch.cuda.max_memory_allocated(dev) / 1e9, 3),
                   iterations=info["iterations"], relative_residual=info["relative_residual"], n=info["n"],
                   nnz=info["nnz"], locations_kept=info.get("locations_kept"),
                   locations_total=info.get("locations_total"),
                   stages_ms={k: round(v, 2) for k, v in f._stage_timer.report().items() if k != "start"})
        print(json.dumps(row), flush=True)
        out = None if q is None else (f.alpha.clone(), f.evaluate_f(q).value.clone())
        del f
        return row, out

    def cloud(n, seed):
        xyz, sensor = bench.make_cloud(args.workload, seed, points=n)
        return xyz.to(dev), sensor.to(dev)

    result = {"gpu": gpu_info(), "workload": args.workload, "rows": []}
    print(json.dumps({"gpu": result["gpu"]}), flush=True)
    xyz, sensor = cloud(args.points, 4)
    g = torch.Generator(device="cpu").manual_seed(0)
    qi = torch.randint(0, xyz.shape[0], (200_000,), generator=g).to(dev)
    q = xyz[qi] + 0.5 * W * torch.randn(qi.shape[0], 3, generator=g).to(dev)
    ops = ("assembled", "matrix_free")
    for op in ops:                                       # warm-up
        step(xyz, sensor, op)
    last = {}
    for run in range(args.runs):
        for op in ops:
            row, out = step(xyz, sensor, op, q if run == args.runs - 1 else None)
            result["rows"].append(row)
            if out is not None:
                last[op] = out
    (a_as, fa), (a_mf, fm) = last["assembled"], last["matrix_free"]
    result["compare"] = dict(
        alpha_max_abs_diff=float((a_as - a_mf).abs().max()), alpha_max_abs=float(a_as.abs().max()),
        query_f_max_abs_diff=float((fa - fm).abs().max()), query_f_max_abs=float(fa.abs().max()))
    print(json.dumps(result["compare"]), flush=True)
    del last, a_as, a_mf, fa, fm
    torch.cuda.empty_cache()
    if args.big_points:
        del xyz, sensor
        torch.cuda.empty_cache()
        xyz, sensor = cloud(args.big_points, 4)
        step(xyz, sensor, "matrix_free")                 # warm-up at this size
        for _ in range(args.runs):
            result["rows"].append(step(xyz, sensor, "matrix_free")[0])
    result["gpu_after"] = gpu_info()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
