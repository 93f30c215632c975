"""Score and time the mesh-quality evaluator (nksr_b200.metrics.MeshEvaluator) on bench.py's scenes.

    python tools/metrics_bench.py --out DIR [--reps 3] [--workloads dev_outdoor_1M cfg3_indoor_1M]

For every workload: bench.py's generator draws the input cloud (seed 4) and bench.py's solver settings reconstruct it
(pool backbone, kNN normals, tree depth 4), then extract_dual_mesh(mise_iter=1).  The ground truth is a second
seeded draw of the same scene (seed 5): a noisy LiDAR-like sample, not the analytic surface, with kNN-PCA normals.
eval_mesh is timed at n_points = 5e5 and 5e6 with CUDA events after one warm-up, split into the sampling, the two
nearest-neighbour passes (hash build included) and the reductions (median of --reps).  The oracle
(oracle/metrics.py: scipy cKDTree in fp64, workers=-1) is timed on the same samples, with the host's core count.
Writes DIR/metrics_bench.json with the GPU's name and power limit, and prints it.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def reconstruct(bench, workload, dev):
    import torch
    import nksr_b200
    cfg = bench.WORKLOADS[workload]
    xyz, sensor = bench.make_cloud(workload, 4)
    rec = nksr_b200.Reconstructor(dev, tree_depth=bench.TREE_DEPTH, adaptive_depth=bench.ADAPTIVE_DEPTH,
                                  kernel_dim=bench.KERNEL_DIM)
    prep = nksr_b200.get_estimate_normal_preprocess_fn(bench.KNN, bench.MAX_ANGLE)
    field = rec.reconstruct(xyz.to(dev), sensor=sensor.to(dev), voxel_size=cfg["voxel_size"], preprocess_fn=prep,
                            **bench.SOLVER)
    mesh = field.extract_dual_mesh(mise_iter=1)
    torch.cuda.synchronize(dev)
    return mesh


def ground_truth(bench, workload, dev):
    from nksr_b200.reconstructor import estimate_normals_knn
    xyz, sensor = bench.make_cloud(workload, 5)
    r = estimate_normals_knn(xyz.to(dev), sensor.to(dev), knn=bench.KNN)
    return r.xyz, r.normal


def time_gpu(mesh, gt, gt_n, n, reps):
    """median ms of each phase of eval_mesh over `reps` runs after one warm-up; the last run's samples and metrics"""
    import torch
    from nksr_b200 import metrics as M
    phases = ("sample", "nn_completeness", "nn_accuracy", "reduce")
    ms = {k: [] for k in phases + ("total",)}
    for rep in range(reps + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(phases) + 1)]
        ev[0].record()
        xyz, nrm, _ = M.sample_surface(mesh.v, mesh.f, n, seed=0)
        ev[1].record()
        comp, _, cdot = M.nearest_neighbours(gt, xyz, gt_n, nrm)
        ev[2].record()
        acc, _, adot = M.nearest_neighbours(xyz, gt, nrm, gt_n)
        ev[3].record()
        out = M.summarise(comp, cdot, acc, adot)
        ev[4].record()
        torch.cuda.synchronize()
        if rep:
            for k, a, b in zip(phases, ev[:-1], ev[1:]):
                ms[k].append(a.elapsed_time(b))
            ms["total"].append(ev[0].elapsed_time(ev[-1]))
    return {k: round(statistics.median(v), 3) for k, v in ms.items()}, xyz, nrm, out


def time_oracle(xyz, nrm, gt, gt_n):
    from oracle import metrics as OM
    t0 = time.perf_counter()
    comp, _, cdot = OM.nearest(gt, xyz, gt_n, nrm)
    t1 = time.perf_counter()
    acc, _, adot = OM.nearest(xyz, gt, nrm, gt_n)
    t2 = time.perf_counter()
    out = OM.summarise(comp, cdot, acc, adot)
    t3 = time.perf_counter()
    return {"nn_completeness": round(1e3 * (t1 - t0), 1), "nn_accuracy": round(1e3 * (t2 - t1), 1),
            "reduce": round(1e3 * (t3 - t2), 1), "total_without_sampling": round(1e3 * (t3 - t0), 1)}, out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workloads", nargs="+", default=["dev_outdoor_1M", "cfg3_indoor_1M"])
    ap.add_argument("--n-points", type=float, nargs="+", default=[5e5, 5e6])
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("metrics_bench.py needs a CUDA device")
    import bench
    dev = torch.device("cuda", 0)
    res = {"gpu": bench.gpu_info(0), "host_cores": os.cpu_count(),
           "host_cores_usable": len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else None,
           "ground_truth": "a second seeded draw of the scene (seed 5) with kNN-PCA normals: noisy, not analytic",
           "runs": []}
    for wl in args.workloads:
        mesh = reconstruct(bench, wl, dev)
        gt, gt_n = ground_truth(bench, wl, dev)
        gt_np, gtn_np = gt.cpu().numpy(), gt_n.cpu().numpy()
        for n in (int(x) for x in args.n_points):
            gpu_ms, xyz, nrm, gpu_out = time_gpu(mesh, gt, gt_n, n, args.reps)
            ora_ms, ora_out = time_oracle(xyz.cpu().numpy(), nrm.cpu().numpy(), gt_np, gtn_np)
            run = {"workload": wl, "n_points": n, "gt_points": int(gt.shape[0]), "mesh_vertices": int(mesh.v.shape[0]),
                   "mesh_triangles": int(mesh.f.shape[0]), "gpu_ms": gpu_ms, "oracle_ckdtree_ms": ora_ms,
                   "nn_speedup": round((ora_ms["nn_completeness"] + ora_ms["nn_accuracy"]) /
                                       (gpu_ms["nn_completeness"] + gpu_ms["nn_accuracy"]), 1),
                   "metrics": {k: gpu_out[k] for k in ("chamfer-L1", "chamfer-L2", "f-score", "f-score-20",
                                                       "f-score-outdoor", "normals")},
                   "max_abs_diff_vs_oracle": max(abs(gpu_out[k] - ora_out[k]) for k in gpu_out
                                                 if gpu_out[k] == gpu_out[k])}
            print(json.dumps(run), flush=True)
            res["runs"].append(run)
        del mesh, gt, gt_n
        torch.cuda.empty_cache()
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "metrics_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({"gpu": res["gpu"], "host_cores": res["host_cores"],
                      "host_cores_usable": res["host_cores_usable"]}))


if __name__ == "__main__":
    main()
