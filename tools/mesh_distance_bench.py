"""Time the closest-triangle query (nksr_b200.metrics.MeshOccupancy.closest / signed_distance, csrc/raycast.cu
k_mesh_closest; DESIGN.md SPEC S21).

    python tools/mesh_distance_bench.py --out DIR [--reps 5]

Workloads: an icosphere of 1.31 M triangles (level 8, R = 1, W = 0.02) with 1 M queries; the dual-MC mesh of bench.py's
cfg3 indoor scene at 1 M points (reconstructed as tools/metrics_bench.py does, W its voxel size) with 1 M queries; a
ShapeNet-sized case, an icosphere of 81,920 triangles (level 6, R = 0.5, W = 0.01) with 100 k queries.  Two query
sets (seed 0): uniform in the mesh's bounding box padded by 10 % per side, and a band of +-2 W around the surface
(area-uniform surface samples moved along their normals by a uniform offset in [-2 W, 2 W]).  The build is timed as
in tools/occupancy_bench.py, then `closest` and `signed_distance` with K = 1 and 3; every number is the median of
--reps runs after one warm-up, timed with CUDA events.  The brute force (tests/distance_oracle.py, numpy) is checked
against the GPU bit for bit on an 8-query subsample of each set.  Writes DIR/mesh_distance_bench.json with the GPU's
name and power limit, read in the same run.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

N_ORACLE = 8


def timed(fn, reps):
    """median CUDA-event time of fn() over reps runs after one warm-up, and its last result"""
    import torch
    ms, out = [], None
    for rep in range(reps + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        if rep:
            ms.append(a.elapsed_time(b))
    return round(statistics.median(ms), 3), out


def run_workload(name, v, f, W, m, reps):
    import numpy as np
    import torch
    from nksr_b200.metrics import sample_surface
    from tests import distance_oracle as D
    from tools.occupancy_bench import build_timed, median_dict
    dev = v.device
    f = f.to(torch.int32).contiguous()
    v = v.to(torch.float32).contiguous()
    builds = [build_timed(v, f) for _ in range(reps + 1)]
    occ = builds[-1][1]
    res = {"workload": name, "triangles": int(f.shape[0]), "W": W,
           "build_ms": median_dict([b[0] for b in builds[1:]]), "query": []}
    lo, hi = v.min(0).values, v.max(0).values
    g = torch.Generator(device=dev).manual_seed(0)
    uniform = lo - 0.1 * (hi - lo) + torch.rand((m, 3), generator=g, device=dev) * 1.2 * (hi - lo)
    xyz, nrm, _ = sample_surface(v, f, m, seed=0)
    band = xyz + nrm * ((torch.rand((m, 1), generator=g, device=dev) * 2.0 - 1.0) * 2.0 * W)
    for qname, q in (("uniform", uniform), ("band_2W", band)):
        row = {"queries": qname, "m": m}
        row["closest_ms"], (dist, point, tri) = timed(lambda: occ.closest(q), reps)
        for k in (1, 3):
            row[f"signed_distance_k{k}_ms"], _ = timed(lambda: occ.signed_distance(q, k), reps)
        row["queries_per_s_closest"] = float(f"{m / (row['closest_ms'] * 1e-3):.4g}")
        row["median_distance"] = round(float(dist.median()), 6)
        sub = torch.randperm(m, generator=g, device=dev)[:N_ORACLE]
        want = D.mesh_closest(v.cpu().numpy(), f.cpu().numpy(), q[sub].cpu().numpy())
        got = (dist[sub].cpu().numpy(), point[sub].cpu().numpy(), tri[sub].cpu().numpy())
        row["oracle_equal"] = all(np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a,
                                                 b.view(np.uint32) if b.dtype == np.float32 else b)
                                  for a, b in zip(got, want))
        res["query"].append(row)
        print(json.dumps({"workload": name, **row}), flush=True)
    print(json.dumps({"workload": name, "build_ms": res["build_ms"]}), flush=True)
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workloads", nargs="+", default=["icosphere8", "cfg3_indoor_1M", "shapenet"])
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mesh_distance_bench.py needs a CUDA device")
    import bench
    from tests.test_cpu_occupancy import icosphere
    dev = torch.device("cuda", 0)
    res = {"gpu": bench.gpu_info(0), "runs": []}
    t = lambda a: torch.from_numpy(a).to(dev)
    for wl in args.workloads:
        if wl == "icosphere8":
            v, f = icosphere(8)
            res["runs"].append(run_workload(wl, t(v), t(f), 0.02, 1_000_000, args.reps))
        elif wl == "shapenet":
            v, f = icosphere(6, 0.5)
            res["runs"].append(run_workload("shapenet_82k", t(v), t(f), 0.01, 100_000, args.reps))
        else:
            from tools.metrics_bench import reconstruct
            mesh = reconstruct(bench, wl, dev)
            W = float(bench.WORKLOADS[wl]["voxel_size"])
            res["runs"].append(run_workload(f"{wl}_dual_mc", mesh.v, mesh.f, W, 1_000_000, args.reps))
            del mesh
        torch.cuda.empty_cache()
    res["gpu_after"] = bench.gpu_info(0)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "mesh_distance_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({"gpu": res["gpu"]}))


if __name__ == "__main__":
    main()
