"""Time the mesh occupancy query (nksr_b200.metrics.MeshOccupancy, csrc/raycast.cu; DESIGN.md SPEC S20).

    python tools/occupancy_bench.py --out DIR [--reps 5]

Workloads: an icosphere of 1.31 M triangles (level 8) with 1 M queries; the dual-MC mesh of bench.py's cfg3 indoor
scene at 1 M points (reconstructed as tools/metrics_bench.py does, extract_dual_mesh(mise_iter=1)) with 1 M and 5 M
queries; a ShapeNet-sized case, an icosphere of 81,920 triangles (level 6) with 100 k queries.  Queries are uniform
in the mesh's bounding box padded by 10 % per side (seed 0).  The build is timed in its three parts (keys + sort,
hierarchy, refit), the query for K = 1, 3, 5; every number is the median of --reps runs after one warm-up, timed with
CUDA events.  The brute-force oracle (tests/occupancy_oracle.py, numpy) is timed on a 50-query subsample with K = 1
only and checked against the GPU's answer there.  Writes DIR/occupancy_bench.json with the GPU's name and power limit.
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

N_ORACLE = 50           # the oracle's subsample: every triangle for every query does not finish at full size


def build_timed(v, f):
    """MeshOccupancy's build, one CUDA event between the parts: (ms per part, the built object)"""
    import torch
    from nksr_b200 import _lib
    from nksr_b200.metrics import MeshOccupancy
    occ = MeshOccupancy.__new__(MeshOccupancy)
    dev, t = v.device, f.shape[0]
    occ.device, occ.n_tri = dev, t
    occ.scene = torch.zeros(8, dtype=torch.float32, device=dev)
    occ.nodes = torch.empty((max(t - 1, 0), 16), dtype=torch.float32, device=dev)
    occ.tris = torch.empty((t, 12), dtype=torch.float32, device=dev)
    keys = torch.empty(t, dtype=torch.int64, device=dev)
    idx = torch.empty(t, dtype=torch.int32, device=dev)
    nb = _lib.call("nksr_bvh_workspace_bytes", t)
    ws = _lib._ws(nb, dev)
    st = _lib.stream_ptr(dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    ev[0].record()
    _lib.call("nksr_bvh_keys", v, f, t, occ.scene, keys, idx, st)
    keys, idx = _lib.sort_pairs(keys, idx)
    ev[1].record()
    _lib.call("nksr_bvh_hierarchy", keys, t, occ.nodes, ws, nb, st)
    ev[2].record()
    _lib.call("nksr_bvh_refit", v, f, idx, t, occ.nodes, occ.tris, ws, nb, st)
    ev[3].record()
    torch.cuda.synchronize(dev)
    return {"keys_sort": ev[0].elapsed_time(ev[1]), "hierarchy": ev[1].elapsed_time(ev[2]),
            "refit": ev[2].elapsed_time(ev[3]), "total": ev[0].elapsed_time(ev[3])}, occ


def median_dict(runs):
    return {k: round(statistics.median(r[k] for r in runs), 3) for k in runs[0]}


def run_workload(name, v, f, n_queries, reps):
    import numpy as np
    import torch
    from nksr_b200.metrics import MeshOccupancy
    from tests import occupancy_oracle as OO
    dev = v.device
    f = f.to(torch.int32).contiguous()
    v = v.to(torch.float32).contiguous()
    builds = [build_timed(v, f) for _ in range(reps + 1)]
    occ = builds[-1][1]
    ref = MeshOccupancy(v, f)                                  # the product's build path, for a bitwise check
    diff = ref.nodes.view(torch.int32) != occ.nodes.view(torch.int32)
    repeat = {"nodes_bitwise_equal": not bool(diff.any()), "node_words_differing": int(diff.sum()),
              "node_columns_differing": torch.nonzero(diff.any(0)).flatten().tolist(),
              "tris_bitwise_equal": bool(torch.equal(ref.tris.view(torch.int32), occ.tris.view(torch.int32)))}
    lo, hi = v.min(0).values, v.max(0).values
    g = torch.Generator(device=dev).manual_seed(0)
    res = {"workload": name, "triangles": int(f.shape[0]), "build_ms": median_dict([b[0] for b in builds[1:]]),
           "rebuild": repeat, "query": []}
    for m in n_queries:
        q = lo - 0.1 * (hi - lo) + torch.rand((m, 3), generator=g, device=dev) * 1.2 * (hi - lo)
        for k in (1, 3, 5):
            ms = []
            for rep in range(reps + 1):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                inside = occ.contains(q, k)
                b.record()
                torch.cuda.synchronize(dev)
                if rep:
                    ms.append(a.elapsed_time(b))
            t = statistics.median(ms)
            repeat.setdefault("answers_equal_across_builds", True)
            repeat["answers_equal_across_builds"] &= bool(torch.equal(ref.contains(q, k), inside))
            res["query"].append({"queries": m, "rays": k, "ms": round(t, 3),
                                 "query_rays_per_s": float(f"{m * k / (t * 1e-3):.4g}"),
                                 "inside_fraction": round(float(inside.float().mean()), 5)})
            print(json.dumps({"workload": name, **res["query"][-1]}), flush=True)
    qs = lo - 0.1 * (hi - lo) + torch.rand((N_ORACLE, 3), generator=g, device=dev) * 1.2 * (hi - lo)
    qn = qs.cpu().numpy()
    t0 = time.perf_counter()
    want = OO.occupancy(v.cpu().numpy(), f.cpu().numpy(), qn, n_rays=1)
    t1 = time.perf_counter()
    res["oracle_subsample"] = {"queries": N_ORACLE, "rays": 1, "ms": round(1e3 * (t1 - t0), 1),
                               "label": f"numpy brute force on {N_ORACLE} queries, K = 1 (host CPU)",
                               "equal_to_gpu": bool(np.array_equal(occ.contains(qs, 1).cpu().numpy(), want))}
    print(json.dumps({"workload": name, "build_ms": res["build_ms"], "rebuild": repeat,
                      "oracle": res["oracle_subsample"]}), flush=True)
    return res


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--workloads", nargs="+", default=["icosphere8", "cfg3_indoor_1M", "shapenet"])
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("occupancy_bench.py needs a CUDA device")
    import bench
    from tests.test_cpu_occupancy import icosphere
    dev = torch.device("cuda", 0)
    res = {"gpu": bench.gpu_info(0), "runs": []}
    for wl in args.workloads:
        if wl == "icosphere8":
            v, f = icosphere(8)
            res["runs"].append(run_workload(wl, torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev),
                                            [1_000_000], args.reps))
        elif wl == "shapenet":
            v, f = icosphere(6, 0.5)
            res["runs"].append(run_workload("shapenet_100k", torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev),
                                            [100_000], args.reps))
        else:
            from tools.metrics_bench import reconstruct
            mesh = reconstruct(bench, wl, dev)
            res["runs"].append(run_workload(f"{wl}_dual_mc", mesh.v, mesh.f, [1_000_000, 5_000_000], args.reps))
            del mesh
        torch.cuda.empty_cache()
    res["gpu_after"] = bench.gpu_info(0)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "occupancy_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({"gpu": res["gpu"]}))


if __name__ == "__main__":
    main()
