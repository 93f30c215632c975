"""Time the first-hit query (nksr_b200.metrics.MeshOccupancy.intersect, csrc/raycast.cu k_mesh_first_hit; DESIGN.md
SPEC S22) and simulated scans (nksr_b200.gt_geometry.scan_mesh).

    python tools/mesh_scan_bench.py --out DIR [--reps 5]

Workloads: the icosphere of 1.31 M triangles (level 8, R = 1) with rays from inside (origins uniform in the ball of
radius 0.99, uniform directions) and from outside (origins at radius 1.5 to 2.5, aimed at the centre with a
N(0, 0.3^2) tilt per component, so most hit and some miss); the closed room of tests/test_gpu_mesh_scan.py (thick
walls and three boxes, 60 triangles) with rays from its air; 1 M and 10 M rays each (seed 0).  Beside every
`intersect` the parity kernel runs at K = 1 on the same origins (`contains(o, 1)`, its built-in direction): a
traversal that counts every crossing against one that stops shrinking at the first.  Then `scan_mesh` of the room with
lidar_directions(64, 1024, (-45, 45)) from 10 poses.  Every number is the median of --reps runs after one warm-up,
timed with CUDA events; the brute force (tests/hit_oracle.py) is checked against the GPU bit for bit on an 8-ray
subsample of each set.  Writes DIR/mesh_scan_bench.json with the GPU's name and power limit, read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

N_ORACLE = 8


def rays(kind, m, dev, g):
    import torch
    u = lambda n: torch.nn.functional.normalize(torch.randn((n, 3), generator=g, device=dev), dim=1)
    if kind == "inside":
        o = u(m) * (torch.rand((m, 1), generator=g, device=dev) * 0.99)
        return o, u(m)
    if kind == "outside":
        o = u(m) * (1.5 + torch.rand((m, 1), generator=g, device=dev))
        return o, torch.nn.functional.normalize(-o, dim=1) + 0.3 * torch.randn((m, 3), generator=g, device=dev)
    from tests.test_gpu_mesh_scan import ROOM_INNER, in_room_air
    lo, hi = torch.tensor(ROOM_INNER[0], device=dev), torch.tensor(ROOM_INNER[1], device=dev)
    o = lo + torch.rand((2 * m, 3), generator=g, device=dev) * (hi - lo)
    o = o[torch.from_numpy(in_room_air(o.cpu().numpy(), 1e-3)).to(dev)][:m].contiguous()
    return o, u(o.shape[0])


def run_set(name, occ, v, f, kind, m, reps):
    import numpy as np
    import torch
    from tests import hit_oracle as H
    from tools.mesh_distance_bench import timed
    g = torch.Generator(device=occ.device).manual_seed(0)
    o, d = rays(kind, m, occ.device, g)
    row = {"workload": name, "rays": kind, "m": int(o.shape[0])}
    row["intersect_ms"], (t, x, n, tri) = timed(lambda: occ.intersect(o, d), reps)
    row["parity_k1_ms"], _ = timed(lambda: occ.contains(o, 1), reps)
    row["rays_per_s"] = float(f"{o.shape[0] / (row['intersect_ms'] * 1e-3):.4g}")
    row["parity_k1_rays_per_s"] = float(f"{o.shape[0] / (row['parity_k1_ms'] * 1e-3):.4g}")
    row["hit_fraction"] = round(float((tri >= 0).double().mean()), 6)
    sub = torch.randperm(o.shape[0], generator=g, device=occ.device)[:N_ORACLE]
    want = H.first_hit(v, f, o[sub].cpu().numpy(), d[sub].cpu().numpy())
    got = tuple(a[sub].cpu().numpy() for a in (t, x, n, tri))
    row["oracle_equal"] = all(np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a,
                                             b.view(np.uint32) if b.dtype == np.float32 else b)
                              for a, b in zip(got, want))
    print(json.dumps(row), flush=True)
    del o, d, t, x, n, tri
    torch.cuda.empty_cache()
    return row


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", type=int, nargs="+", default=[1_000_000, 10_000_000])
    args = ap.parse_args(argv)
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("mesh_scan_bench.py needs a CUDA device")
    import bench
    from nksr_b200.gt_geometry import lidar_directions, scan_mesh
    from nksr_b200.metrics import MeshOccupancy
    from tests.test_cpu_occupancy import icosphere
    from tests.test_gpu_mesh_scan import ROOM_INNER, in_room_air, room_mesh
    from tools.mesh_distance_bench import timed
    dev = torch.device("cuda", 0)
    res = {"gpu": bench.gpu_info(0), "runs": []}
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    for name, (v, f), kinds in (("icosphere8", icosphere(8), ("inside", "outside")),
                                ("room", room_mesh(), ("room_air",))):
        occ = MeshOccupancy(t(v), t(f))
        for kind in kinds:
            for m in args.sizes:
                res["runs"].append(run_set(name, occ, v, f, kind, m, args.reps))
    # a scan: 64 x 1024 directions from 10 poses in the room's air
    v, f = room_mesh()
    occ = MeshOccupancy(t(v), t(f))
    rng = np.random.default_rng(0)
    lo, hi = np.asarray(ROOM_INNER[0]), np.asarray(ROOM_INNER[1])
    p = (lo + rng.random((1000, 3)) * (hi - lo)).astype(np.float32)
    poses = t(p[in_room_air(p, 0.3)][:10])
    dirs = lidar_directions(64, 1024, (-45.0, 45.0)).to(dev)
    ms, scan = timed(lambda: scan_mesh(occ, poses, dirs), args.reps)
    row = {"workload": "room_scan", "poses": int(poses.shape[0]), "directions": int(dirs.shape[0]),
           "returns": int(scan.xyz.shape[0]), "scan_mesh_ms": ms,
           "returns_per_s": float(f"{scan.xyz.shape[0] / (ms * 1e-3):.4g}")}
    print(json.dumps(row), flush=True)
    res["scan"] = row
    res["gpu_after"] = bench.gpu_info(0)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "mesh_scan_bench.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({"gpu": res["gpu"]}))


if __name__ == "__main__":
    main()
