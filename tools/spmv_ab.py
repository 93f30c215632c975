"""Time the PCG's SpMV on the benchmark system: the tile stream with its packed column tiles, the launch that packs
them, and the row kernel; optionally other builds of libnksr_b200.so on the same matrix.

Builds the bench.py system (cfg4 at 5 M points by default, seed 4, bench.SOLVER) and, when reconstruct() reaches its
PCG, times with CUDA events on the same device buffers, for everything streamed (what KernelField does) and for the
two finest levels streamed with the coarse rows by the row kernel ("split"):
  * the first SpMV over a new plan (nksr_spmv_plan_build, then the launch that packs the tiles), and the plan's counts
    of packed tiles and entries;
  * one SpMV (median of --reps runs of 10 launches) through nksr_spmv_stream_planned, and through the row kernel
    nksr_spmv;
  * with --against LIB (repeatable): the same SpMVs of another build.  A build with nksr_spmv_stream_planned is timed
    like this one; an older build through nksr_spmv_stream (its plan build included, a binary search per tile), and
    its y is compared bit for bit with this build's.
It prints the GPU name, power limit and clocks, and one JSON line.

    python tools/spmv_ab.py [--workload cfg4_outdoor_5M] [--reps 5] [--against path/to/libnksr_b200.so ...]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")

import bench  # noqa: E402  (the workload, its seed and SOLVER come from the benchmark itself)
from tools.fill_ab import gpu_info  # noqa: E402

LAUNCHES = 10


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg4_outdoor_5M", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--against", action="append", default=[], help="another build's libnksr_b200.so")
    args = ap.parse_args()

    import torch
    import nksr_b200
    from nksr_b200 import _lib, fields

    dev = torch.device("cuda", 0)
    cfg = bench.WORKLOADS[args.workload]
    xyz, sensor = bench.make_cloud(args.workload, 4)
    xyz, sensor = xyz.to(dev), sensor.to(dev)
    rec = nksr_b200.Reconstructor(dev, network=None, tree_depth=bench.TREE_DEPTH, adaptive_depth=bench.ADAPTIVE_DEPTH,
                                  kernel_dim=bench.KERNEL_DIM)
    prep = nksr_b200.get_estimate_normal_preprocess_fn(bench.KNN, bench.MAX_ANGLE)
    result = {}
    state = {"measure": False}
    orig_call = fields.call

    def ev_time(fn, per=1, reps=None):
        ts = []
        for _ in range(reps or args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(per):
                fn()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b) / per)
        ts.sort()
        return round(ts[len(ts) // 2], 4)

    def bind(lib, name):
        fn = getattr(lib, name)
        fn.restype = ctypes.c_int
        kinds = _lib._SIGNATURES[name][1]
        fn.argtypes = [_lib._T[k] for k in kinds]
        return lambda *a: _check(name, fn(*[_lib._conv(k, v) for k, v in zip(kinds, a)]))

    def _check(name, rc):
        if rc != 0:
            raise RuntimeError(f"{name} returned {rc}")

    def measure(rowptr, col, val, n, nnz, split_row, split_nnz, st):
        x = torch.randn(n, device=dev)
        y = torch.empty_like(x)
        nb = orig_call("nksr_spmv_plan_bytes", nnz)
        plan = torch.empty(nb, dtype=torch.uint8, device=dev)
        stats = (ctypes.c_int64 * 4)()
        ys = {}
        for label, sr, sn in (("all", n, nnz), ("split", split_row, split_nnz)):
            spmv = lambda: orig_call("nksr_spmv_stream_planned", rowptr, col, val, x, y, n, nnz, sr, sn, plan, st)
            first = []
            for _ in range(args.reps):
                orig_call("nksr_spmv_plan_build", rowptr, n, nnz, sr, sn, plan, nb, st)
                first.append(ev_time(spmv, 1, reps=1))
            first.sort()
            result[f"first_launch_ms_{label}"] = first[len(first) // 2]
            orig_call("nksr_spmv_plan_stats", plan, ctypes.addressof(stats), st)
            result[f"packed_{label}"] = {"tiles": stats[0], "entries": stats[1], "streamed_tiles": stats[2],
                                         "streamed_entries": stats[3], "entry_share": round(stats[1] / max(stats[3], 1), 4)}
            result[f"stream_ms_{label}"] = ev_time(spmv, LAUNCHES)
            ys[label] = y.clone()
            for i, path in enumerate(args.against):
                other = ctypes.CDLL(os.path.abspath(path))
                key = f"against{i}_{label}"
                if hasattr(other, "nksr_spmv_stream_planned"):
                    bind(other, "nksr_spmv_plan_build")(rowptr, n, nnz, sr, sn, plan, nb, st)
                    fn = bind(other, "nksr_spmv_stream_planned")
                    result[key + "_ms"] = ev_time(lambda: fn(rowptr, col, val, x, y, n, nnz, sr, sn, plan, st),
                                                  LAUNCHES)
                else:
                    fn = bind(other, "nksr_spmv_stream")
                    result[key + "_ms_with_plan"] = ev_time(lambda: fn(rowptr, col, val, x, y, n, nnz, sr, sn,
                                                                       plan, nb, st), LAUNCHES)
                    result[key + "_bitwise_equal"] = bool(torch.equal(y.view(torch.int32),
                                                                      ys[label].view(torch.int32)))
        result["rows_ms"] = ev_time(lambda: orig_call("nksr_spmv", rowptr, col, val, x, y, n, st), LAUNCHES)
        result.update(n=n, nnz=nnz, split_row=split_row, split_nnz=split_nnz, bytes_raw=8 * nnz + 12 * n,
                      bytes_packed_all=8 * nnz + 12 * n - 2 * result["packed_all"]["entries"])

    def measuring_call(name, *a):
        if state["measure"] and name == "nksr_pcg_solve_stream":
            state["measure"] = False
            rowptr, col, val = a[0], a[1], a[2]
            n, nnz = a[6], a[7]
            split_row = state["svh"].offsets[2] if state["svh"].depth > 2 else n
            split_nnz = int(rowptr[split_row].item()) if split_row < n else nnz
            measure(rowptr, col, val, n, nnz, split_row, split_nnz, a[-1])
            torch.cuda.empty_cache()
        return orig_call(name, *a)

    fields.call = measuring_call
    orig_pcg = fields.KernelField._pcg

    def pcg(self, *a, **kw):
        state["svh"] = self.svh
        return orig_pcg(self, *a, **kw)
    fields.KernelField._pcg = pcg
    solve = dict(bench.SOLVER)
    rec.reconstruct(xyz, sensor=sensor, voxel_size=cfg["voxel_size"], preprocess_fn=prep, **solve)  # warm-up
    torch.cuda.synchronize()
    state["measure"] = True
    rec.reconstruct(xyz, sensor=sensor, voxel_size=cfg["voxel_size"], preprocess_fn=prep, **solve)
    torch.cuda.synchronize()
    if state["measure"]:
        raise RuntimeError("the solve did not go through nksr_pcg_solve_stream (NKSR_SPMV=rows?)")
    result["gpu"] = gpu_info()
    result["workload"] = args.workload
    result["against"] = args.against
    print(json.dumps(result))


if __name__ == "__main__":
    main()
