"""Time one application of the inference operator both ways on the benchmark systems: matrix-free (nksr_op_apply, from
the kernel rows) and assembled (the packed tile-stream SpMV the assembled PCG runs, nksr_spmv_stream_planned over a plan
that has packed its tiles).

For each workload (bench.py's scene, seed 4, bench.SOLVER) it reconstructs once with the assembled operator and keeps
its CSR matrix, then once matrix-free, and inside that solve times the two operators alternated on the same x: the
median of --reps runs of 10 launches each.  Bytes per application: for the assembled matrix 8 nnz + 12 n less 2 bytes
per packed column; for the matrix-free operator the byte model of fields.operator_bytes_per_apply (kernel rows,
containing voxels, nbr27, the planar partial sums written and gathered, z, x and y).  It prints the GPU name, power
limit and clocks, and one JSON line per workload.

    python tools/operator_ab.py [--workload cfg4_outdoor_5M --workload cfg3_indoor_1M] [--reps 5]
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


def run(workload, reps):
    import torch
    import nksr_b200
    from nksr_b200 import fields

    dev = torch.device("cuda", 0)
    cfg = bench.WORKLOADS[workload]
    xyz, sensor = bench.make_cloud(workload, 4)
    xyz, sensor = xyz.to(dev), sensor.to(dev)
    rec = nksr_b200.Reconstructor(dev, network=None, tree_depth=bench.TREE_DEPTH, adaptive_depth=bench.ADAPTIVE_DEPTH,
                                  kernel_dim=bench.KERNEL_DIM)
    prep = nksr_b200.get_estimate_normal_preprocess_fn(bench.KNN, bench.MAX_ANGLE)
    orig_call = fields.call
    state = {}
    result = {"workload": workload}

    def ev_time(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(LAUNCHES):
            fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / LAUNCHES

    def keep_matrix(rowptr, col, val, n, nnz, st):
        """the assembled matrix and a plan whose tiles the first launch has packed"""
        x = torch.randn(n, device=dev)
        y = torch.empty_like(x)
        nb = orig_call("nksr_spmv_plan_bytes", nnz)
        plan = torch.empty(nb, dtype=torch.uint8, device=dev)
        orig_call("nksr_spmv_plan_build", rowptr, n, nnz, n, nnz, plan, nb, st)
        orig_call("nksr_spmv_stream_planned", rowptr, col, val, x, y, n, nnz, n, nnz, plan, st)
        stats = (ctypes.c_int64 * 4)()
        orig_call("nksr_spmv_plan_stats", plan, ctypes.addressof(stats), st)
        state["spmv"] = lambda xx, yy: orig_call("nksr_spmv_stream_planned", rowptr, col, val, xx, yy, n, nnz, n, nnz,
                                                 plan, st)
        state["tensors"] = (rowptr, col, val, plan)
        result.update(n=n, nnz=nnz, assembled_bytes=8 * nnz + 12 * n - 2 * stats[1], packed_entries=stats[1])

    def measure(a):
        svh, feat, cs, base_pos, base_nrm = a[0], a[1], a[2], a[3], a[4]
        op_ws, op_nb, st = a[12], a[13], a[-1]
        n = result["n"]
        x = torch.randn(n, device=dev)
        y_mf, y_as = torch.empty_like(x), torch.empty_like(x)
        apply = lambda: orig_call("nksr_op_apply", svh, feat, cs, base_pos, base_nrm, x, y_mf, op_ws, op_nb, st)
        spmv = lambda: state["spmv"](x, y_as)
        apply()
        spmv()
        t_mf, t_as = [], []
        for _ in range(reps):          # alternated
            t_mf.append(ev_time(apply))
            t_as.append(ev_time(spmv))
        t_mf.sort()
        t_as.sort()
        torch.cuda.synchronize()
        d = (y_mf.double() - y_as.double()).abs().max().item()
        result.update(matrix_free_ms=round(t_mf[len(t_mf) // 2], 4), assembled_ms=round(t_as[len(t_as) // 2], 4),
                      matrix_free_ms_range=[round(t_mf[0], 4), round(t_mf[-1], 4)],
                      assembled_ms_range=[round(t_as[0], 4), round(t_as[-1], 4)],
                      max_abs_diff_over_max_abs=d / max(y_as.abs().max().item(), 1e-30))

    def measuring_call(name, *a):
        if name == "nksr_pcg_solve_stream" and state.get("want") == "assembled":
            state["want"] = None
            keep_matrix(a[0], a[1], a[2], a[6], a[7], a[-1])
        if name == "nksr_pcg_solve_matrix_free" and state.get("want") == "matrix_free":
            state["want"] = None
            measure(a)
        return orig_call(name, *a)

    fields.call = measuring_call
    try:
        for op in ("assembled", "matrix_free"):    # the assembled pass also warms up every stage before the solve
            os.environ["NKSR_OPERATOR"] = op
            state["want"] = op
            f = rec.reconstruct(xyz, sensor=sensor, voxel_size=cfg["voxel_size"], preprocess_fn=prep, **bench.SOLVER)
            if op == "matrix_free":
                result["matrix_free_bytes"] = f.solve_info["operator_bytes_per_apply"]
            del f
            torch.cuda.synchronize()
    finally:
        fields.call = orig_call
        os.environ.pop("NKSR_OPERATOR", None)
        state.clear()
        torch.cuda.empty_cache()
    for k in ("matrix_free", "assembled"):
        result[f"{k}_gbs"] = round(result[f"{k}_bytes"] / (result[f"{k}_ms"] * 1e-3) / 1e9, 1)
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", action="append", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    info = gpu_info()
    print(f"# {info}", flush=True)
    for w in args.workload or ["cfg4_outdoor_5M", "cfg3_indoor_1M"]:
        r = run(w, args.reps)
        r["gpu"] = info
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
