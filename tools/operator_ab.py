"""Time one application of the inference operator both ways on the benchmark systems: matrix-free (nksr_op_apply, from
the kernel rows) and assembled (the packed tile-stream SpMV the assembled PCG runs, nksr_spmv_stream_planned over a plan
that has packed its tiles).

For each workload (bench.py's scene, seed 4, bench.SOLVER) it reconstructs once with the assembled operator and keeps
its CSR matrix, then once matrix-free, and inside that solve times the two operators alternated on the same x: the
median of --reps runs of 10 launches each.  Bytes per application: for the assembled matrix 8 nnz + 12 n less 2 bytes
per packed column; for the matrix-free operator the byte model of fields.operator_bytes_per_apply (kernel rows,
containing voxels, nbr27, the planar partial sums written and gathered, z, x and y).  It prints the GPU name, power
limit and clocks, and one JSON line per workload.

Per kernel: a separate pass under torch.profiler (CUDA activity only, after the timed runs) gives the device time of
every kernel of one matrix-free application (`matrix_free_kernels_ms`: name -> ms per application).  `locations`
describes the work the gather-scatter balances: the constraint locations (positions + normal locations) per voxel of
the top level and of level 1 -- mean, quantiles, maximum and a power-of-two histogram over the voxels that hold any.

    python tools/operator_ab.py [--workload cfg4_outdoor_5M --workload cfg3_indoor_1M] [--reps 5] [--item-size S ...]

With --item-size (repeatable) the matrix-free solve and its measurements are repeated for each item size, and each
line also gives `setup_ms`, the device time of nksr_op_setup.
"""
import argparse
import ctypes
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")

import bench  # noqa: E402  (the workload, its seed and SOLVER come from the benchmark itself)
from tools.fill_ab import gpu_info  # noqa: E402

LAUNCHES = 10


def _histogram(counts):
    """summary of the per-voxel location counts (voxels with at least one location)"""
    import torch
    c = counts[counts > 0].double()
    if c.numel() == 0:
        return {"voxels": 0}
    q = torch.quantile(c[: 1 << 24], torch.tensor([0.5, 0.9, 0.99, 0.999], dtype=torch.float64, device=c.device))
    bins = torch.bincount(torch.log2(c).floor().long()).tolist()
    return {"voxels": int(c.numel()), "mean": round(c.mean().item(), 2), "p50": q[0].item(), "p90": q[1].item(),
            "p99": q[2].item(), "p999": q[3].item(), "max": int(c.max().item()),
            "pow2_hist": {f"{1 << k}-{(2 << k) - 1}": v for k, v in enumerate(bins) if v}}


def _locations(svh, bases):
    """locations per voxel of the top level and of level 1 (both kinds together)"""
    import torch
    out = {}
    for name, l in (("top", svh.depth - 1), ("level1", min(1, svh.depth - 1))):
        cnt = torch.zeros(svh.n[l], dtype=torch.int64, device=bases[0].device)
        for b in bases:
            v = b[l][b[l] >= 0].long()
            cnt += torch.bincount(v, minlength=svh.n[l])
        out[name] = _histogram(cnt)
    return out


def _kernel_split(fn):
    """device ms per call of every kernel `fn` launches, from torch.profiler over LAUNCHES calls"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(LAUNCHES):
            fn()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        t = getattr(e, "device_time", None)
        if t is None:
            t = e.cuda_time
        if not t:
            continue
        name = re.match(r"(?:void\s+)?([\w:]+)", e.name.replace("(anonymous namespace)::", "")).group(1)
        per[name] = per.get(name, 0.0) + t / 1e3 / LAUNCHES
    return {k: round(v, 4) for k, v in sorted(per.items(), key=lambda kv: -kv[1])}


def run(workload, reps, sizes):
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
        result["matrix_free_kernels_ms"] = _kernel_split(apply)
        if "locations" not in result:
            result["locations"] = _locations(svh, [b for b in (base_pos, base_nrm) if b is not None])

    def measuring_call(name, *a):
        if name == "nksr_pcg_solve_stream" and state.get("want") == "assembled":
            state["want"] = None
            keep_matrix(a[0], a[1], a[2], a[6], a[7], a[-1])
        if name == "nksr_pcg_solve_matrix_free" and state.get("want") == "matrix_free":
            state["want"] = None
            measure(a)
        if name == "nksr_op_setup" and state.get("want") == "matrix_free":
            ev = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev[0].record()
            rc = orig_call(name, *a)
            ev[1].record()
            ev[1].synchronize()
            result["setup_ms"] = round(ev[0].elapsed_time(ev[1]), 3)
            return rc
        return orig_call(name, *a)

    fields.call = measuring_call
    out = []
    default_size = fields.OP_ITEM_SIZE
    try:
        # the assembled pass also warms up every stage before the solves; then one matrix-free solve per item size
        for op, size in [("assembled", None)] + [("matrix_free", S) for S in sizes]:
            os.environ["NKSR_OPERATOR"] = op
            fields.OP_ITEM_SIZE = size or default_size
            state["want"] = op
            f = rec.reconstruct(xyz, sensor=sensor, voxel_size=cfg["voxel_size"], preprocess_fn=prep, **bench.SOLVER)
            if op == "matrix_free":
                result.update(item_size=size, matrix_free_bytes=f.solve_info["operator_bytes_per_apply"])
                for k in ("matrix_free", "assembled"):
                    result[f"{k}_gbs"] = round(result[f"{k}_bytes"] / (result[f"{k}_ms"] * 1e-3) / 1e9, 1)
                out.append(dict(result))
            del f
            torch.cuda.synchronize()
    finally:
        fields.call = orig_call
        fields.OP_ITEM_SIZE = default_size
        os.environ.pop("NKSR_OPERATOR", None)
        state.clear()
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", action="append", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--item-size", type=int, action="append",
                    help="locations per work item of the matrix-free walk, one solve each (default fields.OP_ITEM_SIZE)")
    args = ap.parse_args()
    info = gpu_info()
    print(f"# {info}", flush=True)
    for w in args.workload or ["cfg4_outdoor_5M", "cfg3_indoor_1M"]:
        for r in run(w, args.reps, args.item_size or [None]):
            r["gpu"] = info
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
