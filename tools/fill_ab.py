"""Time the Gram fill of the benchmark system per level, and the brick fill against the row fill.

Builds the bench.py system once (cfg4 at 5 M points, seed 4, bench.SOLVER), then, inside the assembly of a second
reconstruct() -- where every buffer of the fill is alive -- times with CUDA events:
  * the row fill (k_gram_fill) on the rows of each level, and on all rows;
  * the brick fill (nksr_gram_fill_brick) on all rows, with the default density threshold and with every level below
    the split level bricked;
  * the brick fill with the threshold set between the levels' densities, so that levels l and up are bricked, for
    every fine level l: the brick time of level l is the difference of two such fills plus the row fill of level l.
It prints n per level, the constraint rows per voxel, the kernel-row lines the row fill loads per level (every source
voxel's lines once per active neighbour row), the GPU name and power limit, and one JSON line.  With --hash it also
prints a SHA-256 of each array of the system the brick fill makes with every fine level bricked (rowptr, col, val,
rhs, diag); with --against LIB, the same for the brick fill of another build of libnksr_b200.so run on the same
buffers, so that two builds are compared bit for bit on one input (the constraint rows of two runs of reconstruct()
need not be in the same order).

    python tools/fill_ab.py [--workload cfg4_outdoor_5M] [--reps 3] [--hash] [--against path/to/libnksr_b200.so]
"""
import argparse
import ctypes
import hashlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("PYTORCH_CUDA_ALLOC_CONF", "expandable_segments:True")

import bench  # noqa: E402  (the workload, its seed and SOLVER come from the benchmark itself)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        q = "nvidia-smi unavailable"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="cfg4_outdoor_5M", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--hash", action="store_true")
    ap.add_argument("--against", default=None, help="another build's libnksr_b200.so (implies --hash)")
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

    ranges = {}
    orig_rows = fields.KernelField._sorted_rows

    def sorted_rows(self, xyz_, mode, *a, **kw):
        out = orig_rows(self, xyz_, mode, *a, **kw)
        ranges[mode] = out[3]
        return out
    fields.KernelField._sorted_rows = sorted_rows

    result = {}
    state = {"measure": False}
    orig_call = fields.call

    def ev_time(fn):
        ts = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b))
        ts.sort()
        return ts[len(ts) // 2]

    def measuring_call(name, *a):
        rc = orig_call(name, *a)
        if not state["measure"] or name not in ("nksr_gram_fill_placed", "nksr_gram_fill_brick"):
            return rc
        state["measure"] = False
        svh_v, feat, cs, cnt, rowptr, place, col, val, rhs, diag = a[:10]
        st = a[-1]
        rows_args = (svh_v, feat, cs, cnt, rowptr, place, col, val, rhs, diag, st)
        brick_args = rows_args[:10] + (float(fields.BRICK_MIN_LOCATIONS_PER_VOXEL), st)
        svh = state["field_svh"]
        offs = list(svh.offsets) + [svh.num_unknowns]
        L = svh.depth
        result["split_level"] = int(cs.split_level)
        per = []
        for l in range(L):
            t = ev_time(lambda: orig_call("nksr_gram_fill_placed_rows", svh_v, feat, cs, cnt, rowptr, place,
                                          offs[l], offs[l + 1], col, val, rhs, diag, st))
            per.append(t)
        result["rows_ms_per_level"] = [round(t, 3) for t in per]
        result["rows_ms"] = round(ev_time(lambda: orig_call("nksr_gram_fill_placed", *rows_args)), 3)
        result["brick_ms"] = round(ev_time(lambda: orig_call("nksr_gram_fill_brick", *brick_args)), 3)
        result["brick_every_level_ms"] = round(ev_time(lambda: orig_call("nksr_gram_fill_brick",
                                                                          *brick_args[:10], 0.0, st)), 3)
        # levels >= l bricked: a threshold just under level l's constraint locations per voxel (density grows with l)
        nsplit = min(int(cs.split_level), L)
        locations = float(cs.n_pos) + float(cs.n_nrm)
        dens = [locations / max(offs[l + 1] - offs[l], 1) for l in range(nsplit)]
        from_level = [ev_time(lambda: orig_call("nksr_gram_fill_brick", *brick_args[:10],
                                                float(min(dens[l:])) * 0.999, st)) for l in range(nsplit)]
        from_level.append(result["rows_ms"])
        result["locations_per_voxel"] = [round(d, 3) for d in dens]
        result["brick_ms_per_level"] = [round(from_level[l] - from_level[l + 1] + per[l], 3) for l in range(nsplit)]
        if args.hash or args.against:
            def hashed(fill):
                for t in (col, val, rhs, diag):
                    t.zero_()
                fill()
                torch.cuda.synchronize()
                return {k: hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()
                        for k, t in (("rowptr", rowptr), ("col", col), ("val", val), ("rhs", rhs), ("diag", diag))}
            this = lambda: orig_call("nksr_gram_fill_brick", *brick_args[:10], 0.0, st)
            result["sha256_every_level_bricked"] = hashed(this)
            if args.against:
                other = ctypes.CDLL(os.path.abspath(args.against))
                fn = other.nksr_gram_fill_brick
                ret, kinds = _lib._SIGNATURES["nksr_gram_fill_brick"]
                fn.restype = ctypes.c_int
                fn.argtypes = [_lib._T[k] for k in kinds]
                conv = [_lib._conv(k, v) for k, v in zip(kinds, brick_args[:10] + (0.0, st))]
                rcs = []
                result["sha256_against"] = hashed(lambda: rcs.append(fn(*conv)))
                result["against_rc"] = rcs[0]
                result["bitwise_equal"] = result["sha256_against"] == result["sha256_every_level_bricked"]
                this()                                   # the solve goes on with this build's system
        # counts from the constraint-row ranges
        n_l, pos_per, nrm_per, lines = [], [], [], []
        for l in range(L):
            lo, hi = offs[l], offs[l + 1]
            n_l.append(hi - lo)
            rp = ranges[0][lo:hi]
            npos = (rp[:, 1] - rp[:, 0]).double()
            nnrm = (ranges[1][lo:hi, 1] - ranges[1][lo:hi, 0]).double() if 1 in ranges else torch.zeros_like(npos)
            pos_per.append(round(float(npos.mean()), 3) if hi > lo else 0.0)
            nrm_per.append(round(float(nnrm.mean()), 3) if hi > lo else 0.0)
            nb = (svh.nbr27[l] >= 0).sum(1).double()           # rows that visit voxel u = its active neighbours
            nlev = L - l
            lines.append(float((nb * (npos * nlev + nnrm * 3 * nlev)).sum()) if l < cs.split_level else None)
        result.update(n_per_level=n_l, pos_rows_per_voxel=pos_per, nrm_rows_per_voxel=nrm_per,
                      row_fill_lines_per_level=lines)
        return rc

    fields.call = measuring_call
    orig_assemble = fields.KernelField.assemble

    def assemble(self, *a, **kw):
        state["field_svh"] = self.svh
        return orig_assemble(self, *a, **kw)
    fields.KernelField.assemble = assemble

    rec.reconstruct(xyz, sensor=sensor, voxel_size=cfg["voxel_size"], preprocess_fn=prep, **bench.SOLVER)  # warm-up
    torch.cuda.synchronize()
    state["measure"] = True
    rec.reconstruct(xyz, sensor=sensor, voxel_size=cfg["voxel_size"], preprocess_fn=prep, **bench.SOLVER)
    torch.cuda.synchronize()
    result["gpu"] = gpu_info()
    result["workload"] = args.workload
    result["fill"] = os.environ.get("NKSR_FILL", "default")
    result["row_layout"] = os.environ.get("NKSR_ROW_LAYOUT", "default")
    if "rows_ms_per_level" in result:
        below = sum(result["rows_ms_per_level"][:max(result["split_level"], 0)])
        result["rows_share_below_split"] = round(below / max(sum(result["rows_ms_per_level"]), 1e-9), 3)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
