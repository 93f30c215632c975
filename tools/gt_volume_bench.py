"""Time the PointTSDFVolume builder (nksr_b200.gt_geometry.PointTSDFVolume.from_sensor_rays, csrc/tsdf_volume.cu,
DESIGN.md SPEC S19) on crops of the cfg4 outdoor scene.

    python tools/gt_volume_bench.py [--points 200000 1000000 4000000] [--reps 5] [--out DIR]

Each crop (tests/scenes.crop, the 10 M-point cfg4 cloud at its own density) is taken with its sensor positions and
the kNN normals of train_unet.py; the volume has node spacing h = W (0.1), truncation tau = 2 W and a margin of one
depth-4 top-level voxel (0.8), as `train_unet.py --vol-sup` builds it.  Reported per crop: the grid, the median over
--reps of the whole builder call (CUDA events, after one warm-up), and from a separate torch.profiler run the device
time of each kernel: k_tsdf_init, k_tsdf_near (pass 1), k_tsdf_free (pass 2) and k_tsdf_finalise.  The GPU's name and
power limit are printed with the numbers.
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

KERNELS = ("k_tsdf_init", "k_tsdf_near", "k_tsdf_free", "k_tsdf_finalise")


def kernel_ms(build):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        build()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in KERNELS}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                out[k] += ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3
    return {k: round(v, 3) for k, v in out.items()}


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--points", type=int, nargs="+", default=[200_000, 1_000_000, 4_000_000])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--depth", type=int, default=4)
    ap.add_argument("--out", default=None, help="also write DIR/gt_volume_bench.json")
    args = ap.parse_args(argv)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("gt_volume_bench.py needs a CUDA device")
    from bench import gpu_info
    from tools.train_unet import build_volume, cfg4_crop
    dev = torch.device("cuda:0")
    res = {"gpu": gpu_info(0), "runs": []}
    print(json.dumps(res["gpu"]), flush=True)
    for n in args.points:
        px, pn, ps, W = cfg4_crop(n, dev)
        build = lambda: build_volume(px, pn, ps, W, args.depth)
        gt = build()
        ms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            build()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        run = dict(points=n, rays=int(px.shape[0]), dims=list(gt.volume.shape), nodes=gt.volume.numel(),
                   build_ms_median=round(statistics.median(ms), 3), build_ms=[round(v, 3) for v in ms],
                   kernel_ms=kernel_ms(build),
                   fractions={k: round(v, 5) for k, v in gt.class_fractions().items()})
        print(json.dumps(run), flush=True)
        res["runs"].append(run)
        del gt, px, pn, ps
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "gt_volume_bench.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
