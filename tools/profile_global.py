"""One reconstruct_global() of a bench workload on ONE GPU (world size 1: same step kernels, no collectives), for
profiler launch lists of the distributed-CG kernels.  usage: python tools/profile_global.py [workload]"""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench, nksr_b200
from nksr_b200 import dist_solve
wl = sys.argv[1] if len(sys.argv) > 1 else "cfg4_outdoor_5M"
dev = torch.device("cuda:0")
xyz, sensor = bench.make_cloud(wl, 4, 0)
rec = nksr_b200.Reconstructor(dev)
prep = nksr_b200.get_estimate_normal_preprocess_fn(64, 85.0)
os.environ["NKSR_STAGE_TIMES"] = "1"
f = dist_solve.reconstruct_global(rec, xyz.to(dev), None, bench.WORKLOADS[wl]["voxel_size"], sensor=sensor.to(dev),
                                  preprocess_fn=prep, approx_kernel_grad=True, solver_tol=1e-4, distributed_input=True)
print(json.dumps({k: v for k, v in f.solve_info.items() if k != "slab"}))
print(f._stage_timer.report())
