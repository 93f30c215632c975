"""One reconstruct() (+ optional mesh) of a bench workload, for profiler captures.
usage: python tools/profile_run.py [workload] [points] [mesh]"""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench, nksr_b200
wl = sys.argv[1] if len(sys.argv) > 1 else "dev_outdoor_1M"
pts = int(sys.argv[2]) if len(sys.argv) > 2 else None
dev = torch.device("cuda:0")
xyz, sensor = bench.make_cloud(wl, 4, 0, points=pts)
rec = nksr_b200.Reconstructor(dev)
prep = nksr_b200.get_estimate_normal_preprocess_fn(64, 85.0)
os.environ["NKSR_STAGE_TIMES"] = "1"
f = rec.reconstruct(xyz.to(dev), sensor=sensor.to(dev), voxel_size=bench.WORKLOADS[wl]["voxel_size"], preprocess_fn=prep, **bench.SOLVER)
print(json.dumps(rec.last_stats))
if len(sys.argv) > 3:
    m = f.extract_dual_mesh(mise_iter=1)
    torch.cuda.synchronize()
    print("mesh", m.v.shape, m.f.shape)
