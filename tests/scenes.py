"""Crops of the BASELINE.json benchmark scenes (bench.py's seeded generators) at their own point density (cfg4: the
10 M-point cloud of BASELINE.json, denser than the 5 M points bench.py runs on one GPU), shared by the large-scale
parity tests: a box in x-y around an anchor holding exactly `n` points."""
import functools

import numpy as np

_ANCHOR = {"cfg4_outdoor": ("cfg4_outdoor_5M", (0.0, 14.0), 10_000_000),
           "cfg3_indoor": ("cfg3_indoor_1M", (2.0, 2.0), 1_000_000)}


@functools.lru_cache(maxsize=2)
def _full(scene):
    import bench
    workload, _, points = _ANCHOR[scene]
    xyz, sensor = bench.make_cloud(workload, 4, points=points)
    return xyz.numpy(), sensor.numpy(), float(bench.WORKLOADS[workload]["voxel_size"])


def crop(scene, n, with_sensor=False):
    xyz, sensor, W = _full(scene)
    ax, ay = _ANCHOR[scene][1]
    d = np.maximum(np.abs(xyz[:, 0] - ax), np.abs(xyz[:, 1] - ay))
    idx = np.sort(np.argpartition(d, n)[:n])            # keep the generator's (random) point order
    if with_sensor:
        return np.ascontiguousarray(xyz[idx]), np.ascontiguousarray(sensor[idx]), W
    return np.ascontiguousarray(xyz[idx]), W
