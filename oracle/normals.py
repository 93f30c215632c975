"""CPU restatement of the normal-estimation preprocess -- TEST / BASELINE INFRASTRUCTURE ONLY.

Follows the reference's open CPU twin line by line (examples/recons_waymo_cpu.py:21-41), which is what
`nksr.get_estimate_normal_preprocess_fn(64, 85.0)` does on the GPU (examples/recons_waymo.py:36):

    :26  indices, normal = pcu.estimate_point_cloud_normals_knn(xyz, 64)    kNN (k = 64) PCA normals
    :32-33 view_dir = (sensor - xyz) / (|sensor - xyz| + 1e-6)
    :34-36 flip normals with  <view_dir, normal> < 0
    :38-39 keep |cos| > cos(85 deg)

`point_cloud_utils` is a third-party dependency absent from the reference tree (environment.yml pins no
version); its published algorithm is restated here: the k nearest neighbours of a point INCLUDING the point
itself, the 3x3 covariance of those neighbours about their mean, the unit eigenvector of the smallest
eigenvalue.  Parity unpinned (no golden vectors in the reference).  scipy's cKDTree does the search.
"""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree


def knn_indices(xyz: np.ndarray, k: int, workers: int = -1):
    """(N,k) indices and (N,k) distances of the k nearest points (self included), nearest first."""
    tree = cKDTree(np.asarray(xyz, np.float64))
    d, idx = tree.query(np.asarray(xyz, np.float64), k=k, workers=workers)
    return idx.reshape(xyz.shape[0], -1), d.reshape(xyz.shape[0], -1)


def _pca_block(p64, idx):
    p = p64[idx]                                                 # (n,k,3)
    c = p - p.mean(axis=1, keepdims=True)
    cov = np.einsum('nki,nkj->nij', c, c) / idx.shape[1]
    w, v = np.linalg.eigh(cov)
    return v[:, :, 0], w


def pca_normals(xyz: np.ndarray, idx: np.ndarray, workers: int = -1):
    """unit eigenvector of the smallest eigenvalue of the neighbourhood covariance (float64);
    also returns the eigenvalues (ascending) so that tests can skip degenerate neighbourhoods.
    Points are independent, so blocks of them go to a thread pool (numpy releases the GIL in the gathers, einsum and
    eigh): the same arithmetic per point whatever the block size, on all host cores like the kNN search."""
    import os
    from concurrent.futures import ThreadPoolExecutor
    p64 = np.asarray(xyz, np.float64)
    n = idx.shape[0]
    nw = (os.cpu_count() or 1) if workers is None or workers < 0 else max(1, int(workers))
    block = 8192                                                 # ~40 MB of temporaries per worker
    if nw == 1 or n <= block:
        return _pca_block(p64, idx)
    spans = [(s, min(s + block, n)) for s in range(0, n, block)]
    with ThreadPoolExecutor(max_workers=nw) as ex:
        parts = list(ex.map(lambda ab: _pca_block(p64, idx[ab[0]:ab[1]]), spans))
    return np.concatenate([q[0] for q in parts]), np.concatenate([q[1] for q in parts])


def estimate_normal_preprocess(xyz: np.ndarray, sensor: np.ndarray, knn: int = 64, max_angle_deg: float = 85.0,
                               workers: int = -1):
    """Returns xyz', normal' (float32) of the kept points, the keep mask, and (normals of ALL points, cos, eigvals)."""
    idx, _ = knn_indices(xyz, min(knn, xyz.shape[0]), workers)
    n, ev = pca_normals(xyz, idx, workers)
    view = np.asarray(sensor, np.float64) - np.asarray(xyz, np.float64)
    view = view / (np.linalg.norm(view, axis=-1, keepdims=True) + 1e-6)
    cos = np.sum(view * n, axis=1)
    n = np.where((cos < 0.0)[:, None], -n, n)
    keep = np.abs(cos) > np.cos(np.deg2rad(max_angle_deg))
    return (np.ascontiguousarray(xyz[keep], np.float32), np.ascontiguousarray(n[keep], np.float32), keep,
            (n, cos, ev))
