"""Parity at the sizes and settings the benchmark runs (VERDICT r1 item 1): >= 200 K-point crops of the
BASELINE.json scenes cfg3 (indoor, W = 0.02) and cfg4 (outdoor, W = 0.1, full 10 M-point density), the CUDA
path against the C++/OpenMP restatement (oracle/nksr_oracle_cpu.cpp) with the AUTOMATIC Gram-block split
level, the sort-free placement and the default graph-replayed PCG:

  * voxel keys of every level                                   bit-exact
  * CSR pattern: row lengths == SPEC S6 counts, no duplicates, sampled rows column-exact, oracle nonzeros
    all present                                                 exact
  * CSR values, rhs, diagonal                                   <= RTOL_GRAM (4e-6) of the largest entry of the same
                                                                level-pair block (rhs, diagonal: of the same level);
                                                                the C++ restatement gives no per-entry magnitude
                                                                scale, so the per-entry bounds of the smaller
                                                                oracle tests (test_gpu_parity.py) are not used here
  * PCG solution (bench tolerance 1e-4) on the ORACLE's system  residual <= 2e-4 ||b||
  * f (and grad f) at 10 K queries                              evaluation <= 2e-3 of max |f| against the
                                                                oracle evaluating the same coefficients
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import cpu_port as P
from tests import scenes
from tests.bounds import assert_blockwise

pytestmark = pytest.mark.gpu

# max |diff| / max |ref| per level block; worst measured on an H100 (400 W): 9.9e-7 (rhs, cfg4_outdoor)
RTOL_GRAM = 4e-6


def _np(t):
    return t.detach().cpu().numpy()


def _gpu_csr(s):
    n = s.rowptr.numel() - 1
    return sp.csr_matrix((_np(s.val).astype(np.float64), _np(s.col), _np(s.rowptr)), shape=(n, n))


@pytest.mark.parametrize("scene,approx", [("cfg4_outdoor", True), ("cfg3_indoor", False)])
def test_assembly_solve_evaluate_at_bench_scale(cuda, scene, approx):
    import nksr_b200
    xyz, W = scenes.crop(scene, 220_000)
    L, C = 4, 4
    assert xyz.shape[0] >= 200_000
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_point_splatting(t(xyz))
    osvh = P.CpuSvh(xyz, W, L)
    for l in range(L):
        assert np.array_equal(_np(svh.keys[l]), osvh.keys(l)), f"voxel keys of level {l} differ"
    rng = np.random.default_rng(17)
    feats = [(0.5 + 0.2 * rng.normal(size=(osvh.n(l), C))).astype(np.float32) for l in range(L)]
    field = nksr_b200.KernelField(svh, None, [t(f) for f in feats], approx)
    nxyz = np.concatenate([osvh.centers(0), osvh.centers(1)])
    nval = rng.normal(size=nxyz.shape).astype(np.float32)
    nval /= np.linalg.norm(nval, axis=1, keepdims=True)
    pw, nw, rw = 1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * W * W, 1.0
    n = svh.num_unknowns
    # the settings of Reconstructor._reconstruct_one / bench.py: automatic split level, structural placement
    field.solver_config.update(keep_system=True, tol=1e-4, max_iter=2000)
    field.solve(t(xyz), t(nxyz), t(nval), pw, nw, rw)
    s = field.system
    assert field.solve_info["relative_residual"] <= 1e-4

    ref = P.CpuSystem(osvh, feats, xyz, nxyz, nval, pw, nw, rw, approx)
    A_ref, b_ref = ref.to_scipy()
    # ---- pattern
    cnt = osvh.structural_counts()
    rowptr = _np(s.rowptr)
    assert np.array_equal(np.diff(rowptr), cnt.astype(np.int64)), "row lengths differ from SPEC S6"
    A = _gpu_csr(s)
    col = _np(s.col)
    for r in np.random.default_rng(3).integers(0, n, 3000):
        got = np.sort(col[rowptr[r]:rowptr[r + 1]])
        assert np.array_equal(got, osvh.structural_row(r, cnt[r])), f"columns of row {r}"
    A.sum_duplicates()
    assert A.nnz == rowptr[-1], "duplicate column inside a row"
    # ---- values (entries absent from the oracle are structural zeros: the difference covers both sides)
    offs = osvh.offsets()
    assert_blockwise(A, A_ref, offs, RTOL_GRAM, f"Gram values ({scene})")
    assert abs(A - A.T).max() <= 1e-6 * abs(A_ref).max()
    assert_blockwise(_np(s.rhs), b_ref, offs, RTOL_GRAM, f"rhs ({scene})")
    assert_blockwise(_np(s.diag), A_ref.diagonal(), offs, RTOL_GRAM, f"diagonal ({scene})")
    # ---- the GPU solution solves the ORACLE's system to the requested tolerance
    alpha = _np(field.alpha)
    res = np.linalg.norm(A_ref @ alpha.astype(np.float64) - b_ref) / np.linalg.norm(b_ref)
    assert res <= 2e-4, res
    # ---- evaluation at 10 K queries: near the surface, off the band, at voxel centres
    q = np.concatenate([xyz[:6000] + rng.normal(size=(6000, 3)).astype(np.float32) * np.float32(0.3 * W),
                        xyz[6000:8000] + rng.normal(size=(2000, 3)).astype(np.float32) * np.float32(6 * W),
                        osvh.centers(0)[:1500], osvh.centers(2)[:500]]).astype(np.float32)
    r = field.evaluate_f(t(q), grad=True)
    fo, go = osvh.evaluate(feats, alpha, q, grad=True, approx=approx)
    assert np.abs(_np(r.value) - fo).max() <= 2e-3 * np.abs(fo).max()
    assert np.abs(_np(r.gradient) - go).max() <= 2e-3 * np.abs(go).max()


def test_reconstructor_matches_oracle_pipeline(cuda):
    """SURVEY 8 row a8: Reconstructor.reconstruct (stand-in network, sensor feature, normal constraints at
    the voxel centres, Jacobi-PCG) against the CPU restatement of the same wiring (oracle/pipeline.py) on a
    200 K-point cfg4 crop: same hierarchy, same features (to fp32 pooling order), same field."""
    import copy
    import nksr_b200
    from oracle import pipeline
    xyz, sensor, W = scenes.crop("cfg4_outdoor", 200_000, with_sensor=True)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    rec = nksr_b200.Reconstructor(cuda)
    field = rec.reconstruct(t(xyz), sensor=t(sensor), voxel_size=W, approx_kernel_grad=True, solver_tol=1e-6)
    net_cpu = copy.deepcopy(rec.network).cpu()
    ref = pipeline.reconstruct(xyz, sensor=sensor, voxel_size=W, depth=4, adaptive_depth=2, network=net_cpu,
                               approx_kernel_grad=True, solver_tol=1e-7)
    osvh = ref["svh"]
    for l in range(4):
        assert np.array_equal(_np(field.svh.keys[l]), osvh.keys(l))
        z = _np(field.z[l])
        assert np.abs(z - ref["feats"][l]).max() <= 1e-4 * np.abs(ref["feats"][l]).max(), f"features level {l}"
    # (the CUDA path stores every STRUCTURAL slot of SPEC S6, the C++ restatement only the products that occur)
    assert field.solve_info["n"] == ref["system"].n and field.solve_info["nnz"] >= ref["system"].nnz
    # same field: values and gradients at the input points and around them
    rng = np.random.default_rng(5)
    q = np.concatenate([xyz[:5000], xyz[5000:10000] + rng.normal(size=(5000, 3)).astype(np.float32) * np.float32(W)])
    r = field.evaluate_f(t(q), grad=True)
    fo, go = osvh.evaluate(ref["feats"], ref["alpha"], q, grad=True, approx=True)
    fs = max(np.abs(fo).max(), 1e-6)
    assert np.abs(_np(r.value) - fo).max() <= 5e-3 * fs
    assert np.abs(_np(r.gradient) - go).max() <= 2e-2 * np.abs(go).max()
    # the reference's own training checks on the solved field (models/loss.py:188-198): |f| small at the
    # points, gradient along the (estimated) outward direction
    # (a sanity bound on the fit, not a parity bound: the oracle's own field sits at the same level)
    assert np.abs(_np(r.value[:5000])).mean() <= 0.1 * fs
    assert abs(np.abs(_np(r.value[:5000])).mean() - np.abs(fo[:5000]).mean()) <= 0.02 * fs
