"""SURVEY 8(f) row 4 -- the reference's GT-SDF generator ext.sdfgen.sdf_from_points (ext/sdfgen/sdf_from_points.cu,
ext/common/kdtree_cuda.cu), the ONE piece of this path whose source is in the reference tree:

  * nksr_b200.sdfgen.sdf_from_points (csrc/sdfgen.cu: voxel-hash kNN + vote in one kernel)
  * oracle/sdfgen.py (numpy + cKDTree restatement, line by line)
  * the UNMODIFIED reference sources, compiled by oracle/Makefile.ref and run once on an H100: a seeded sample of their
    outputs on these same inputs is stored in tests/golden/sdfgen/reference_outputs.npz (tests/golden/make_sdfgen_golden.py)

are compared pairwise on the GPU with the reference's own argument sets (dataset/av_gt_geometry.py:67-70: nb_points=8,
stdv=3.0, adaptive_knn=8; models/loss.py:85: 8, 0.02) plus the IMLS variant.  The rule is discontinuous where the nearest
distance crosses stdv*ref_std, where a vote d_k crosses 0 and where the k-th / (k+1)-th neighbours swap: queries within a
rounding error of such a point are excluded from the exact comparison (and counted: they must be rare)."""
import os

import numpy as np
import pytest
import torch

from oracle import sdfgen as OS
from tests import clouds, scenes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sdfgen", "reference_outputs.npz")


def _np(t):
    return t.detach().cpu().numpy()


def _case(name):
    rng = np.random.default_rng(5)
    if name == "sphere":
        xyz, nrm = clouds.sphere(40_000, noise=0.001)
        q = (xyz[rng.integers(0, xyz.shape[0], 60_000)] + rng.normal(size=(60_000, 3)) * 0.05).astype(np.float32)
        q[:2000] = rng.uniform(-2, 2, size=(2000, 3))                        # far from the data
    else:
        xyz, sensor, _ = scenes.crop("cfg4_outdoor", 150_000, with_sensor=True)
        from oracle import normals as ON
        idx, _ = ON.knn_indices(xyz, 16)
        nrm, _ = ON.pca_normals(xyz, idx)
        view = sensor - xyz
        nrm = np.where((np.sum(view * nrm, axis=1) < 0)[:, None], -nrm, nrm).astype(np.float32)
        q = (xyz[rng.integers(0, xyz.shape[0], 80_000)] + rng.normal(size=(80_000, 3)) * 0.15).astype(np.float32)
    return xyz.astype(np.float32), nrm.astype(np.float32), q


ARGS = [dict(nb_points=8, stdv=3.0, adaptive_knn=8, imls=False),        # dataset/av_gt_geometry.py:67-70
        dict(nb_points=8, stdv=0.02, adaptive_knn=0, imls=False),       # models/loss.py:85
        dict(nb_points=16, stdv=0.05, adaptive_knn=0, imls=True),
        dict(nb_points=33, stdv=2.0, adaptive_knn=40, imls=False)]
ARG_IDS = ["gt_geometry", "loss", "imls", "k33"]
CASES = ["sphere", "cfg4"]


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("args", ARGS, ids=ARG_IDS)
def test_sdf_from_points_matches_reference_and_oracle(cuda, case, args):
    import nksr_b200
    xyz, nrm, q = _case(case)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    kw = dict(args)
    out = nksr_b200.sdfgen.sdf_from_points(t(q), t(xyz), t(nrm), kw["nb_points"], kw["stdv"], True, kw["imls"],
                                           kw["adaptive_knn"])
    sdf, grad = _np(out[0]), _np(out[1])
    assert sdf.shape == (q.shape[0],) and grad.shape == (q.shape[0], 3) and np.isfinite(sdf).all()
    o_sdf, o_grad = OS.sdf_from_points(q, xyz, nrm, kw["nb_points"], kw["stdv"], True, kw["imls"], kw["adaptive_knn"])
    a, b, c = OS.decision_margins(q, xyz, nrm, kw["nb_points"], kw["stdv"], kw["adaptive_knn"])
    scale = max(np.abs(o_sdf).max(), 1e-6)
    clear = (c > 1e-6) if kw["imls"] else ((a > 1e-4) & (b > 1e-6 * scale) & (c > 1e-6))
    assert clear.mean() > 0.97
    tol = 2e-5 * scale + 2e-5 * np.abs(o_sdf)
    assert (np.abs(sdf - o_sdf)[clear] <= tol[clear]).all(), np.abs(sdf - o_sdf)[clear].max()
    assert np.abs(grad - o_grad)[clear].max() <= 2e-4
    assert (np.abs(sdf - o_sdf) <= tol).mean() >= 0.99
    key = f"{case}_{ARG_IDS[ARGS.index(args)]}"
    with np.load(GOLDEN) as g:
        i, r_q, r_sdf, r_grad = g[key + "_idx"], g[key + "_q"], g[key + "_sdf"], g[key + "_grad"]
    assert np.array_equal(q[i], r_q), "the inputs are no longer the ones the reference binary ran on"
    sdf, grad, o_sdf, clear, tol = sdf[i], grad[i], o_sdf[i], clear[i], tol[i]
    # the oracle is pinned by the reference binary, and so is the kernel (on the stored sample of the queries)
    assert (np.abs(o_sdf - r_sdf)[clear] <= tol[clear]).all(), np.abs(o_sdf - r_sdf)[clear].max()
    assert (np.abs(sdf - r_sdf)[clear] <= tol[clear]).all(), np.abs(sdf - r_sdf)[clear].max()
    assert np.abs(grad - r_grad)[clear].max() <= 2e-4
    assert (np.abs(sdf - r_sdf) <= tol).mean() >= 0.99


def test_sdf_sign_convention_and_default_return(cuda):
    """sdf_from_points(...)[0] without gradient; the reference negates it at its call sites (inside = positive there):
    on a sphere with outward normals the raw value is positive outside."""
    import nksr_b200
    xyz, nrm = clouds.sphere(20_000, noise=0.0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    q = np.array([[0.0, 0.0, 0.0], [0.0, 0.0, 0.6], [0.3, 0.0, 0.0], [0.0, 0.5, 0.0]], np.float32)
    out = nksr_b200.sdfgen.sdf_from_points(t(q), t(xyz), t(nrm), 8, 0.02, False)
    assert len(out) == 1
    s = _np(out[0])
    assert s[0] < 0 and s[2] < 0 and s[1] > 0 and s[3] > 0
    assert abs(abs(s[1]) - 0.25) < 5e-3 and abs(abs(s[0]) - 0.35) < 5e-3
