"""Whole-pipeline parity (SURVEY 8 rows a7/a8): BASELINE.json configs[0] -- the reference's own asset
assets/bunny.ply run the way examples/recons_simple.py:20-27 runs it (detail_level=1.0, extract_dual_mesh(mise_iter=1))
-- through the CUDA path and through the CPU restatement (oracle/pipeline.py), compared as FIELDS and as SURFACES.
Unlike tests/test_gpu_parity.py::test_dual_mesh_matches_oracle (which feeds the oracle's MC driver the GPU field values to
pin the MC bookkeeping exactly), the oracle mesh here comes from the oracle's own evaluator on the oracle's own
coefficients, so the whole chain is compared end to end."""
import copy

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

from oracle import nksr_oracle as O
from oracle import pipeline
from tests import clouds

pytestmark = pytest.mark.gpu


def _np(t):
    return t.detach().cpu().numpy()


def _oracle_mesh(ref, adaptive_depth, mise):
    osvh, svh = ref["osvh"], ref["svh"]

    def mask(v):                                 # LayerField(svh, adaptive_depth), models/nksr_net.py:132
        b = svh.locate(v.astype(np.float32))
        return (b[:adaptive_depth] >= 0).any(axis=0)
    return O.extract_dual_mesh(osvh, lambda q: svh.evaluate(ref["feats"], ref["alpha"], q), 1, mise, mask)


def _surface_distance(va, vb):
    d1 = cKDTree(vb).query(va)[0]
    d2 = cKDTree(va).query(vb)[0]
    return d1, d2


def test_cfg1_bunny_field_and_mesh_match_oracle(cuda):
    import nksr_b200
    xyz, nrm = clouds.bunny()
    assert xyz.shape == (10000, 3)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    rec = nksr_b200.Reconstructor(cuda)
    field = rec.reconstruct(t(xyz), t(nrm), detail_level=1.0, solver_tol=1e-6)        # examples/recons_simple.py:26
    W = rec.last_stats["voxel_size"]
    mesh = field.extract_dual_mesh(mise_iter=1)                                        # examples/recons_simple.py:27
    ref = pipeline.reconstruct(xyz, normal=nrm, voxel_size=W, depth=4, adaptive_depth=2,
                               network=copy.deepcopy(rec.network).cpu(), solver_tol=1e-8)
    for l in range(4):
        assert np.array_equal(_np(field.svh.keys[l]), ref["svh"].keys(l))
    # field
    rng = np.random.default_rng(0)
    q = np.concatenate([xyz[:3000], xyz[:3000] + rng.normal(size=(3000, 3)).astype(np.float32) * np.float32(W)])
    r = field.evaluate_f(t(q), grad=True)
    fo, go = ref["svh"].evaluate(ref["feats"], ref["alpha"], q, grad=True)
    fs = np.abs(fo).max()
    assert np.abs(_np(r.value) - fo).max() <= 5e-3 * fs
    assert np.abs(_np(r.gradient) - go).max() <= 2e-2 * np.abs(go).max()
    # surface: same mesh up to the cells whose corner values sit within rounding of zero
    vo, fo_ = _oracle_mesh(ref, 2, 1)
    v = _np(mesh.v).astype(np.float64)
    assert abs(mesh.f.shape[0] - fo_.shape[0]) <= 0.01 * fo_.shape[0] + 8
    d1, d2 = _surface_distance(v, vo.astype(np.float64))
    cell = W / 2                                                 # final cell size after one MISE round
    assert np.quantile(d1, 0.99) <= 0.02 * cell and np.quantile(d2, 0.99) <= 0.02 * cell
    assert max(d1.max(), d2.max()) <= 1.8 * cell                 # differing cells stay within a cell diagonal
    # manifold: no edge of the (mask-trimmed, hence open at the band boundary) mesh is shared by more than two faces
    f = _np(mesh.f)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    assert cnt.max() <= 2 and (cnt == 2).mean() > 0.8


def test_mesh_of_solved_field_matches_oracle_mesh_as_surface(cuda):
    """a7 end to end on the noisy-sphere setup of the parity tests: GPU mesh of the GPU solution against the oracle's
    mesh of the oracle's solution, for mise_iter = 0, 1, 2 and grid_upsample = 2."""
    import nksr_b200
    xyz, nrm = clouds.sphere(4000, noise=0.002)
    W, L = 0.05, 3
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    rec = nksr_b200.Reconstructor(cuda, tree_depth=L)
    field = rec.reconstruct(t(xyz), t(nrm), voxel_size=W, solver_tol=1e-7)
    ref = pipeline.reconstruct(xyz, normal=nrm, voxel_size=W, depth=L, adaptive_depth=2,
                               network=copy.deepcopy(rec.network).cpu(), solver_tol=1e-9)
    osvh, svh = ref["osvh"], ref["svh"]
    mask = lambda v: (svh.locate(v.astype(np.float32))[:2] >= 0).any(axis=0)
    ev = lambda q: svh.evaluate(ref["feats"], ref["alpha"], q)
    for g, mise in ((1, 0), (1, 1), (1, 2), (2, 1)):
        mesh = field.extract_dual_mesh(grid_upsample=g, mise_iter=mise)
        vo, fo = O.extract_dual_mesh(osvh, ev, g, mise, mask)
        cell = W / (g * 2 ** mise)
        assert abs(mesh.f.shape[0] - fo.shape[0]) <= 0.01 * fo.shape[0] + 8, (g, mise)
        d1, d2 = _surface_distance(_np(mesh.v).astype(np.float64), vo.astype(np.float64))
        assert np.quantile(d1, 0.99) <= 0.02 * cell and np.quantile(d2, 0.99) <= 0.02 * cell, (g, mise)
        r = np.linalg.norm(_np(mesh.v), axis=1)
        assert abs(np.median(r) - 0.35) < 0.004


def _boundary(v, faces):
    """(lengths of the edges used by exactly one triangle, number of edges used by more than two)"""
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    e.sort(axis=1)
    u, c = np.unique(e, axis=0, return_counts=True)
    b = u[c == 1]
    return np.linalg.norm(v[b[:, 0]] - v[b[:, 1]], axis=1), int((c > 2).sum())


@pytest.mark.parametrize("g,mise", [(1, 1), (2, 0), (1, 0)])
def test_adaptive_hierarchy_meshes_without_holes_or_cracks(cuda, g, mise):
    """VERDICT r1 missing #6 / models/nksr_net.py:175-179,214: a hierarchy whose finest voxels were pruned (coarse
    leaves) must still be meshed everywhere.  Half of a densely sampled sphere loses its level-0 voxels; leaves count
    as subdivided ("virtual" finest voxels), so the cells form ONE lattice: the CUDA mesher equals the oracle's
    restatement cell for cell (same vertices to 1e-5, same faces), the surface is closed (every edge in exactly two
    triangles -- no holes where level 0 is missing, no cracks at the level transition), whereas the finest-level-only
    extraction of the same hierarchy is open."""
    import nksr_b200
    xyz, _ = clouds.sphere(60_000, noise=0.0005)
    W, L = 0.04, 3
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    osvh = O.OracleSVH(W, L).build_point_splatting(xyz)
    keys = list(osvh.keys)
    keys[0] = keys[0][O.key_to_ijk(keys[0], 0)[:, 0] >= 0]           # x < 0: level-1 voxels become leaves
    osvh = O.OracleSVH(W, L).build_from_keys(keys)
    svh = nksr_b200.SparseFeatureHierarchy(W, L, cuda).build_from_keys([t(k) for k in keys])

    class Analytic(nksr_b200.fields.BaseField):                      # f = r0 - |x|: the mesher alone is under test
        def evaluate_f(self, q, grad=False):
            return nksr_b200.fields.EvaluationResult(value=0.35 - q.norm(dim=1), gradient=None)

    field = Analytic(svh)
    ev = lambda q: 0.35 - np.linalg.norm(q.astype(np.float32), axis=1).astype(np.float32)
    from nksr_b200.meshing import extract_dual_mesh
    m_fine = extract_dual_mesh(field, g, mise, multi_level=False)
    m_all = extract_dual_mesh(field, g, mise, multi_level=True)
    vo, fo = O.extract_dual_mesh(osvh, ev, g, mise, coarse_levels=L)
    v, f = _np(m_all.v), _np(m_all.f)
    assert v.shape == vo.shape and f.shape == fo.shape
    assert np.abs(v - vo).max() <= 1e-5 and np.array_equal(f, fo)
    # no open boundary is added by the pruning: the data band itself leaves small holes where the sphere clips a cell
    # that holds no data point (the unpruned hierarchy has them too); the finest-level-only extraction of the pruned
    # hierarchy has a macroscopic hole -- the whole x < 0 half
    b_all, nm_all = _boundary(v, f)
    b_fine, _ = _boundary(_np(m_fine.v), _np(m_fine.f))
    full = O.OracleSVH(W, L).build_point_splatting(xyz)
    b_full, _ = _boundary(*O.extract_dual_mesh(full, ev, g, mise))
    assert nm_all == 0
    assert b_all.sum() <= b_full.sum() + 1e-6 and (b_all.size == 0 or b_all.max() <= 0.75 * W)
    assert b_fine.sum() >= 1.5                                       # ~ the great circle at x = 0 (2 pi 0.35 = 2.2)
    assert (v[:, 0] < -0.3).any() and not (_np(m_fine.v)[:, 0] < -0.1).any()
    assert np.abs(np.linalg.norm(v, axis=1) - 0.35).max() <= 0.02 * W


def test_chunked_reconstruction_blends_and_welds(cuda):
    """Chunk mode (examples/recons_by_chunk.py:27-29, NKSR-USAGE.md:88-120,146-167): a sphere cut into 2 x 2 x 2 chunks.
    With every chunk at hand the field is the partition-of-unity blend of the chunk solutions and ONE mesh is extracted
    over it: no cracks along the chunk faces (the clipped per-chunk meshes of round 1 left ~130 units of open edges
    there), on the sphere, and close to the un-chunked reconstruction; the blend is continuous across a seam.
    `chunk_tmp_device = cpu` parks the solved chunks in host memory and gives the same mesh."""
    import nksr_b200
    xyz, nrm = clouds.sphere(60_000, radius=3.5, noise=0.005)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    rec = nksr_b200.Reconstructor(cuda)
    field = rec.reconstruct(t(xyz), t(nrm), detail_level=None, chunk_size=4.0, solver_tol=1e-5)
    assert len(field.fields) == 8 and field.blended
    mesh = field.extract_dual_mesh(mise_iter=1)
    v, f = _np(mesh.v), _np(mesh.f)
    r = np.linalg.norm(v, axis=1)
    assert f.shape[0] > 5000 and abs(np.median(r) - 3.5) < 0.02 and np.percentile(np.abs(r - 3.5), 99) < 0.08
    # against the un-chunked reconstruction: same surface within a fraction of a voxel, and no more open edges
    whole = rec.reconstruct(t(xyz), t(nrm), detail_level=None, voxel_size=0.1, solver_tol=1e-5)
    mw = whole.extract_dual_mesh(mise_iter=1)
    vw = _np(mw.v)
    d_ab, d_ba = _surface_distance(v, vw)
    assert max(np.percentile(d_ab, 99), np.percentile(d_ba, 99)) < 0.05
    blen, over = _boundary(v, f)
    blen_w, over_w = _boundary(vw, _np(mw.f))
    assert blen.sum() <= blen_w.sum() + 1.0 and over <= over_w + 2
    # the unblended union (what a rank of the multi-GPU chunk mapping has) does leave the seams open
    field.blended = False
    mc = field.extract_dual_mesh(mise_iter=1)
    field.blended = True
    assert _boundary(_np(mc.v), _np(mc.f))[0].sum() > blen.sum() + 20.0
    # continuity across the seam x = 0.  The plane is also a voxel face, where ANY single field may jump (a containing
    # voxel active on one side only -- the un-chunked field does too), so the property of the blend is pointwise: with
    # continuous weights, f(a) - f(b) = sum_k w_k(a) (f_k(a) - f_k(b)) + O(|a - b|): for two points 1e-4 apart on the two
    # sides of the seam the blend jumps no more than the largest jump among the chunk fields it blends there (an
    # owner-takes-all union jumps by f_A - f_B instead)
    rng = np.random.default_rng(0)
    q = (xyz[rng.integers(0, xyz.shape[0], 4000)] * rng.uniform(0.995, 1.005, (4000, 1))).astype(np.float32)
    qa, qb = q.copy(), q.copy()
    qa[:, 0], qb[:, 0] = -5e-5, 5e-5
    fa, fb = field.evaluate_f(t(qa)).value, field.evaluate_f(t(qb)).value
    scale = float(whole.evaluate_f(t(q * 1.03)).value.abs().median())
    bound = torch.zeros_like(fa)
    n_blend = torch.zeros_like(fa)
    for k, fk in enumerate(field.fields):
        wk = field._weights(t(qa), k)
        jk = (fk.evaluate_f(t(qa)).value - fk.evaluate_f(t(qb)).value).abs()
        bound = torch.maximum(bound, torch.where(wk > 0, jk, torch.zeros_like(jk)))
        n_blend += (wk > 0).float()
    assert float(n_blend.min()) >= 2                                           # every query sits in a cross-fade band
    assert bool(((fa - fb).abs() <= bound + 0.01 * max(scale, 1e-6)).all())
    # (the blend is NOT the un-chunked function value for value: a chunk's weights are normalised by ITS point counts,
    # models/nksr_net.py:103-111, so the data-to-regulariser balance differs; the zero level sets agree -- checked above)
    # chunk_tmp_device = cpu: the solved chunks wait in host memory, visit the GPU per evaluation, return to the host
    rec.chunk_tmp_device = torch.device("cpu")
    parked = rec.reconstruct(t(xyz), t(nrm), detail_level=None, chunk_size=4.0, solver_tol=1e-5)
    assert all(f_.svh.device.type == "cpu" and f_.alpha.device.type == "cpu" for f_ in parked.fields)
    mp = parked.extract_dual_mesh(mise_iter=1)
    assert all(f_.svh.device.type == "cpu" for f_ in parked.fields)
    # same faces; the vertices move by the run-to-run difference of two solves to tol = 1e-5
    assert torch.equal(mp.f, mesh.f) and torch.allclose(mp.v, mesh.v, atol=1e-3)
