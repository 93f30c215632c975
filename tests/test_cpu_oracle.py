"""CPU tests: oracle self-consistency, MC table properties, library surface (no GPU needed)."""
import ctypes
import os
import re

import numpy as np
import pytest

from oracle import nksr_oracle as O
from tests import clouds

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_morton_roundtrip_and_parent():
    rng = np.random.default_rng(0)
    u = rng.integers(0, 1 << 21, size=(1000, 3))
    k = O.morton_encode(u)
    assert (O.morton_decode(k) == u).all()
    ijk = rng.integers(-(1 << 18), 1 << 18, size=(1000, 3))
    for l in range(3):
        assert (O.voxel_key(ijk >> (l + 1), l + 1) == (O.voxel_key(ijk >> l, l) >> 3)).all()


def test_quantisation_matches_reference_formula():
    # models/nksr_net.py:66: floor(xyz / voxel_size); ours: floor(x/(W/2)) >> 1
    xyz, _ = clouds.offset_blob(5000)
    for W in (0.1, 0.02, 0.37):
        h = O.quantize_half(xyz, W)
        ref = np.floor(xyz / np.float32(W)).astype(np.int32)
        assert (h >> 1 == ref).all()


def test_svh_parent_closed_and_contains_points():
    xyz, _ = clouds.shapenet_like(3000)
    svh = O.OracleSVH(0.02, 4).build_point_splatting(xyz)
    for l in range(3):
        par = np.unique(svh.keys[l] >> 3)
        assert np.isin(par, svh.keys[l + 1]).all()
    assert (svh.locate(xyz) >= 0).all()


def _small_system(C=4, seed=1):
    xyz, nrm = clouds.sphere(800, seed=seed)
    svh = O.OracleSVH(0.05, 3).build_point_splatting(xyz)
    rng = np.random.default_rng(seed)
    feats = [(0.5 + 0.1 * rng.normal(size=(svh.n(l), C))).astype(np.float32) for l in range(3)]
    nxyz = svh.centers(0)
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True))
    A, b, E = O.build_system(svh, feats, xyz, nxyz, nval, 1e4 / 800, 1e4 / nxyz.shape[0] * 0.05 ** 2, 1.0)
    return svh, feats, xyz, A, b


def test_system_is_spd_and_inside_pattern():
    svh, feats, xyz, A, b = _small_system()
    assert abs(A - A.T).max() < 1e-9 * abs(A).max()
    rng = np.random.default_rng(0)
    for _ in range(5):
        v = rng.normal(size=A.shape[0])
        assert v @ (A @ v) > 0
    P = O.structural_pattern(svh)
    assert (A - A.multiply(P)).count_nonzero() == 0
    assert abs(P - P.T).max() == 0


def test_pcg_matches_dense_solve_and_field_vanishes_on_points():
    svh, feats, xyz, A, b = _small_system()
    x, it, res = O.pcg(A, b, 1e-10, 5000)
    assert res <= 1e-10
    xd = np.linalg.solve(A.toarray(), b)
    assert np.linalg.norm(x - xd) <= 1e-6 * np.linalg.norm(xd)
    f, g = O.evaluate_f(svh, feats, x, xyz, grad=True)
    assert np.abs(f).mean() < 5e-3
    outward = xyz / np.linalg.norm(xyz, axis=1, keepdims=True)
    assert np.mean(np.sum(-g * outward, axis=1)) > 0.8       # grad f = -normal


def test_chronopoulos_gear_reference_has_the_pcg_iterates():
    """oracle.pcg_cg (the distributed solve's arrangement) against oracle.pcg, both fp64, on the fp32 values of the
    sphere system of the GPU solver tests (4000 points, W 0.05, 3 levels): the first 20 iterates and residuals agree to
    1e-10 relative.  At tol 1e-6 (about 165 iterations, long after orthogonality is lost) the two stop within 3
    iterations of each other (164 and 166)."""
    xyz, _ = clouds.sphere(4000)
    W = 0.05
    svh = O.OracleSVH(W, 3).build_point_splatting(xyz)
    rng = np.random.default_rng(11)
    feats = [(0.5 + 0.2 * rng.normal(size=(svh.n(l), 4))).astype(np.float32) for l in range(3)]
    nxyz = np.concatenate([svh.centers(0), svh.centers(1)])
    rng = np.random.default_rng(3)
    nval = rng.normal(size=nxyz.shape).astype(np.float32)
    nval /= np.linalg.norm(nval, axis=1, keepdims=True)
    A, b, _ = O.build_system(svh, feats, xyz, nxyz, nval, 1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * W * W, 1.0)
    A32, b32 = A.astype(np.float32).astype(np.float64), b.astype(np.float32).astype(np.float64)
    h_pcg, h_cg = [], []
    O.pcg(A32, b32, 0.0, 20, history=h_pcg)
    O.pcg_cg(A32, b32, 0.0, 20, history=h_cg)
    assert len(h_pcg) == len(h_cg) == 20
    for k, ((x1, r1), (x2, r2)) in enumerate(zip(h_pcg, h_cg), 1):
        assert np.linalg.norm(x1 - x2) <= 1e-10 * np.linalg.norm(x1), k
        assert abs(r1 - r2) <= 1e-10 * r1, k
    _, it1, res1 = O.pcg(A32, b32, 1e-6, 5000)
    _, it2, res2 = O.pcg_cg(A32, b32, 1e-6, 5000)
    assert abs(it1 - it2) <= 3 and res1 <= 1e-6 and res2 <= 1e-6


def test_gradient_matches_finite_differences():
    svh, feats, xyz, A, b = _small_system()
    x, _, _ = O.pcg(A, b, 1e-8, 3000)
    q = (xyz[:50] + 0.003).astype(np.float32)
    _, g = O.evaluate_f(svh, feats, x, q, grad=True)
    eps = 1e-4
    for a in range(3):
        d = np.zeros(3, np.float32); d[a] = eps
        fd = (O.evaluate_f(svh, feats, x, q + d) - O.evaluate_f(svh, feats, x, q - d)) / (2 * eps)
        ok = np.abs(fd - g[:, a]) < 2e-2 * (1 + np.abs(g[:, a]))
        assert ok.mean() > 0.9          # kinks of the trilinear phi make a few samples disagree


def test_mc_table_is_watertight_and_oriented():
    tab, cnt = O.build_mc_table()
    assert cnt.max() == 5 and cnt[0] == 0 and cnt[255] == 0
    # every case: each crossing edge is used by exactly two triangle sides, once per direction
    for case in range(1, 255):
        tris = tab[case][: 3 * cnt[case]].reshape(-1, 3)
        crossing = {e for e, (a, b, _) in enumerate(O.MC_EDGES) if ((case >> a) & 1) != ((case >> b) & 1)}
        assert set(tris.reshape(-1).tolist()) == crossing
    # random smooth field on a grid: closed, consistently oriented surface
    rng = np.random.default_rng(3)
    n = 12
    c = rng.uniform(3, 8, size=(4, 3))
    g = np.stack(np.meshgrid(*[np.arange(n)] * 3, indexing="ij"), -1).reshape(-1, 3).astype(np.float64)
    f = (np.exp(-((g[:, None] - c[None]) ** 2).sum(-1) / 6.0)).sum(1) - 0.6
    keys = O.voxel_key(g.astype(np.int64), 0)
    order = np.argsort(keys)
    svh = O.OracleSVH(1.0, 1).build_from_keys([keys[order]])
    fsorted = f[order]

    def ev(q):
        ijk = np.floor(q.astype(np.float64)).astype(np.int64)      # lattice points are voxel centres i+0.5
        return fsorted[svh.lookup(0, ijk)]
    v, tri = O.extract_dual_mesh(svh, ev, 1, 0)
    assert tri.shape[0] > 50
    e = np.concatenate([tri[:, [0, 1]], tri[:, [1, 2]], tri[:, [2, 0]]])
    fw = set(map(tuple, e.tolist()))
    assert len(fw) == e.shape[0]
    assert all((b, a) in fw for a, b in fw)


def test_oracle_mesh_sphere_radius():
    xyz, nrm = clouds.sphere(20000, noise=0.001)
    W = 0.05
    svh = O.OracleSVH(W, 3).build_point_splatting(xyz)
    feats = [np.full((svh.n(l), 4), 0.5, np.float32) for l in range(3)]
    nxyz = np.concatenate([svh.centers(0), svh.centers(1)])
    nval = -(nxyz / np.linalg.norm(nxyz, axis=1, keepdims=True))
    A, b, _ = O.build_system(svh, feats, xyz, nxyz, nval, 1e4 / xyz.shape[0], 1e4 / nxyz.shape[0] * W * W, 1.0)
    x, it, res = O.pcg(A, b, 1e-6, 3000)
    v, tri = O.extract_dual_mesh(svh, lambda q: O.evaluate_f(svh, feats, x, q), 1, 1)
    r = np.linalg.norm(v, axis=1)
    assert abs(r.mean() - 0.35) < 0.005 and r.min() > 0.33 and r.max() < 0.37
    n = np.cross(v[tri[:, 1]] - v[tri[:, 0]], v[tri[:, 2]] - v[tri[:, 0]])
    assert (np.sum(n * v[tri].mean(1), axis=1) > 0).mean() > 0.99


def test_library_exports_every_declared_symbol():
    import nksr_b200._lib as L
    path = L.library_path()
    assert os.path.exists(path), "build the library first (__graft_entry__.build())"
    lib = ctypes.CDLL(path)
    header = open(os.path.join(ROOT, "include", "nksr_b200.h")).read()
    declared = sorted(set(re.findall(r"NKSR_API [\w\* ]+?(nksr_\w+)\(", header)))
    assert declared == L.exported_symbols()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.nksr_version


def test_ctypes_signatures_match_the_header_prototypes():
    """Every prototype of include/nksr_b200.h against the argument kinds nksr_b200/_lib.py binds: same count,
    pointer where the header has a pointer, the right scalar width elsewhere."""
    import nksr_b200._lib as L
    header = open(os.path.join(ROOT, "include", "nksr_b200.h")).read()
    header = re.sub(r"/\*.*?\*/", " ", header, flags=re.S)
    protos = re.findall(r"NKSR_API\s+([\w\s\*]+?)\b(nksr_\w+)\s*\(([^;]*?)\)\s*;", header, flags=re.S)
    assert len(protos) == len(L._SIGNATURES)
    scalar = {"int64_t": "q", "int32_t": "i", "int": "i", "float": "f", "size_t": "z"}
    struct = {"nksr_svh_t": "S", "nksr_feat_t": "F", "nksr_constraints_t": "K", "nksr_placement_t": "P"}
    for ret, name, params in protos:
        kinds = L._SIGNATURES[name][1]
        plist = [p.strip() for p in params.replace("\n", " ").split(",")] if params.strip() not in ("", "void") else []
        assert len(plist) == len(kinds), name
        for p, k in zip(plist, kinds):
            if "*" in p:
                base = re.sub(r"\bconst\b", "", p).split("*")[0].strip()
                # double*: `info` is a HOST array (ctypes double array), every other one a device buffer
                want = struct.get(base, "d" if (base == "double" and p.split("*")[-1].strip() == "info") else "p")
                assert k == want, (name, p, k)
            else:
                assert k == scalar[p.split()[-2] if len(p.split()) > 1 else p], (name, p, k)
        rk = L._SIGNATURES[name][0]
        ret = ret.strip()
        assert rk == {"int": "i", "size_t": "z", "int64_t": "q", "const char*": "s", "const char *": "s"}[ret], (name, ret)


def test_every_python_call_site_passes_the_declared_number_of_arguments():
    """Static check of the host mirror: each call("nksr_...", ...) in nksr_b200/*.py, bench.py, tools/ and
    __graft_entry__.py has as many arguments as the entry point declares (paths a CPU run never executes)."""
    import ast
    import nksr_b200._lib as L
    files = [os.path.join(ROOT, "nksr_b200", f) for f in os.listdir(os.path.join(ROOT, "nksr_b200")) if f.endswith(".py")]
    files += [os.path.join(ROOT, "bench.py"), os.path.join(ROOT, "__graft_entry__.py")]
    files += [os.path.join(ROOT, "tools", f) for f in os.listdir(os.path.join(ROOT, "tools")) if f.endswith(".py")]
    seen = 0
    for path in files:
        for node in ast.walk(ast.parse(open(path).read())):
            if not isinstance(node, ast.Call) or not node.args:
                continue
            fn = node.func
            fname = fn.id if isinstance(fn, ast.Name) else (fn.attr if isinstance(fn, ast.Attribute) else None)
            first = node.args[0]
            if fname != "call" or not (isinstance(first, ast.Constant) and isinstance(first.value, str)
                                       and first.value.startswith("nksr_")):
                continue
            assert first.value in L._SIGNATURES, (path, first.value)
            if any(isinstance(a, ast.Starred) for a in node.args):
                continue
            assert len(node.args) - 1 == len(L._SIGNATURES[first.value][1]), (os.path.basename(path), node.lineno,
                                                                             first.value)
            seen += 1
    assert seen >= 50


def test_ctypes_mirrors_match_the_header_layout(tmp_path):
    """The structs that cross the C-ABI by pointer: sizeof and every field offset of the ctypes mirror in
    nksr_b200/_lib.py equal what a C compiler makes of include/nksr_b200.h (the header is plain C)."""
    import subprocess
    import nksr_b200._lib as L
    pairs = {"nksr_svh_t": L.SvhT, "nksr_feat_t": L.FeatT, "nksr_constraints_t": L.ConstraintsT,
             "nksr_placement_t": L.PlacementT}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "nksr_b200.h"', "int main(void) {"]
    for cname, mirror in pairs.items():
        lines.append(f'  printf("{cname} %zu\\n", sizeof({cname}));')
        for fname, _ in mirror._fields_:
            lines.append(f'  printf("{cname}.{fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    for cname, mirror in pairs.items():
        assert int(got[cname]) == ctypes.sizeof(mirror), cname
        for fname, _ in mirror._fields_:
            assert int(got[f"{cname}.{fname}"]) == getattr(mirror, fname).offset, f"{cname}.{fname}"


def test_product_does_not_import_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "nksr_b200")):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, fn)).read()
                assert "import oracle" not in src and "from oracle" not in src, fn


def test_no_cpu_fallback():
    import torch
    import nksr_b200
    with pytest.raises(RuntimeError):
        nksr_b200.Reconstructor(torch.device("cpu"))
    svh = nksr_b200.SparseFeatureHierarchy(0.1, 4, "cpu")
    with pytest.raises(RuntimeError):
        svh.build_point_splatting(torch.zeros(10, 3))


def test_mc_tables_inc_is_current():
    import subprocess, sys
    inc = os.path.join(ROOT, "nksr_b200", "csrc", "mc_tables.inc")
    before = open(inc).read()
    subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "gen_mc_tables.py")], stdout=subprocess.DEVNULL)
    assert open(inc).read() == before
    from nksr_b200 import mc_tables
    t, c = mc_tables.build_tables()
    to, co = O.build_mc_table()
    assert (t == to).all() and (c == co).all() and (mc_tables.EDGES == O.MC_EDGES).all()
