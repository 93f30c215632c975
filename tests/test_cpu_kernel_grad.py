"""The fp64 kernel-field VJPs (tests/grad_oracle.py) against fp64 central differences: row functionals of value and
gradient rows (full and approx), the regulariser, and a whole solve followed by an evaluation loss.  No GPU."""
import numpy as np
import pytest
import scipy.sparse.linalg as spla

from oracle import nksr_oracle as O
from tests import clouds
from tests import grad_oracle as G

H = 1e-6


def _setup(L, C, seed=0, n=120, W=0.1):
    xyz, nrm = clouds.sphere(n)
    xyz = xyz.astype(np.float32)
    svh = O.OracleSVH(W, L).build_point_splatting(xyz)
    rng = np.random.default_rng(seed)
    feats = [0.5 + 0.3 * rng.normal(size=(svh.n(l), C)) for l in range(L)]
    # normal constraints at voxel centres (the tent snap zone) of the two finest levels, plus off-centre locations
    cen = np.concatenate([svh.centers(l) for l in range(min(2, L))])[:60]
    off = (xyz[:30] + np.float32(0.13 * W)).astype(np.float32)
    return svh, feats, xyz, np.concatenate([cen, off]).astype(np.float32), rng


def _fd(fun, feats, rng, k=12):
    """central differences of fun(feats) on k random entries of every level: list of (level, row, col, value)"""
    out = []
    for l, f in enumerate(feats):
        for _ in range(k):
            i, c = int(rng.integers(f.shape[0])), int(rng.integers(f.shape[1]))
            fp = [g.copy() for g in feats]
            fm = [g.copy() for g in feats]
            fp[l][i, c] += H
            fm[l][i, c] -= H
            out.append((l, i, c, (fun(fp) - fun(fm)) / (2 * H)))
    return out


def _check(fd, dz, tol=1e-6):
    for l, i, c, v in fd:
        assert abs(dz[l][i, c] - v) <= tol * (1 + abs(v)), (l, i, c, dz[l][i, c], v)


def _functional(svh, xyz, mode, approx, coef, vecs):
    """Q(z) = sum_q sum_s omega_{q,s} E_q[n_s] through the oracle's kernel rows"""
    offs = svh.offsets()

    def q(feats):
        base = svh.locate(xyz)
        tot = 0.0
        for l in range(svh.depth):
            if svh.n(l) == 0:
                continue
            nbr, K, dK = O.level_rows(svh, l, xyz, base[l], feats[l], mode == 1, approx)
            g = np.maximum(nbr, 0) + offs[l]
            ok = nbr >= 0
            if mode == 0:
                om = sum(coef[:, k, None] * v[g] for k, v in enumerate(vecs))
                tot += np.sum(np.where(ok, om * K, 0.0))
            else:
                om = sum(coef[:, k, :, None] * v[g][:, None, :] for k, v in enumerate(vecs))
                tot += np.sum(np.where(ok[:, None, :], om * dK, 0.0))
        return tot
    return q


@pytest.mark.parametrize("L,C", [(1, 1), (2, 4), (3, 5)])
@pytest.mark.parametrize("mode,approx", [(0, False), (1, False), (1, True)])
def test_feature_vjp_matches_central_differences(L, C, mode, approx):
    svh, feats, xyz, nxyz, rng = _setup(L, C, seed=L * 10 + C)
    loc = xyz[:80] if mode == 0 else nxyz
    n = int(svh.offsets()[-1])
    vecs = [rng.normal(size=n), rng.normal(size=n)]
    coef = rng.normal(size=(loc.shape[0], 2) if mode == 0 else (loc.shape[0], 2, 3))
    dz = G.feature_vjp(svh, feats, loc, mode, approx, coef, vecs)
    _check(_fd(_functional(svh, loc, mode, approx, coef, vecs), feats, rng), dz)


@pytest.mark.parametrize("L,C", [(1, 4), (3, 5)])
@pytest.mark.parametrize("mode", [0, 1])
def test_evaluate_adjoint_is_the_transpose_evaluation(L, C, mode):
    svh, feats, xyz, nxyz, rng = _setup(L, C, seed=3)
    n = int(svh.offsets()[-1])
    coef = rng.normal(size=(nxyz.shape[0],) if mode == 0 else (nxyz.shape[0], 3))
    d = G.evaluate_adjoint(svh, feats, nxyz, mode, False, coef)
    for _ in range(10):
        j = int(rng.integers(n))
        e = np.zeros(n)
        e[j] = 1.0
        out = O.evaluate_f(svh, feats, e, nxyz, grad=mode == 1)
        want = np.sum(coef * out) if mode == 0 else np.sum(coef * out[1])
        assert abs(d[j] - want) <= 1e-12 * (1 + abs(want))


@pytest.mark.parametrize("L,C", [(1, 1), (3, 4)])
def test_regulariser_vjp_matches_central_differences(L, C):
    svh, feats, _, _, rng = _setup(L, C, seed=5)
    n = int(svh.offsets()[-1])
    lam, alpha = rng.normal(size=n), rng.normal(size=n)
    dz = G.regulariser_vjp(svh, feats, lam, alpha)
    _check(_fd(lambda f: lam @ (O.build_regulariser(svh, f) @ alpha), feats, rng), dz)


@pytest.mark.parametrize("L,C,approx", [(1, 4, False), (2, 1, False), (3, 5, False), (3, 4, True)])
def test_solve_then_evaluate_matches_central_differences(L, C, approx):
    """L = sum h f(x_q) + sum h' . grad f(x_q) with alpha = A(z)^-1 b(z, t): the VJP in z and in the normal targets t"""
    svh, feats, xyz, nxyz, rng = _setup(L, C, seed=7, n=80)
    t = rng.normal(size=(nxyz.shape[0], 3))
    pw, nw, rw = 2.0, 0.05, 0.5
    qx = np.concatenate([xyz[:40] + np.float32(0.02), nxyz[:20]]).astype(np.float32)
    hv, hg = rng.normal(size=qx.shape[0]), rng.normal(size=(qx.shape[0], 3))

    def loss(f, tt=t):
        A, b, _ = O.build_system(svh, f, xyz, nxyz, tt, pw, nw, rw, approx)
        a = spla.spsolve(A.tocsc(), b)
        fv, gv = O.evaluate_f(svh, f, a, qx, grad=True, approx_kernel_grad=approx)
        return hv @ fv + np.sum(hg * gv)

    A, b, _ = O.build_system(svh, feats, xyz, nxyz, t, pw, nw, rw, approx)
    alpha = spla.spsolve(A.tocsc(), b)
    g_alpha = G.evaluate_adjoint(svh, feats, qx, 0, approx, hv) + G.evaluate_adjoint(svh, feats, qx, 1, approx, hg)
    out = G.solve_vjp(svh, feats, xyz, nxyz, t, pw, nw, rw, approx, g_alpha)
    ev = G.feature_vjp(svh, feats, qx, 0, approx, hv[:, None], [alpha])
    eg = G.feature_vjp(svh, feats, qx, 1, approx, hg[:, None, :], [alpha])
    dz = [a + b_ + c for a, b_, c in zip(out["dz"], ev, eg)]
    _check(_fd(loss, feats, rng, k=6), dz, tol=1e-5)
    for _ in range(6):
        j, a = int(rng.integers(t.shape[0])), int(rng.integers(3))
        tp, tm = t.copy(), t.copy()
        tp[j, a] += H
        tm[j, a] -= H
        v = (loss(feats, tp) - loss(feats, tm)) / (2 * H)
        assert abs(out["dt"][j, a] - v) <= 1e-5 * (1 + abs(v))
