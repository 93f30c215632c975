"""fp64 vector-Jacobian products of the kernel field (DESIGN.md 4.6): the reference the backward kernels
(csrc/field_bwd.cu) are held to.  Built on the fp64 oracle's basis functions (oracle/nksr_oracle.py); every function
can also return an `abs_terms` scale -- the same expression with every weight, feature and coefficient replaced by
its absolute value -- the per-entry magnitude against which the fp32 kernels' rounding error is bounded."""
import numpy as np
import scipy.sparse.linalg as spla

from oracle import nksr_oracle as O

_B3C = (lambda b: (b[:, None, None] * b[None, :, None] * b[None, None, :]).reshape(27))(np.array([0.125, 0.75, 0.125]))


def _weights(svh, l, xyz, base, absw):
    """per (location, slot): nbr (M,27), B, T (M,27), dB, dT (M,3,27) in x units; T, dT zero on absent slots"""
    nbr, tau = O._level_tau(svh, l, xyz, base)
    bs, tn = (O._bspline_abs, O._tent_abs) if absw else (O._bspline, O._tent)
    Bw, dBw = zip(*[bs(tau[:, a]) for a in range(3)])
    Tw, dTw = zip(*[tn(tau[:, a]) for a in range(3)])
    W = svh.level_w(l)
    ok = nbr >= 0
    B, T = O._prod3(*Bw), np.where(ok, O._prod3(*Tw), 0.0)
    dB, dT = np.zeros((xyz.shape[0], 3, 27)), np.zeros((xyz.shape[0], 3, 27))
    for a in range(3):
        b, t = list(Bw), list(Tw)
        b[a], t[a] = dBw[a], dTw[a]
        dB[:, a] = O._prod3(*b) / W
        dT[:, a] = np.where(ok, O._prod3(*t) / W, 0.0)
    return nbr, B, T, dB, dT


def _feature_vjp_level(svh, l, xyz, base, z, mode, approx, omega, absw):
    nbr, B, T, dB, dT = _weights(svh, l, xyz, base, absw)
    ok = nbr >= 0
    zn = np.where(ok[:, :, None], z[np.maximum(nbr, 0)], 0.0)                         # (M,27,C)
    phi = np.einsum('ms,msc->mc', T, zn)
    if mode == 0:
        om = np.where(ok, omega, 0.0)
        psi = np.einsum('ms,msc->mc', om * B, zn)
        contrib = (om * B)[:, :, None] * phi[:, None, :] + T[:, :, None] * psi[:, None, :]
    else:
        om = np.where(ok[:, None, :], omega, 0.0)                                     # (M,3,27)
        psi0 = np.einsum('ms,msc->mc', np.sum(om * dB, axis=1), zn)
        contrib = np.sum(om * dB, axis=1)[:, :, None] * phi[:, None, :] + T[:, :, None] * psi0[:, None, :]
        if not approx:
            dphi = np.einsum('mas,msc->mac', dT, zn)
            psia = np.einsum('mas,msc->mac', om * B[:, None, :], zn)
            contrib += np.einsum('mas,mac->msc', om * B[:, None, :], dphi)
            contrib += np.einsum('mas,mac->msc', dT, psia)
    dz = np.zeros(z.shape)
    np.add.at(dz, nbr[ok], contrib[ok])
    return dz


def feature_vjp(svh, feats, xyz, mode, approx, coef, vecs, abs_terms=False):
    """d/dz sum_q sum_s omega_{q,(a,)s} E_q[n_s] per level, omega = sum_k coef[q,k(,a)] vecs[k][n_s].
    mode 0: value rows, coef (M, K); mode 1: gradient rows, coef (M, K, 3).  Returns the list of (n_l, C) arrays
    (and their abs-term scales)."""
    offs = svh.offsets()
    base = svh.locate(xyz)
    out, outa = [], []
    for l in range(svh.depth):
        z = np.asarray(feats[l], np.float64)
        if svh.n(l) == 0:
            out.append(np.zeros(z.shape)); outa.append(np.zeros(z.shape))
            continue
        nbr = O._level_tau(svh, l, xyz, base[l])[0]
        g = np.maximum(nbr, 0) + offs[l]
        if mode == 0:
            om = sum(coef[:, k, None] * np.asarray(v, np.float64)[g] for k, v in enumerate(vecs))
            oma = sum(np.abs(coef[:, k, None]) * np.abs(np.asarray(v, np.float64)[g]) for k, v in enumerate(vecs))
        else:
            om = sum(coef[:, k, :, None] * np.asarray(v, np.float64)[g][:, None, :] for k, v in enumerate(vecs))
            oma = sum(np.abs(coef[:, k, :, None]) * np.abs(np.asarray(v, np.float64)[g])[:, None, :]
                      for k, v in enumerate(vecs))
        out.append(_feature_vjp_level(svh, l, xyz, base[l], z, mode, approx, om, False))
        if abs_terms:
            outa.append(_feature_vjp_level(svh, l, xyz, base[l], np.abs(z), mode, approx, oma, True))
    return (out, outa) if abs_terms else out


def evaluate_adjoint(svh, feats, xyz, mode, approx, coef, abs_terms=False):
    """dalpha = sum_q coef_q E_q: value rows coef (M,), gradient rows coef (M,3); (n,) and its abs-term scale"""
    offs = svh.offsets()
    base = svh.locate(xyz)
    n = int(offs[-1])
    d, da = np.zeros(n), np.zeros(n)
    for l in range(svh.depth):
        if svh.n(l) == 0:
            continue
        nbr, K, dK, Ka, dKa = O.level_rows(svh, l, xyz, base[l], feats[l], mode == 1, approx, abs_terms=True)
        ok = nbr >= 0
        if mode == 0:
            v, va = coef[:, None] * K, np.abs(coef[:, None]) * Ka
        else:
            v, va = np.einsum('ma,mas->ms', coef, dK), np.einsum('ma,mas->ms', np.abs(coef), dKa)
        np.add.at(d, nbr[ok] + offs[l], v[ok])
        np.add.at(da, nbr[ok] + offs[l], va[ok])
    return (d, da) if abs_terms else d


def regulariser_vjp(svh, feats, lam, alpha, abs_terms=False):
    """d/dz (lam^T R alpha) per level: sum_{i' in N27(i)} B3c(i'-i) (lam_i alpha_i' + alpha_i lam_i') z_i'"""
    offs = svh.offsets()
    out, outa = [], []
    for l in range(svh.depth):
        z = np.asarray(feats[l], np.float64)
        if svh.n(l) == 0:
            out.append(np.zeros(z.shape)); outa.append(np.zeros(z.shape))
            continue
        nbr = svh.nbr27(l)
        ok = nbr >= 0
        li, ai = lam[offs[l]:offs[l + 1]], alpha[offs[l]:offs[l + 1]]
        ln, an = li[np.maximum(nbr, 0)], ai[np.maximum(nbr, 0)]
        zn = np.where(ok[:, :, None], z[np.maximum(nbr, 0)], 0.0)
        w = np.where(ok, _B3C[None] * (li[:, None] * an + ai[:, None] * ln), 0.0)
        out.append(np.einsum('ns,nsc->nc', w, zn))
        if abs_terms:
            wa = np.where(ok, _B3C[None] * (np.abs(li[:, None] * an) + np.abs(ai[:, None] * ln)), 0.0)
            outa.append(np.einsum('ns,nsc->nc', wa, np.abs(zn)))
    return (out, outa) if abs_terms else out


def solve_vjp(svh, feats, pos, nrm, t, pw, nw, rw, approx, g_alpha, alpha=None, abs_terms=False):
    """Backward of alpha = A(z)^-1 b(z, t) (SPEC S5) for the upstream gradient g_alpha, all in fp64:
    lambda = A^-1 g_alpha, dz = sum_j w_j [(t_j - E_j alpha) d(E_j lambda) - (E_j lambda) d(E_j alpha)]
    - reg d(lambda^T R alpha), dt = w_nrm E_nrm lambda.  alpha: the solution to linearise at (default: the fp64 solve).
    Returns dict(alpha, lam, dz (list), dt (K,3)[, dz_abs])."""
    A, b, E = O.build_system(svh, feats, pos, nrm, t, pw, nw, rw, approx)
    A = A.tocsc()
    if alpha is None:
        alpha = spla.spsolve(A, b)
    lam = spla.spsolve(A, np.asarray(g_alpha, np.float64))
    N, K = pos.shape[0], nrm.shape[0]
    ea, el = E @ alpha, E @ lam
    fa, fl = ea[:N], el[:N]
    ga, gl = ea[N:].reshape(K, 3), el[N:].reshape(K, 3)
    vecs = [lam, alpha]
    dz, dza = feature_vjp(svh, feats, pos, 0, approx, np.stack([-pw * fa, -pw * fl], 1), vecs, True)
    if K:
        t = np.asarray(t, np.float64).reshape(K, 3)
        dn, dna = feature_vjp(svh, feats, nrm, 1, approx, np.stack([nw * (t - ga), -nw * gl], 1), vecs, True)
        dz = [a + b_ for a, b_ in zip(dz, dn)]
        dza = [a + b_ for a, b_ in zip(dza, dna)]
    dr, dra = regulariser_vjp(svh, feats, lam, alpha, True)
    dz = [a - rw * b_ for a, b_ in zip(dz, dr)]
    dza = [a + abs(rw) * b_ for a, b_ in zip(dza, dra)]
    out = dict(alpha=alpha, lam=lam, dz=dz, dt=nw * gl)
    if abs_terms:
        out["dz_abs"] = dza
    return out
