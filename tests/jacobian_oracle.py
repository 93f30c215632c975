"""fp64 restatement of the neural field's interpolation u(x) and its position Jacobian J = du/dx (DESIGN.md SPEC S17,
S17a), and of the Jacobian's VJP with respect to the features, built from the oracle's hierarchy (locate, _level_tau,
_tent).  Each comes with its error scale: the same sums with every term replaced by its absolute value
(tests/bounds.py's convention)."""
import numpy as np

from oracle import nksr_oracle as O


def level_weights(osvh, l, q):
    """per query: the level-l neighbour rows (M, 27), fp64 tent weights T_s (M, 27), their derivatives
    dT_s / dx_a (M, 3, 27) -- the tent derivative of SPEC S4 divided by W_l -- and the error scale of those: the
    same products with every tent factor t replaced by |t| + 2^-28 (|x_b| / W_l + 1).  That term is the fp64
    rounding of the local coordinate (at most 2^-52 (|x| / W_l + 1) between the device's x (1 / W_l) - c and this
    x / W_l - c), in units of 2^-24: it bounds what a factor that is 0 here, e.g. at a voxel centre, may be on the
    device.  All are 0 where the slot is absent."""
    base = osvh.locate(q)[l]
    nbr, tau = O._level_tau(osvh, l, q, base)
    t, dt = zip(*(O._tent(tau[:, a]) for a in range(3)))
    eps = 2.0 ** -28 * (np.abs(q.astype(np.float64)) / osvh.level_w(l) + 1.0)
    ta = [np.abs(t[a]) + eps[:, a, None] for a in range(3)]
    ok = nbr >= 0
    w = np.where(ok, O._prod3(*t), 0.0)
    dw = np.stack([np.where(ok, O._prod3(*[dt[b] if b == a else t[b] for b in range(3)]), 0.0) / osvh.level_w(l)
                   for a in range(3)], axis=1)
    dw_abs = np.stack([np.where(ok, O._prod3(*[np.abs(dt[b]) if b == a else ta[b] for b in range(3)]), 0.0)
                       / osvh.level_w(l) for a in range(3)], axis=1)
    return nbr, w, dw, dw_abs


def interp64(osvh, feats, levels, q):
    """u(x) in fp64, (M, C |G|); a given level without voxels gives C zero columns"""
    cols = []
    for l in levels:
        F = feats[l].astype(np.float64)
        if osvh.n(l) == 0:
            cols.append(np.zeros((q.shape[0], F.shape[1])))
            continue
        nbr, w, _, _ = level_weights(osvh, l, q)
        cols.append(np.einsum("ms,msc->mc", w, F[np.where(nbr >= 0, nbr, 0)]))
    return np.concatenate(cols, 1)


def jacobian64(osvh, feats, levels, q):
    """J (M, 3, C |G|) in fp64 and its error scale sum_s |dT_s / dx_a| |F_s| (level_weights' scale of dT_s)"""
    cols, scale = [], []
    for l in levels:
        F = feats[l].astype(np.float64)
        if osvh.n(l) == 0:
            cols.append(np.zeros((q.shape[0], 3, F.shape[1])))
            scale.append(np.zeros((q.shape[0], 3, F.shape[1])))
            continue
        nbr, _, dw, dw_abs = level_weights(osvh, l, q)
        g = F[np.where(nbr >= 0, nbr, 0)]                       # (M, 27, C)
        cols.append(np.einsum("mas,msc->mac", dw, g))
        scale.append(np.einsum("mas,msc->mac", dw_abs, np.abs(g)))
    return np.concatenate(cols, 2), np.concatenate(scale, 2)


def jacobian_vjp64(osvh, levels, channels, q, g):
    """dF_l = sum_q sum_a dT_{slot(v),a}(q) / W_l g[q][a][col(l)] for every given level: {l: (ref (n_l, C), scale)},
    the scale with level_weights' scale of dT"""
    out = {}
    for j, l in enumerate(levels):
        ref = np.zeros((osvh.n(l), channels))
        sc = np.zeros((osvh.n(l), channels))
        if osvh.n(l) == 0:
            out[l] = (ref, sc)
            continue
        nbr, _, dw, dw_abs = level_weights(osvh, l, q)
        gl = g[:, :, j * channels:(j + 1) * channels]           # (M, 3, C)
        for s in range(27):
            ok = nbr[:, s] >= 0
            np.add.at(ref, nbr[ok, s], np.einsum("ma,mac->mc", dw[ok, :, s], gl[ok]))
            np.add.at(sc, nbr[ok, s], np.einsum("ma,mac->mc", dw_abs[ok, :, s], np.abs(gl[ok])))
        out[l] = (ref, sc)
    return out
