"""Numpy restatement (fp64) of DESIGN.md SPEC S19: the PointTSDFVolume built from sensor rays (csrc/tsdf_volume.cu).

The kernel walks each ray's cells with a 3D-DDA; here each ray is clipped to the box by the slab test and split at
every crossing of a cell-boundary plane, and each piece lies in one cell (found from its midpoint).  The signed
distances are the same IEEE fp64 expressions as the kernel's (which is compiled without fused multiply-adds).

Besides the volume, `tsdf_volume` reports the nodes whose value or class an fp64 restatement cannot pin, because a
decision on the way was within rounding of its threshold:
* a ray's overlap with the node's cell is under 1e-3 h;
* |sdf - tau| or |sdf + tau| is under 1e-5 tau;
* the ray enters two cells at (nearly) the same parameter, which leaves a piece under 1e-3 h between them: every
  cell the walk could enter instead (the box spanned by the cells before and after that piece) is flagged;
* pass 2 (free space) reached the node after a node on the same ray that may or may not hold a near observation, and
  so may stop the ray or not.
"""
from __future__ import annotations

import numpy as np

OVERLAP_EPS = 1e-3      # x h
TAU_EPS = 1e-5          # x tau
NO_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)


def _rays(xyz, sensor):
    s = np.asarray(sensor, np.float32).astype(np.float64)
    p = np.asarray(xyz, np.float32).astype(np.float64)
    v = p - s
    with np.errstate(invalid="ignore", over="ignore"):
        r = np.sqrt(v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1] + v[:, 2] * v[:, 2])
        ok = np.isfinite(r) & (r > 0.0)
        d = v / np.where(ok, r, 1.0)[:, None]
    return s, d, r, ok


def _clip(s, d, r, lo, h, dims, tau, t_lo):
    """slab test of [t_lo, r + tau] against the box [lo - h/2, lo + (dims - 1/2) h]"""
    t0 = np.full(r.shape, t_lo) if np.isscalar(t_lo) else t_lo.copy()
    t1 = r + tau
    ok = np.ones(r.shape, bool)
    for a in range(3):
        blo, bhi = lo[a] - 0.5 * h, lo[a] + (dims[a] - 0.5) * h
        zero = d[:, a] == 0.0
        ok &= ~(zero & ((s[:, a] < blo) | (s[:, a] > bhi)))
        with np.errstate(divide="ignore", invalid="ignore"):
            ta = (blo - s[:, a]) / d[:, a]
            tb = (bhi - s[:, a]) / d[:, a]
        tmin, tmax = np.where(zero, -np.inf, np.minimum(ta, tb)), np.where(zero, np.inf, np.maximum(ta, tb))
        t0, t1 = np.maximum(t0, tmin), np.minimum(t1, tmax)
    return t0, t1, ok & (t0 < t1)


def _pieces(s, d, t0, t1, lo, h, dims):
    """every (ray, cell) piece of the clipped rays, in order of entry parameter within each ray: ray index, cell
    (n, 3), entry and exit parameter"""
    m = s.shape[0]
    g_lo = np.asarray(lo, np.float64) - 0.5 * h
    ts, rid = [t0, t1], [np.arange(m), np.arange(m)]
    for a in range(3):
        x0, x1 = s[:, a] + t0 * d[:, a], s[:, a] + t1 * d[:, a]
        k0 = np.floor((np.minimum(x0, x1) - g_lo[a]) / h).astype(np.int64)
        k1 = np.ceil((np.maximum(x0, x1) - g_lo[a]) / h).astype(np.int64)
        k0, k1 = np.maximum(k0, 1), np.minimum(k1, dims[a] - 1)
        cnt = np.where(d[:, a] != 0.0, np.maximum(k1 - k0 + 1, 0), 0)
        ray = np.repeat(np.arange(m), cnt)
        k = np.arange(cnt.sum()) - np.repeat(np.cumsum(cnt) - cnt, cnt) + np.repeat(k0, cnt)
        t = (lo[a] + (k.astype(np.float64) - 0.5) * h - s[ray, a]) / d[ray, a]
        keep = (t > t0[ray]) & (t < t1[ray])
        ts.append(t[keep])
        rid.append(ray[keep])
    t, ray = np.concatenate(ts), np.concatenate(rid)
    order = np.lexsort((t, ray))
    t, ray = t[order], ray[order]
    piece = ray[:-1] == ray[1:]
    ta, tb, pr = t[:-1][piece], t[1:][piece], ray[:-1][piece]
    tm = 0.5 * (ta + tb)
    x = s[pr] + tm[:, None] * d[pr]
    cell = np.floor((x - g_lo) / h).astype(np.int64)
    cell = np.clip(cell, 0, np.asarray(dims) - 1)
    return pr, cell, ta, tb


def _tie_cells(ray, cell, ta, tb, h):
    """the cells a walk may enter instead, around every piece shorter than OVERLAP_EPS h (where the ray enters two
    cells at nearly the same parameter): every cell of the box spanned by the pieces before and after it"""
    tiny = np.nonzero((tb - ta) < OVERLAP_EPS * h)[0]
    prev = np.where((tiny > 0) & (ray[np.maximum(tiny - 1, 0)] == ray[tiny]), tiny - 1, tiny)
    nxt = np.where((tiny + 1 < ray.size) & (ray[np.minimum(tiny + 1, ray.size - 1)] == ray[tiny]), tiny + 1, tiny)
    a, b = cell[prev], cell[nxt]
    lo, ext = np.minimum(a, b), np.minimum(np.abs(b - a), 1)
    cells = np.concatenate([lo + np.array([(o >> 2) & 1, (o >> 1) & 1, o & 1])[None] * ext for o in range(8)])
    return np.tile(ray[tiny], 8), cells


def _sdf(s, d, r, ray, cell, lo, h):
    c = [lo[a] + cell[:, a].astype(np.float64) * h - s[ray, a] for a in range(3)]
    return r[ray] - (c[0] * d[ray, 0] + c[1] * d[ray, 1] + c[2] * d[ray, 2])


def tsdf_volume(xyz, sensor, volume_min, h, dims, tau, chunk=20000):
    """(volume float32 [X][Y][Z], ambiguous bool [X][Y][Z]) of SPEC S19; volume_min, h and tau are taken as fp32
    values, as the C-ABI takes them"""
    lo = np.asarray(volume_min, np.float32).astype(np.float64)
    h, tau = float(np.float32(h)), float(np.float32(tau))
    dims = tuple(int(v) for v in dims)
    n_nodes = dims[0] * dims[1] * dims[2]
    s, d, r, valid = _rays(xyz, sensor)
    rays = np.nonzero(valid)[0]
    node = lambda c: (c[:, 0] * dims[1] + c[:, 1]) * dims[2] + c[:, 2]
    key = np.full(n_nodes, NO_KEY, np.uint64)
    amb = np.zeros(n_nodes, bool)
    amb_near = np.zeros(n_nodes, bool)     # ambiguous whether the node holds a near observation

    def chunk_pieces(idx):
        t0, t1, ok = _clip(s[idx], d[idx], r[idx], lo, h, dims, tau, 0.0)
        idx, t0, t1 = idx[ok], t0[ok], t1[ok]
        pr, cell, ta, tb = _pieces(s[idx], d[idx], t0, t1, lo, h, dims)
        return idx[pr], cell, ta, tb

    # pass 1: near observations, and every piece's ambiguity
    for c0 in range(0, rays.size, chunk):
        ray, cell, ta, tb = chunk_pieces(rays[c0:c0 + chunk])
        sdf = _sdf(s, d, r, ray, cell, lo, h)
        v = node(cell)
        tr, tc = _tie_cells(ray, cell, ta, tb, h)
        amb[node(tc)] = True
        amb_near[node(tc)[np.abs(_sdf(s, d, r, tr, tc, lo, h)) < tau * (1.0 + TAU_EPS)]] = True
        edge = v[(np.abs(sdf - tau) < TAU_EPS * tau) | (np.abs(sdf + tau) < TAU_EPS * tau)]
        amb[edge] = True
        amb_near[edge] = True
        near = np.abs(sdf) < tau
        q = (np.abs(sdf[near]) / tau).astype(np.float32).view(np.uint32).astype(np.uint64)
        np.minimum.at(key, v[near], (q << np.uint64(32)) | ray[near].astype(np.uint64))
    # pass 2: free space up to the first near node of each ray
    free = np.zeros(n_nodes, bool)
    for c0 in range(0, rays.size, chunk):
        ray, cell, _, _ = chunk_pieces(rays[c0:c0 + chunk])
        if ray.size == 0:
            continue
        v = node(cell)
        sdf = _sdf(s, d, r, ray, cell, lo, h)
        first = np.r_[True, ray[1:] != ray[:-1]]
        start = np.maximum.accumulate(np.where(first, np.arange(ray.size), 0))

        def seen(flag):              # flag at or before this piece, within the ray
            cs = np.cumsum(flag)
            return cs - cs[start] + flag[start] > 0
        isnear = key[v] != NO_KEY
        free[v[~seen(isnear) & (sdf >= tau)]] = True
        # from a node that may or may not be near, the ray may stop or go on, up to the first certain near node
        definite = seen(isnear & ~amb_near[v])
        past_definite = np.r_[False, definite[:-1]] & ~first
        amb[v[seen(amb_near[v]) & ~past_definite & (sdf >= tau * (1.0 - TAU_EPS))]] = True
    vol = np.full(n_nodes, np.nan, np.float32)
    vol[free] = 1.0
    nz = np.nonzero(key != NO_KEY)[0]
    j = (key[nz] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    cell = np.stack([nz // (dims[1] * dims[2]), (nz // dims[2]) % dims[1], nz % dims[2]], axis=1)
    vol[nz] = (_sdf(s, d, r, j, cell, lo, h) / tau).astype(np.float32)
    return vol.reshape(dims), amb.reshape(dims)
