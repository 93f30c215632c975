"""Host reference (numpy, TEST INFRASTRUCTURE ONLY) for the sort-free placement of the transposed
cross-level Gram entries (DESIGN.md SPEC S6b).

Setting: fine voxel j (level l, offset-space coords u) stores an entry for coarse voxel c (level l+k) iff
c lies in box_k(j) = [((u-1)>>k) - 1, ((u+1)>>k) + 1] per axis (SPEC S6).  With a = u >> k the ancestor of j,
    (u-1)>>k = a - [u mod 2^k == 0]        ("low edge" of the ancestor block on that axis)
    (u+1)>>k = a + [u mod 2^k == 2^k - 1]  ("high edge")
so  c - a in {-1,0,1} always qualifies, c - a = -2 needs the low edge, c - a = +2 the high edge.
Hence the fine voxels reaching c are, for each of the 125 ancestors a = c - d (d in {-2..2}^3), the
descendants of a in an edge class that depends only on d; descendants of one ancestor are contiguous
in Morton order.  Ordering c's transposed segment by (slot of d, Morton index of j) gives

    position(j -> c) = prefix[c][slot(d)] + rank of j among the class(d) descendants of a

and both tables come from linear prefix sums -- no atomics, no sort.  Finer levels come first (ascending), so the
whole segment of c is ordered by (level, slot of d, Morton index); transposed_order gives that order for a whole
hierarchy, and the GPU assembly is checked against it.  tests/test_cpu_placement.py checks the formula and
transposed_order against a brute-force sort on real hierarchies."""
from __future__ import annotations

import numpy as np

from . import nksr_oracle as O

_D5 = np.array([[a, b, c] for a in range(-2, 3) for b in range(-2, 3) for c in range(-2, 3)], np.int64)
_OFF4 = np.array([[a, b, c] for a in range(4) for b in range(4) for c in range(4)], np.int64)


def _edge_class(d):
    """per axis: 0 = any, 1 = low edge required (c - a = -2), 2 = high edge required (c - a = +2)."""
    return np.where(d == -2, 1, np.where(d == 2, 2, 0))


def placement_by_structure(svh: O.OracleSVH, l: int, k: int):
    """-> dict {(c, j): position} for every transposed entry from level l into level l+k."""
    lu = l + k
    fine = svh.ijk(l).astype(np.int64) + O.level_offset(l)              # offset-space coords, Morton order
    nf = fine.shape[0]
    anc_coord = fine >> k
    anc = svh.lookup(lu, anc_coord - O.level_offset(lu))                 # ancestor index of every fine voxel
    assert (anc >= 0).all()
    m = (1 << k) - 1
    low = (fine & m) == 0
    high = (fine & m) == m
    # class membership of every fine voxel for the 27 per-axis requirement combinations
    member = np.ones((27, nf), bool)
    for cls in range(27):
        req = [(cls // 9) % 3, (cls // 3) % 3, cls % 3]
        for ax in range(3):
            if req[ax] == 1:
                member[cls] &= low[:, ax]
            elif req[ax] == 2:
                member[cls] &= high[:, ax]
    # rank of j inside its ancestor block per class, and class counts per ancestor (prefix sums in Morton order)
    first = np.full(svh.n(lu), nf, np.int64)
    np.minimum.at(first, anc, np.arange(nf))
    cum = np.concatenate([np.zeros((27, 1), np.int64), np.cumsum(member, axis=1)], axis=1)      # (27, nf+1)
    rank = cum[:, :-1] - cum[:, first[anc]]                                                    # (27, nf)
    last = np.zeros(svh.n(lu), np.int64)
    np.maximum.at(last, anc, np.arange(nf) + 1)
    count = np.where(first[None] < nf, cum[:, np.minimum(last, nf)] - cum[:, np.minimum(first, nf)], 0)   # (27, n_coarse)
    # prefix over the 125 ancestors of every coarse voxel c (a = c - d)
    coarse = svh.ijk(lu).astype(np.int64) + O.level_offset(lu)
    out = {}
    cls_of_d = (_edge_class(_D5) * np.array([9, 3, 1])).sum(axis=1)                             # (125,)
    nbr = svh.lookup(lu, (coarse[:, None, :] - _D5[None]) - O.level_offset(lu))                  # (n_c, 125) ancestor index or -1
    cnt = np.where(nbr >= 0, count[cls_of_d[None, :], np.maximum(nbr, 0)], 0)                    # (n_c, 125)
    prefix = np.concatenate([np.zeros((coarse.shape[0], 1), np.int64), np.cumsum(cnt, axis=1)], axis=1)
    for c in range(coarse.shape[0]):
        for s in range(125):
            a = nbr[c, s]
            if a < 0 or cnt[c, s] == 0:
                continue
            js = np.nonzero((anc == a) & member[cls_of_d[s]])[0]
            for j in js:
                out[(c, int(j))] = int(prefix[c, s] + rank[cls_of_d[s], j])
    return out, prefix[:, -1]


def placement_by_sort(svh: O.OracleSVH, l: int, k: int):
    """brute force: enumerate box_k(j) for every fine voxel, then sort each coarse segment by
    (slot of d = c - a ... in the same canonical order, Morton index)."""
    lu = l + k
    fine = svh.ijk(l).astype(np.int64) + O.level_offset(l)
    coarse_lookup = lambda q: svh.lookup(lu, q - O.level_offset(lu))
    entries = {}
    for j in range(fine.shape[0]):
        u = fine[j]
        lo = ((u - 1) >> k) - 1
        hi = ((u + 1) >> k) + 1
        a = u >> k
        for x in range(lo[0], hi[0] + 1):
            for y in range(lo[1], hi[1] + 1):
                for z in range(lo[2], hi[2] + 1):
                    c = int(coarse_lookup(np.array([[x, y, z]]))[0])
                    if c < 0:
                        continue
                    d = np.array([x, y, z]) - a                      # c - a
                    slot = int(((d[0] + 2) * 25 + (d[1] + 2) * 5 + (d[2] + 2)))
                    entries.setdefault(c, []).append((slot, j))
    out = {}
    for c, lst in entries.items():
        for pos, (_, j) in enumerate(sorted(lst)):
            out[(c, j)] = pos
    return out


def transposed_order(svh: O.OracleSVH):
    """-> (row, col): every transposed entry of the hierarchy (global unknown indices, levels concatenated), in the
    storage order of SPEC S6b -- by row, then finer level (ascending), then slot of d = c - a, then Morton index."""
    offs = svh.offsets()
    rows, cols, lev, slot = [], [], [], []
    for l in range(svh.depth):
        fine = svh.ijk(l).astype(np.int64)
        for lu in range(l + 1, svh.depth):
            k = lu - l
            cand = (((fine - 1) >> k) - 1)[:, None, :] + _OFF4[None]                 # the 4^3 box of every fine voxel
            c = svh.lookup(lu, cand)
            m = (c >= 0) & np.all(cand <= (((fine + 1) >> k) + 1)[:, None, :], axis=-1)
            d = cand - (fine >> k)[:, None, :]
            j = np.broadcast_to(np.arange(fine.shape[0])[:, None], m.shape)
            rows.append(c[m] + offs[lu])
            cols.append(j[m] + offs[l])
            lev.append(np.full(int(m.sum()), l))
            slot.append(((d + 2) * np.array([25, 5, 1])).sum(axis=-1)[m])
    if not rows:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    rows, cols, lev, slot = (np.concatenate(a) for a in (rows, cols, lev, slot))
    order = np.lexsort((cols, slot, lev, rows))
    return rows[order], cols[order]
