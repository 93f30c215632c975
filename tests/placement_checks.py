"""The SPEC S6b checks of an assembled Gram system against the host reference (oracle/placement_proto.py), shared by
the parity tests of every depth."""
import numpy as np
import scipy.sparse as sp

from oracle import nksr_oracle as O
from oracle import placement_proto as PP
from tests.bounds import level_of


def assert_structural_placement(osvh, rp, col, val, cnt, cnt_down, what):
    """cnt / cnt_down split the structural pattern at the level offsets, every slot is written once (no slot twice,
    none left out), every row's finer-level segment follows placement_proto.transposed_order, and every transposed
    copy (c, j) is bitwise the value row j stores for column c.  Arrays as numpy (rowptr, col, val, cnt, cnt_down)."""
    pattern = O.structural_pattern(osvh)
    P = pattern.tocoo()
    offs = osvh.offsets()
    n = int(offs[-1])
    finer = level_of(offs, P.col) < level_of(offs, P.row)
    cnt_ref = np.bincount(P.row[~finer], minlength=n)
    down_ref = np.bincount(P.row[finer], minlength=n)
    bad = np.nonzero((cnt != cnt_ref) | (cnt_down != down_ref))[0]
    assert bad.size == 0, f"{what}: row lengths differ in {bad.size} rows, first at row {bad[0]} level " \
                          f"{level_of(offs, bad[0])}: cnt {cnt[bad[0]]} / {cnt_ref[bad[0]]}, " \
                          f"down {cnt_down[bad[0]]} / {down_ref[bad[0]]}"
    assert np.array_equal(rp, np.concatenate([[0], np.cumsum(cnt_ref + down_ref)])), what
    A = sp.csr_matrix((np.ones(col.shape[0]), col, rp), shape=(n, n), copy=True)   # (sum_duplicates sorts in place)
    A.sum_duplicates()
    assert A.nnz == rp[-1] and (A - pattern).count_nonzero() == 0, f"{what}: pattern"
    order_rows, order_cols = PP.transposed_order(osvh)
    row_of = np.repeat(np.arange(n), np.diff(rp))
    down = np.arange(rp[-1]) - rp[row_of] >= cnt[row_of]
    assert order_cols.shape[0] == int(down.sum()) > 0, what
    wrong = np.nonzero((row_of[down] != order_rows) | (col[down] != order_cols))[0]
    if wrong.size:
        r, c = int(order_rows[wrong[0]]), int(order_cols[wrong[0]])
        raise AssertionError(f"{what}: {wrong.size} transposed entries out of S6b order, first in row {r} (level "
                             f"{level_of(offs, r)}), expected column {c} (level {level_of(offs, c)}), "
                             f"got {col[down][wrong[0]]}")
    own_key = row_of[~down] * n + col[~down]
    srt = np.argsort(own_key)
    src_key = col[down].astype(np.int64) * n + row_of[down]
    at = np.minimum(np.searchsorted(own_key[srt], src_key), own_key.size - 1)
    assert np.array_equal(own_key[srt][at], src_key), f"{what}: a transposed entry without its source entry"
    assert np.array_equal(val[~down][srt][at].view(np.uint32), val[down].view(np.uint32)), \
        f"{what}: a transposed copy differs from its source entry"
