"""The matrix-free walk steps over each work item in windows of 32 merged locations (csrc/operator.cu): item sizes
around one window (31, 32, 33 locations, so that runs start at a window's first location and items end inside a
window, on it, or one past it) against the fp64 oracle, for the 4- and 8-level walks and the 3-line gradient rows,
on the cloud of tests/test_gpu_matrix_free_items.py."""
import pytest

from oracle import nksr_oracle as O
from tests.test_gpu_matrix_free import _check_against, _np, _t
from tests.test_gpu_matrix_free_items import _system

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("L,approx,S", [(4, True, 31), (4, True, 32), (4, True, 33), (8, True, 33), (4, False, 31),
                                        (4, False, 33)])
def test_window_sized_items_match_oracle(cuda, L, approx, S):
    field, osvh, feats, xyz, nxyz, nval, w = _system(cuda, L=L, approx=approx)
    op = field.matrix_free_system(_t(cuda, xyz), _t(cuda, nxyz), _t(cuda, nval), *w, item_size=S)
    items = _np(field.operator_items(op)[2])
    assert (items[:, 1] - items[:, 0] > 32).any()           # items over more than one window
    A_ref, b_ref, _, A_abs, b_abs = O.build_system(osvh, feats, xyz, nxyz, nval, *w, approx, abs_terms=True)
    _check_against(field, cuda, op, A_ref, A_abs, b_ref, b_abs, A_ref.diagonal(), A_abs.diagonal(),
                   f"L={L} approx={approx} item size {S}")
