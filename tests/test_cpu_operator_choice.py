"""Which operator KernelField.solve uses when the caller does not name one (fields.KernelField._operator): matrix-free
only for approx_kernel_grad systems of at least MATRIX_FREE_MIN_UNKNOWNS unknowns, and never when a Gram fill is
chosen explicitly; an explicit operator wins over both."""
from types import SimpleNamespace

import pytest

from nksr_b200 import fields


def _choice(monkeypatch, n, approx, config=None, env=None):
    for k in ("NKSR_OPERATOR", "NKSR_FILL"):
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    me = SimpleNamespace(svh=SimpleNamespace(num_unknowns=n), approx_kernel_grad=approx, solver_config=config or {})
    return fields.KernelField._operator(me)


def test_default_operator(monkeypatch):
    big, small = fields.MATRIX_FREE_MIN_UNKNOWNS, fields.MATRIX_FREE_MIN_UNKNOWNS - 1
    assert _choice(monkeypatch, big, True) == "matrix_free"
    assert _choice(monkeypatch, small, True) == "assembled"
    assert _choice(monkeypatch, big, False) == "assembled"
    # a chosen fill asks for the assembled matrix
    assert _choice(monkeypatch, big, True, {"fill": "brick"}) == "assembled"
    assert _choice(monkeypatch, big, True, env={"NKSR_FILL": "rows"}) == "assembled"


def test_explicit_operator_wins(monkeypatch):
    assert _choice(monkeypatch, 10, False, {"operator": "matrix_free"}) == "matrix_free"
    assert _choice(monkeypatch, 10, True, {"fill": "rows"}, {"NKSR_OPERATOR": "matrix_free"}) == "matrix_free"
    assert _choice(monkeypatch, fields.MATRIX_FREE_MIN_UNKNOWNS, True, env={"NKSR_OPERATOR": "assembled"}) == "assembled"
    with pytest.raises(ValueError):
        _choice(monkeypatch, 10, True, {"operator": "csr"})
