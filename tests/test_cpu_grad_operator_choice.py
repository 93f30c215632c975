"""Which operator a grad-recording KernelField.solve uses (fields.KernelField._grad_operator): the matrix-free operator
only when solver_config['operator'] or NKSR_OPERATOR names it, whatever the size rule of inference would choose, and
never with keep_system."""
from types import SimpleNamespace

import pytest

from nksr_b200 import fields


def _choice(monkeypatch, n, approx, config=None, env=None):
    for k in ("NKSR_OPERATOR", "NKSR_FILL"):
        monkeypatch.delenv(k, raising=False)
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    me = SimpleNamespace(svh=SimpleNamespace(num_unknowns=n), approx_kernel_grad=approx, solver_config=config or {})
    return fields.KernelField._grad_operator(me)


def test_grad_solves_assemble_unless_the_operator_is_named(monkeypatch):
    big = fields.MATRIX_FREE_MIN_UNKNOWNS
    assert _choice(monkeypatch, big, True) == "assembled"        # the inference size rule does not apply
    assert _choice(monkeypatch, 10, False) == "assembled"
    assert _choice(monkeypatch, 10, False, {"operator": "matrix_free"}) == "matrix_free"
    assert _choice(monkeypatch, 10, True, env={"NKSR_OPERATOR": "matrix_free"}) == "matrix_free"
    assert _choice(monkeypatch, big, True, {"operator": "assembled"}, {"NKSR_OPERATOR": "matrix_free"}) == "assembled"


def test_keep_system_assembles_and_unknown_names_are_refused(monkeypatch):
    assert _choice(monkeypatch, 10, True, {"operator": "matrix_free", "keep_system": True}) == "assembled"
    assert _choice(monkeypatch, 10, True, {"keep_system": True}, {"NKSR_OPERATOR": "matrix_free"}) == "assembled"
    with pytest.raises(ValueError):
        _choice(monkeypatch, 10, True, {"operator": "csr"})
    with pytest.raises(ValueError):
        _choice(monkeypatch, 10, True, env={"NKSR_OPERATOR": "csr"})
