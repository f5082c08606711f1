"""CPU: the restatement of cg_lanczos_shift! and cgls_lanczos_shift! (oracle/shift_oracle.py) against the reference's
own assertions (test/test_cg_lanczos_shift.jl, test/test_cgls_lanczos_shift.jl), against cg_lanczos! at σ = 0, and
against its frozen output (tests/golden/oracle_shift.json)."""
import json
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as sla

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from oracle import oracle as O  # noqa: E402
from oracle import shift_oracle as S  # noqa: E402
from oracle.lsq_oracle import lsq_test  # noqa: E402

SHIFTS = [1.0, 2.0, 3.0, 4.0, 5.0, 6.0]


def _direct(K, rhs):
    return sla.spsolve(sp.csc_matrix(K), rhs)


def test_cg_lanczos_shift_solves_each_system():
    A, b = O.symmetric_definite()
    n = A.shape[0]
    xs, st = S.cg_lanczos_shift(A, b, SHIFTS, itmax=n)
    assert st["solved"] and len(xs) == len(SHIFTS)
    for s, x in zip(SHIFTS, xs):
        K = A + s * sp.eye(n)
        assert np.linalg.norm(b - K @ x) / np.linalg.norm(b) <= 1e-6
        assert np.linalg.norm(x - _direct(K, b)) <= 1e-6 * np.linalg.norm(x)


def test_negative_curvature_flags():
    A, b = O.symmetric_definite()
    _, st = S.cg_lanczos_shift(A, b, [-4.0, -3.0, 2.0], check_curvature=True, itmax=A.shape[0])
    assert st["indefinite"] == [True, True, False]


@pytest.mark.parametrize("name", ["cg_lanczos_shift", "cgls_lanczos_shift"])
def test_zero_rhs(name):
    A, b = O.zero_rhs()
    xs, st = getattr(S, name)(A, b, SHIFTS)
    assert all(np.linalg.norm(x) == 0 for x in xs)
    assert st["status"] == "x is a zero-residual solution" and st["niter"] == 0 and st["solved"]


def test_diagonal_preconditioner():
    A, b, M = O.square_preconditioned()
    n = A.shape[0]
    xs, st = S.cg_lanczos_shift(A, b, SHIFTS, M=M)
    assert st["solved"]
    for s, x in zip(SHIFTS, xs):
        assert np.linalg.norm(b - (A + s * sp.eye(n)) @ x) / np.linalg.norm(b) <= 1e-6


@pytest.mark.parametrize("name", ["cg_lanczos_shift", "cgls_lanczos_shift"])
def test_callback_exit(name):
    A, b = O.symmetric_definite()
    seen = []
    _, st = getattr(S, name)(A, b, SHIFTS, atol=0.0, rtol=0.0, callback=lambda it: seen.append(it) or it >= 2)
    assert st["status"] == "user-requested exit" and st["niter"] == 2 and seen == [1, 2]


@pytest.mark.parametrize("npower", [1, 2, 3, 4])
def test_cgls_lanczos_shift_solves_each_system(npower):
    b, A = lsq_test(40, 40, 4, npower, 0)[:2]
    n = A.shape[1]
    xs, st = S.cgls_lanczos_shift(A, b, SHIFTS)
    assert st["solved"] and st["indefinite"] == [False] * len(SHIFTS)
    Atb = A.T @ b
    for s, x in zip(SHIFTS, xs):
        K = A.T @ A + s * sp.eye(n)
        assert np.linalg.norm(Atb - K @ x) / np.linalg.norm(Atb) <= 1e-6
        assert np.linalg.norm(x - _direct(K, Atb)) <= 1e-6 * np.linalg.norm(x)


def test_cgls_refuses_a_preconditioner():
    b, A = lsq_test(40, 40, 4, 1, 0)[:2]
    with pytest.raises(ValueError, match="Preconditioner `M` is not supported."):
        S.cgls_lanczos_shift(A, b, SHIFTS, M=np.ones(A.shape[0]))
    with pytest.raises(TypeError):
        S.cgls_lanczos_shift(A, b, SHIFTS, check_curvature=True)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_zero_shift_column_is_cg_lanczos(dtype):
    """σ = 0 with M = I runs cg_lanczos!'s iteration operation for operation: x byte for byte."""
    A = O.get_div_grad(6, 6, 6)
    b = np.ones(A.shape[0])
    xs, st = S.cg_lanczos_shift(A, b, [0.0, 3.0, 0.25], atol=0.0, rtol=0.0, itmax=10, dtype=dtype)
    x0, s0 = O.cg_lanczos(A, b, atol=0.0, rtol=0.0, itmax=10, dtype=dtype)
    assert st["niter"] == s0["niter"] == 10
    assert xs[0].tobytes() == x0.tobytes()
    assert np.array_equal(st["residuals"][0], s0["residuals"])


def test_history_only_for_active_shifts():
    """Each shift's history has one entry per iteration it was active in, plus the initial one."""
    A = O.get_div_grad(6, 6, 6)
    b = np.ones(A.shape[0])
    _, st = S.cg_lanczos_shift(A, b, [0.0, 10.0, 1000.0])
    lens = [len(r) for r in st["residuals"]]
    assert lens[0] == st["niter"] + 1 and lens[0] > lens[1] > lens[2]


def test_golden():
    import gen_golden_shift as G
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "oracle_shift.json")))
    for name, f, A, b, shifts, kw in G.cases():
        _, st = f(A, b, shifts, **kw)
        g = gold[name]
        assert st["niter"] == g["niter"] and st["status"] == g["status"] and st["indefinite"] == g["indefinite"], name
        for r, rg in zip(st["residuals"], g["residuals"]):
            assert np.array_equal(r, np.asarray(rg)), name
