"""CPU: the oracle of the Krylov processes (oracle/krylov_oracle_processes.h) meets the real-case assertions of the
reference's test/test_processes.jl, raises the reference's breakdown messages at the reference's iteration, writes
zero columns under allow_breakdown, and reproduces its frozen fixture bit for bit.  The CSC structure the Python API
gives the coefficient matrices is the reference's."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import processes_oracle as P
from process_cases import K, check_identities, path3, problems

import krylov_b200 as kb

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_processes.json")
NAMES = ("hermitian_lanczos", "arnoldi", "golub_kahan", "nonhermitian_lanczos", "saunders_simon_yip")


def run(name, A, b, c, k, **kw):
    f = getattr(P, name)
    return f(A, b, c, k, **kw) if c is not None else f(A, b, k, **kw)


def as_matrices(name, out, k):
    """nzval outputs -> the reference's sparse matrices, through the Python API's CSC structure."""
    if name == "hermitian_lanczos":
        V, beta, T = out
        return V, beta, kb._csc(T, kb._tridiag_structure(k), (k + 1, k))
    if name == "arnoldi":
        return out
    if name == "golub_kahan":
        V, U, beta, L = out
        return V, U, beta, kb._csc(L, kb._bidiag_structure(k), (k + 1, k + 1))
    V, beta, T, U, gamma, Th = out
    s = kb._tridiag_structure(k)
    return V, beta, kb._csc(T, s, (k + 1, k)), U, gamma, kb._csc(Th, s, (k + 1, k))


@pytest.mark.parametrize("reorth", [False, True])
@pytest.mark.parametrize("name", NAMES)
def test_reference_assertions(name, reorth):
    if reorth and name not in ("hermitian_lanczos", "arnoldi"):
        pytest.skip("reorthogonalization is a keyword of hermitian_lanczos and arnoldi only")
    A, b, c = problems()[name]
    kw = {"reorthogonalization": True} if reorth else {}
    check_identities(name, A, b, c, as_matrices(name, run(name, A, b, c, K, **kw), K))


def _structure_reference(k, bidiag):
    """colptr / rowval of krylov_processes.jl, 1-based, restated loop for loop."""
    if bidiag:
        colptr, rowval = [0] * (k + 2), [0] * (2 * k + 1)
        colptr[0] = 1
        for i in range(1, k + 2):
            pos = colptr[i - 1]
            if i <= k:
                colptr[i] = pos + 2
                rowval[pos - 1], rowval[pos] = i, i + 1
            else:
                colptr[i] = pos + 1
                rowval[pos - 1] = i
        return colptr, rowval
    colptr, rowval = [0] * (k + 1), [0] * (3 * k - 1)
    colptr[0] = 1
    for i in range(1, k + 1):
        pos = colptr[i - 1]
        colptr[i] = 3 * i
        if i == 1:
            rowval[pos - 1], rowval[pos] = i, i + 1
        else:
            rowval[pos - 1], rowval[pos], rowval[pos + 1] = i - 1, i, i + 1
    return colptr, rowval


@pytest.mark.parametrize("k", [1, 2, 3, 7, 20])
def test_coefficient_structure_is_the_reference(k):
    for bidiag, fn in ((False, kb._tridiag_structure), (True, kb._bidiag_structure)):
        colptr, rowval = fn(k)
        ref_c, ref_r = _structure_reference(k, bidiag)
        assert list(colptr + 1) == ref_c and list(rowval + 1) == ref_r


MESSAGES_AT_ZERO = {"hermitian_lanczos": "Exact breakdown β₁ == 0.", "arnoldi": "Exact breakdown β == 0.",
                    "golub_kahan": "Exact breakdown β₁ == 0.", "nonhermitian_lanczos": "Exact breakdown β₁γ₁ == 0.",
                    "saunders_simon_yip": "Exact breakdown β₁ == 0."}
MESSAGES_PATH = {"hermitian_lanczos": "Exact breakdown βᵢ₊₁ == 0 at iteration i = 3.",
                 "arnoldi": "Exact breakdown Hᵢ₊₁.ᵢ == 0 at iteration i = 3.",
                 "golub_kahan": "Exact breakdown αᵢ₊₁ == 0 at iteration i = 1.",
                 "nonhermitian_lanczos": "Exact breakdown βᵢ₊₁γᵢ₊₁ == 0 at iteration i = 3.",
                 "saunders_simon_yip": "Exact breakdown βᵢ₊₁ == 0 at iteration i = 3."}


def breakdown_case(name, zero):
    A, e1 = path3()
    b = np.zeros_like(e1) if zero else e1
    c = e1 if name in ("nonhermitian_lanczos", "saunders_simon_yip") else None
    return A, b, c


@pytest.mark.parametrize("zero", [True, False])
@pytest.mark.parametrize("name", NAMES)
def test_breakdown_messages_and_zero_columns(name, zero):
    A, b, c = breakdown_case(name, zero)
    with pytest.raises(P.ProcessBreakdown) as e:
        run(name, A, b, c, 5)
    assert str(e.value) == (MESSAGES_AT_ZERO if zero else MESSAGES_PATH)[name]
    out = run(name, A, b, c, 5, allow_breakdown=True)
    for x in out:
        assert np.all(np.isfinite(x))
    V = out[0]
    if not zero and name != "golub_kahan":
        assert np.all(V[:, 3:] == 0) and np.all(np.any(V[:, :3] != 0, axis=0))   # v₄ = 0 and every later column
    if zero:
        assert np.all(V[:, 0] == 0)


def _golden_cases():
    return json.load(open(GOLDEN))


def test_golden_fixture_reproduced_bit_for_bit():
    from golden.gen_golden_processes import compute
    g = _golden_cases()
    assert compute() == g
