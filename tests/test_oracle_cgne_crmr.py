"""The CPU oracle's cgne and crmr (oracle/krylov_oracle_cgne.h) against the reference's own assertions
(test/test_cgne.jl and test/test_crmr.jl, real case, same tolerance), against a dense restatement of both recurrences,
against the frozen histories of tests/golden/oracle_cgne_crmr.json (tests/golden/gen_golden_cgne_crmr.py), and on the
reference's quirks the GPU must repeat."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import cgne_oracle as O
from parity import golden_module

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1.0e-6                                                         # cgne_tol, crmr_tol
G = golden_module("cgne_crmr")
GOLD = json.load(open(os.path.join(HERE, "golden", "oracle_cgne_crmr.json")))
SOLVERS = ["cgne", "crmr"]


def _solve(solver, A, b, **kw):
    return getattr(O, solver)(A, b, **kw)


def _resid(A, b, x, lam=0.0):
    """test_cgne / test_crmr: r = b - A x; with λ > 0, s = r / √λ and r = r - √λ s."""
    r = b - A @ x
    if lam > 0:
        s = r / np.sqrt(lam)
        r = r - np.sqrt(lam) * s
    return np.linalg.norm(r) / np.linalg.norm(b)


def _check_min_norm(A, b, x, lam=0.0):
    """check_min_norm (test/test_utils.jl): the least-norm solution of [A √λI] [x; s] = b from a QR factorization."""
    Ad = A.toarray()
    if lam > 0:
        Ad = np.hstack([Ad, np.sqrt(lam) * np.eye(Ad.shape[0])])
        x = np.concatenate([x, (b - A @ x) / np.sqrt(lam)])
    Q, R = np.linalg.qr(Ad.T)
    xmin = Q @ np.linalg.lstsq(R.T, b, rcond=None)[0]
    return x, xmin, np.linalg.norm(xmin)


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("name", ["under_consistent", "square_consistent", "over_consistent"])
def test_consistent_systems(solver, name):
    A, b = getattr(O, name)()
    x, st = _solve(solver, A, b)
    assert _resid(A, b, x) <= TOL
    assert st["solved"]
    xI, xmin, xmin_norm = _check_min_norm(A, b, x)
    assert np.linalg.norm(xI - xmin) <= np.linalg.cond(A.toarray()) * TOL * xmin_norm


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("name", ["under_inconsistent", "square_inconsistent", "over_inconsistent"])
def test_inconsistent_systems(solver, name):
    A, b = getattr(O, name)()
    x, st = _solve(solver, A, b, history=True)
    assert st["inconsistent"] and not st["solved"]
    if solver == "crmr":
        assert st["Aresiduals"][-1] <= TOL
        assert st["status"] == "system probably inconsistent but least squares/norm solution found"
    else:
        assert st["status"] == "system probably inconsistent"


@pytest.mark.parametrize("solver", SOLVERS)
def test_regularization(solver):
    A, b = O.over_inconsistent()
    x, st = _solve(solver, A, b, lambda_=1e-3)
    assert _resid(A, b, x, 1e-3) <= TOL
    assert st["solved"]
    xI, xmin, xmin_norm = _check_min_norm(A, b, x, 1e-3)
    assert np.linalg.norm(xI - xmin) <= np.linalg.cond(A.toarray()) * TOL * xmin_norm


@pytest.mark.parametrize("solver", SOLVERS)
def test_zero_rhs(solver):
    """b = 0 exits before the loop; CRMR alone pushes one ‖Aᵀr‖ entry of 0 at that exit."""
    A, b = O.zero_rhs()
    x, st = _solve(solver, A, b, lambda_=1e-3 if solver == "cgne" else 0.0, history=True)
    assert np.linalg.norm(x) == 0 and st["status"] == "x is a zero-residual solution"
    assert st["niter"] == 0 and st["solved"] and not st["inconsistent"]
    assert list(st["residuals"]) == [0.0]
    if solver == "crmr":
        assert list(st["Aresiduals"]) == [0.0]
    else:
        assert "Aresiduals" not in st


@pytest.mark.parametrize("solver", SOLVERS)
def test_preconditioned(solver):
    cases = [G.mass_transfer()]
    if solver == "cgne":                                             # test_cgne.jl alone runs square_preconditioned
        cases.append(O.square_preconditioned())
    for A, b, N in cases:
        x, st = _solve(solver, A, b, N=N)
        assert _resid(A, b, x) <= TOL
        assert st["solved"]
        xI, xmin, xmin_norm = _check_min_norm(A, b, x)
        assert np.linalg.norm(xI - xmin) <= np.linalg.cond(A.toarray()) * TOL * xmin_norm


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("t", [False, True])
def test_extra_vector_dimensions(solver, t):
    """small_sp: N (m x m) and λ = 1 on a rectangular A -- the m-dimensional s and z / Nq run without a size error."""
    A, b, c, D = O.small_sp(t)
    x, st = _solve(solver, A, b, N=1.0 / D, lambda_=1.0)
    assert x.shape == (A.shape[1],) and np.all(np.isfinite(x))


@pytest.mark.parametrize("solver", SOLVERS)
def test_callback_stops(solver):
    A, b = O.over_consistent()
    seen = []
    x, st = _solve(solver, A, b, callback=lambda it: seen.append(it) or True)
    assert st["status"] == "user-requested exit" and st["niter"] == 1 and seen == [1]


def _dense(solver, A, b, N=None, lam=0.0, iters=5):
    """cgne.jl / crmr.jl restated densely in NumPy, for `iters` iterations: the residual (and ‖Aᵀr‖) history."""
    A = A.toarray()
    m, n = A.shape
    Nm = np.diag(N) if N is not None else np.eye(m)
    x = np.zeros(n)
    if solver == "cgne":
        r = b.copy()
        z = Nm @ r
        res = [np.linalg.norm(r)]
        s = r.copy()
        p = A.T @ z
        gamma = r @ z
        for _ in range(iters):
            q = A @ p + lam * s
            delta = p @ p + lam * (s @ s)
            alpha = gamma / delta
            x = x + alpha * p
            r = r - alpha * q
            z = Nm @ r
            gnext = r @ z
            beta = gnext / gamma
            p = A.T @ z + beta * p
            s = r + beta * s
            gamma = gnext
            res.append(np.sqrt(gnext))
        return x, res, None
    r = Nm @ b
    rNorm = np.linalg.norm(r)
    res, ares = [rNorm], []
    s = r.copy()
    Ar = A.T @ r
    p = Ar.copy()
    gamma = Ar @ Ar + lam * rNorm * rNorm
    ares.append(np.sqrt(gamma))
    for _ in range(iters):
        q = A @ p + lam * s
        Nq = Nm @ q
        alpha = gamma / (q @ Nq)
        x = x + alpha * p
        r = r - alpha * Nq
        rNorm = np.linalg.norm(r)
        Ar = A.T @ r
        gnext = Ar @ Ar + lam * rNorm * rNorm
        beta = gnext / gamma
        p = Ar + beta * p
        s = r + beta * s
        gamma = gnext
        res.append(rNorm)
        ares.append(np.sqrt(gamma))
    return x, res, ares


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("variant", ["plain", "N", "lambda", "N_lambda", "N_ldiv"])
def test_recurrences_match_a_dense_restatement(solver, variant):
    """With N ≠ I, CGNE's first entry is ‖b‖ and every later one √⟨r, N r⟩; CRMR's r is N (b - A x) and its first
    ‖Aᵀr‖ entry carries λ ‖r‖² (from the rounded ‖r‖) under the root."""
    rng = np.random.default_rng(7)
    A = sp.csr_matrix(rng.standard_normal((12, 30)))
    b = rng.standard_normal(12)
    d = np.linspace(0.5, 2.0, 12)
    N = d if "N" in variant else None
    lam = 0.3 if "lambda" in variant else 0.0
    ldiv = variant == "N_ldiv"
    x, st = _solve(solver, A, b, N=N, lambda_=lam, ldiv=ldiv, itmax=5, atol=0.0, rtol=0.0, history=True)
    xd, res, ares = _dense(solver, A, b, N=(1.0 / d if ldiv else d) if N is not None else None, lam=lam)
    assert st["niter"] == 5 and st["status"] == "maximum number of iterations exceeded"
    np.testing.assert_allclose(st["residuals"], res, rtol=1e-10)
    if solver == "crmr":
        np.testing.assert_allclose(st["Aresiduals"], ares, rtol=1e-10)
    np.testing.assert_allclose(x, xd, rtol=1e-9, atol=1e-12 * np.linalg.norm(xd))
    if solver == "cgne" and N is not None:
        assert st["residuals"][0] == pytest.approx(np.linalg.norm(b), rel=1e-15)


def test_only_cgne_stops_on_machine_precision():
    """resid_decrease_mach (rNorm + 1 ≤ 1) is CGNE's alone: with atol = rtol = 0 and a tiny b, CGNE stops as solved
    after one iteration while CRMR runs on to itmax."""
    rng = np.random.default_rng(3)
    A = sp.csr_matrix(rng.standard_normal((8, 20)))
    b = 1e-20 * rng.standard_normal(8)
    _, sc = O.cgne(A, b, atol=0.0, rtol=0.0, itmax=6)
    _, sr = O.crmr(A, b, atol=0.0, rtol=0.0, itmax=6)
    assert (sc["niter"], sc["solved"], sc["status"]) == (1, True, "solution good enough given atol and rtol")
    assert (sr["niter"], sr["solved"], sr["status"]) == (6, False, "maximum number of iterations exceeded")


def test_status_precedence():
    """Both rank 'inconsistent' above 'tired': a run that is both at once reports each solver's own inconsistent
    status."""
    A, b = O.square_inconsistent()
    for solver, want in (("cgne", "system probably inconsistent"),
                         ("crmr", "system probably inconsistent but least squares/norm solution found")):
        _, st = _solve(solver, A, b, itmax=1)                     # tired and inconsistent at once
        assert st["niter"] == 1 and st["inconsistent"] and st["status"] == want


def test_float32_runs():
    A, b = O.under_consistent()
    for solver in SOLVERS:
        x, st = _solve(solver, A, b.astype(np.float32), dtype=np.float32)
        assert x.dtype == np.float32 and st["solved"]


@pytest.mark.parametrize("name", sorted(GOLD))
def test_oracle_reproduces_golden(name):
    solver, A, b, kw = G.cases()[name]
    x, st = G.run(solver, A, b, **kw)
    want = GOLD[name]
    assert (st["niter"], st["solved"], st["inconsistent"], st["status"]) == \
        (want["niter"], want["solved"], want["inconsistent"], want["status"])
    np.testing.assert_allclose(st["residuals"], want["residuals"], rtol=1e-12, atol=0)
    np.testing.assert_allclose(st.get("Aresiduals", []), want["Aresiduals"], rtol=1e-12, atol=0)
    np.testing.assert_allclose(x[:6], want["x_head"], rtol=1e-12, atol=0)
