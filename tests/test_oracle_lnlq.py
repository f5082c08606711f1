"""The CPU oracle's lnlq (oracle/krylov_oracle_lnlq.h) against the reference's own assertions (test/test_lnlq.jl,
real case, same tolerance, transfer_to_craig false and true), against the frozen histories of
tests/golden/oracle_lnlq.json (tests/golden/gen_golden_lnlq.py), and on the reference's quirks the GPU must repeat."""
import json
import os

import numpy as np
import pytest

from oracle import lnlq_oracle as O
from parity import golden_module

HERE = os.path.dirname(os.path.abspath(__file__))
TOL = 1.0e-6                                                         # lnlq_tol
G = golden_module("lnlq")
GOLD = json.load(open(os.path.join(HERE, "golden", "oracle_lnlq.json")))
TRANSFER = [False, True]


def _min_norm(A, b, x):
    """check_min_norm.jl (λ = 0): the least-norm solution from a QR factorization of Aᵀ."""
    Q, R = np.linalg.qr(A.toarray().T)
    xmin = Q @ np.linalg.lstsq(R.T, b, rcond=None)[0]
    return x, xmin, np.linalg.norm(xmin)


def test_zero_rhs():
    A, b = O.zero_rhs()
    x, y, st = O.lnlq(A, b)
    assert np.linalg.norm(x) == 0 and np.linalg.norm(y) == 0
    assert st["status"] == "x is a zero-residual solution" and st["niter"] == 0 and st["solved"]


@pytest.mark.parametrize("transfer", TRANSFER)
@pytest.mark.parametrize("name", ["under_consistent", "square_consistent", "over_consistent"])
def test_consistent_systems(name, transfer):
    A, b = getattr(O, name)()
    x, y, st = O.lnlq(A, b, transfer_to_craig=transfer, utolx=0.0, utoly=0.0)
    assert np.linalg.norm(x - A.T @ y) <= TOL * np.linalg.norm(x)
    assert np.linalg.norm(b - A @ x) / np.linalg.norm(b) <= TOL
    assert st["solved"]
    cond = np.linalg.cond(A.toarray())
    xI, xmin, xmin_norm = _min_norm(A, b, x)
    assert np.linalg.norm(xI - xmin) <= cond * TOL * xmin_norm
    xs, _, ss = O.lnlq(A, b, transfer_to_craig=transfer, atol=0.0, rtol=0.0, sigma=0.5)
    xI, xmin, xmin_norm = _min_norm(A, b, xs)
    assert np.linalg.norm(xI - xmin) <= cond * TOL * xmin_norm
    assert len(ss["error_bnd_x"]) == len(ss["error_bnd_y"]) == ss["niter"]   # one pair before the loop, one per pass


@pytest.mark.parametrize("transfer", TRANSFER)
def test_regularization(transfer):
    A, b, lam = O.regularization()
    runs = (O.lnlq(A, b, lambda_=lam, transfer_to_craig=transfer, utolx=0.0, utoly=0.0),
            O.lnlq(A, b, transfer_to_craig=transfer, atol=0.0, rtol=0.0, utolx=1e-10, utoly=1e-10, lambda_=lam))
    for x, y, _ in runs:
        s = lam * y
        assert np.linalg.norm(b - (A @ x + lam * s)) / np.linalg.norm(b) <= TOL
        assert np.linalg.norm(b - (A @ (A.T @ y) + lam ** 2 * y)) / np.linalg.norm(b) <= TOL


@pytest.mark.parametrize("transfer", TRANSFER)
def test_saddle_point_with_N(transfer):
    A, b, D = O.saddle_point()
    for kw in ({}, dict(atol=0.0, rtol=0.0, sigma=0.001)):
        x, y, _ = O.lnlq(A, b, N=1.0 / D, transfer_to_craig=transfer, **kw)
        assert np.linalg.norm(b - A @ x) / np.linalg.norm(b) <= TOL
        assert np.linalg.norm(b - A @ ((A.T @ y) / D)) / np.linalg.norm(b) <= TOL


@pytest.mark.parametrize("transfer", TRANSFER)
def test_two_preconditioners(transfer):
    A, b, Mi, Ni = O.two_preconditioners()
    for kw in ({}, dict(atol=0.0, rtol=0.0, sigma=0.5)):
        x, y, _ = O.lnlq(A, b, M=Mi, N=Ni, sqd=False, transfer_to_craig=transfer, **kw)
        r = b - A @ x
        assert np.sqrt(r @ (Mi * r)) / np.linalg.norm(b) <= TOL
        assert np.linalg.norm(x - Ni * (A.T @ y)) <= TOL * np.linalg.norm(x)


@pytest.mark.parametrize("transfer", TRANSFER)
def test_sqd_and_lambda4_with_M_N(transfer):
    A, b, M, N = O.sqd()
    for kw in ({}, dict(atol=0.0, rtol=0.0, sigma=0.5)):
        x, y, _ = O.lnlq(A, b, M=1.0 / M, N=1.0 / N, sqd=True, transfer_to_craig=transfer, **kw)
        assert np.linalg.norm(b - (A @ x + M * y)) / np.linalg.norm(b) <= TOL
        assert np.linalg.norm(b - (A @ ((A.T @ y) / N) + M * y)) / np.linalg.norm(b) <= TOL
    lam = 4.0
    for kw in ({}, dict(atol=0.0, rtol=0.0, sigma=0.5)):
        x, y, _ = O.lnlq(A, b, M=1.0 / M, N=1.0 / N, lambda_=lam, transfer_to_craig=transfer, **kw)
        assert np.linalg.norm(b - (A @ x + lam ** 2 * M * y)) / np.linalg.norm(b) <= TOL
        assert np.linalg.norm(b - (A @ ((A.T @ y) / N) + lam ** 2 * M * y)) / np.linalg.norm(b) <= TOL


@pytest.mark.parametrize("transfer", TRANSFER)
@pytest.mark.parametrize("t", [False, True])
def test_extra_vector_dimensions(t, transfer):
    """small_sp and small_sqd in both orientations: the lazily sized vectors (u, v, q) have the right lengths."""
    A, b, c, D = O.small_sp(t)
    x, y, _ = O.lnlq(A.T.tocsr(), c, N=1.0 / D, transfer_to_craig=transfer)
    assert x.shape == (A.shape[0],) and y.shape == (A.shape[1],)
    A, b, c, M, N = O.small_sqd(t)
    x, y, _ = O.lnlq(A, b, M=1.0 / M, N=1.0 / N, sqd=True, transfer_to_craig=transfer)
    assert x.shape == (A.shape[1],) and y.shape == (A.shape[0],)
    assert np.all(np.isfinite(x)) and np.all(np.isfinite(y))


def test_small_least_norm():
    A, b = O.small_ln()
    x, y, st = O.lnlq(A, b)
    assert st["solved"]
    assert np.linalg.norm(b - A @ x) / np.linalg.norm(b) <= TOL
    assert np.linalg.norm(x - A.T @ y) <= TOL * np.linalg.norm(x)


def test_sqd_with_lambda_raises():
    A, b = O.small_ln()
    with pytest.raises(ValueError, match="sqd cannot be set to true if λ ≠ 0 !"):
        O.lnlq(A, b, sqd=True, lambda_=1.0)


@pytest.mark.parametrize("transfer", TRANSFER)
def test_tired_run_reports_one_more_than_the_passes(transfer):
    """`iter` is incremented before the loop and after every pass, so itmax = k reports niter = k + 1; the first pass
    pushes ‖b‖ again, so the history starts with ‖b‖ twice and has niter entries."""
    A, b = O.over_consistent()
    passes = []
    _, _, st = O.lnlq(A, b, itmax=4, atol=0.0, rtol=0.0, utolx=0.0, utoly=0.0, transfer_to_craig=transfer,
                      callback=lambda it: passes.append(it) and False)
    assert st["status"] == "maximum number of iterations exceeded"
    assert st["niter"] == 4 + 1 and passes == [1, 2, 3, 4]
    r = st["residuals"]
    assert r[0] == r[1] == np.linalg.norm(b) and len(r) == st["niter"]


def test_bounds_met_before_the_loop_report_one_iteration():
    """σ > 0 with bounds already below utolx / utoly: zero passes, niter = 1, one pair of bounds."""
    A, b = O.over_consistent()
    _, _, st = O.lnlq(A, b, sigma=0.5, utolx=1e10, utoly=1e10)
    assert st["niter"] == 1 and st["solved"] and len(st["residuals"]) == 1
    assert len(st["error_bnd_x"]) == len(st["error_bnd_y"]) == 1


def test_callback_stops_and_sees_the_iteration():
    A, b = O.over_consistent()
    seen = []
    _, _, st = O.lnlq(A, b, callback=lambda it: seen.append(it) or True)
    assert st["status"] == "user-requested exit" and seen == [1] and st["niter"] == 2


def test_error_bounds_latch_once_complex():
    """Once a discriminant goes negative, no bound is pushed any more (error_with_bnd); the stale ones still count."""
    A, b, M, N = O.sqd()
    _, _, st = O.lnlq(A, b, M=1.0 / M, N=1.0 / N, sqd=True, atol=0.0, rtol=0.0, sigma=0.5)
    assert st["error_with_bnd"]
    assert 0 < len(st["error_bnd_x"]) < st["niter"]


@pytest.mark.parametrize("name", sorted(GOLD))
def test_oracle_reproduces_golden(name):
    A, b, kw = G.cases()[name]
    x, y, st = G.run(A, b, **kw)
    g = GOLD[name]
    assert (st["niter"], st["solved"], st["status"], st["error_with_bnd"]) == (g["niter"], g["solved"], g["status"],
                                                                              g["error_with_bnd"])
    for key in ("residuals", "error_bnd_x", "error_bnd_y"):                  # NaN matches NaN (small_ln, LNLQ point)
        np.testing.assert_array_equal(np.asarray(st[key], dtype=np.float64), np.asarray(g[key], dtype=np.float64), key)
    np.testing.assert_array_equal(x[:6], np.asarray(g["x_head"]))
    np.testing.assert_array_equal(y[:6], np.asarray(g["y_head"]))
