"""ctypes front-end of the CPU restatement of the Krylov processes -- TEST INFRASTRUCTURE ONLY.

Same status as oracle/oracle.py (only tests/ may import it; the product never does).  The processes live in
krylov_oracle_processes.h, built into the oracle library that oracle.py builds and loads, so oracle.dot_mode
(re-exported here) switches their dot products too.
Each function returns the reference's outputs with the coefficient matrices as their nzval arrays (dense H for
arnoldi); an exact breakdown without allow_breakdown raises ProcessBreakdown with the reference's message.
Parity pinning: tests/test_oracle_processes.py and tests/golden/oracle_processes.json.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import scipy.sparse as sp

from oracle.oracle import _csr, _p, _suf, _vec, dot_mode, lib  # noqa: F401

# the reference's messages, in the order each process checks them (kind 1, 2, ...)
MESSAGES = {
    "hermitian_lanczos": ["Exact breakdown β₁ == 0.", "Exact breakdown βᵢ₊₁ == 0 at iteration i = {}."],
    "arnoldi": ["Exact breakdown β == 0.", "Exact breakdown Hᵢ₊₁.ᵢ == 0 at iteration i = {}."],
    "golub_kahan": ["Exact breakdown β₁ == 0.", "Exact breakdown α₁ == 0.", "Exact breakdown βᵢ₊₁ == 0 at iteration i = {}.",
                    "Exact breakdown αᵢ₊₁ == 0 at iteration i = {}."],
    "nonhermitian_lanczos": ["Exact breakdown β₁γ₁ == 0.", "Exact breakdown βᵢ₊₁γᵢ₊₁ == 0 at iteration i = {}."],
    "saunders_simon_yip": ["Exact breakdown β₁ == 0.", "Exact breakdown γ₁ᴴ == 0.", "Exact breakdown βᵢ₊₁ == 0 at iteration i = {}.",
                           "Exact breakdown γᵢ₊₁ == 0 at iteration i = {}."],
}


class ProcessBreakdown(RuntimeError):
    """The reference's ErrorException on an exact breakdown with allow_breakdown = false."""



def _call(name, dtype, args):
    suf, real = _suf(dtype)
    f = getattr(lib(), f"oracle_{name}_{suf}")
    brk = C.c_int(0)
    cargs = []
    for a in args:
        if isinstance(a, np.ndarray):
            cargs.append(_p(a))
        elif isinstance(a, C._SimpleCData) or isinstance(a, C.Array):
            cargs.append(C.byref(a))
        else:
            cargs.append(C.c_int(int(a)))
    f.restype = C.c_int
    kind = f(*cargs, C.byref(brk))
    if kind:
        raise ProcessBreakdown(MESSAGES[name][kind - 1].format(brk.value))


def _ops(A, dtype, adjoint):
    A = sp.csr_matrix(A)
    m, n = A.shape
    _, rp, ci, va = _csr(A, dtype)
    if not adjoint:
        return m, n, [rp, ci, va]
    _, trp, tci, tva = _csr(A.T, dtype)
    return m, n, [rp, ci, va, trp, tci, tva]


def hermitian_lanczos(A, b, k, allow_breakdown=False, reorthogonalization=False, dtype=np.float64):
    """-> V (n x (k+1)), β, nzval of T ((k+1) x k, 3k-1 entries)."""
    _, real = _suf(dtype)
    m, n, ops = _ops(A, dtype, False)
    V, T, beta = np.zeros((n, k + 1), dtype, order="F"), np.zeros(3 * k - 1, dtype), real(0)
    _call("hermitian_lanczos", dtype, [n, *ops, _vec(b, dtype), k, allow_breakdown, reorthogonalization, V, beta, T])
    return V, float(beta.value), T


def arnoldi(A, b, k, allow_breakdown=False, reorthogonalization=False, dtype=np.float64):
    """-> V (n x (k+1)), β, H (dense (k+1) x k)."""
    _, real = _suf(dtype)
    m, n, ops = _ops(A, dtype, False)
    V, H, beta = np.zeros((n, k + 1), dtype, order="F"), np.zeros((k + 1, k), dtype, order="F"), real(0)
    _call("arnoldi", dtype, [n, *ops, _vec(b, dtype), k, allow_breakdown, reorthogonalization, V, beta, H])
    return V, float(beta.value), H


def golub_kahan(A, b, k, allow_breakdown=False, dtype=np.float64):
    """-> V (n x (k+1)), U (m x (k+1)), β, nzval of L ((k+1) x (k+1), 2k+1 entries)."""
    _, real = _suf(dtype)
    m, n, ops = _ops(A, dtype, True)
    V, U = np.zeros((n, k + 1), dtype, order="F"), np.zeros((m, k + 1), dtype, order="F")
    L, beta = np.zeros(2 * k + 1, dtype), real(0)
    _call("golub_kahan", dtype, [m, n, *ops, _vec(b, dtype), k, allow_breakdown, V, U, beta, L])
    return V, U, float(beta.value), L


def nonhermitian_lanczos(A, b, c, k, allow_breakdown=False, dtype=np.float64):
    """-> V, β, nzval of T, U, γᴴ, nzval of Tᴴ."""
    _, real = _suf(dtype)
    m, n, ops = _ops(A, dtype, True)
    V, U = np.zeros((n, k + 1), dtype, order="F"), np.zeros((n, k + 1), dtype, order="F")
    T, Th, beta, gamma = np.zeros(3 * k - 1, dtype), np.zeros(3 * k - 1, dtype), real(0), real(0)
    _call("nonhermitian_lanczos", dtype, [n, *ops, _vec(b, dtype), _vec(c, dtype), k, allow_breakdown, V, U, beta, gamma, T, Th])
    return V, float(beta.value), T, U, float(gamma.value), Th


def saunders_simon_yip(A, b, c, k, allow_breakdown=False, dtype=np.float64):
    """-> V (m x (k+1)), β, nzval of T, U (n x (k+1)), γᴴ, nzval of Tᴴ."""
    _, real = _suf(dtype)
    m, n, ops = _ops(A, dtype, True)
    V, U = np.zeros((m, k + 1), dtype, order="F"), np.zeros((n, k + 1), dtype, order="F")
    T, Th, beta, gamma = np.zeros(3 * k - 1, dtype), np.zeros(3 * k - 1, dtype), real(0), real(0)
    _call("saunders_simon_yip", dtype, [m, n, *ops, _vec(b, dtype), _vec(c, dtype), k, allow_breakdown, V, U, beta, gamma, T, Th])
    return V, float(beta.value), T, U, float(gamma.value), Th
