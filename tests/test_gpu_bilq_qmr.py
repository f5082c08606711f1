"""GPU parity of bilq! and qmr! on square operators against the CPU oracle (oracle/krylov_oracle_biorth.h), Float64:
same iteration count, `solved` and status; residual histories within 1e-6 relative at every iteration (or 10x the
oracle's own sensitivity to a few-ulp change of b, where that is larger); x within the same bar.  Float32 within the
measured dot-rounding envelope (DESIGN.md §5).  The fused path (3 launches per iteration) against the primitive one."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp

import parity
from krylov_b200 import _lib
from krylov_b200 import problems as P
from parity import TOL

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
SOLVERS = ["bilq", "qmr"]
G = parity.golden_module("bilq_qmr")


@pytest.fixture(scope="module")
def O():
    """The CPU restatement of bilq! / qmr! (oracle/biorth_oracle.py; test infrastructure)."""
    from oracle import biorth_oracle
    biorth_oracle.lib()
    return biorth_oracle


def _compare(O, kb, solver, A, b, **kw):
    """Run the oracle and the library on the same problem and compare them.  Where the oracle's own iteration count
    moves under a few-ulp change of b (polar_poisson: 411 to 537 BiLQ iterations, 429 to 755 QMR ones, loss of
    biorthogonality), the library's count must lie in that range, with the same status, and x must meet the reference's
    residual assertion; histories are then compared where the oracle's own sensitivity allows."""
    return parity.compare(getattr(O, solver), getattr(kb, solver), A, b, keys=("residuals",), flags=("solved",),
                          floor=1e-12, unsteady="range", check_length=False, xtol=None, **kw)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("name", sorted(G.cases()))
def test_known_answer_problems_match_oracle(kb, O, solver, name, fused):
    A, b, kw = G.cases()[name]
    _compare(O, kb, solver, A, b, fused=fused, **kw)


def _big(O):
    A, b = O.kron_unsymmetric(12)
    return A, np.asarray(b)


@pytest.mark.parametrize("solver", SOLVERS)
def test_options_match_oracle(kb, O, solver):
    A, b = _big(O)
    n = A.shape[0]
    d = np.linspace(0.5, 2.0, n)
    c = np.cos(np.arange(n))                                           # c != b
    _compare(O, kb, solver, A, b, c=c, itmax=60)
    _compare(O, kb, solver, A, b, M=d, itmax=60)
    _compare(O, kb, solver, A, b, N=1 / d, itmax=60)
    _compare(O, kb, solver, A, b, M=d, N=d, ldiv=True, itmax=60)
    _compare(O, kb, solver, A, b, x0=np.sin(np.arange(n)), itmax=60)  # warm start
    _compare(O, kb, solver, A, b, x0=np.sin(np.arange(n)), M=d, itmax=60)
    if solver == "bilq":
        _compare(O, kb, solver, A, b, transfer_to_bicg=False, itmax=60)


@pytest.mark.parametrize("solver", SOLVERS)
def test_callbacks_and_device_pointers(kb, O, solver):
    from scipy.sparse.linalg import aslinearoperator
    A, b = _big(O)
    n = A.shape[0]
    d = np.linspace(0.5, 2.0, n)
    _compare(O, kb, solver, A, b, gpu_A=aslinearoperator(A), itmax=60)                      # A and Aᵀ as host callbacks
    _compare(O, kb, solver, A, b, gpu_A=(lambda x: A @ x, lambda y: A.T @ y), M=d, itmax=60)
    xo, so = getattr(O, solver)(A, b, M=d, N=d, itmax=60)                                  # M, N as host callables
    x, st = getattr(kb, solver)(A, b, M=lambda v: d * v, N=lambda v: d * v, itmax=60, history=True)
    assert (st.niter, st.status) == (so["niter"], so["status"]) and np.linalg.norm(x - xo) <= TOL * np.linalg.norm(xo)
    _compare(O, kb, solver, A, b, device_b=True, c=np.cos(np.arange(n)), itmax=60)          # device-pointer workspace


@pytest.mark.parametrize("solver", SOLVERS)
def test_exits(kb, O, solver):
    A, b = O.polar_poisson()
    ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64)
    seen = []
    ws.solve(A, b, callback=lambda w: (seen.append(w.stats.niter) or len(seen) >= 3))
    assert ws.stats.status == "user-requested exit" and ws.stats.niter == 3 and seen == [1, 2, 3]
    ws.solve(A, b, timemax=0.0)
    assert ws.stats.status == "time limit exceeded" and ws.stats.niter == 1
    with pytest.raises(TypeError):
        ws.solve(A, b, callback=lambda w: "string", history=True)
    ws.free()


def test_c_abi_rules(kb):
    L = _lib.lib()
    for sid in (12, 13):
        for dt in (_lib.KRYLOV_FLOAT32, _lib.KRYLOV_FLOAT64):
            ws = C.c_void_p()
            assert L.krylov_workspace_create(sid, 4, 4, dt, 0, None, C.byref(ws)) == 0
            assert L.krylov_workspace_free(ws) == 0
        for dt in (2, 3):                                                                   # complex types
            assert L.krylov_workspace_create(sid, 4, 4, dt, 0, None, C.byref(C.c_void_p())) == -2
        ws = C.c_void_p()
        assert L.krylov_workspace_create(sid, 4, 4, _lib.KRYLOV_FLOAT64, 0, None, C.byref(ws)) == 0
        f = _lib.MATVEC(lambda x, y, u: None)
        b = np.ones(4)
        assert L.krylov_solve(ws, f, _lib.MATVEC(), _lib.MATVEC(), _lib.MATVEC(), b.ctypes.data_as(C.c_void_p), None, None, None) == -1
        assert "matvec_At" in _lib.last_error()
        assert L.krylov_get_y(ws, None, 4) == -2
        assert L.krylov_warm_start2(ws, None, None, 4, 4) == -2
        assert L.krylov_warm_start(ws, np.zeros(4).ctypes.data_as(C.c_void_p), 4) == 0
        assert L.krylov_b200_dist_init(ws, 0, 1, 0, None, None) == -1
        assert "row-partitioned" in _lib.last_error()
        assert L.krylov_workspace_free(ws) == 0
    assert L.krylov_workspace_create(14, 4, 4, _lib.KRYLOV_FLOAT64, 0, None, C.byref(C.c_void_p())) == -2   # USYMLQ


@pytest.mark.parametrize("solver", SOLVERS)
def test_float32_within_dot_rounding_envelope(kb, O, solver):
    A, b = _big(O)
    xo, so = getattr(O, solver)(A, b, dtype=np.float32, itmax=40)
    with O.dot_mode(1):
        _, s1 = getattr(O, solver)(A, b, dtype=np.float32, itmax=40)
    r0, r1 = np.asarray(so["residuals"], float), np.asarray(s1["residuals"], float)
    env = np.maximum.accumulate(np.abs(r0 - r1) / np.maximum(r0, 1e-300))
    x, st = getattr(kb, solver)(A, b.astype(np.float32), itmax=40, history=True)
    assert st.niter == so["niter"]
    res = np.asarray(st.residuals)
    tol = np.maximum(4 * 1.2e-7, 10 * env)
    assert np.all(np.abs(res - r0) <= tol * r0 + 1e-6 * r0[0])


@pytest.mark.parametrize("solver", SOLVERS)
def test_grouped_passes_equal_the_primitive_path(kb, O, solver):
    """fused=True runs an iteration as 3 launches (B1, B2, U); every element update repeats the k* sequence it
    replaces, so against fused=False: same iteration count and status, histories equal to dot-product rounding, and
    far fewer launches."""
    A, b = _big(O)
    out = {}
    for fused in (True, False):
        ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64)
        ws.solve(A, b, itmax=3, fused=fused)                  # forms and caches Aᵀ outside the count
        l0 = ws.launches
        ws.solve(A, b, history=True, fused=fused)
        out[fused] = (ws.x, ws.stats, ws.launches - l0)
        ws.free()
    (x1, s1, l1), (x0, s0, l0) = out[True], out[False]
    assert s1.niter == s0.niter and s1.status == s0.status
    assert np.allclose(s1.residuals, s0.residuals, rtol=1e-7, atol=1e-12 * s0.residuals[0])
    assert np.linalg.norm(x1 - x0) <= 1e-8 * np.linalg.norm(x0)
    assert l1 < 0.3 * l0, (l1, l0)


@pytest.mark.parametrize("solver", SOLVERS)
def test_benchmark_size_matches_oracle(kb, O, solver):
    """60 iterations on kron_unsymmetric(215) with b = A 1 (test/test_utils.jl), all tolerances 0, fused path: the
    history against the oracle's within 1e-6 relative, or 10x the oracle's own change under a 1-ulp perturbation of b
    where that is larger (the estimates of this strongly non-normal operator grow, and so does their sensitivity)."""
    import torch
    n1 = 215
    rp, ci, va = P.kron_unsymmetric_csr(n1, xp=torch, device="cuda")
    n = n1 ** 3
    A = sp.csr_matrix((va.cpu().numpy(), ci.cpu().numpy(), rp.cpu().numpy()), shape=(n, n))
    bh = A @ np.ones(n)
    ws = kb.krylov_workspace(solver, n, n, np.float64, device="cuda")
    ws.solve((rp, ci, va), torch.tensor(bh, device="cuda"), atol=0.0, rtol=0.0, itmax=60, history=True)
    st = ws.stats
    ws.free()
    _, so = getattr(O, solver)(A, bh, atol=0.0, rtol=0.0, itmax=60)
    sign = np.random.default_rng(0).choice([-1.0, 1.0], size=n)
    _, s1 = getattr(O, solver)(A, bh * (1 + 2.2e-16 * sign), atol=0.0, rtol=0.0, itmax=60)
    ro, rg, r1 = np.asarray(so["residuals"]), np.asarray(st.residuals), np.asarray(s1["residuals"])
    assert st.niter == so["niter"] == 60 and len(rg) == len(ro)
    tol = np.maximum(TOL, 10 * np.maximum.accumulate(np.abs(r1 - ro) / np.abs(ro)))
    rel = np.abs(rg - ro) / np.abs(ro)
    assert np.all(rel <= tol), (rel.max(), tol[np.argmax(rel > tol)])


def test_reference_test_all_solvers_bilq_qmr_rows():
    import subprocess
    path = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "test_all_solvers")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/test_all_solvers was not built (reference tree absent at build time)")
    out = subprocess.run([path], capture_output=True, text=True, timeout=600)
    rows = [l for l in out.stdout.splitlines() if l.split() and l.split()[0].lower() in ("bilq", "qmr")]
    assert len(rows) >= 2, out.stdout[-2000:]
    for l in rows:
        assert "PASS" in l, l
