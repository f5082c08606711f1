"""GPU parity of cgls! and crls! on rectangular operators against the CPU oracle (oracle/krylov_oracle_cgls.h), Float64:
same iteration count, status and `inconsistent`; residual and Aᴴ-residual histories within 1e-6 relative at every
iteration (or 10x the oracle's own sensitivity to a few-ulp change of b, where that is larger); x within 1e-6."""
import ctypes as C
import functools
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
SOLVERS = ["cgls", "crls"]
G = parity.golden_module("cgls")


@pytest.fixture(scope="module")
def CO():
    """The CPU restatement of cgls! / crls! (oracle/cgls_oracle.py; test infrastructure)."""
    from oracle import cgls_oracle
    cgls_oracle.lib()
    return cgls_oracle


def _compare(CO, kb, solver, A, b, **kw):
    """Solve on the GPU (operator gpu_A, default A) and with the oracle; assert the parity bar."""
    return parity.compare(getattr(CO, solver), functools.partial(getattr(kb, solver), n=A.shape[1]), A, b,
                          keys=("residuals", "Aresiduals"), flags=("inconsistent",), floor=1e-9, **kw)


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("shape", ["square", "tall_lstp", "wide_lstp", "ddx", "grad7", "tall_gaps", "wide_gaps"])
@pytest.mark.parametrize("fused", [True, False])
def test_shapes_match_oracle(kb, CO, solver, shape, fused):
    A, b = parity.shapes()[shape]
    _compare(CO, kb, solver, A, b, fused=fused, itmax=200)


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("fused", [True, False])
def test_options_match_oracle(kb, CO, solver, fused):
    A, b = parity.shapes()["tall_gaps"]
    m = A.shape[0]
    dm = np.linspace(0.5, 2.0, m)
    _compare(CO, kb, solver, A, b, lambda_=1e-2, itmax=300, fused=fused)        # lambda > 0 stays fused
    _compare(CO, kb, solver, A, b, M=dm, itmax=300, fused=fused)                # M: primitive path
    _compare(CO, kb, solver, A, b, M=dm, ldiv=True, itmax=300, fused=fused)
    _compare(CO, kb, solver, A, b, M=dm, lambda_=1e-2, itmax=300, fused=fused)
    xs, _, _ = _compare(CO, kb, solver, A, b, itmax=300, fused=fused)
    _, st, _ = _compare(CO, kb, solver, A, b, radius=0.5 * np.linalg.norm(xs), itmax=300, fused=fused)
    assert st.status == "on trust-region boundary"
    for key in sorted(G.cases()):                               # the reference's known-answer problems
        Ak, bk, kw = G.cases()[key]
        # Their last iterations sit at the √eps stopping threshold, where the oracle's own iteration count moves by one
        # under a few-ulp change of b: histories are compared up to two iterations before the oracle stops.  On the
        # nearly singular 5 x 5 matrices x itself moves far more than the residuals: its bar is 10x the oracle's own
        # change under the same perturbations.
        _, so = getattr(CO, solver)(Ak, bk, **kw)
        it = max(so["niter"] - 2, 1)
        _compare(CO, kb, solver, Ak, bk, fused=fused, itmax=it, xtol=None, **kw)
        x, st = getattr(kb, solver)(Ak, bk, fused=fused, **kw)
        assert st.solved and abs(st.niter - so["niter"]) <= 2, (key, st.niter, so["niter"])


@pytest.mark.parametrize("fused", [True, False])
def test_crls_zero_curvature(kb, CO, fused):
    b, A, *_ = CO.lsq_test(40, 40, 4, 1, 0)
    _, st, _ = _compare(CO, kb, "crls", A, b, radius=1.0e3, atol=1.0, rtol=0.0, fused=fused)
    assert st.status == "zero-curvature encountered" and st.niter == 0
    A, b = G.psd_problem()                                      # test/test_crls.jl's assertions (rank-deficient A)
    x, st = kb.crls(A, b, radius=10.0, fused=fused)
    assert st.solved and st.status in ("zero-curvature encountered", "on trust-region boundary")
    assert np.linalg.norm(x) <= 10.0 * (1 + 1e-12)


@pytest.mark.parametrize("solver", SOLVERS)
def test_host_callbacks_and_device_b(kb, CO, solver):
    import torch
    from scipy.sparse.linalg import aslinearoperator
    A, b = parity.shapes()["grad7"]
    _compare(CO, kb, solver, A, b, gpu_A=aslinearoperator(A), itmax=100)
    _compare(CO, kb, solver, A, b, gpu_A=(lambda x: A @ x, lambda y: A.T @ y), itmax=100)
    dm = np.linspace(0.5, 2.0, A.shape[0])
    _compare(CO, kb, solver, A, b, gpu_A=aslinearoperator(A), M=dm, itmax=100)
    xo, so = getattr(CO, solver)(A, b, M=dm, itmax=100)
    x, st = getattr(kb, solver)(A, b, M=lambda v: dm * v, itmax=100, history=True)   # M as a host callable
    assert st.niter == so["niter"] and np.linalg.norm(x - xo) <= TOL * np.linalg.norm(xo)
    xo, so = getattr(CO, solver)(A, b, itmax=100)
    x, st = getattr(kb, solver)(A, torch.tensor(b, device="cuda"), itmax=100, history=True)
    assert x.is_cuda and st.niter == so["niter"] and st.status == so["status"]
    assert np.linalg.norm(x.cpu().numpy() - xo) <= TOL * np.linalg.norm(xo)


@pytest.mark.parametrize("solver", SOLVERS)
@pytest.mark.parametrize("fused", [True, False])
def test_zero_rhs_and_zero_adjoint_residual(kb, CO, solver, fused):
    n = 20
    A = sp.csr_matrix(sp.vstack([sp.identity(n), sp.csr_matrix((3, n))]))
    b = np.zeros(n + 3)
    _, st, _ = _compare(CO, kb, solver, A, b, fused=fused)
    assert st.status == "x is a zero-residual solution" and st.niter == 0
    b[n + 1] = 1.0                                              # b orthogonal to range(A): Aᴴb = 0
    x, st, _ = _compare(CO, kb, solver, A, b, fused=fused)
    assert st.status == "solution good enough given atol and rtol" and st.niter == 0 and not x.any()


@pytest.mark.parametrize("solver", SOLVERS)
def test_callback_user_exit_and_type(kb, CO, solver):
    A, b = parity.shapes()["grad7"]
    seen = []

    def cb(ws):
        seen.append(1)
        return len(seen) >= 3
    x, st = getattr(kb, solver)(A, b, callback=cb, history=True)
    assert st.status == "user-requested exit" and st.niter == 3 and len(st.residuals) == 4
    with pytest.raises(TypeError):
        getattr(kb, solver)(A, b, callback=lambda ws: "string", history=True)


@pytest.mark.parametrize("solver", SOLVERS)
def test_unsupported_kwargs_and_right_preconditioner(kb, CO, solver):
    A, b = parity.shapes()["grad7"]
    for kw in (dict(N=np.ones(A.shape[1])), dict(sigma=1.0), dict(sqd=True), dict(etol=1e-3)):
        with pytest.raises(kb.B200Error):
            getattr(kb, solver)(A, b, **kw)
    L = _lib.lib()
    ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64)
    ws.set_operator(A)
    d = np.ones(A.shape[1])
    assert L.krylov_b200_set_preconditioner_diag(ws._h, 1, d.ctypes.data_as(C.c_void_p), 0) == 0
    bb = np.ascontiguousarray(b)
    null = _lib.MATVEC()
    assert L.krylov_solve(ws._h, null, null, null, null, bb.ctypes.data_as(C.c_void_p), None, None, None) == -1
    assert "right preconditioner" in _lib.last_error()
    ws.free()


@pytest.mark.parametrize("solver", SOLVERS)
def test_fused_against_primitives(kb, CO, solver):
    rp, ci, va = P.grad_csr(24)
    m, n = len(rp) - 1, 24 ** 3
    b = np.random.default_rng(1).standard_normal(m)
    for lam in (0.0, 1e-2):
        kw = dict(atol=0.0, rtol=0.0, lambda_=lam, history=True)
        out, launches = {}, {}
        for fused in (True, False):
            ws = kb.krylov_workspace(solver, m, n, np.float64)
            ws.set_operator((rp, ci, va))
            counts = []
            for itmax in (10, 30):
                l0 = ws.launches
                ws.solve(None, b, itmax=itmax, fused=fused, **kw)
                counts.append(ws.launches - l0)
            launches[fused] = (counts[1] - counts[0]) / 20
            out[fused] = (ws.x, ws.stats)
            ws.free()
        (xf, sf), (xp, spr) = out[True], out[False]
        assert (sf.niter, sf.status) == (spr.niter, spr.status)
        for key in ("residuals", "Aresiduals"):
            a, c = np.asarray(getattr(sf, key)), np.asarray(getattr(spr, key))
            assert np.all(np.abs(a - c) <= 1e-12 * np.abs(c) + 1e-14 * c[0]), key
        assert np.linalg.norm(xf - xp) <= 1e-10 * np.linalg.norm(xp)
        assert launches[True] == 4 and launches[False] >= 8, launches


@pytest.mark.parametrize("solver", SOLVERS)
def test_bench_size_parity(kb, CO, solver):
    """The benchmark workload (gradient of the 215^3 grid, m = 29 676 450, n = 9 938 375) over 4 iterations."""
    N = 215
    rp, ci, va = P.grad_csr(N)
    m, n = len(rp) - 1, N ** 3
    A = sp.csr_matrix((va, ci, rp), shape=(m, n))
    b = np.random.default_rng(0).standard_normal(m)
    _compare(CO, kb, solver, A, b, gpu_A=(rp, ci, va), atol=0.0, rtol=0.0, itmax=4)


@pytest.mark.parametrize("solver", SOLVERS)
def test_float32(kb, CO, solver):
    A, _ = parity.shapes()["square"]
    b = A @ np.ones(A.shape[1])
    A32, b32 = A.astype(np.float32), b.astype(np.float32)
    xo, so = getattr(CO, solver)(A32, b32, dtype=np.float32)
    x, st = getattr(kb, solver)(A32, b32)
    assert st.solved and abs(st.niter - so["niter"]) <= 1, (st.niter, so["niter"])
    r = b - A @ x.astype(np.float64)
    assert np.linalg.norm(A.T @ r) <= 1e-3 * np.linalg.norm(A.T @ b)


def test_c_abi_rules(kb):
    L = _lib.lib()
    for sid in (_lib.KRYLOV_CGLS, _lib.KRYLOV_CRLS):
        ws = C.c_void_p()
        assert L.krylov_workspace_create(sid, 5, 3, _lib.KRYLOV_FLOAT64, 0, None, C.byref(ws)) == 0
        f = _lib.MATVEC(lambda x, y, u: None)
        b = np.ones(5)
        assert L.krylov_solve(ws, f, _lib.MATVEC(), _lib.MATVEC(), _lib.MATVEC(), b.ctypes.data_as(C.c_void_p), None, None, None) == -1
        assert "matvec_At" in _lib.last_error()
        assert L.krylov_get_y(ws, None, 5) == -2
        assert L.krylov_warm_start(ws, np.zeros(3).ctypes.data_as(C.c_void_p), 3) == -1
        assert L.krylov_b200_dist_init(ws, 0, 1, 0, None, None) == -1
        blocks = np.ones((2, 2, 2))
        assert L.krylov_b200_set_preconditioner_blockdiag(ws, 0, 2, blocks.ctypes.data_as(C.c_void_p), 0) == -1
        assert L.krylov_workspace_free(ws) == 0


def test_reference_test_all_solvers_least_squares_rows():
    import subprocess
    path = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "test_all_solvers")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/test_all_solvers was not built (reference tree absent at build time)")
    out = subprocess.run([path], capture_output=True, text=True, timeout=600)
    rows = [l for l in out.stdout.splitlines() if l.split() and l.split()[0].lower() in ("cgls", "crls", "lslq", "lsqr", "lsmr")]
    assert len(rows) >= 5, out.stdout[-2000:]
    for l in rows:
        assert "PASS" in l, l
