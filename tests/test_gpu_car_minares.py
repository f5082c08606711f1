"""GPU parity of car! and minares! on symmetric operators against the CPU oracle (oracle/krylov_oracle_ares.h),
Float64: same iteration count, `solved` and status; residual and A-residual histories within 1e-6 relative at every
iteration (or 10x the oracle's own sensitivity to a few-ulp change of b, where that is larger); x within the same bar.
Float32 within the measured dot-rounding envelope (DESIGN.md §5).  The fused path (3 launches per iteration) against
the primitive one."""
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
SOLVERS = ["car", "minares"]
G = parity.golden_module("car_minares")
KAT = [(s, name) for s, cs in G.cases().items() for name in sorted(cs)]


@pytest.fixture(scope="module")
def O():
    """The CPU restatement of car! / minares! (oracle/ares_oracle.py; test infrastructure)."""
    from oracle import ares_oracle
    ares_oracle.lib()
    return ares_oracle


def _compare(O, kb, solver, A, b, **kw):
    """Run the oracle and the library on the same problem and compare them.  Where the oracle's own iteration count
    moves under a few-ulp change of b (almost_singular: 228 to 234 MINARES iterations, loss of orthogonality in the
    Lanczos process), the library's count must lie in that range widened by its own spread, with the same status, and x
    must meet the reference's residual assertion (scaled by ‖A‖‖x‖ for MINARES); histories are then compared up to the
    point where the oracle's own history moves by 1e-3."""
    return parity.compare(getattr(O, solver), getattr(kb, solver), A, b, keys=("residuals", "Aresiduals"),
                          flags=("solved",), floor=1e-12, unsteady="widened", scaled_resid=solver == "minares",
                          xtol=None, **kw)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("solver,name", KAT)
def test_known_answer_problems_match_oracle(kb, O, solver, name, fused):
    A, b, kw = G.cases()[solver][name]
    _compare(O, kb, solver, A, b, fused=fused, **kw)


def _big(O):
    A, b = O.sparse_laplacian(24)
    return sp.csr_matrix(A), np.asarray(b)


def test_car_options_match_oracle(kb, O):
    A, b = _big(O)
    n = A.shape[0]
    d = np.linspace(0.5, 2.0, n)
    _compare(O, kb, "car", A, b, M=d, itmax=60)                               # diagonal M
    _compare(O, kb, "car", A, b, M=d, ldiv=True, itmax=60)
    _compare(O, kb, "car", A, b, x0=np.sin(np.arange(n)), itmax=60)          # warm start
    _compare(O, kb, "car", A, b, x0=np.sin(np.arange(n)), M=d, itmax=60)
    _compare(O, kb, "car", A, b, itmax=7)
    xo, so = O.car(A, b, M=d, itmax=60)                                       # M as a host callable
    x, st = kb.car(A, b, M=lambda v: d * v, itmax=60, history=True)
    assert (st.niter, st.status) == (so["niter"], so["status"]) and np.linalg.norm(x - xo) <= TOL * np.linalg.norm(xo)


def test_minares_options_match_oracle(kb, O):
    A, b = _big(O)
    n = A.shape[0]
    _compare(O, kb, "minares", A, b, lambda_=0.5, itmax=60)                   # shift
    _compare(O, kb, "minares", A, b, x0=np.sin(np.arange(n)), itmax=60)      # warm start
    _compare(O, kb, "minares", A, b, x0=np.sin(np.arange(n)), lambda_=0.5, itmax=60)   # warm start with λ
    _compare(O, kb, "minares", A, b, atol=0.0, rtol=0.0, artol=1e-4)         # Artol
    _compare(O, kb, "minares", A, b, itmax=7)
    with pytest.raises(Exception, match="Preconditioners are not yet supported"):
        kb.minares(A, b, M=np.ones(n))


@pytest.mark.parametrize("solver", SOLVERS)
def test_callback_operator_and_device_pointers(kb, O, solver):
    import torch
    A, b = _big(O)
    kw = dict(lambda_=0.5) if solver == "minares" else {}
    _compare(O, kb, solver, A, b, gpu_A=lambda v: A @ v, itmax=60, **kw)             # A as a host callback
    xo, so = getattr(O, solver)(A, b, itmax=60, **kw)
    x, st = getattr(kb, solver)((torch.tensor(A.indptr, dtype=torch.int32, device="cuda"),
                                 torch.tensor(A.indices, dtype=torch.int32, device="cuda"),
                                 torch.tensor(A.data, device="cuda")), torch.tensor(b, device="cuda"), itmax=60, **kw)
    x = x.cpu().numpy()
    assert (st.niter, st.status) == (so["niter"], so["status"]) and np.linalg.norm(x - xo) <= TOL * np.linalg.norm(xo)


@pytest.mark.parametrize("solver", SOLVERS)
def test_exits(kb, O, solver):
    A, b = O.sparse_laplacian()
    ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64)
    seen = []
    ws.solve(A, b, callback=lambda w: (seen.append(w.stats.niter) or len(seen) >= 3))
    assert ws.stats.status == "user-requested exit" and ws.stats.niter == 3 and seen == [1, 2, 3]
    # the reference's TestCallbackN2: stop once ‖b - A x‖ ≤ tol
    ws.solve(A, b, atol=0.0, rtol=0.0, callback=lambda w: bool(np.linalg.norm(b - A @ w.x) <= 1e-1))
    assert ws.stats.status == "user-requested exit" and np.linalg.norm(b - A @ ws.x) <= 1e-1
    ws.solve(A, b, timemax=0.0)
    assert ws.stats.status == "time limit exceeded" and ws.stats.niter == 1
    with pytest.raises(TypeError):
        ws.solve(A, b, callback=lambda w: "string", history=True)
    ws.free()


def test_c_abi_rules(kb):
    L = _lib.lib()
    for sid in (32, 33):
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
        assert L.krylov_solve(ws, f, _lib.MATVEC(), _lib.MATVEC(), f, b.ctypes.data_as(C.c_void_p), None, None, None) == -1
        assert "matvec_N" in _lib.last_error()
        assert L.krylov_get_y(ws, None, 4) == -2
        assert L.krylov_warm_start2(ws, None, None, 4, 4) == -2
        assert L.krylov_warm_start(ws, np.zeros(4).ctypes.data_as(C.c_void_p), 4) == 0
        assert L.krylov_b200_dist_init(ws, 0, 1, 0, None, None) == -1
        assert "row-partitioned" in _lib.last_error()
        p = C.c_void_p()
        names = ("r", "p", "s", "q", "t", "u") if sid == 32 else ("vₖ", "vₖ₊₁", "v_next", "wₖ₋₂", "w_prev2", "wₖ₋₁", "w_prev",
                                                                  "dₖ₋₂", "d_prev2", "dₖ₋₁", "d_prev", "q")
        for nm in names:
            assert L.krylov_b200_get_vector(ws, nm.encode(), C.byref(p)) == 0 and p.value, nm
        assert L.krylov_workspace_free(ws) == 0
    for sid in (2, 4):                                                                     # SYMMLQ, MINRES-QLP
        assert L.krylov_workspace_create(sid, 4, 4, _lib.KRYLOV_FLOAT64, 0, None, C.byref(C.c_void_p())) == -2


@pytest.mark.parametrize("solver", SOLVERS)
def test_float32_within_dot_rounding_envelope(kb, O, solver):
    A, b = _big(O)
    xo, so = getattr(O, solver)(A, b, dtype=np.float32, itmax=40)
    with O.dot_mode(1):
        _, s1 = getattr(O, solver)(A, b, dtype=np.float32, itmax=40)
    x, st = getattr(kb, solver)(A, b.astype(np.float32), itmax=40, history=True)
    assert st.niter == so["niter"]
    for key, got in (("residuals", st.residuals), ("Aresiduals", st.Aresiduals)):
        r0, r1 = np.asarray(so[key], float), np.asarray(s1[key], float)
        env = np.maximum.accumulate(np.abs(r0 - r1) / np.maximum(r0, 1e-300))
        res = np.asarray(got)
        tol = np.maximum(4 * 1.2e-7, 10 * env)
        assert np.all(np.abs(res - r0) <= tol * r0 + 1e-6 * r0[0]), key


@pytest.mark.parametrize("solver", SOLVERS)
def test_grouped_passes_equal_the_primitive_path(kb, O, solver):
    """fused=True runs an iteration as 3 launches (C1-C3 / M1-M3); every element update repeats the k* sequence it
    replaces, so against fused=False: same iteration count and status, histories equal to dot-product rounding, and
    fewer than 0.3x the launches."""
    A, b = _big(O)
    out = {}
    for fused in (True, False):
        ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64)
        ws.solve(A, b, itmax=3, fused=fused)
        l0 = ws.launches
        ws.solve(A, b, history=True, fused=fused)
        out[fused] = (ws.x, ws.stats, ws.launches - l0)
        ws.free()
    (x1, s1, l1), (x0, s0, l0) = out[True], out[False]
    assert s1.niter == s0.niter and s1.status == s0.status
    assert np.allclose(s1.residuals, s0.residuals, rtol=1e-7, atol=1e-12 * s0.residuals[0])
    assert np.allclose(s1.Aresiduals, s0.Aresiduals, rtol=1e-7, atol=1e-12 * s0.Aresiduals[0])
    assert np.linalg.norm(x1 - x0) <= 1e-8 * np.linalg.norm(x0)
    assert l1 < 0.3 * l0, (l1, l0)


@pytest.mark.parametrize("solver", SOLVERS)
def test_benchmark_size_matches_oracle(kb, O, solver):
    """60 fused iterations on get_div_grad(215) with b = ones, all tolerances 0: the histories against the oracle's
    within 1e-6 relative, or 10x the oracle's own change under a 1-ulp perturbation of b where that is larger."""
    import torch
    n1 = 215
    rp, ci, va = P.div_grad_csr(n1, xp=torch, device="cuda")
    n = n1 ** 3
    A = sp.csr_matrix((va.cpu().numpy(), ci.cpu().numpy(), rp.cpu().numpy()), shape=(n, n))
    bh = np.ones(n)
    kw = dict(atol=0.0, rtol=0.0, itmax=60) | (dict(artol=0.0) if solver == "minares" else {})
    ws = kb.krylov_workspace(solver, n, n, np.float64, device="cuda")
    ws.solve((rp, ci, va), torch.tensor(bh, device="cuda"), history=True, **kw)
    st = ws.stats
    ws.free()
    _, so = getattr(O, solver)(A, bh, **kw)
    sign = np.random.default_rng(0).choice([-1.0, 1.0], size=n)
    _, s1 = getattr(O, solver)(A, bh * (1 + 2.2e-16 * sign), **kw)
    assert st.niter == so["niter"] == 60
    for key, got in (("residuals", st.residuals), ("Aresiduals", st.Aresiduals)):
        ro, rg, r1 = np.asarray(so[key]), np.asarray(got), np.asarray(s1[key])
        assert len(rg) == len(ro)
        tol = np.maximum(TOL, 10 * np.maximum.accumulate(np.abs(r1 - ro) / np.abs(ro)))
        rel = np.abs(rg - ro) / np.abs(ro)
        assert np.all(rel <= tol), (key, rel.max(), tol[np.argmax(rel > tol)])


def test_reference_test_all_solvers_car_minares_rows():
    import subprocess
    path = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "test_all_solvers")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/test_all_solvers was not built (reference tree absent at build time)")
    out = subprocess.run([path], capture_output=True, text=True, timeout=600)
    rows = [l for l in out.stdout.splitlines() if l.split() and l.split()[0].lower() in ("car", "minares")]
    assert len(rows) >= 2, out.stdout[-2000:]
    for l in rows:
        assert "PASS" in l, l
