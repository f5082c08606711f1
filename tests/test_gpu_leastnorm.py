"""GPU parity of craig! and craigmr! against the CPU oracle (oracle/krylov_oracle_leastnorm.h), Float64: same iteration
count, status, solved and inconsistent flags; the histories within parity.TOL relative at every iteration (or 10x the
oracle's own sensitivity to a few-ulp change of b, where that is larger); x and y within 1e-6 relative where the
counts are steady.  Both paths: the fused one (CRAIG: 2 launches per iteration, CRAIGMR: 3) and fused = 0."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp

import parity
from krylov_b200 import _lib
from parity import TOL

pytestmark = pytest.mark.gpu
SOLVERS = ["craig", "craigmr"]
KEYS = {"craig": ("residuals",), "craigmr": ("residuals", "Aresiduals")}
FLAGS = ("solved", "inconsistent")


@pytest.fixture(scope="module")
def O():
    from oracle import leastnorm_oracle
    leastnorm_oracle.lib()
    return leastnorm_oracle


@pytest.fixture(scope="module")
def kb():
    import krylov_b200
    if krylov_b200.device_count() < 1:
        pytest.skip("no CUDA device")
    return krylov_b200


def compare(O, kb, solver, A, b, *, unsteady=None, xtol=TOL, **kw):
    """parity.compare on x, then y against the oracle's y where the counts match.  xtol=None: the solve ends on noise
    (CRAIG's exits on an inconsistent system), x is held to 10x the oracle's own change under the perturbations of b
    and y is not compared."""
    ys = {}

    def oracle(A_, b_, **kw_):
        x, y, st = getattr(O, solver)(A_, b_, **kw_)
        ys.setdefault("oracle", y)
        return x, st

    def gpu(A_, b_, **kw_):
        x, y, st = getattr(kb, solver)(A_, b_, **kw_)
        ys["gpu"] = y.cpu().numpy() if hasattr(y, "cpu") else y
        return x, st

    x, st, so = parity.compare(oracle, gpu, A, b, keys=KEYS[solver], flags=FLAGS, floor=1e-9, unsteady=unsteady, xtol=xtol,
                               **kw)
    if st.niter == so["niter"] and xtol is not None:
        yo = ys["oracle"]
        assert np.linalg.norm(ys["gpu"] - yo) <= TOL * max(np.linalg.norm(yo), 1e-300)
    return x, ys["gpu"], st, so


def oracle_cases(O):
    """name -> (A, b, kwargs): the problems of the reference's test_craig.jl / test_craigmr.jl."""
    out = {}
    for name in ("under_consistent", "under_inconsistent", "square_consistent", "square_inconsistent", "over_consistent",
                 "over_inconsistent", "small_ln"):
        out[name] = getattr(O, name)() + ({},)
    A, b = O.zero_rhs()
    out["zero_rhs"] = (A, b, dict(lambda_=1.0e-3))
    A, b, lam = O.regularization()
    out["regularization"] = (A, b, dict(lambda_=lam))
    A, b, D = O.saddle_point()
    out["saddle_point"] = (A, b, dict(N=1.0 / D))
    A, b, Mi, Ni = O.two_preconditioners()
    out["two_preconditioners"] = (A, b, dict(M=Mi, N=Ni))
    A, b, M, N = O.sqd()
    out["sqd"] = (A, b, dict(M=1.0 / M, N=1.0 / N, sqd=True))
    out["sqd_lambda4"] = (A, b, dict(M=1.0 / M, N=1.0 / N, lambda_=4.0))
    for t in (False, True):
        A, b, c, D = O.small_sp(t)
        out[f"small_sp_{int(t)}"] = (sp.csr_matrix(A.T), c, dict(N=1.0 / D))
    return out


CASES = ["under_consistent", "under_inconsistent", "square_consistent", "square_inconsistent", "over_consistent",
         "over_inconsistent", "small_ln", "zero_rhs", "regularization", "saddle_point", "two_preconditioners", "sqd",
         "sqd_lambda4", "small_sp_0", "small_sp_1"]


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("solver", SOLVERS)
def test_oracle_cases(O, kb, solver, case, fused):
    A, b, kw = oracle_cases(O)[case]
    # on these inconsistent systems CRAIG's last steps run on alpha or beta of the size of rounding noise, and x with them
    noisy = solver == "craig" and case in ("under_inconsistent", "square_inconsistent", "over_inconsistent", "small_sp_1")
    compare(O, kb, solver, A, b, fused=fused, xtol=None if noisy else TOL, **kw)


def consistent_shapes():
    """parity.shapes() with b = A z: consistent systems on m > n, m < n, m = n and operators with empty rows and
    columns (the least-norm problem is the meaningful one there)."""
    rng = np.random.default_rng(11)
    return {k: (A, A @ rng.standard_normal(A.shape[1])) for k, (A, _) in parity.shapes().items()}


def zero_tol(solver):
    """Tolerances 0 (CRAIG: btol = 0, conlim = 0): the solve runs itmax iterations."""
    return dict(atol=0.0, rtol=0.0, **({"btol": 0.0, "conlim": 0.0} if solver == "craig" else {}))


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("shape", sorted(parity.shapes()))
@pytest.mark.parametrize("solver", SOLVERS)
def test_shapes(O, kb, solver, shape, fused):
    A, b = consistent_shapes()[shape]
    # the lstp operators are built with a wide spread of singular values: after 10 iterations x moves by more than 1e-6
    # under a few-ulp change of b, so it is held to 10x the oracle's own change
    compare(O, kb, solver, A, b, fused=fused, itmax=10, xtol=None if "lstp" in shape else TOL, **zero_tol(solver))


@pytest.mark.parametrize("solver", SOLVERS)
def test_fused_path_runs_and_untiled_twin_matches(O, kb, solver):
    """At most 3 launches per iteration on a staged operator (CRAIG 2, CRAIGMR 3), and as many on its untiled twin,
    the gradient with a dense row (A untiled) or a dense column (Aᵀ untiled), whose results match the oracle."""
    G = parity.grad(24)
    rng = np.random.default_rng(3)
    b = G @ rng.standard_normal(G.shape[1])
    want = {"craig": 2, "craigmr": 3}[solver]
    assert parity.launches_per_iteration(kb, solver, G, b, **zero_tol(solver)) == want
    assert parity.launches_per_iteration(kb, solver, G, b, fused=False, **zero_tol(solver)) > want
    for row in (True, False):
        U = parity.dense_line(parity.grad(24), row)
        bu = U @ rng.standard_normal(U.shape[1])
        assert parity.launches_per_iteration(kb, solver, U, bu, **zero_tol(solver)) == want
        compare(O, kb, solver, U, bu, fused=True, itmax=40, xtol=None, **zero_tol(solver))


@pytest.mark.parametrize("solver", SOLVERS)
def test_ring_depth_changes_no_bit(kb, monkeypatch, solver):
    """On an operator of about 10⁶ rows, at 3, 2 and 1 CTAs per SM, every ring depth gives byte-identical x, y,
    histories, niter and status (parity.assert_ring_depth_changes_no_bit)."""
    G = parity.grad(72)                                         # 1 119 744 rows, 373 248 columns
    A = sp.csr_matrix(G.T) if solver == "craig" else G          # both orientations of the gradient pair
    b = A @ np.cos(np.arange(A.shape[1], dtype=np.float64))
    kw = dict(itmax=20, history=True, **zero_tol(solver))

    def run():
        x, y, st = getattr(kb, solver)(A, b, **kw)
        return (x.tobytes(), y.tobytes(), np.asarray(st.residuals).tobytes(), np.asarray(st.Aresiduals).tobytes(),
                st.niter, st.status)
    parity.assert_ring_depth_changes_no_bit(monkeypatch, run)


@pytest.mark.parametrize("solver", SOLVERS)
def test_options_against_oracle(O, kb, solver):
    A, b = O.over_consistent()
    Au, bu = O.under_consistent()
    compare(O, kb, solver, A, b, itmax=1)                                          # itmax
    compare(O, kb, solver, Au, bu, lambda_=1e-2, fused=True)                       # λ > 0 (primitive path)
    compare(O, kb, solver, Au, bu, M=np.linspace(1, 2, Au.shape[0]), N=np.linspace(1, 3, Au.shape[1]))   # diagonal M / N
    if solver == "craig":
        A2, b2, lam = O.regularization()
        compare(O, kb, solver, A2, b2, lambda_=lam, transfer_to_lsqr=True)
        compare(O, kb, solver, Au, bu, btol=1e-3)
        compare(O, kb, solver, Au, bu, conlim=10.0)
    x, y, st = getattr(kb, solver)(Au, bu, timemax=0.0)
    assert st.status == "time limit exceeded" and st.niter == 1


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("solver", SOLVERS)
def test_callback_reads_current_x(O, kb, solver, fused):
    """The callback sees the x of the iteration it is called after (CRAIG's fused x update is flushed before it)."""
    A, b = O.over_consistent()
    seen = []
    ws = getattr(kb, solver.capitalize() + "Workspace")(A.shape[0], A.shape[1], np.float64)
    try:
        ws.solve(A, b, fused=fused, callback=lambda w: seen.append(w.x.copy()) or len(seen) >= 2)
        assert ws.stats.status == "user-requested exit" and ws.stats.niter == 2
        xo, _, _ = getattr(O, solver)(A, b, itmax=2)
        assert np.linalg.norm(seen[-1] - xo) <= TOL * np.linalg.norm(xo)
        xo1, _, _ = getattr(O, solver)(A, b, itmax=1)
        assert np.linalg.norm(seen[0] - xo1) <= TOL * np.linalg.norm(xo1)
    finally:
        ws.free()


@pytest.mark.parametrize("solver", SOLVERS)
def test_float32_within_dot_rounding_envelope(O, kb, solver):
    A, b = consistent_shapes()["tall_gaps"]
    kw = dict(itmax=15, atol=0.0, rtol=0.0)
    _, _, s0 = getattr(O, solver)(A, b, dtype=np.float32, **kw)
    with O.dot_mode(1):
        _, _, s1 = getattr(O, solver)(A, b, dtype=np.float32, **kw)
    for fused in (True, False):
        _, _, st = getattr(kb, solver)(A, b.astype(np.float32), history=True, fused=fused, **kw)
        r0, r1, rg = (np.asarray(v, dtype=np.float64) for v in (s0["residuals"], s1["residuals"], st.residuals))
        k = min(len(r0), len(r1), len(rg))
        env = np.maximum(np.abs(r1[:k] - r0[:k]), 1e-5 * np.abs(r0[:k]))
        assert np.all(np.abs(rg[:k] - r0[:k]) <= 10 * np.maximum.accumulate(env / np.abs(r0[:k])) * np.abs(r0[:k]))


@pytest.mark.parametrize("solver", SOLVERS)
def test_torch_device_inputs(O, kb, solver):
    import torch
    A, b = O.under_consistent()
    x, y, st = getattr(kb, solver)(A, torch.tensor(b, device="cuda"))
    xo, yo, so = getattr(O, solver)(A, b)
    assert st.niter == so["niter"] and st.status == so["status"]
    assert np.linalg.norm(x.cpu().numpy() - xo) <= TOL * np.linalg.norm(xo)
    assert np.linalg.norm(y.cpu().numpy() - yo) <= TOL * np.linalg.norm(yo)


@pytest.mark.parametrize("solver", SOLVERS)
def test_c_abi_contract(kb, solver):
    L = _lib.lib()
    sid = _lib.SOLVER_IDS[solver]
    h = C.c_void_p()
    assert L.krylov_workspace_create(sid, 3, 4, 2, _lib.KRYLOV_CPU, None, C.byref(h)) == -2        # Complex
    assert L.krylov_workspace_create(sid, 3, 4, 3, _lib.KRYLOV_CPU, None, C.byref(h)) == -2
    ws = getattr(kb, solver.capitalize() + "Workspace")(3, 4, np.float64)
    try:
        A = sp.csr_matrix(np.array([[1.0, 0, 2, 0], [0, 1.0, 0, 3], [1.0, 1, 0, 0]]))
        null = _lib.MATVEC()
        f = _lib.MATVEC(lambda x, y, u: None)
        b = np.ones(3)
        rc = L.krylov_solve(ws._h, f, null, null, null, b.ctypes.data_as(C.c_void_p), None, None, None)
        assert rc == -1 and f"{solver} applies the adjoint of A" in _lib.last_error()
        ws.solve(A, b)
        y = np.empty(3)
        assert L.krylov_get_y(ws._h, y.ctypes.data_as(C.c_void_p), 3) == 0
        np.testing.assert_allclose(ws.x, A.T @ y, rtol=1e-10)
        x0 = np.zeros(4)
        assert L.krylov_warm_start(ws._h, x0.ctypes.data_as(C.c_void_p), 4) == -1
        assert "does not support warm-start" in _lib.last_error()
        assert L.krylov_warm_start2(ws._h, x0.ctypes.data_as(C.c_void_p), y.ctypes.data_as(C.c_void_p), 4, 3) == -2
        assert L.krylov_b200_dist_init(ws._h, 0, 2, 0, None, None) == -1
        blocks = np.ones((2, 2, 2))
        assert L.krylov_b200_set_preconditioner_blockdiag(ws._h, 0, 2, blocks.ctypes.data_as(C.c_void_p), 0) == -1
        for name in ("x", "y", "Nv", "Mu", "w") + (("d", "wbar", "w̄") if solver == "craigmr" else ()):
            p = C.c_void_p()
            assert L.krylov_b200_get_vector(ws._h, name.encode(), C.byref(p)) == 0 and p.value, name
    finally:
        ws.free()
    lsqr = kb.LsqrWorkspace(3, 4, np.float64)                  # single-solution workspaces still answer -2
    try:
        y = np.empty(3)
        assert L.krylov_get_y(lsqr._h, y.ctypes.data_as(C.c_void_p), 3) == -2
    finally:
        lsqr.free()


def test_sqd_with_lambda_raises(kb):
    with pytest.raises(kb.B200Error, match="sqd cannot be set to true if λ ≠ 0 !"):
        kb.craig(sp.csr_matrix(np.eye(2)), np.ones(2), sqd=True, lambda_=1.0)


def test_reference_c_programs():
    """The rows of the least-norm solvers (craig, craigmr, lnlq, cgne, crmr) in the reference's test_all_solvers.c
    (built into oracle/_ref/ by build()) pass, and so does every row that passed before."""
    import subprocess
    exe = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "test_all_solvers")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/test_all_solvers was not built (reference tree absent at build time)")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    rows = {ln.split()[0].lower(): ln for ln in out.stdout.splitlines() if ln.split()}
    for name in ("craig", "craigmr", "lnlq", "cgne", "crmr"):
        assert name in rows and "PASS" in rows[name], out.stdout[-3000:]
    for name in ("cg", "cr", "minres", "gmres", "fom", "fgmres", "bicgstab", "cgs", "bilq", "qmr", "lsqr", "lsmr", "lslq",
                 "cgls", "crls", "car", "minares", "diom", "dqgmres", "bilqr", "trilqr"):
        if name in rows:
            assert "PASS" in rows[name], rows[name]
