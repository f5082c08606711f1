"""GPU parity of cgne! and crmr! against the CPU oracle (oracle/krylov_oracle_cgne.h), Float64: same iteration count,
status, solved and inconsistent flags; the residual history (and CRMR's ‖Aᵀr‖ history) within parity.TOL relative at
every iteration (or 10x the oracle's own sensitivity to a few-ulp change of b, where that is larger); x within 1e-6
relative where the counts are steady.  Both paths: the fused one (2 launches per CGNE iteration, 4 per CRMR iteration)
and fused = 0."""
import ctypes as C
import importlib.util
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp

import parity
from krylov_b200 import _lib
from krylov_b200 import problems as P
from parity import TOL

pytestmark = pytest.mark.gpu
FLAGS = ("solved", "inconsistent")
SOLVERS = ["cgne", "crmr"]
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "oracle_cgne_crmr.json")))
ZERO_TOL = dict(atol=0.0, rtol=0.0)


@pytest.fixture(scope="module")
def O():
    from oracle import cgne_oracle
    cgne_oracle.lib()
    return cgne_oracle


@pytest.fixture(scope="module")
def kb():
    import krylov_b200
    if krylov_b200.device_count() < 1:
        pytest.skip("no CUDA device")
    return krylov_b200


def keys_of(solver):
    return ("residuals", "Aresiduals") if solver == "crmr" else ("residuals",)


def compare(O, kb, solver, A, b, **kw):
    return parity.compare(getattr(O, solver), getattr(kb, solver), A, b, keys=keys_of(solver), flags=FLAGS, floor=1e-9,
                          **kw)


def golden_cases():
    spec = importlib.util.spec_from_file_location("gen_golden_cgne_crmr",
                                                  os.path.join(HERE, "golden", "gen_golden_cgne_crmr.py"))
    G = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(G)
    return G.cases()


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("case", sorted(GOLD))
def test_oracle_cases(O, kb, case, fused):
    """The problems of test_cgne.jl / test_crmr.jl; those with N or λ > 0 run the primitive path whatever `fused`."""
    solver, A, b, kw = golden_cases()[case]
    # small_sp runs a 5-iteration CGNE to itmax on an inconsistent system: its last steps work on rounding noise
    compare(O, kb, solver, A, b, fused=fused, xtol=None if "small_sp" in case else TOL, **kw)


def consistent_shapes():
    """parity.shapes() with b = A z: consistent systems on m > n, m < n, m = n and operators with empty rows and
    columns."""
    rng = np.random.default_rng(11)
    return {k: (A, A @ rng.standard_normal(A.shape[1])) for k, (A, _) in parity.shapes().items()}


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("shape", sorted(parity.shapes()))
@pytest.mark.parametrize("solver", SOLVERS)
def test_shapes(O, kb, solver, shape, fused):
    A, b = consistent_shapes()[shape]
    compare(O, kb, solver, A, b, fused=fused, itmax=10, xtol=None if "lstp" in shape else TOL, **ZERO_TOL)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("solver", SOLVERS)
def test_inconsistent_shapes(O, kb, solver, fused):
    """Tall systems of parity.shapes() with their own, inconsistent, right-hand sides: CRMR detects the inconsistency
    (after 40 and 38 iterations) and CGNE runs to itmax, as the oracle does."""
    for shape in ("tall_gaps", "grad7"):
        A, b = parity.shapes()[shape]
        compare(O, kb, solver, A, b, fused=fused, itmax=60, xtol=None)


@pytest.mark.parametrize("solver", SOLVERS)
def test_options_against_oracle(O, kb, solver):
    """λ > 0, diagonal N (mul and ldiv), itmax and timemax = 0 on the primitive path."""
    A, b = O.under_consistent()
    Ao, bo = O.over_consistent()
    d = np.linspace(1, 2, A.shape[0])
    compare(O, kb, solver, Ao, bo, itmax=1)
    compare(O, kb, solver, A, b, lambda_=1e-2)
    compare(O, kb, solver, A, b, N=d)
    compare(O, kb, solver, A, b, N=d, ldiv=True)
    compare(O, kb, solver, A, b, N=d, lambda_=0.5, itmax=3, **ZERO_TOL)
    x, st = getattr(kb, solver)(A, b, timemax=0.0)
    assert st.status == "time limit exceeded" and st.niter == 1


@pytest.mark.parametrize("solver", SOLVERS)
def test_callback_preconditioner_matches_its_diagonal(O, kb, solver):
    """N given as a host callable on the m-dimensional residual space runs as the same diagonal does."""
    A, b = consistent_shapes()["grad7"]
    d = np.linspace(1, 3, A.shape[0])
    xo, so = getattr(O, solver)(A, b, N=d, itmax=5, **ZERO_TOL)
    x, st = getattr(kb, solver)(A, b, N=lambda v: d * v, itmax=5, history=True, **ZERO_TOL)
    assert (st.niter, st.status) == (so["niter"], so["status"])
    for key in keys_of(solver):
        np.testing.assert_allclose(getattr(st, key), so[key], rtol=TOL)
    assert np.linalg.norm(x - xo) <= TOL * np.linalg.norm(xo)


def _launches(kb, solver, A, b, fused, itmax):
    ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64)
    try:
        ws.solve(A, b, fused=fused, itmax=itmax, **ZERO_TOL)
        assert ws.stats.niter == itmax, ws.stats.status
        return ws.launches
    finally:
        ws.free()


def launches_per_iteration(kb, solver, A, b, fused=True):
    return (_launches(kb, solver, A, b, fused, 12) - _launches(kb, solver, A, b, fused, 6)) / 6


def _grad(N):
    rp, ci, va = P.grad_csr(N)
    return sp.csr_matrix((va, ci, rp), shape=(len(rp) - 1, N ** 3))


def _div(N):
    return sp.csr_matrix(_grad(N).T)


def _dense_line(A, row):
    """A plus a dense row (row=True) or column: long enough that its tile, or the tile of Aᵀ, is untiled."""
    A = sp.lil_matrix(A)
    line = 1.0 + np.arange(A.shape[1 if row else 0]) / A.shape[1 if row else 0]
    if row:
        A[0, :] = line
    else:
        A[:, 0] = line.reshape(-1, 1)
    return sp.csr_matrix(A)


@pytest.mark.parametrize("solver,want", [("cgne", 2), ("crmr", 4)])
def test_fused_path_runs_and_untiled_twin_matches(O, kb, solver, want):
    """2 (CGNE) and 4 (CRMR) launches per iteration on a staged operator (the divergence of the 24³ grid, m < n), and
    as many on its untiled twins (with a dense row: A untiled; with a dense column: Aᵀ untiled), whose first three
    iterations match the oracle.  From the fourth on, the dense line's outlying singular value makes both solvers'
    histories depend on the order of the sums (a NumPy restatement departs from the oracle there too)."""
    D = _div(24)
    rng = np.random.default_rng(3)
    b = D @ rng.standard_normal(D.shape[1])
    assert launches_per_iteration(kb, solver, D, b) == want
    assert launches_per_iteration(kb, solver, D, b, fused=False) > want
    for row in (True, False):
        U = _dense_line(_div(24), row)
        bu = U @ rng.standard_normal(U.shape[1])
        assert launches_per_iteration(kb, solver, U, bu) == want
        compare(O, kb, solver, U, bu, fused=True, itmax=3, **ZERO_TOL)


RING_ENV = ("KB200_STAGES", "KB200_CTAS_PER_SM")


@pytest.mark.parametrize("solver", SOLVERS)
def test_ring_depth_changes_no_bit(kb, solver):
    """On an operator of about 10⁶ columns, at 3, 2 and 1 CTAs per SM, every ring depth gives byte-identical x,
    histories, niter and status; the default plan is compared with the same plan forced."""
    A = _div(72)                                                # 373 248 rows, 1 119 744 columns
    b = A @ np.cos(np.arange(A.shape[1], dtype=np.float64))
    kw = dict(itmax=20, history=True, **ZERO_TOL)
    ref = {}
    saved = {k: os.environ.get(k) for k in RING_ENV}
    try:
        for cps in (None, 3, 2, 1):
            for stages in ((None,) if cps is None else (1, 2, 3, 4)):
                for k in RING_ENV:
                    os.environ.pop(k, None)
                if cps is not None:
                    os.environ["KB200_CTAS_PER_SM"], os.environ["KB200_STAGES"] = str(cps), str(stages)
                x, st = getattr(kb, solver)(A, b, **kw)
                out = (x.tobytes(), np.asarray(st.residuals).tobytes(), np.asarray(st.Aresiduals).tobytes(), st.niter,
                       st.status)
                if cps is None:
                    ref["default"] = out
                    continue
                if out == ref["default"]:
                    ref.setdefault("default_cps", cps)
                assert out == ref.setdefault(cps, out), (cps, stages)
        assert "default_cps" in ref
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("solver", SOLVERS)
def test_callback_reads_current_x(O, kb, solver, fused):
    """The callback sees the x of the iteration it is called after: the oracle's x after k iterations."""
    A, b = consistent_shapes()["tall_gaps"]
    seen = []
    ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64)
    try:
        ws.solve(A, b, fused=fused, callback=lambda w: seen.append(w.x.copy()) or len(seen) >= 3, **ZERO_TOL)
        assert ws.stats.status == "user-requested exit" and ws.stats.niter == 3
        for k in (1, 2, 3):
            xo, so = getattr(O, solver)(A, b, itmax=k, **ZERO_TOL)
            assert so["niter"] == k
            assert np.linalg.norm(seen[k - 1] - xo) <= TOL * np.linalg.norm(xo)
    finally:
        ws.free()


@pytest.mark.parametrize("solver", SOLVERS)
def test_float32_within_dot_rounding_envelope(O, kb, solver):
    """On the 7³ gradient, where the oracle's Float32 history moves by less than 1e-5 between its two summation modes,
    the GPU's stays within 10x that envelope on both paths."""
    A, b = consistent_shapes()["grad7"]
    kw = dict(itmax=15, **ZERO_TOL)
    _, s0 = getattr(O, solver)(A, b, dtype=np.float32, **kw)
    with O.dot_mode(1):
        _, s1 = getattr(O, solver)(A, b, dtype=np.float32, **kw)
    for fused in (True, False):
        _, st = getattr(kb, solver)(A, b.astype(np.float32), history=True, fused=fused, **kw)
        for key in keys_of(solver):
            r0, r1, rg = (np.asarray(v, dtype=np.float64) for v in (s0[key], s1[key], getattr(st, key)))
            k = min(len(r0), len(r1), len(rg))
            env = np.maximum(np.abs(r1[:k] - r0[:k]), 1e-5 * np.abs(r0[:k]))
            assert np.all(np.abs(rg[:k] - r0[:k]) <= 10 * np.maximum.accumulate(env / np.abs(r0[:k])) * np.abs(r0[:k]))


@pytest.mark.parametrize("solver", SOLVERS)
def test_torch_device_inputs(O, kb, solver):
    A, b = O.under_consistent()
    compare(O, kb, solver, A, b, device_b=True)


@pytest.mark.parametrize("solver,sid", [("cgne", 26), ("crmr", 27)])
def test_c_abi_contract(O, kb, solver, sid):
    L = _lib.lib()
    assert _lib.SOLVER_IDS[solver] == sid
    h = C.c_void_p()
    assert L.krylov_workspace_create(sid, 3, 4, 2, _lib.KRYLOV_CPU, None, C.byref(h)) == -2        # Complex
    assert L.krylov_workspace_create(sid, 3, 4, 3, _lib.KRYLOV_CPU, None, C.byref(h)) == -2
    for dt in (np.float32, np.float64):
        w = kb.krylov_workspace(solver, 3, 4, dt)
        w.free()
    ws = kb.krylov_workspace(solver, 3, 4, np.float64)
    try:
        A = sp.csr_matrix(np.array([[1.0, 0, 2, 0], [0, 1.0, 0, 3], [1.0, 1, 0, 0]]))
        null = _lib.MATVEC()
        f = _lib.MATVEC(lambda x, y, u: None)
        b = np.array([1.0, 2.0, 3.0])
        rc = L.krylov_solve(ws._h, f, null, null, null, b.ctypes.data_as(C.c_void_p), None, None, None)
        assert rc == -1 and f"{solver} applies the adjoint of A" in _lib.last_error()
        ws.solve(A, b)
        assert ws.stats.solved
        np.testing.assert_allclose(A @ ws.x, b, rtol=1e-10)
        # λ travels in KrylovOptions.lambda
        xo, so = getattr(O, solver)(A, b, lambda_=0.25)
        ws.solve(A, b, lambda_=0.25)
        assert ws.stats.niter == so["niter"] and np.linalg.norm(ws.x - xo) <= TOL * np.linalg.norm(xo)
        # M is refused, as a callback and as an attached diagonal; N is the only preconditioner
        opts = L.krylov_default_options()
        rc = L.krylov_solve(ws._h, null, null, f, null, b.ctypes.data_as(C.c_void_p), None, None, C.byref(opts))
        assert rc == -1 and "takes no preconditioner M" in _lib.last_error() and "N" in _lib.last_error()
        dm = np.ones(3)
        assert L.krylov_b200_set_preconditioner_diag(ws._h, 0, dm.ctypes.data_as(C.c_void_p), 0) == 0
        rc = L.krylov_solve(ws._h, null, null, null, null, b.ctypes.data_as(C.c_void_p), None, None, C.byref(opts))
        assert rc == -1 and "takes no preconditioner M" in _lib.last_error()
        assert L.krylov_b200_set_preconditioner_diag(ws._h, 0, None, 0) == 0
        # an N diagonal has m entries
        dn = np.array([1.0, 2.0, 4.0])
        ws.solve(A, b, N=dn, itmax=2, atol=0.0, rtol=0.0)
        xo, so = getattr(O, solver)(A, b, N=dn, itmax=2, atol=0.0, rtol=0.0)
        assert np.linalg.norm(ws.x - xo) <= TOL * np.linalg.norm(xo)
        x0 = np.zeros(4)
        y = np.zeros(3)
        assert L.krylov_warm_start(ws._h, x0.ctypes.data_as(C.c_void_p), 4) == -1
        assert f"{solver} does not support warm-start (it takes no x0)" in _lib.last_error()
        assert L.krylov_warm_start2(ws._h, x0.ctypes.data_as(C.c_void_p), y.ctypes.data_as(C.c_void_p), 4, 3) == -2
        assert L.krylov_get_y(ws._h, y.ctypes.data_as(C.c_void_p), 3) == -2
        assert L.krylov_b200_dist_init(ws._h, 0, 2, 0, None, None) == -1
        blocks = np.ones((2, 2, 2))
        assert L.krylov_b200_set_preconditioner_blockdiag(ws._h, 1, 2, blocks.ctypes.data_as(C.c_void_p), 0) == -1
        names = ("x", "p", "Aᴴz", "r", "q") if solver == "cgne" else ("x", "p", "Aᴴr", "r", "q")
        for name in names:
            p = C.c_void_p()
            assert L.krylov_b200_get_vector(ws._h, name.encode(), C.byref(p)) == 0 and p.value, name
        lazy = ("s", "z") if solver == "cgne" else ("s", "Nq")   # allocated by the solves that need them (N, λ > 0)
        for name in lazy:
            p = C.c_void_p()
            assert L.krylov_b200_get_vector(ws._h, name.encode(), C.byref(p)) == 0 and p.value, name
    finally:
        ws.free()


def test_reference_c_programs():
    """The cgne and crmr rows of the reference's test_all_solvers.c (built into oracle/_ref/ by build()) pass, and so
    does every row that passed before."""
    import subprocess
    exe = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "test_all_solvers")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/test_all_solvers was not built (reference tree absent at build time)")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    rows = {ln.split()[0].lower(): ln for ln in out.stdout.splitlines() if ln.split()}
    for name in ("cgne", "crmr"):
        assert name in rows and "PASS" in rows[name], out.stdout[-3000:]
    for name in ("cg", "cr", "minres", "gmres", "fom", "fgmres", "bicgstab", "cgs", "bilq", "qmr", "lsqr", "lsmr", "lslq",
                 "cgls", "crls", "car", "minares", "diom", "dqgmres", "bilqr", "trilqr", "craig", "craigmr", "lnlq"):
        if name in rows:
            assert "PASS" in rows[name], rows[name]
