"""GPU parity of bilqr! and trilqr! against the CPU oracle (oracle/krylov_oracle_adjoint.h), Float64: same iteration
count, status, solved_primal and solved_dual; both residual histories within parity.TOL relative at every iteration (or
10x the oracle's own sensitivity to a few-ulp change of b and c, where that is larger); x and y within 1e-6 relative.
Both paths: the fused one (3 launches per iteration) and fused = 0.  Float32 within the measured dot-rounding envelope."""
import ctypes as C
import importlib.util
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
SOLVERS = ["bilqr", "trilqr"]
KEYS = ("residuals_primal", "residuals_dual")
_spec = importlib.util.spec_from_file_location("gen_golden_adjoint", os.path.join(HERE, "golden", "gen_golden_adjoint.py"))
G = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(G)


@pytest.fixture(scope="module")
def O():
    """The CPU restatement of bilqr! / trilqr! (oracle/adjoint_oracle.py; test infrastructure)."""
    from oracle import adjoint_oracle
    adjoint_oracle.lib()
    return adjoint_oracle


def compare(O, kb, solver, A, b, c, *, gpu_A=None, device=False, xtol=TOL, floor=1e-9, **kw):
    """parity.compare's bar on the pair as one block system: K = diag(A, Aᵀ) with right-hand side [b; c] and solution
    [x; y], so that parity.compare perturbs b and c together, checks the residual of both systems and compares both
    histories ("keys") and both flags.  Counts that move under those perturbations (the SSY process on the dense and
    inconsistent pairs, the loss of biorthogonality of long BiLQR solves) take parity.compare's "widened" range.  Where
    the counts are steady, x and y are also checked one by one against the unperturbed oracle run, within xtol (None:
    only parity.compare's check of [x; y], within 10x the oracle's own change under the perturbations)."""
    m, n = A.shape
    K = sp.block_diag((A, sp.csr_matrix(A.T)), format="csr")
    first = {}

    def oracle(K_, bc, **kw_):
        x, y, st = getattr(O, solver)(A, bc[:m], bc[m:], **kw_)
        first.setdefault("xy", (x, y))
        return np.concatenate([x, y]), st

    def gpu(op, bc, **kw_):
        x, y, st = getattr(kb, solver)(op, bc[:m], bc[m:], **kw_)
        first["gpu"] = tuple(v.cpu().numpy() if hasattr(v, "cpu") else v for v in (x, y))
        return np.concatenate(first["gpu"]), st

    _, st, so = parity.compare(oracle, gpu, K, np.concatenate([b, c]), keys=KEYS, flags=("solved_primal", "solved_dual"),
                               floor=floor, unsteady="widened", check_length=True, xtol=xtol,
                               gpu_A=A if gpu_A is None else gpu_A, device_b=device, **kw)
    x, y = first["gpu"]
    if st.niter == so["niter"] and xtol is not None:
        for got_v, want_v in zip((x, y), first["xy"]):
            assert np.linalg.norm(got_v - want_v) <= xtol * max(np.linalg.norm(want_v), 1e-300)
    return x, y, st, so


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", sorted(G.cases()))
def test_known_answer_problems_match_oracle(kb, O, name, fused):
    solver, A, b, c, kw = G.cases()[name]
    if name == "trilqr/overdetermined_adjoint":
        # a dense 200 x 100 operator: below 1e-5 of their first entries both estimates follow the rounding of the
        # products' sums (the fused and the primitive path alike move there, away from the oracle's, by up to 1e-5)
        kw = dict(kw, floor=5e-5, xtol=1e-5)
    if name == "bilqr/adjoint_pde":
        # the oracle's count (210) does not move under few-ulp changes of b and c, but from about iteration 130 on the
        # biorthogonality is lost and the device's dot-product rounding moves it (194 on both paths): parity over the
        # first 120 iterations here, and the full solve against the reference's assertions below
        kw = dict(kw, itmax=120)
    compare(O, kb, solver, A, b, c, fused=fused, **kw)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("name", sorted(n for n in G.cases() if n != "bilqr/bc_breakdown"))
def test_known_answer_problems_meet_the_reference_assertions(kb, O, name, fused):
    """test_bilqr.jl / test_trilqr.jl on the full solves: both halves solved, with the oracle's status, and both
    relative residuals within 1e-6 (an inconsistent dual: ‖A s‖ / ‖A c‖), or within 10 atol where one is set."""
    solver, A, b, c, kw = G.cases()[name]
    x, y, st = getattr(kb, solver)(A, b, c, fused=fused, **kw)
    _, _, so = getattr(O, solver)(A, b, c, **kw)
    assert (st.solved_primal, st.solved_dual, st.status) == (True, True, so["status"]), st
    atol = kw.get("atol", 0.0)
    assert np.linalg.norm(b - A @ x) <= max(1e-6 * np.linalg.norm(b), 10 * atol)
    s_ = c - A.T @ y
    assert (np.linalg.norm(s_) <= max(1e-6 * np.linalg.norm(c), 10 * atol)
            or np.linalg.norm(A @ s_) <= 1e-6 * np.linalg.norm(A @ c))


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("shape", sorted(parity.shapes()))
def test_trilqr_on_rectangular_shapes(kb, O, shape, fused):
    """m > n, m < n, m = n and operators with empty rows and columns; c a random n-vector."""
    A, b = parity.shapes()[shape]
    c = np.random.default_rng(7).standard_normal(A.shape[1])
    compare(O, kb, "trilqr", A, b, c, fused=fused, itmax=40, xtol=None)   # 40 iterations: x and y are not converged


def _kron(O):
    A, b = O.kron_unsymmetric(12)
    return A, np.asarray(b), np.cos(np.arange(A.shape[0]))


@pytest.mark.parametrize("solver", SOLVERS)
def test_options_match_oracle(kb, O, solver):
    A, b, c = _kron(O)
    if solver == "trilqr":
        A = A[:, : A.shape[1] - 100].tocsr()                     # m > n
        c = c[: A.shape[1]]
    n, m = A.shape[1], A.shape[0]
    tkey = "transfer_to_bicg" if solver == "bilqr" else "transfer_to_usymcg"
    for fused in (True, False):
        compare(O, kb, solver, A, b, c, fused=fused, itmax=60)
        compare(O, kb, solver, A, b, c, fused=fused, itmax=60, **{tkey: False})
        compare(O, kb, solver, A, b, c, fused=fused, itmax=60, x0=np.sin(np.arange(n)), y0=np.cos(np.arange(m)))
        compare(O, kb, solver, A, b, c, fused=fused, itmax=60, device=True)


@pytest.mark.parametrize("solver", SOLVERS)
def test_zero_right_hand_sides(kb, O, solver):
    A, b, c = O.adjoint_ode(30)
    for bb, cc in ((0 * b, c), (b, 0 * c)):
        for fused in (True, False):
            x, y, st = getattr(kb, solver)(A, bb, cc, history=True, fused=fused, itmax=20)
            xo, yo, so = getattr(O, solver)(A, bb, cc, itmax=20)
            assert (st.niter, st.status, st.solved_primal, st.solved_dual) == \
                (so["niter"], so["status"], so["solved_primal"], so["solved_dual"])
            if solver == "bilqr":
                assert st.status == "Breakdown bᴴc = 0"


@pytest.mark.parametrize("solver", SOLVERS)
def test_warm_start2_takes_fewer_iterations(kb, O, solver):
    A, b, c = O.adjoint_pde(20, 20)
    tol = dict(atol=1e-7 * min(np.linalg.norm(b), np.linalg.norm(c)), rtol=0.0)
    ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64)
    ws.solve(A, b, c, **tol)
    cold, x, y = ws.stats.niter, ws.x, ws.y
    ws.warm_start(x + 1e-6, y - 1e-6)
    ws.solve(A, b, c, history=True, **tol)
    st = ws.stats
    xo, yo, so = getattr(O, solver)(A, b, c, x0=x + 1e-6, y0=y - 1e-6, **tol)
    assert st.niter < cold and st.niter == so["niter"] and st.status == so["status"]
    assert np.linalg.norm(ws.x - xo) <= TOL * np.linalg.norm(xo) and np.linalg.norm(ws.y - yo) <= TOL * np.linalg.norm(yo)
    with pytest.raises(kb.B200Error):
        ws.warm_start(x[:-1], y)                                   # warm_start2: lengths must match
    ws.free()


@pytest.mark.parametrize("solver", SOLVERS)
def test_split_convergence_freezes_the_solved_half(kb, O, solver):
    """One half converges well before the other: the "Only the ..." point is reached with the same flags, and the
    solved half's vector stops moving (its history stops growing) while the other half keeps iterating."""
    for case in ("primal_first", "dual_first"):
        _, A, b, c, kw = G.cases()[f"{solver}/{case}"]
        for fused in (True, False):
            x, y, st, so = compare(O, kb, solver, A, b, c, fused=fused, **kw)
        lp, ld = len(so["residuals_primal"]), len(so["residuals_dual"])
        assert (lp < ld) if case == "primal_first" else (ld < lp)
        k = min(lp, ld) - 1                                      # the iteration where the first half is solved
        ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64)
        ws.solve(A, b, c, itmax=k, **kw)
        st = ws.stats
        frozen = ws.x if case == "primal_first" else ws.y
        _, _, sk = getattr(O, solver)(A, b, c, itmax=k, **kw)
        assert (st.niter, st.status, st.solved_primal, st.solved_dual) == \
            (sk["niter"], sk["status"], sk["solved_primal"], sk["solved_dual"])
        assert (st.solved_primal, st.solved_dual) == ((True, False) if case == "primal_first" else (False, True))
        want = "Only the primal solution" if case == "primal_first" else "Only the dual solution"
        assert st.status.startswith(want), st.status
        ws.solve(A, b, c, itmax=k + 5, **kw)
        now = ws.x if case == "primal_first" else ws.y
        assert np.array_equal(now, frozen)
        ws.free()


@pytest.mark.parametrize("solver", SOLVERS)
def test_exits_and_callback(kb, O, solver):
    A, b, c = O.adjoint_pde()
    ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64)
    seen = []

    def cb(w):                                                     # TestCallbackN2Adjoint(A, b, c; tol = 0.1)
        seen.append(w.stats.niter)
        return bool(np.linalg.norm(A @ w.x - b) <= 0.1 and np.linalg.norm(A.T @ w.y - c) <= 0.1)
    ws.solve(A, b, c, atol=0.0, rtol=0.0, callback=cb)
    assert ws.stats.status == "user-requested exit" and cb(ws)
    assert seen[:3] == [1, 2, 3]
    ws.solve(A, b, c, timemax=0.0)
    assert ws.stats.status == "time limit exceeded" and ws.stats.niter == 1
    with pytest.raises(TypeError):
        ws.solve(A, b, c, callback=lambda w: "string", history=True)
    ws.free()


@pytest.mark.parametrize("solver", SOLVERS)
def test_float32_within_dot_rounding_envelope(kb, O, solver):
    A, b, c = _kron(O)
    kw = dict(dtype=np.float32, itmax=40)
    xo, yo, so = getattr(O, solver)(A, b, c, **kw)
    with O.dot_mode(1):
        _, _, s1 = getattr(O, solver)(A, b, c, **kw)
    x, y, st = getattr(kb, solver)(A, b.astype(np.float32), c.astype(np.float32), itmax=40, history=True)
    assert st.niter == so["niter"]
    for key in KEYS:
        r0, r1 = np.asarray(so[key], float), np.asarray(s1[key], float)
        env = np.maximum.accumulate(np.abs(r0 - r1) / np.maximum(r0, 1e-300))
        res = np.asarray(getattr(st, key))
        tol = np.maximum(4 * 1.2e-7, 10 * env)
        assert len(res) == len(r0) and np.all(np.abs(res - r0) <= tol * r0 + 1e-6 * r0[0]), key


@pytest.mark.parametrize("solver", SOLVERS)
def test_fused_launch_budget_and_equality_with_primitive_path(kb, O, solver):
    """fused = 1 runs an iteration as 3 launches; over a 100-iteration solve at most 3.1 per iteration.  Given the same
    scalars the element updates repeat the k* sequence, so against fused = 0 the histories agree to dot rounding."""
    A, b, c = O.adjoint_pde()                                     # neither half converges within 100 iterations
    out = {}
    for fused in (True, False):
        ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64)
        ws.solve(A, b, c, itmax=3, fused=fused)                    # forms and caches Aᵀ outside the count
        l0 = ws.launches
        ws.solve(A, b, c, atol=0.0, rtol=0.0, itmax=100, history=True, fused=fused)
        out[fused] = (ws.x, ws.y, ws.stats, ws.launches - l0)
        ws.free()
    (x1, y1, s1, l1), (x0, y0, s0, l0) = out[True], out[False]
    assert s1.niter == s0.niter == 100 and s1.status == s0.status
    assert l1 <= 3.1 * 100, l1
    for key in KEYS:
        a, b_ = np.asarray(getattr(s1, key)), np.asarray(getattr(s0, key))
        assert np.allclose(a, b_, rtol=1e-7, atol=1e-12 * b_[0]), key
    assert np.linalg.norm(x1 - x0) <= 1e-8 * np.linalg.norm(x0) and np.linalg.norm(y1 - y0) <= 1e-8 * np.linalg.norm(y0)


def test_callbacks_as_operator(kb, O):
    from scipy.sparse.linalg import aslinearoperator
    A, b, c = _kron(O)
    compare(O, kb, "bilqr", A, b, c, gpu_A=aslinearoperator(A), itmax=60)
    At = A[:, :-30].tocsr()
    compare(O, kb, "trilqr", At, b, c[: At.shape[1]], gpu_A=(lambda x: At @ x, lambda y: At.T @ y), itmax=60)


def test_c_abi_rules(kb):
    L = _lib.lib()
    for sid in (18, 19):
        for dt in (_lib.KRYLOV_FLOAT32, _lib.KRYLOV_FLOAT64):
            ws = C.c_void_p()
            assert L.krylov_workspace_create(sid, 4, 4, dt, 0, None, C.byref(ws)) == 0
            assert L.krylov_workspace_free(ws) == 0
        for dt in (2, 3):                                                                   # complex types
            assert L.krylov_workspace_create(sid, 4, 4, dt, 0, None, C.byref(C.c_void_p())) == -2
        ws = C.c_void_p()
        assert L.krylov_workspace_create(sid, 4, 4, _lib.KRYLOV_FLOAT64, 0, None, C.byref(ws)) == 0
        f = _lib.MATVEC(lambda x, y, u: None)
        null = _lib.MATVEC()
        b = np.ones(4)
        pb = b.ctypes.data_as(C.c_void_p)
        assert L.krylov_solve(ws, f, null, null, null, pb, pb, None, None) == -1
        assert "matvec_At" in _lib.last_error()
        assert L.krylov_solve(ws, f, f, null, null, pb, None, None, None) == -1                 # c is required
        assert "c must be given" in _lib.last_error()
        assert L.krylov_solve(ws, f, f, f, null, pb, pb, None, None) == -1                      # no M
        assert "preconditioner" in _lib.last_error()
        assert L.krylov_solve(ws, f, f, null, f, pb, pb, None, None) == -1                      # no N
        assert L.krylov_b200_set_preconditioner_diag(ws, 0, pb, 0) == 0
        assert L.krylov_solve(ws, f, f, null, null, pb, pb, None, None) == -1                   # nor an attached M
        assert L.krylov_b200_set_preconditioner_diag(ws, 0, None, 0) == 0
        assert L.krylov_warm_start(ws, pb, 4) == -1
        assert "krylov_warm_start2" in _lib.last_error()
        assert L.krylov_warm_start2(ws, pb, pb, 3, 4) == -1
        assert L.krylov_warm_start2(ws, pb, pb, 4, 4) == 0
        assert L.krylov_b200_dist_init(ws, 0, 1, 0, None, None) == -1
        assert "row-partitioned" in _lib.last_error()
        assert L.krylov_workspace_free(ws) == 0
    ws = C.c_void_p()                                        # single-solution workspaces keep answering -2
    assert L.krylov_workspace_create(12, 4, 4, _lib.KRYLOV_FLOAT64, 0, None, C.byref(ws)) == 0
    assert L.krylov_get_y(ws, None, 4) == -2 and L.krylov_warm_start2(ws, None, None, 4, 4) == -2
    assert L.krylov_workspace_free(ws) == 0
    for sid in (14, 15, 16, 17, 23, 31):                     # USYMLQ, USYMQR, TriCG, TriMR, USYMLQR, GPMR
        assert L.krylov_workspace_create(sid, 4, 4, _lib.KRYLOV_FLOAT64, 0, None, C.byref(C.c_void_p())) == -2


@pytest.mark.parametrize("solver", SOLVERS)
def test_benchmark_size_runs_fused(kb, O, solver):
    """30 iterations of the benchmark problems of profiles/bench_adjoint.py at a reduced size, device vectors."""
    import torch
    if solver == "bilqr":
        n1 = 40
        rp, ci, va = P.kron_unsymmetric_csr(n1, xp=torch, device="cuda")
        n = m = n1 ** 3
    else:
        n1 = 30
        rp, ci, va = P.grad_csr(n1, xp=torch, device="cuda")
        m, n = int(rp.shape[0]) - 1, n1 ** 3
    A = sp.csr_matrix((va.cpu().numpy(), ci.cpu().numpy(), rp.cpu().numpy()), shape=(m, n))
    b, c = A @ np.cos(np.arange(n)), A.T @ np.cos(np.arange(m))
    ws = kb.krylov_workspace(solver, m, n, np.float64, device="cuda")
    ws.solve((rp, ci, va), torch.tensor(b, device="cuda"), torch.tensor(c, device="cuda"), atol=0.0, rtol=0.0, itmax=30,
             history=True)
    st = ws.stats
    ws.free()
    kw = dict(atol=0.0, rtol=0.0, itmax=30)
    _, _, so = getattr(O, solver)(A, b, c, **kw)
    sign = np.random.default_rng(0).choice([-1.0, 1.0], size=m + n)   # the estimates' own sensitivity to 1 ulp of b, c
    bc = np.concatenate([b, c]) * (1 + 2.2e-16 * sign)
    runs = [(None, getattr(O, solver)(A, bc[:m], bc[m:], **kw)[2])]
    assert st.niter == so["niter"] == 30
    for key in KEYS:
        ro, rg = np.asarray(so[key]), np.asarray(getattr(st, key))
        assert len(rg) == len(ro), key
        tol = np.maximum(TOL, 10 * parity.sens(ro, runs, key))
        assert np.all(np.abs(rg - ro) <= tol * np.abs(ro)), key


def test_reference_test_all_solvers_rows():
    import subprocess
    path = os.path.join(os.path.dirname(HERE), "oracle", "_ref", "test_all_solvers")
    if not os.path.exists(path):
        pytest.skip("oracle/_ref/test_all_solvers was not built (reference tree absent at build time)")
    out = subprocess.run([path], capture_output=True, text=True, timeout=600)
    rows = {l.split()[0].lower(): l for l in out.stdout.splitlines() if l.split()}
    for name in ("bilqr", "trilqr"):
        assert name in rows and "PASS" in rows[name], out.stdout[-3000:]
    for name in ("cg", "cr", "minres", "gmres", "fom", "fgmres", "bicgstab", "cgs", "bilq", "qmr", "lsqr", "lsmr", "lslq",
                 "cgls", "crls", "car", "minares", "diom", "dqgmres"):
        if name in rows:
            assert "PASS" in rows[name], rows[name]
