"""GPU: block-Jacobi preconditioner (SURVEY.md 8f-1; docs/src/preconditioners.md:33,159) -- dense b x b diagonal
blocks, b in {2, 4, 8} (+ a block size with a ragged last block) -- through the C ABI vs the CPU oracle.
cg! carries it inside the persistent fused kernel (z = M r formed block by block in the r-update phase); gmres!,
bicgstab!, minres! apply it as one extra kernel per product; ldiv = true applies the inverted blocks."""
import ctypes as C
import functools
import os

import numpy as np
import pytest
import scipy.sparse as sp

import parity
import test_gpu_tile_plans as TP
from krylov_b200 import _lib
from krylov_b200 import problems as P

pytestmark = pytest.mark.gpu


def _diag_blocks(A, bs):
    """(nblocks, bs, bs) diagonal blocks of A (zero-padded last block with a unit diagonal in the padding)."""
    n = A.shape[0]
    nb = (n + bs - 1) // bs
    D = np.zeros((nb, bs, bs))
    C = sp.coo_matrix(A)
    keep = C.row // bs == C.col // bs
    D[C.row[keep] // bs, C.row[keep] % bs, C.col[keep] % bs] = C.data[keep]
    for i in range(n - (nb - 1) * bs, bs):
        D[-1, i, i] = 1.0
    return D


@pytest.mark.parametrize("bs", [2, 4, 8, 3])
def test_cg_block_jacobi_fused_matches_oracle(kb, O, bs):
    A, b = O.sparse_laplacian(12)                       # n = 1728
    A = sp.csr_matrix(A + sp.diags(np.linspace(0.0, 2.0, A.shape[0])))
    n = A.shape[0]
    Minv = np.linalg.inv(_diag_blocks(A, bs))           # the operator the solver applies: P^-1 (SPD blocks)
    with O.precond_block(bs):
        xo, so = O.cg(A, b, M=Minv.reshape(-1), atol=0.0, rtol=1e-10)
    ws = kb.CgWorkspace(n, n, np.float64)
    for fused in (True, False):                         # persistent fused kernel / primitive path
        ws.solve(A, b, M=Minv, atol=0.0, rtol=1e-10, history=True, fused=fused)
        st = ws.stats
        assert st.niter == so["niter"] and st.status == so["status"], (fused, st.niter, so["niter"])
        assert np.allclose(st.residuals, so["residuals"], rtol=1e-6, atol=1e-9 * so["residuals"][0])
        assert np.linalg.norm(ws.x - xo) <= 1e-6 * np.linalg.norm(xo)
        if fused:
            launches_fused = ws.launches
    # fewer iterations than unpreconditioned CG, and the fused path launches far less than the primitive one
    x1, s1 = kb.cg(A, b, atol=0.0, rtol=1e-10)
    assert st.niter < s1.niter
    l0 = ws.launches
    ws.solve(A, b, M=Minv, atol=0.0, rtol=1e-10, fused=True)
    assert ws.launches - l0 < 20 + st.niter              # one persistent launch per 16 iterations + prologue
    ws.free()


def test_cg_block_jacobi_without_x_update_in_k1_falls_back(kb, O, monkeypatch):
    """KB200_XUP=0 rules out the persistent kernel, the only fused kernel that carries a block-Jacobi M: the solve
    must take the primitive path (same iterations, status and x as fused=False) instead of failing."""
    A, b = O.sparse_laplacian(12)
    A = sp.csr_matrix(A + sp.diags(np.linspace(0.0, 2.0, A.shape[0])))
    n = A.shape[0]
    Minv = np.linalg.inv(_diag_blocks(A, 4))
    ws = kb.CgWorkspace(n, n, np.float64)
    ws.solve(A, b, M=Minv, atol=0.0, rtol=1e-10, fused=False)
    ref = (ws.stats.niter, ws.stats.status, np.array(ws.x))
    monkeypatch.setenv("KB200_XUP", "0")
    ws.solve(A, b, M=Minv, atol=0.0, rtol=1e-10, fused=True)
    assert (ws.stats.niter, ws.stats.status) == ref[:2]
    assert np.array_equal(ws.x, ref[2])
    ws.free()


def test_block_jacobi_ldiv_and_other_solvers(kb, O):
    Ak, bk = O.kron_unsymmetric(9)                       # n = 729 = 3^6: ragged last block for bs = 4, 8
    Ak = sp.csr_matrix(Ak + sp.diags(np.linspace(0.0, 3.0, Ak.shape[0])))
    n = Ak.shape[0]
    for bs in (4, 8):
        P = _diag_blocks(Ak, bs)
        Pinv = np.linalg.inv(P)
        with O.precond_block(bs):
            ref = {"gmres": O.gmres(Ak, bk, M=Pinv.reshape(-1), memory=30), "bicgstab": O.bicgstab(Ak, bk, M=Pinv.reshape(-1)),
                   "gmres_ldiv": O.gmres(Ak, bk, M=P.reshape(-1), ldiv=True, memory=30),
                   "gmres_right": O.gmres(Ak, bk, N=Pinv.reshape(-1), memory=30)}
        runs = {"gmres": ("gmres", dict(M=Pinv, memory=30)), "bicgstab": ("bicgstab", dict(M=Pinv)),
                "gmres_ldiv": ("gmres", dict(M=P, ldiv=True, memory=30)), "gmres_right": ("gmres", dict(N=Pinv, memory=30))}
        for name, (solver, kw) in runs.items():
            mem = kw.pop("memory", 0)
            ws = kb.krylov_workspace(solver, n, n, np.float64, memory=mem)
            ws.solve(Ak, bk, history=True, **kw)
            xo, so = ref[name]
            st = ws.stats
            assert st.niter == so["niter"] and st.status == so["status"], (name, bs, st.niter, so["niter"])
            tol = 1e-5 if solver == "bicgstab" or "ldiv" in name else 1e-6
            assert np.allclose(st.residuals, so["residuals"], rtol=tol, atol=1e-9 * so["residuals"][0]), (name, bs)
            assert np.linalg.norm(ws.x - xo) <= 1e-6 * np.linalg.norm(xo), (name, bs)
            ws.free()


def test_block_jacobi_argument_checks(kb):
    ws = kb.CgWorkspace(10, 10, np.float64)
    with pytest.raises(kb.B200Error):
        ws._set_diag(0, np.zeros((2, 4, 4)))            # 10 rows need ceil(10/4) = 3 blocks
    with pytest.raises(kb.B200Error):
        ws._set_diag(0, np.zeros((1, 16, 16)))          # block size must be in 2..8
    ws.free()


# ----------------------------------------------------------------------------------------------------------------------
# Every solver that takes the blocks, against the oracle, at every block size, both types, fused and not
# ----------------------------------------------------------------------------------------------------------------------
SPD = ["cg", "cr", "minres", "car", "cg_lanczos"]
UNSYM_M = ["diom", "dqgmres", "fom", "gmres", "fgmres", "bicgstab", "cgs"]     # these take block N as well
OPTS = {"gmres": dict(memory=20), "fom": dict(memory=20), "fgmres": dict(memory=20), "dqgmres": dict(memory=6),
        "diom": dict(memory=6)}
CASES = [(s, "M") for s in SPD + UNSYM_M] + [(s, "N") for s in UNSYM_M]


@functools.cache
def operators(n):
    """The SPD operator and a nonsymmetric one on n rows.  n = 841 = 29² ≡ 1 (mod 840): every bs in 2..8 leaves a
    one-row last block.  n = 839: its leading 839 x 839 part, whose last block has bs - 1 rows for every bs.  The
    diagonal shift keeps every diagonal block, and the nonsymmetric operator's, well away from singular."""
    S = sp.csr_matrix(sp.csr_matrix((lambda c: (c[2], c[1], c[0]))(P.div_grad_csr(29, 29, 1)), shape=(841, 841)))
    S = sp.csr_matrix(S + sp.diags(np.linspace(0.0, 2.0, 841)))
    U = sp.csr_matrix(S + 0.5 * sp.triu(S, 1))
    S, U = sp.csr_matrix(S[:n, :n]), sp.csr_matrix(U[:n, :n])
    S.sort_indices()
    U.sort_indices()
    return S, U


def _oracle_fn(O, solver):
    if solver == "car":
        from oracle import ares_oracle
        return ares_oracle
    return O


def compare_blocks(O, kb, solver, A, b, bs, side, P, ldiv=False, **kw):
    """parity.compare with the dense blocks P as M or N (side), with the bar of the solver family's own tests; ldiv:
    P is applied by its inverse, which the GPU precomputes and the oracle does not, so x gets the bar of the oracle's
    own perturbed runs."""
    mod = _oracle_fn(O, solver)

    def oracle(A_, b_, **kw_):
        with O.precond_block(bs):
            return getattr(mod, solver)(A_, b_, **{side: P.reshape(-1)}, ldiv=ldiv, **kw_)

    def gpu(A_, b_, **kw_):
        return getattr(kb, solver)(A_, b_, **{side: P}, ldiv=ldiv, **kw_)
    kw = dict(OPTS.get(solver, {}), **kw)
    if solver == "car":
        bar = dict(keys=("residuals", "Aresiduals"), flags=("solved",), floor=1e-12, unsteady="widened", xtol=None)
    else:
        bar = dict(keys=("residuals",), flags=("solved", "inconsistent"), floor=1e-9,
                   xtol=None if ldiv or solver == "cgs" else parity.TOL)
    return parity.compare(oracle, gpu, A, b, **bar, **kw)


def _stop(solver):
    """Default tolerances with an iteration cap, as the families' own tests run them.  CR with a preconditioner
    tracks ‖r‖ by the reference's recurrence √|ρ + ω| √|ρ - ω|, which cancels near convergence: there the oracle's own
    count moves from 13 to 150 under a one-ulp change of b, so CR runs a fixed 12 iterations instead."""
    if solver == "cr":
        return dict(atol=0.0, rtol=0.0, itmax=12)
    return dict(itmax=60 if solver == "cgs" else 150)


def _problem(solver, n, bs, ldiv=False):
    S, U = operators(n)
    A = S if solver in SPD else U
    assert n % bs != 0
    Pb = _diag_blocks(A, bs)
    b = np.ones(n) if solver in SPD else A @ np.cos(np.arange(n))
    return A, b, (Pb if ldiv else np.linalg.inv(Pb))


@pytest.mark.parametrize("n", [841, 839])
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("bs", range(2, 9))
@pytest.mark.parametrize("solver,side", CASES)
def test_block_jacobi_matches_oracle(kb, O, solver, side, bs, fused, n):
    A, b, Minv = _problem(solver, n, bs)
    assert (n - 1) % bs == (0 if n == 841 else bs - 2)          # last block: 1 row (n = 841), bs - 1 rows (n = 839)
    compare_blocks(O, kb, solver, A, b, bs, side, Minv, fused=fused, **_stop(solver))


@pytest.mark.parametrize("n", [841, 839])
@pytest.mark.parametrize("bs", range(2, 9))
@pytest.mark.parametrize("solver,side", CASES)
def test_block_jacobi_ldiv_matches_oracle(kb, O, solver, side, bs, n):
    """ldiv = true: the GPU multiplies by the inverses formed at attach time, the oracle eliminates block by block."""
    A, b, Pb = _problem(solver, n, bs, ldiv=True)
    compare_blocks(O, kb, solver, A, b, bs, side, Pb, ldiv=True, **_stop(solver))


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("bs", range(2, 9))
@pytest.mark.parametrize("solver,side", CASES)
def test_block_jacobi_float32_matches_oracle(kb, O, solver, side, bs, fused):
    """Float32 on n = 841, 12 iterations, all tolerances 0, within the dot-rounding envelope of the oracle (its Float32
    run against the same run with double-accumulated dots)."""
    A, b, Minv = _problem(solver, 841, bs)
    b32, M32 = b.astype(np.float32), Minv.astype(np.float32)
    kw = dict(atol=0.0, rtol=0.0, itmax=12, **OPTS.get(solver, {}))
    with O.precond_block(bs):
        so, s1 = TP._f32_envelope(_oracle_fn(O, solver), solver, A, b32, **{side: M32.reshape(-1)}, **kw)
    x, st = getattr(kb, solver)(A.astype(np.float32), b32, **{side: M32}, history=True, fused=fused, **kw)
    assert x.dtype == np.float32
    assert (st.niter, st.status) == (so["niter"], so["status"])
    assert TP._within_envelope(st.residuals, so["residuals"], s1["residuals"])


# ----------------------------------------------------------------------------------------------------------------------
# CG: the persistent kernel, warm starts, device blocks, the fallbacks to the primitive path
# ----------------------------------------------------------------------------------------------------------------------
def _cg_launches(kb, A, b, Minv, fused, dt=np.float64):
    ws = kb.CgWorkspace(A.shape[0], A.shape[0], dt)
    ws.solve(A, (1e8 * b).astype(dt), M=Minv.astype(dt), atol=0.0, rtol=0.0, itmax=64, fused=fused)
    out = ws.launches, ws.stats.niter
    ws.free()
    return out


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("bs", range(2, 9))
def test_cg_block_jacobi_runs_the_persistent_kernel(kb, bs, dt):
    """Block sizes 2, 4, 8 (compiled) and 3, 5, 6, 7 (run-time size), ragged last block: one launch per batch of
    iterations, far fewer than the primitive path's several per iteration.  (b is scaled so that the absolute stop
    ‖r‖ + 1 <= 1 of cg! comes late.)"""
    A, b, Minv = _problem("cg", 841, bs)
    lf, it = _cg_launches(kb, A, b, Minv, True, dt)
    lp, itp = _cg_launches(kb, A, b, Minv, False, dt)
    assert it == itp >= 20, (it, itp)
    assert 2 * lf < it and 4 * lf < lp, (lf, lp, it)


@pytest.fixture(scope="module")
def large():
    """div_grad(841, 841, 1): 707 281 rows, so at bs = 2 phase B's loop over blocks (stride grid x 288) takes several
    trips per thread."""
    A = sp.csr_matrix((lambda c: (c[2], c[1], c[0]))(P.div_grad_csr(841, 841, 1)), shape=(841 * 841,) * 2)
    A = sp.csr_matrix(A + sp.diags(np.linspace(0.0, 2.0, A.shape[0])))
    A.sort_indices()
    return A


@pytest.mark.parametrize("bs", [2, 3])
def test_cg_block_jacobi_multi_trip_matches_oracle(kb, O, large, bs):
    A = large
    n = A.shape[0]
    nb = (n + bs - 1) // bs
    grid = TP.plan_of(A, np.float64)["grid"]                   # the persistent grid is at most the plan's
    assert n % bs and nb > 2 * grid * 288, (nb, grid)
    Minv = np.linalg.inv(_diag_blocks(A, bs))
    b = np.cos(np.arange(n))
    compare_blocks(O, kb, "cg", A, b, bs, "M", Minv, fused=True, atol=0.0, rtol=0.0, itmax=100)
    ws = kb.CgWorkspace(n, n, np.float64)
    ws.solve(A, b, M=Minv, atol=0.0, rtol=0.0, itmax=100)
    assert 4 * ws.launches < ws.stats.niter, (ws.launches, ws.stats.niter)    # the persistent kernel ran
    ws.free()


@pytest.mark.parametrize("bs", [2, 5])
def test_cg_block_jacobi_warm_start_and_device_blocks(kb, O, bs):
    import torch
    A, b, Minv = _problem("cg", 841, bs)
    x0 = np.sin(np.arange(841))
    for fused in (True, False):
        compare_blocks(O, kb, "cg", A, b, bs, "M", Minv, fused=fused, x0=x0, rtol=1e-10)
    # the blocks as a CUDA tensor (copied device to device at attach time) give the same bytes as host blocks
    x1, s1 = kb.cg(A, b, M=Minv, rtol=1e-10, history=True)
    x2, s2 = kb.cg(A, b, M=torch.tensor(Minv, device="cuda"), rtol=1e-10, history=True)
    assert x1.tobytes() == x2.tobytes() and s1.residuals == s2.residuals and s1.niter == s2.niter


def _untiled_spd(N1=593, N2=17):
    """div_grad(593, 17, 1) (n = 10 081 ≡ 1 mod 840) with a dense first row and column, the corner raised above its
    row's sum: SPD, and its first tile holds more nonzeros than any ring takes (untiled)."""
    n = N1 * N2
    A = sp.csr_matrix((lambda c: (c[2], c[1], c[0]))(P.div_grad_csr(N1, N2, 1)), shape=(n, n))
    w = (1.0 + np.random.default_rng(1).random(n)) / n
    w[0] = w[1:].sum() + 1.0
    R = sp.csr_matrix((w, (np.zeros(n, np.int64), np.arange(n))), shape=(n, n))
    A = sp.csr_matrix(A + R + sp.csr_matrix(R.T) - sp.csr_matrix(([w[0]], ([0], [0])), shape=(n, n)))
    A.sort_indices()
    return A


def test_cg_block_jacobi_fallbacks_match_the_primitive_path(kb, O, monkeypatch):
    """Wherever the persistent kernel cannot run -- fused = 2, KB200_XUP=0, a callback, an untiled operator -- a
    block-Jacobi CG takes the primitive path: the same niter, status and x bytes as fused = False."""
    for A in (operators(841)[0], _untiled_spd()):
        n = A.shape[0]
        bs = 7
        assert n % bs == 1
        Minv = np.linalg.inv(_diag_blocks(A, bs))
        b = np.ones(n)

        def run(**kw):
            x, st = kb.cg(A, b, M=Minv, atol=0.0, rtol=1e-10, history=True, **kw)
            return st.niter, st.status, x.tobytes()
        ref = run(fused=False)
        untiled = not TP.plan_of(A, np.float64)["tma_ok"]
        assert untiled == (n != 841)
        if untiled:
            assert run(fused=True) == ref
            compare_blocks(O, kb, "cg", A, b, bs, "M", Minv, fused=True, rtol=1e-10)
            continue
        assert run(fused=2) == ref
        assert run(callback=lambda ws: False) == ref
        monkeypatch.setenv("KB200_XUP", "0")
        assert run(fused=True) == ref
        monkeypatch.delenv("KB200_XUP")


# ----------------------------------------------------------------------------------------------------------------------
# The block kernel on every tile plan
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("bs", [2, 7])
def test_cg_block_jacobi_on_every_tile_plan(kb, O, monkeypatch, dt, bs):
    """Block-Jacobi CG, 20 iterations, all tolerances 0, on the 102³ grid (bs = 7: a one-row last block) at 3, 2 and 1
    CTAs per SM and every ring depth: identical bytes within a CTA count, and each CTA count against the oracle."""
    A = TP.ring_operator("div_grad")
    n = A.shape[0]
    assert (bs == 2) == (n % bs == 0)
    Minv = np.linalg.inv(_diag_blocks(A, bs)).astype(dt)
    b = np.cos(np.arange(n)).astype(dt)
    isz = np.dtype(dt).itemsize
    seen = {}

    def run():
        cps, s = (int(os.environ[k]) if k in os.environ else None for k in ("KB200_CTAS_PER_SM", "KB200_STAGES"))
        if cps is not None and s in TP.ring_depths("div_grad", cps, isz):
            TP.assert_plan(A, dt, (cps, s))
        op = kb.CsrOperator.from_scipy(A, dtype=dt)
        ws = kb.CgWorkspace(n, n, dt)
        ws.solve(op, b, M=Minv, atol=0.0, rtol=0.0, itmax=20, history=True)
        out = ws.x.tobytes(), np.asarray(ws.stats.residuals).tobytes(), ws.stats.niter, ws.stats.status
        l0 = ws.launches
        ws.free()
        op.free()
        assert l0 < 20, l0                                       # the persistent kernel ran
        seen.setdefault(cps, out)
        return out
    parity.assert_ring_depth_changes_no_bit(monkeypatch, run)
    kw = dict(atol=0.0, rtol=0.0, itmax=20)
    if dt == np.float64:
        with O.precond_block(bs):
            xo, so = O.cg(A, b, M=Minv.reshape(-1), **kw)
        for cps, (x, res, niter, status) in seen.items():
            r = np.frombuffer(res)
            assert (niter, status) == (so["niter"], so["status"])
            parity.assert_history("residuals", r, so["residuals"], lambda: np.zeros(len(r)), 1e-9 * so["residuals"][0])
            assert np.linalg.norm(np.frombuffer(x) - xo) <= parity.TOL * np.linalg.norm(xo), cps
    else:
        with O.precond_block(bs):
            so, s1 = TP._f32_envelope(O, "cg", A, b, M=Minv.reshape(-1), **kw)
        for cps, (x, res, niter, status) in seen.items():
            assert niter == so["niter"] and TP._within_envelope(np.frombuffer(res), so["residuals"], s1["residuals"]), cps


# ----------------------------------------------------------------------------------------------------------------------
# Refusals, and singular blocks under ldiv = true
# ----------------------------------------------------------------------------------------------------------------------
SQ, LS, LN = (6, 6), (6, 4), (4, 6)
REFUSED = {   # solver: (shape, refused at attach, the text for M, the text for N)
    "minares": (SQ, False, "Preconditioners are not yet supported", "car and minares take no right preconditioner N"),
    "bilq": (SQ, False, "bilq and qmr apply M^H and N^H: block-Jacobi", "bilq and qmr apply M^H and N^H: block-Jacobi"),
    "qmr": (SQ, False, "bilq and qmr apply M^H and N^H: block-Jacobi", "bilq and qmr apply M^H and N^H: block-Jacobi"),
    "bilqr": (SQ, False, "bilqr takes no preconditioner", "bilqr takes no preconditioner"),
    "trilqr": (LS, False, "trilqr takes no preconditioner", "trilqr takes no preconditioner"),
    **{s: (LS if s in ("lsqr", "lsmr", "lslq", "cgls", "crls") else LN, True, "not available on least-squares",
           "not available on least-squares")
       for s in ("lsqr", "lsmr", "lslq", "cgls", "crls", "cgne", "crmr", "craig", "craigmr", "lnlq")},
}


@pytest.mark.parametrize("solver", sorted(REFUSED))
def test_block_jacobi_refusals(solver):
    L = _lib.lib()
    (m, n), at_attach, text_m, text_n = REFUSED[solver]
    A = np.eye(m, n) * 4.0 + np.eye(m, n, 1)
    nz = np.nonzero(A)
    rowptr = np.concatenate([[0], np.cumsum(np.count_nonzero(A, axis=1))]).astype(np.int32)
    colind, vals = nz[1].astype(np.int32), A[nz]
    b, c = np.ones(m), np.ones(n)
    blocks = np.tile(np.eye(3), (4, 1, 1))
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    ws = C.c_void_p()
    assert L.krylov_workspace_create(_lib.SOLVER_IDS[solver], m, n, _lib.KRYLOV_FLOAT64, _lib.KRYLOV_CPU, None,
                                     C.byref(ws)) == 0
    try:
        assert L.krylov_b200_set_operator_csr(ws, m, len(colind), ptr(rowptr), ptr(colind), ptr(vals), 0, 4, 0) == 0
        null = _lib.MATVEC()
        for which, text in ((0, text_m), (1, text_n)):
            rc = L.krylov_b200_set_preconditioner_blockdiag(ws, which, 3, ptr(blocks), 0)
            if not at_attach:
                assert rc == 0, _lib.last_error()
                rc = L.krylov_solve(ws, null, null, null, null, ptr(b), ptr(c), None, None)
            assert rc == -1 and text in _lib.last_error(), _lib.last_error()
            assert L.krylov_b200_set_preconditioner_blockdiag(ws, which, 3, None, 0) == 0
    finally:
        L.krylov_workspace_free(ws)


@pytest.mark.parametrize("solver,side", [("gmres", "M"), ("gmres", "N"), ("cg", "M"), ("bicgstab", "N")])
def test_singular_block_refuses_ldiv(kb, O, solver, side):
    """A singular diagonal block is accepted; ldiv = true then fails naming the first singular block, as the
    reference's factorization raises, while ldiv = false applies the blocks as given and matches the oracle."""
    bs, n = 3, 841
    A, b, Pb = _problem(solver, n, bs, ldiv=True)
    Ps = Pb.copy()
    Ps[5, 1, :] = 0.0                                          # a zero row
    Ps[9, 2, :] = Ps[9, 0, :]                                  # two equal rows
    ws = kb.krylov_workspace(solver, n, n, np.float64, memory=20 if solver == "gmres" else 0)
    with pytest.raises(kb.B200Error, match=rf"block-Jacobi {side} with ldiv = true: diagonal block 5 \(rows 15 "):
        ws.solve(A, b, **{side: Ps}, ldiv=True)
    ws.solve(A, b, **{side: Pb}, ldiv=True, history=True)      # re-attached without singular blocks: no refusal
    assert ws.stats.solved
    ws.free()
    # ldiv = false: the singular blocks are just the operator applied
    if solver == "gmres":
        compare_blocks(O, kb, solver, A, b, bs, side, Ps, fused=False, atol=0.0, rtol=0.0, itmax=20)
