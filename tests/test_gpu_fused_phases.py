"""GPU: the fused iteration phases of bicgstab!/minres!/gmres! (csrc/fused_phases.cu) run the same arithmetic as
the primitive path (one kernel per k* call): same iteration count, same history, fewer launches."""
import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu

NAMES = ["bicgstab_kron10", "bicgstab_random3000_f32", "minres_divgrad16", "minres_shift", "minres_indefinite",
         "gmres_kron10_restart30", "gmres_divgrad16_mem10_restart", "gmres_divgrad16_mem10_norestart"]


def run(kb, name, fused):
    solver, A, b, kw, dt = cases.build(name)
    kw = dict(kw)
    mem = kw.pop("memory", 0)
    ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], dt, memory=mem)
    ws.solve(A, b.astype(dt), history=True, fused=fused, **kw)
    out = ws.x, ws.stats, ws.launches
    ws.free()
    return out


@pytest.mark.parametrize("name", NAMES)
def test_fused_phases_equal_primitive_path(kb, name):
    x1, s1, l1 = run(kb, name, True)
    x0, s0, l0 = run(kb, name, False)
    dt = cases.build(name)[4]
    assert s1.status == s0.status
    if dt == np.float64:
        assert s1.niter == s0.niter
        tight = 1e-9 if "mem10_restart" not in name else 1e-3      # restarted GMRES(10) amplifies reduction-order noise
        assert np.allclose(s1.residuals, s0.residuals, rtol=tight, atol=1e-9 * s0.residuals[0])
        assert np.linalg.norm(x1 - x0) <= max(tight, 1e-8) * np.linalg.norm(x0)
    else:
        assert abs(s1.niter - s0.niter) <= 2
    assert l1 < l0, (l1, l0)


def test_minres_history_vectors_fused(kb, O):
    A, b = O.sparse_laplacian(10)
    x, st = kb.minres(A, b, history=True)
    xo, so = O.minres(A, b)
    assert st.niter == so["niter"] and np.allclose(st.residuals, so["residuals"], rtol=1e-6)
    assert np.allclose(st.Aresiduals, so["Aresiduals"], rtol=1e-5, atol=1e-12) and np.allclose(st.Acond, so["Acond"], rtol=1e-6)
    assert np.allclose(x, xo, rtol=1e-7)


def test_gmres_fused_beyond_state_capacity(kb, O):
    """Non-restarted GMRES past the 120 h-slots of the fused state block falls back to the primitive path mid-solve."""
    A, b = O.kron_unsymmetric(7)
    x, st = kb.gmres(A, b, memory=5, rtol=1e-13, atol=0.0, itmax=160, history=True)
    xo, so = O.gmres(A, b, memory=5, rtol=1e-13, atol=0.0, itmax=160)
    assert st.niter == so["niter"]
    k = min(60, len(so["residuals"]))
    assert np.allclose(st.residuals[:k], so["residuals"][:k], rtol=1e-6)


def test_fused_cg_with_jacobi_preconditioner(kb, O):
    """Diagonal M folded into the two CG kernels (SURVEY.md 8f-1) == primitive path == oracle."""
    import scipy.sparse as sp
    A, b = O.sparse_laplacian(12)
    A = sp.csr_matrix(A + sp.diags(np.linspace(0.0, 5.0, A.shape[0])))      # non-constant diagonal
    d = 1.0 / A.diagonal()
    out = {}
    for fused in (True, False):
        ws = kb.CgWorkspace(A, b)
        ws.solve(A, b, M=d, history=True, fused=fused)
        out[fused] = (ws.x, ws.stats, ws.launches)
        ws.free()
    xo, so = O.cg(A, b, M=d)
    for fused in (True, False):
        x, st, _ = out[fused]
        assert st.niter == so["niter"] and np.allclose(st.residuals, so["residuals"], rtol=1e-6)
        assert np.linalg.norm(x - xo) <= 1e-7 * np.linalg.norm(xo)
    assert out[True][2] < out[False][2]


def _arrow_csr(N, dt):
    """div_grad(N) with a dense first row and column of small entries (corner raised above the row's sum): its first
    tile does not fit the shared-memory ring in either type, so CG runs cg_k1_rows."""
    import scipy.sparse as sp
    from krylov_b200 import problems as P
    rp, ci, va = P.div_grad_csr(N)
    n = N ** 3
    w = 1e-4 * (1.0 + np.arange(n) % 5)
    w[0] = w[1:].sum() + 1.0
    R = sp.csr_matrix((w, (np.zeros(n, np.int64), np.arange(n))), shape=(n, n))
    A = sp.csr_matrix(sp.csr_matrix((va, ci, rp), shape=(n, n)) + R + R.T - sp.csr_matrix(([w[0]], ([0], [0])), shape=(n, n)))
    A.sort_indices()
    return A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.astype(dt)


def test_cg_x_update_in_k1_is_bit_identical(kb):
    """Moving x += alpha p from K2 into the next K1 (XUP) changes no arithmetic: x, r and the residual history are
    bit-identical to the K2 placement, for convergence exits, itmax exits and Float32, on a staged operator
    (cg_k1_tma) and on an untiled one (cg_k1_rows)."""
    import os
    from krylov_b200 import problems as P
    for op, dt, kw in ((op, dt, kw) for op in ("stencil", "arrow") for dt, kw in (
            (np.float64, dict(atol=0.0, rtol=1e-8)), (np.float64, dict(atol=0.0, rtol=0.0, itmax=7)),
            (np.float64, dict(atol=0.0, rtol=0.0, itmax=8)), (np.float32, dict()))):
        rp, ci, va = P.div_grad_csr(20, dtype=dt) if op == "stencil" else _arrow_csr(31, dt)
        n = len(rp) - 1
        b = (np.arange(n) % 7 + 1).astype(dt)
        outs = []
        for flag in ("1", "0"):
            os.environ["KB200_XUP"] = flag
            ws = kb.CgWorkspace(n, n, dt)
            # fused=2: the two-launch kernels for both placements (the persistent kernel always carries the update
            # in phase A and sums <r,r> over a different grid, so it is not bit-comparable with the K2 placement)
            ws.solve((rp, ci, va), b, history=True, fused=2, **kw)
            outs.append((ws.x, ws.vector("r"), ws.stats))
            ws.free()
        os.environ.pop("KB200_XUP", None)
        (x1, r1, s1), (x0, r0, s0) = outs
        assert s1.niter == s0.niter and s1.residuals == s0.residuals and s1.status == s0.status
        assert np.array_equal(x1, x0) and np.array_equal(r1, r0)


def _jacobi_problem(O, kind):
    import scipy.sparse as sp
    if kind == "sym":
        A, b = O.sparse_laplacian(12)
        A = sp.csr_matrix(A + sp.diags(np.linspace(0.0, 5.0, A.shape[0])))
    else:
        A, b = O.kron_unsymmetric(9)
        A = sp.csr_matrix(A + sp.diags(np.linspace(0.0, 3.0, A.shape[0])))
    return A, b, 1.0 / A.diagonal()


@pytest.mark.parametrize("solver", ["bicgstab", "gmres", "gmres_restart", "minres"])
def test_fused_phases_with_jacobi_preconditioner(kb, O, solver):
    """Left diagonal M folded into the SpMV epilogues / the Lanczos stream pass (SURVEY.md 8f-1): the fused phases,
    the primitive path (M as its own kernel) and the oracle agree; the fused path launches fewer kernels."""
    name = solver.split("_")[0]
    A, b, d = _jacobi_problem(O, "sym" if name == "minres" else "unsym")
    kw = dict(M=d)
    okw = dict(M=d)
    mem = 0
    if name == "gmres":
        mem = 20
        kw["restart"] = okw["restart"] = solver.endswith("restart")
        okw["memory"] = mem
    out = {}
    for fused in (True, False):
        ws = kb.krylov_workspace(name, A.shape[0], A.shape[1], np.float64, memory=mem)
        ws.solve(A, b, history=True, fused=fused, **kw)
        out[fused] = (ws.x, ws.stats, ws.launches)
        ws.free()
    xo, so = getattr(O, name)(A, b, **okw)
    tol = 1e-5 if name == "bicgstab" else 1e-6
    for fused in (True, False):
        x, st, _ = out[fused]
        assert st.status == so["status"], (fused, st.status, so["status"])
        assert st.niter == so["niter"], (fused, st.niter, so["niter"])
        assert np.allclose(st.residuals, so["residuals"], rtol=tol, atol=1e-9 * so["residuals"][0]), fused
        assert np.linalg.norm(x - xo) <= 1e-6 * np.linalg.norm(xo), fused
    assert out[True][2] < out[False][2], (out[True][2], out[False][2])
    if name == "minres":
        assert np.allclose(out[True][1].Aresiduals, so["Aresiduals"], rtol=1e-5, atol=1e-12)
        assert np.allclose(out[True][1].Acond, so["Acond"], rtol=1e-6)
