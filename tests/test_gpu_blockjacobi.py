"""GPU: block-Jacobi preconditioner (SURVEY.md 8f-1; docs/src/preconditioners.md:33,159) -- dense b x b diagonal
blocks, b in {2, 4, 8} (+ a block size with a ragged last block) -- through the C ABI vs the CPU oracle.
cg! carries it inside the persistent fused kernel (z = M r formed block by block in the r-update phase); gmres!,
bicgstab!, minres! apply it as one extra kernel per product; ldiv = true applies the inverted blocks."""
import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu


def _diag_blocks(A, bs):
    """(nblocks, bs, bs) diagonal blocks of A (zero-padded last block with a unit diagonal in the padding)."""
    n = A.shape[0]
    nb = (n + bs - 1) // bs
    D = np.zeros((nb, bs, bs))
    Ad = sp.csr_matrix(A)
    for k in range(nb):
        r0, r1 = k * bs, min(n, (k + 1) * bs)
        D[k, :r1 - r0, :r1 - r0] = Ad[r0:r1, r0:r1].toarray()
        for i in range(r1 - r0, bs):
            D[k, i, i] = 1.0
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
