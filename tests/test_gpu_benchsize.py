"""GPU parity at the BENCHMARK sizes of BASELINE.json (configs 2, 3, 4), through the C ABI vs the CPU oracle.

The small-case parity tests (test_gpu_solvers.py) pin flags and statuses; these pin the residual histories where
the performance numbers are quoted: n ~ 1e7 (7-point stencils) and n = 5e6 / nnz ~ 1.05e8 (random CSR, Float32).
The oracle is sequential, so each case costs it 0.5-2 minutes on the host; iteration counts are bounded
accordingly (fixed-iteration runs, atol = rtol = 0 -- the same way bench.py runs them).
Reference loops: src/cg.jl:195-268, src/gmres.jl:237-355, src/bicgstab.jl:215-256."""
import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu
F64_TOL = 1e-6
# block_gmres! on the host oracle (one thread): p = 8 on get_div_grad(215) takes about 14 s for 2 block iterations and
# 33 s for 4; p = 32 on get_div_grad(127) about 40 s for 2.
BLOCK_ITERS_P8, BLOCK_ITERS_P32 = 4, 2


def _mat(csr):
    rp, ci, va = csr
    n = len(rp) - 1
    return sp.csr_matrix((va, ci, rp), shape=(n, n))


def _rel(a, b):
    a, b = np.asarray(a, float), np.asarray(b, float)
    return np.abs(a - b) / np.maximum(np.abs(b), 1e-300)


def test_cfg2_cg_poisson215_history_matches_oracle(kb, O):
    """BASELINE config 2: cg! on get_div_grad(215,215,215) (n = 9 938 375), b = ones, 40 fixed iterations -- the
    persistent fused kernel AND the two-launch kernels against the sequential oracle, 1e-6 at every iteration."""
    from krylov_b200 import problems as P
    N, iters = 215, 40
    csr = P.div_grad_csr(N)
    n = N ** 3
    b = np.ones(n)
    xo, so = O.cg(_mat(csr), b, atol=0.0, rtol=0.0, itmax=iters)
    assert so["niter"] == iters
    ws = kb.CgWorkspace(n, n, np.float64)
    for fused in (True, 2):
        ws.solve(csr, b, atol=0.0, rtol=0.0, itmax=iters, history=True, fused=fused)
        st = ws.stats
        assert st.niter == so["niter"] and st.status == so["status"]
        assert len(st.residuals) == len(so["residuals"])
        assert _rel(st.residuals, so["residuals"]).max() <= F64_TOL
        assert np.linalg.norm(ws.x - xo) <= F64_TOL * np.linalg.norm(xo)
    ws.free()


def test_cfg3_gmres30_kron215_history_matches_oracle(kb, O):
    """BASELINE config 3: gmres!(memory = 30, restart = true) on kron_unsymmetric(215), b = A*ones; 40 inner
    iterations = one full cycle, the restart, and 10 iterations of the second cycle."""
    from krylov_b200 import problems as P
    N, iters = 215, 40
    csr = P.kron_unsymmetric_csr(N)
    A = _mat(csr)
    n = N ** 3
    b = A @ np.ones(n)
    xo, so = O.gmres(A, b, memory=30, restart=True, atol=0.0, rtol=0.0, itmax=iters)
    ws = kb.GmresWorkspace(n, n, np.float64, memory=30)
    ws.solve(csr, b, atol=0.0, rtol=0.0, itmax=iters, restart=True, history=True)
    st = ws.stats
    assert st.niter == so["niter"] == iters and st.status == so["status"]
    assert len(st.residuals) == len(so["residuals"])
    assert _rel(st.residuals, so["residuals"]).max() <= F64_TOL
    assert np.linalg.norm(ws.x - xo) <= F64_TOL * np.linalg.norm(xo)
    ws.free()


def test_cfg4_bicgstab_f32_random5e6_history_matches_oracle(kb, O):
    """BASELINE config 4: bicgstab! Float32 on the random CSR (n = 5e6, 20 draws per row + diagonal), b = A*ones,
    25 fixed iterations.  Tolerance = 10x the oracle's own sensitivity to the rounding of its dot products
    (sequential fp32 sums vs the same sums accumulated in double), floor 4 ulp(f32) -- measured, not hand-set."""
    from krylov_b200 import problems as P
    n, iters = 5_000_000, 25
    csr = P.random_csr(n, 20, seed=1234, dtype=np.float32)
    A = _mat(csr)
    b = (A @ np.ones(n, np.float32)).astype(np.float32)
    xo, so = O.bicgstab(A, b, dtype=np.float32, atol=0.0, rtol=0.0, itmax=iters)
    with O.dot_mode(1):
        xa, sa = O.bicgstab(A, b, dtype=np.float32, atol=0.0, rtol=0.0, itmax=iters)
    r0, r1 = np.asarray(so["residuals"], float), np.asarray(sa["residuals"], float)
    k = min(len(r0), len(r1))
    env = np.maximum.accumulate(np.abs(r0[:k] - r1[:k]) / np.maximum(r0[:k], 1e-300))
    ws = kb.BicgstabWorkspace(n, n, np.float32)
    ws.solve(csr, b, atol=0.0, rtol=0.0, itmax=iters, history=True)
    st = ws.stats
    assert abs(st.niter - so["niter"]) <= abs(so["niter"] - sa["niter"]) + 1
    res = np.asarray(st.residuals, float)
    k = min(k, len(res))
    tol = np.maximum(5e-7, 10 * env[:k])
    dev = np.abs(res[:k] - r0[:k])
    ok = dev <= tol * r0[:k] + 1e-6 * r0[0]
    assert np.all(ok), (f"iteration {np.argmax(~ok)}: deviation {(dev / r0[:k])[np.argmax(~ok)]:.3e}, "
                        f"allowed {tol[np.argmax(~ok)]:.3e}")
    # (a sequential Float32 sum of 5e6 squares is itself off by ~2e-3 -- the envelope starts there, at iteration 0.)
    # Against the double-accumulated variant of the oracle the GPU's tree sums must be much closer: same envelope
    # allowance, and in the first iterations (before the recurrence amplifies anything) within 1e-4.
    devA = np.abs(res[:k] - r1[:k]) / np.maximum(r1[:k], 1e-300)
    assert np.all(devA <= tol + 1e-6), devA.max()
    assert devA[:3].max() <= 1e-4, devA[:3]
    ws.free()


@pytest.mark.parametrize("N,p,iters", [(215, 8, BLOCK_ITERS_P8), (127, 32, BLOCK_ITERS_P32)])
def test_block_gmres_benchsize_history_matches_oracle(kb, O, N, p, iters):
    """block_gmres! at the sizes profiles/bench_block.py times: p = 8 on get_div_grad(215) (n = 9 938 375, n = 7 mod 8:
    ragged last tiles of every panel kernel, hundreds of partial Gram blocks per reduction) and p = 32 on
    get_div_grad(127) (n = 2 048 383), a fixed number of block iterations (atol = rtol = 0), seeded random B.
    Iteration count, status and the residual history within 1e-6 of the oracle, X within 1e-6."""
    from krylov_b200 import problems as P
    A = _mat(P.div_grad_csr(N))
    n = N ** 3
    B = np.random.default_rng(N).standard_normal((n, p))
    Xo, so = O.block_gmres(A, B, memory=iters, atol=0.0, rtol=0.0, itmax=iters)
    assert so["niter"] == iters
    ws = kb.BlockGmresWorkspace(n, n, p, memory=iters)
    ws.solve(A, B, atol=0.0, rtol=0.0, itmax=iters, history=True)
    st, X = ws.stats, ws.x
    ws.free()
    assert st.niter == so["niter"] and st.status == so["status"]
    assert len(st.residuals) == len(so["residuals"])
    assert _rel(st.residuals, so["residuals"]).max() <= F64_TOL
    assert np.linalg.norm(X - Xo) <= F64_TOL * np.linalg.norm(Xo)


def test_device_assembled_random_csr_equals_scipy_assembly(kb):
    """bench.py assembles the config-4 matrix on the GPU (only the random draws happen on the host): entry by
    entry equal to problems.random_csr (SciPy COO -> CSR, duplicates summed, + 3 I)."""
    import sys, os
    import torch
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    from krylov_b200 import problems as P
    n = 20_000
    rp, ci, va = P.random_csr(n, 20, seed=1234, dtype=np.float32)
    drp, dci, dva = bench.device_random_csr(torch, torch.device("cuda", 0), n)
    assert np.array_equal(drp.cpu().numpy(), rp) and np.array_equal(dci.cpu().numpy(), ci)
    assert np.array_equal(dva.cpu().numpy(), va)
