"""Shared cases of the Krylov-process tests (tests/test_oracle_processes.py on the CPU oracle, tests/test_gpu_processes.py on
the GPU): the seeded problems of the reference's test/test_processes.jl (m = 250, n = 500, k = 20, s = 5, real case) and
its identities, written for dense NumPy outputs."""
import numpy as np
import scipy.sparse as sp

M, N, K, S = 250, 500, 20, 5


def approx(x, y, rtol=None):
    """Julia's x ≈ y for arrays: ‖x - y‖ ≤ √eps · max(‖x‖, ‖y‖)."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    rtol = rtol if rtol is not None else np.sqrt(np.finfo(np.float64).eps)
    return np.linalg.norm(x - y) <= rtol * max(np.linalg.norm(x), np.linalg.norm(y))


def problems(seed=0, m=M, n=N):
    """name -> (A as CSR, b, c) with rand(n, n) / rand(m, n) matrices as the reference draws them."""
    r = np.random.default_rng(seed)
    B = r.random((n, n))
    return {"hermitian_lanczos": (sp.csr_matrix(B.T @ B), r.random(n), None),
            "arnoldi": (sp.csr_matrix(r.random((n, n))), r.random(n), None),
            "nonhermitian_lanczos": (sp.csr_matrix(r.random((n, n))), r.random(n), r.random(n)),
            "golub_kahan": (sp.csr_matrix(r.random((m, n))), r.random(m), None),
            "saunders_simon_yip": (sp.csr_matrix(r.random((m, n))), r.random(m), r.random(n))}


def dense(x):
    return x.toarray() if sp.issparse(x) else np.asarray(x)


def check_identities(name, A, b, c, out, k=K, s=S, rtol=None, orth=1e-4):
    """The real-case assertions of test/test_processes.jl for one process's outputs (coefficients as dense or sparse)."""
    A = dense(A).astype(np.float64)
    I = np.eye(s)
    if name in ("hermitian_lanczos", "arnoldi"):
        V, beta, T = out
        V, T = np.asarray(V, np.float64), dense(T)
        assert np.linalg.norm(V[:, :s].T @ V[:, :s] - I) <= orth
        assert approx(beta * V[:, 0], b, rtol)
        assert approx(A @ V[:, :k], V @ T, rtol)
    elif name == "golub_kahan":
        V, U, beta, L = out
        V, U, L = np.asarray(V, np.float64), np.asarray(U, np.float64), dense(L)
        B = L[:k + 1, :k]
        assert np.linalg.norm(V[:, :s].T @ V[:, :s] - I) <= orth
        assert np.linalg.norm(U[:, :s].T @ U[:, :s] - I) <= orth
        assert approx(beta * U[:, 0], b, rtol)
        assert approx(A @ V[:, :k], U @ B, rtol)
        assert approx(A.T @ U, V @ L.T, rtol)
        assert approx(A.T @ A @ V[:, :k], V @ L.T @ B, rtol)
        assert approx(A @ A.T @ U[:, :k], U @ B @ L[:k, :k].T, rtol)
    else:
        V, beta, T, U, gamma, Th = out
        V, U, T, Th = np.asarray(V, np.float64), np.asarray(U, np.float64), dense(T), dense(Th)
        if name == "nonhermitian_lanczos":
            assert np.linalg.norm(V[:, :s].T @ U[:, :s] - I) <= orth
            assert np.linalg.norm(U[:, :s].T @ V[:, :s] - I) <= orth
            assert approx(A @ V[:, :k], V @ T, rtol)
            assert approx(A.T @ U[:, :k], U @ Th, rtol)
        else:
            assert np.linalg.norm(V[:, :s].T @ V[:, :s] - I) <= orth
            assert np.linalg.norm(U[:, :s].T @ U[:, :s] - I) <= orth
            assert approx(A @ U[:, :k], V @ T, rtol)
            assert approx(A.T @ V[:, :k], U @ Th, rtol)
            assert approx(A.T @ A @ U[:, :k - 1], U @ Th @ T[:k, :k - 1], rtol)
            assert approx(A @ A.T @ V[:, :k - 1], V @ T @ Th[:k, :k - 1], rtol)
        assert approx(beta * V[:, 0], b, rtol)
        assert approx(gamma * U[:, 0], c, rtol)
        assert approx(T[:k, :k], Th[:k, :k].T, rtol)


def path3(n=6):
    """Exact breakdown in exact arithmetic that floating point reproduces: the path graph on e₁, e₂, e₃ (entries 0 and 1)
    next to a diagonal block, with b = c = e₁.  Every product, dot and division is exact, so the Krylov space closes
    exactly: Lanczos, Arnoldi, non-Hermitian Lanczos and SSY meet a zero coefficient at iteration 3, Golub-Kahan its
    αᵢ₊₁ at iteration 1."""
    A = np.zeros((n, n))
    A[0, 1] = A[1, 0] = A[1, 2] = A[2, 1] = 1.0
    for j in range(3, n):
        A[j, j] = float(j)
    e1 = np.zeros(n)
    e1[0] = 1.0
    return sp.csr_matrix(A), e1
