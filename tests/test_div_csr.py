"""CPU: problems.div_csr(N), the divergence of the N³ grid assembled in closed form, equals grad_csr(N).T entry by
entry, column order included, with NumPy and with torch (on the CPU here; the benchmark assembles it on the GPU)."""
import numpy as np
import pytest
import scipy.sparse as sp

from krylov_b200.problems import div_csr, grad_csr


@pytest.mark.parametrize("N", [2, 3, 4, 7])
def test_div_is_the_transpose_of_grad(N):
    rp, ci, va = grad_csr(N)
    G = sp.csr_matrix((va, ci, rp), shape=(len(rp) - 1, N ** 3))
    T = G.T.tocsr()
    T.sort_indices()
    r, c, v = div_csr(N)
    assert r.dtype == np.int32 and c.dtype == np.int32
    np.testing.assert_array_equal(r, T.indptr)
    np.testing.assert_array_equal(c, T.indices)
    np.testing.assert_array_equal(v, T.data)
    torch = pytest.importorskip("torch")
    r2, c2, v2 = div_csr(N, xp=torch, device="cpu")
    np.testing.assert_array_equal(r2.numpy(), r)
    np.testing.assert_array_equal(c2.numpy(), c)
    np.testing.assert_array_equal(v2.numpy(), v)
