"""GPU: the k* primitives (src/krylov_utils.jl:309-349) and the CSR SpMV against the oracle / NumPy.

Vector updates and SpMV are required to be BIT-EXACT (non-contracted mul/add, ascending-column row sums);
dots and norms are tree reductions and are held to 1e-13 (f64) / 1e-5 (f32) relative."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from krylov_b200 import _lib
from krylov_b200 import problems as P

pytestmark = pytest.mark.gpu
DT = {np.float64: _lib.KRYLOV_FLOAT64, np.float32: _lib.KRYLOV_FLOAT32}


class Dev:
    def __init__(self):
        self.L = _lib.lib()
        self.ctx = self.L.kb200_ctx_create(-1)
        assert self.ctx
        self.bufs = []

    def put(self, a):
        a = np.ascontiguousarray(a)
        p = self.L.kb200_alloc(max(a.nbytes, 8))
        assert p
        self.L.kb200_h2d(p, a.ctypes.data_as(C.c_void_p), a.nbytes)
        self.bufs.append(p)
        return p

    def get(self, p, n, dt):
        out = np.empty(n, dt)
        self.L.kb200_sync(self.ctx)
        self.L.kb200_d2h(out.ctypes.data_as(C.c_void_p), p, out.nbytes)
        return out

    def close(self):
        for p in self.bufs:
            self.L.kb200_free(p)
        self.L.kb200_ctx_destroy(self.ctx)


@pytest.fixture()
def dev():
    d = Dev()
    yield d
    d.close()


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("n", [1, 7, 1000, 1 << 20, (1 << 20) + 13])
def test_blas1(dev, dt, n):
    rng = np.random.default_rng(n)
    x, y = rng.standard_normal(n).astype(dt), rng.standard_normal(n).astype(dt)
    L, ctx, d = dev.L, dev.ctx, DT[dt]
    s, t = dt(0.37), dt(-1.25)
    px, py = dev.put(x), dev.put(y)
    r = C.c_double()
    rtol = 1e-13 if dt == np.float64 else 2e-5
    L.kb200_dot(ctx, d, n, px, py, C.byref(r))
    ref = float(np.dot(x.astype(np.float64), y.astype(np.float64)))
    scale = float(np.linalg.norm(x.astype(np.float64)) * np.linalg.norm(y.astype(np.float64)))
    assert abs(r.value - ref) <= rtol * scale
    L.kb200_nrm2(ctx, d, n, px, C.byref(r))
    assert abs(r.value - np.linalg.norm(x.astype(np.float64))) <= rtol * np.linalg.norm(x.astype(np.float64))
    # y += s x  (bit-exact: product rounded, then add)
    L.kb200_axpy(ctx, d, n, float(s), px, py)
    exp = (y + (s * x).astype(dt)).astype(dt)
    assert np.array_equal(dev.get(py, n, dt), exp)
    # y = s x + t y
    L.kb200_axpby(ctx, d, n, float(s), px, float(t), py)
    exp = ((s * x).astype(dt) + (t * exp).astype(dt)).astype(dt)
    assert np.array_equal(dev.get(py, n, dt), exp)
    L.kb200_scal(ctx, d, n, float(t), py)
    exp = (t * exp).astype(dt)
    assert np.array_equal(dev.get(py, n, dt), exp)
    L.kb200_scalcopy(ctx, d, n, py, float(s), px)
    assert np.array_equal(dev.get(py, n, dt), (s * x).astype(dt))
    L.kb200_divcopy(ctx, d, n, py, px, float(s))
    assert np.array_equal(dev.get(py, n, dt), (x / s).astype(dt))
    L.kb200_copy(ctx, d, n, py, px)
    assert np.array_equal(dev.get(py, n, dt), x)
    L.kb200_fill(ctx, d, n, py, 2.5)
    assert np.all(dev.get(py, n, dt) == dt(2.5))
    L.kb200_fill(ctx, d, n, py, 0.0)
    assert np.all(dev.get(py, n, dt) == 0)


def test_dot_is_run_to_run_deterministic(dev):
    n = 3_000_001
    x = np.random.default_rng(1).standard_normal(n)
    px = dev.put(x)
    vals = set()
    r = C.c_double()
    for _ in range(5):
        dev.L.kb200_dot(dev.ctx, _lib.KRYLOV_FLOAT64, n, px, px, C.byref(r))
        vals.add(r.value)
    assert len(vals) == 1


def _spmv_case(dev, O, A, dt, variant, base=0, ibytes=4):
    A = sp.csr_matrix(A).astype(dt)
    A.sort_indices()
    n = A.shape[0]
    x = np.random.default_rng(7).standard_normal(n).astype(dt)
    referenced = np.zeros(n, bool)
    referenced[A.indices] = True
    x[~referenced] = np.nan          # entries no row reads: a gather that is issued but must be discarded (empty rows)
    it = np.int32 if ibytes == 4 else np.int64
    rp, ci = (A.indptr + base).astype(it), (A.indices + base).astype(it)
    va = np.ascontiguousarray(A.data, dtype=dt)
    L = dev.L
    csr = L.kb200_csr_create(dev.ctx, DT[dt], n, A.nnz, rp.ctypes.data_as(C.c_void_p), ci.ctypes.data_as(C.c_void_p),
                             va.ctypes.data_as(C.c_void_p), base, ibytes, 0)
    assert csr, _lib.last_error()
    plan = (C.c_longlong * 7)()
    L.kb200_csr_plan(csr, plan)
    px, py = dev.put(x), dev.put(np.zeros(n, dt))
    if variant == 2 and not plan[3]:
        L.kb200_csr_destroy(csr)
        pytest.skip("tile plan does not fit")
    assert L.kb200_spmv_csr(dev.ctx, csr, px, py, variant) == 0, _lib.last_error()
    y = dev.get(py, n, dt)
    L.kb200_csr_destroy(csr)
    assert np.array_equal(y, O.spmv(A, x, dtype=dt)), "SpMV is not bit-identical to the sequential oracle"
    return plan


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("variant", [1, 2])
def test_spmv_bit_exact_stencils(dev, O, dt, variant):
    # (70, 70, 70): 1340 tiles, several per CTA of the persistent grid (at most 3 CTAs on each of 132 SMs)
    for dims in ((16, 16, 16), (7, 5, 3), (1, 1, 1), (33, 9, 2), (40, 40, 40), (70, 70, 70)):
        rp, ci, va = P.div_grad_csr(*dims, dtype=dt)
        n = len(rp) - 1
        _spmv_case(dev, O, sp.csr_matrix((va, ci, rp), shape=(n, n)), dt, variant)
    rp, ci, va = P.kron_unsymmetric_csr(12, dtype=dt)
    _spmv_case(dev, O, sp.csr_matrix((va, ci, rp), shape=(1728, 1728)), dt, variant)


@pytest.mark.parametrize("variant", [1, 2])
def test_spmv_ragged_rows_and_index_conventions(dev, O, variant):
    rng = np.random.default_rng(3)
    n = 5000
    # empty rows, a few long rows, random pattern
    A = sp.random(n, n, density=0.002, format="lil", random_state=5, dtype=np.float64)
    A[17, :] = 0
    A[4999, :] = 0
    A[100, ::7] = rng.standard_normal(len(range(0, n, 7)))
    A[:, 0] = 0                      # column 0 unreferenced: x[0] is NaN, the gather target of empty rows
    A = sp.csr_matrix(A)
    A.eliminate_zeros()
    _spmv_case(dev, O, A, np.float64, variant)
    # Julia's SparseMatrixCSC{Float64,Int64}: 1-based, 64-bit
    _spmv_case(dev, O, A, np.float64, variant, base=1, ibytes=8)
    _spmv_case(dev, O, A, np.float32, variant, base=1, ibytes=4)
    rp, ci, va = P.random_csr(20000, 20, dtype=np.float32)
    plan = _spmv_case(dev, O, sp.csr_matrix((va, ci, rp), shape=(20000, 20000)), np.float32, variant)
    assert plan[1] >= 20 * 256 * 0.9


def test_spmv_linearity_at_scale(dev):
    """Size-independent property at a benchmark-like size: A(ax) == a(Ax) exactly for a = 2 (power of two)
    and row sums of get_div_grad are 0 in the interior / positive on the boundary."""
    N = 96
    rp, ci, va = P.div_grad_csr(N)
    n = N ** 3
    L = dev.L
    csr = L.kb200_csr_create(dev.ctx, _lib.KRYLOV_FLOAT64, n, len(va), rp.ctypes.data_as(C.c_void_p),
                             ci.ctypes.data_as(C.c_void_p), va.ctypes.data_as(C.c_void_p), 0, 4, 0)
    x = np.random.default_rng(0).standard_normal(n)
    px, p2, py, pz = dev.put(x), dev.put(2 * x), dev.put(np.zeros(n)), dev.put(np.zeros(n))
    for variant in (1, 2):
        L.kb200_spmv_csr(dev.ctx, csr, px, py, variant)
        L.kb200_spmv_csr(dev.ctx, csr, p2, pz, variant)
        y, z = dev.get(py, n, np.float64), dev.get(pz, n, np.float64)
        assert np.array_equal(2 * y, z)
    ones = dev.put(np.ones(n))
    L.kb200_spmv_csr(dev.ctx, csr, ones, py, 0)
    s = dev.get(py, n, np.float64).reshape(N, N, N)
    assert np.all(s[1:-1, 1:-1, 1:-1] == 0) and s.min() >= 0 and s[0, 0, 0] == 3
    L.kb200_csr_destroy(csr)
