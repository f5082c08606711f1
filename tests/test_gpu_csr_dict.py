"""GPU: the constant-coefficient encoding of square CSR operators (CsrDict: at most 8 (column - row, value) pairs,
one mask byte per row) -- which operators it takes, y = A x through it, and the persistent CG kernel on it, which
must reproduce the CSR path bit for bit."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

import krylov_b200 as kb
from krylov_b200 import _lib
from krylov_b200 import problems as P

pytestmark = pytest.mark.gpu


def dict_pairs(A):
    """NumPy restatement of the rule: the distinct (column - row, value bits) pairs, or None when the operator does not
    qualify (not square, more than 8 pairs, or a row whose columns do not ascend strictly)."""
    A = sp.csr_matrix(A)
    if A.shape[0] != A.shape[1]:
        return None
    rows = np.repeat(np.arange(A.shape[0]), np.diff(A.indptr))
    same_row = rows[1:] == rows[:-1]
    if np.any(same_row & (A.indices[1:] <= A.indices[:-1])):
        return None
    bits = A.data.view(np.uint64 if A.data.dtype == np.float64 else np.uint32).astype(np.uint64)
    pairs = set(zip((A.indices - rows).tolist(), bits.tolist()))
    return pairs if 0 < len(pairs) <= 8 else None


def raw_csr(rp, ci, va, n):
    """A CSR object from arrays exactly as given (no sorting, no summing of duplicates)."""
    ctx = _lib.lib().kb200_ctx_create(-1)
    rp, ci, va = (np.ascontiguousarray(a) for a in (rp.astype(np.int32), ci.astype(np.int32), va))
    h = _lib.lib().kb200_csr_create(ctx, _lib.KRYLOV_FLOAT64 if va.dtype == np.float64 else _lib.KRYLOV_FLOAT32, n, len(va),
                                    rp.ctypes.data_as(C.c_void_p), ci.ctypes.data_as(C.c_void_p), va.ctypes.data_as(C.c_void_p),
                                    0, 4, 0)
    assert h, _lib.last_error()
    return kb.CsrOperator(h, ctx, va.dtype)


def encoded(op):
    npairs = C.c_int(-1)
    rc = _lib.lib().kb200_csr_dict(op._csr, C.byref(npairs))
    assert rc in (0, 1) and (rc == 1) == (npairs.value > 0)
    return npairs.value


def stencil(dims, dtype=np.float64):
    rp, ci, va = P.div_grad_csr(*dims, dtype=dtype)
    n = int(np.prod(dims))
    return sp.csr_matrix((va, ci, rp), shape=(n, n))


def kron_unsymmetric(N):
    rp, ci, va = P.kron_unsymmetric_csr(N)
    return sp.csr_matrix((va, ci, rp), shape=(N ** 3, N ** 3))


def signed_zeros(n=1000):
    """Stored 0.0 below and -0.0 above the diagonal, every 17th row empty: three pairs."""
    rows, cols, vals = [], [], []
    for i in range(n):
        if i % 17 == 3:
            continue
        for off, v in ((-1, 0.0), (0, 2.0), (1, -0.0)):
            if 0 <= i + off < n:
                rows.append(i); cols.append(i + off); vals.append(v)
    A = sp.csr_matrix((np.array(vals), (rows, cols)), shape=(n, n))
    assert A.nnz == len(vals)                             # the explicit zeros are stored
    return A


ENCODED = {
    "div_grad_1x1x1": lambda: stencil((1, 1, 1)),
    "div_grad_7x5x3": lambda: stencil((7, 5, 3)),
    "div_grad_33x9x2": lambda: stencil((33, 9, 2)),
    "div_grad_70x70x70": lambda: stencil((70, 70, 70)),            # several tiles per CTA
    "kron_unsymmetric_9": lambda: kron_unsymmetric(9),
    "div_grad_f32": lambda: stencil((11, 6, 5), np.float32),
    "signed_zeros": signed_zeros,
}


@pytest.mark.parametrize("name", sorted(ENCODED))
def test_encoding_detected(name):
    A = ENCODED[name]()
    want = dict_pairs(A)
    assert want is not None
    op = raw_csr(A.indptr, A.indices, A.data, A.shape[0])
    try:
        assert encoded(op) == len(want)
        assert len(want) == {"div_grad_1x1x1": 1, "signed_zeros": 3}.get(name, 7)
    finally:
        op.free()


def test_not_encoded():
    n = 300
    A = stencil((10, 6, 5))
    cases = {"non-constant diagonal": A + sp.diags(np.linspace(0.0, 1.0, n)),
             "nine pairs": A + sp.diags([np.full(n - 7, 0.5), np.full(n - 8, 0.25)], [7, 8])}
    for what, M in cases.items():
        assert dict_pairs(M) is None, what
        op = kb.CsrOperator.from_scipy(M)
        assert encoded(op) == 0, what
        op.free()
    # unsorted row: row 1 holds columns (2, 0)
    rp, ci, va = np.array([0, 1, 3, 4]), np.array([0, 2, 0, 2]), np.array([1.0, 1.0, 1.0, 1.0])
    op = raw_csr(rp, ci, va, 3)
    assert encoded(op) == 0
    op.free()
    # rectangular operators keep the CSR path
    op = kb.CsrOperator.from_scipy(sp.csr_matrix(np.ones((3, 4))))
    assert encoded(op) == 0
    op.free()


def test_signed_zeros_are_distinct_pairs():
    """0.0 and -0.0 are different pairs: a dictionary that merged them would hold 2."""
    A = signed_zeros()
    assert len({v for _, v in dict_pairs(A)}) == 3


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["div_grad_7x5x3", "div_grad_33x9x2", "kron_unsymmetric_9", "signed_zeros"])
def test_spmv_variant3_bit_identical(O, dt, name):
    A = ENCODED[name]()
    A = sp.csr_matrix(A).astype(dt)
    A.sort_indices()
    n = A.shape[0]
    x = np.random.default_rng(3).standard_normal(n).astype(dt)
    read = np.zeros(n, bool)
    read[A.indices] = True
    x[~read] = np.nan                                    # a masked slot whose value leaked would poison its row
    op = raw_csr(A.indptr, A.indices, A.data, n)
    L = _lib.lib()
    try:
        assert encoded(op) > 0
        px, py = L.kb200_alloc(x.nbytes), L.kb200_alloc(x.nbytes)
        L.kb200_h2d(px, x.ctypes.data_as(C.c_void_p), x.nbytes)
        assert L.kb200_spmv_csr(op._ctx, op._csr, px, py, 3) == 0, _lib.last_error()
        y = np.empty(n, dt)
        L.kb200_sync(op._ctx)
        L.kb200_d2h(y.ctypes.data_as(C.c_void_p), py, y.nbytes)
        L.kb200_free(px); L.kb200_free(py)
        assert np.array_equal(y.view(np.uint8), O.spmv(A, x, dtype=dt).view(np.uint8)), "variant 3 differs from the oracle"
    finally:
        op.free()


def test_spmv_variant3_refuses_unencoded():
    op = kb.CsrOperator.from_scipy(stencil((4, 4, 4)) + sp.diags(np.linspace(0.0, 1.0, 64)))
    L = _lib.lib()
    p = L.kb200_alloc(64 * 8)
    try:
        assert L.kb200_spmv_csr(op._ctx, op._csr, p, p, 3) == -1
        assert "encoding" in _lib.last_error()
    finally:
        L.kb200_free(p)
        op.free()


def _cg_outputs(A, b, dict_on, monkeypatch, **kw):
    monkeypatch.setenv("KB200_CSR_DICT", "1" if dict_on else "0")
    op = kb.CsrOperator.from_scipy(A, dtype=b.dtype)
    monkeypatch.delenv("KB200_CSR_DICT")
    assert (encoded(op) > 0) == dict_on
    ws = kb.krylov_workspace("cg", A.shape[0], A.shape[0], b.dtype)
    try:
        ws.solve(op, b, history=True, **kw)
        st = ws.stats
        return dict(x=np.ascontiguousarray(ws.x).tobytes(), niter=st.niter, status=st.status, solved=st.solved,
                    inconsistent=st.inconsistent, residuals=[float(v).hex() for v in st.residuals], launches=ws.launches)
    finally:
        ws.free()
        op.free()


CG_CASES = {
    "one_batch": dict(dims=(20, 17, 9), kw=dict(itmax=20, atol=0.0, rtol=0.0)),
    "across_batches": dict(dims=(33, 9, 2), kw=dict(itmax=150, atol=0.0, rtol=0.0)),
    "rtol_exit_mid_batch": dict(dims=(40, 40, 40), kw=dict(rtol=1e-6)),
    "jacobi": dict(dims=(30, 20, 10), kw=dict(itmax=100, atol=0.0, rtol=0.0), M=True),
    "float32": dict(dims=(30, 20, 10), kw=dict(rtol=1e-4), dtype=np.float32),
    "float32_jacobi": dict(dims=(30, 20, 10), kw=dict(rtol=1e-4), dtype=np.float32, M=True),
    "several_tiles_per_cta": dict(dims=(70, 70, 70), kw=dict(itmax=70, atol=0.0, rtol=0.0)),
}


@pytest.mark.parametrize("case", sorted(CG_CASES))
def test_persistent_cg_bit_identical_to_csr(case, monkeypatch):
    c = CG_CASES[case]
    dt = c.get("dtype", np.float64)
    A = stencil(c["dims"], dt)
    n = A.shape[0]
    b = np.random.default_rng(11).standard_normal(n).astype(dt)
    kw = dict(c["kw"])
    if c.get("M"):
        kw["M"] = (1.0 / np.linspace(5.0, 7.0, n)).astype(dt)    # Diagonal M, applied inside the kernel
    on = _cg_outputs(A, b, True, monkeypatch, **kw)
    off = _cg_outputs(A, b, False, monkeypatch, **kw)
    assert on["niter"] > 0
    if case == "rtol_exit_mid_batch":
        assert on["solved"] and on["niter"] % 32 != 0
    assert on == off
