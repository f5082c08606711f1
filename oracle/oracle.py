"""ctypes front-end of the CPU oracle -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
reference legs may import this module.  The product (krylov.jl_b200/) never
does.  The solver entry points follow Krylov.jl v0.10.8 (src/cg.jl,
src/gmres.jl, src/bicgstab.jl, src/minres.jl); the problem generators are
literal SciPy transcriptions of test/get_div_grad.jl and test/test_utils.jl.

Parity pinning: scalar helpers + solver end states are checked against the
reference's own known-answer tests (tests/test_oracle_kat.py).  Per-iteration
residual histories on the benchmark configs: parity unpinned (no Julia here).
"""
from __future__ import annotations

import ctypes as C
import glob
import math
import os
import subprocess

import numpy as np
import scipy.sparse as sp

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_SOURCES = "krylov_oracle*.[ch]", "Makefile"    # the one translation unit, every family's header, the recipe
_ITER_CB = C.CFUNCTYPE(C.c_int, C.c_int, C.c_void_p)    # oracle_iter_cb: nonzero stops the solve


class Stats(C.Structure):
    _fields_ = [("niter", C.c_int), ("solved", C.c_int), ("inconsistent", C.c_int),
                ("indefinite", C.c_int), ("npcCount", C.c_int), ("nres", C.c_int),
                ("nAres", C.c_int), ("error", C.c_int), ("status", C.c_char * 96)]


class Opts(C.Structure):
    _fields_ = [("atol", C.c_double), ("rtol", C.c_double), ("itmax", C.c_int), ("history", C.c_int),
                ("radius", C.c_double), ("linesearch", C.c_int), ("lambda_", C.c_double),
                ("etol", C.c_double), ("conlim", C.c_double), ("window", C.c_int), ("memory", C.c_int),
                ("restart", C.c_int), ("reorthogonalization", C.c_int), ("ldiv", C.c_int),
                ("hist_cap", C.c_int)]


def build(force: bool = False) -> str:
    """Compile oracle/libkrylov_oracle.so, every solver family's oracle, with the committed Makefile (when missing or
    older than its sources)."""
    so = os.path.join(_HERE, "libkrylov_oracle.so")
    srcs = [f for pattern in _SOURCES for f in glob.glob(os.path.join(_HERE, pattern))]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", _HERE, "-s"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        for suf in ("f64", "f32"):
            getattr(_LIB, f"oracle_dot_{suf}").restype = C.c_double if suf == "f64" else C.c_float
    return _LIB


def _suf(dtype):
    dtype = np.dtype(dtype)
    if dtype == np.float64:
        return "f64", C.c_double
    if dtype == np.float32:
        return "f32", C.c_float
    raise TypeError(f"oracle supports float32/float64, got {dtype}")


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _csr(A, dtype):
    A = sp.csr_matrix(A)
    A.sort_indices()
    return (A.shape[0], np.ascontiguousarray(A.indptr, dtype=np.int32),
            np.ascontiguousarray(A.indices, dtype=np.int32), np.ascontiguousarray(A.data, dtype=dtype))


def _vec(v, dtype):
    return None if v is None else np.ascontiguousarray(v, dtype=dtype)


def _opts(n, kw, default_hist):
    o = Opts()
    o.atol = kw.pop("atol", math.nan)
    o.rtol = kw.pop("rtol", math.nan)
    o.itmax = kw.pop("itmax", 0)
    o.history = int(kw.pop("history", True))
    o.radius = kw.pop("radius", 0.0)
    o.linesearch = int(kw.pop("linesearch", False))
    o.lambda_ = kw.pop("lambda_", 0.0)
    o.etol = kw.pop("etol", math.nan)
    o.conlim = kw.pop("conlim", math.nan)
    o.window = kw.pop("window", 0)
    o.memory = kw.pop("memory", 0)
    o.restart = int(kw.pop("restart", False))
    o.reorthogonalization = int(kw.pop("reorthogonalization", False))
    o.ldiv = int(kw.pop("ldiv", False))
    itmax = o.itmax if o.itmax > 0 else 2 * n
    o.hist_cap = kw.pop("hist_cap", min(itmax + 2, default_hist))
    if kw:
        raise TypeError(f"unknown options {sorted(kw)}")
    return o


def _result(st, x, res, extra=None):
    out = dict(niter=st.niter, solved=bool(st.solved), inconsistent=bool(st.inconsistent),
               indefinite=bool(st.indefinite), npcCount=st.npcCount, error=st.error,
               status=st.status.decode("utf-8"), residuals=res[:min(st.nres, len(res))].copy())
    if extra:
        out.update(extra)
    return x, out


class dot_mode:
    """with dot_mode(1): ...  -- the oracle's dot products, in every solver family, accumulate in double and round once
    (test knob, krylov_oracle_impl.h: kdot); the default 0 is the restatement's sequential sum in the working precision;
    2 sums in the order of the device's one-CTA reduction tree (n <= 256, NaN beyond)."""

    def __init__(self, mode):
        self.mode = int(mode)

    def __enter__(self):
        lib().oracle_set_dot_mode(self.mode)

    def __exit__(self, *a):
        lib().oracle_set_dot_mode(0)


class precond_block:
    """with precond_block(bs): ...  -- M / N arrays handed to the solvers are read as ceil(n/bs) dense bs x bs diagonal
    blocks (row-major, flattened) instead of a diagonal: the block-Jacobi twin of the product's
    krylov_b200_set_preconditioner_blockdiag (test knob, krylov_oracle_impl.h: bdiagmul)."""

    def __init__(self, bs):
        self.bs = int(bs)

    def __enter__(self):
        lib().oracle_set_precond_block(self.bs)

    def __exit__(self, *a):
        lib().oracle_set_precond_block(0)


def cg(A, b, x0=None, M=None, dtype=np.float64, **kw):
    """cg! (src/cg.jl:120-291).  M: None or the diagonal of a Diagonal preconditioner."""
    suf, _ = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    b, x0, M = _vec(b, dtype), _vec(x0, dtype), _vec(M, dtype)
    o = _opts(n, kw, 1 << 22)
    x = np.zeros(n, dtype)
    res = np.zeros(o.hist_cap, dtype)
    npc = np.zeros(n, dtype)
    st = Stats()
    getattr(lib(), f"oracle_cg_{suf}")(n, _p(rp), _p(ci), _p(va), _p(b), _p(x0), _p(M), C.byref(o),
                                        _p(x), _p(res), _p(npc), C.byref(st))
    return _result(st, x, res, dict(npc_dir=npc))


def bicgstab(A, b, c=None, x0=None, M=None, N=None, dtype=np.float64, **kw):
    """bicgstab! (src/bicgstab.jl:125-277)."""
    suf, _ = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    b, c, x0, M, N = (_vec(v, dtype) for v in (b, c, x0, M, N))
    o = _opts(n, kw, 1 << 22)
    x = np.zeros(n, dtype)
    res = np.zeros(o.hist_cap, dtype)
    st = Stats()
    getattr(lib(), f"oracle_bicgstab_{suf}")(n, _p(rp), _p(ci), _p(va), _p(b), _p(c), _p(x0), _p(M), _p(N),
                                              C.byref(o), _p(x), _p(res), C.byref(st))
    return _result(st, x, res)


def gmres(A, b, x0=None, M=None, N=None, dtype=np.float64, **kw):
    """gmres! (src/gmres.jl:121-384)."""
    suf, _ = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    b, x0, M, N = (_vec(v, dtype) for v in (b, x0, M, N))
    o = _opts(n, kw, 1 << 22)
    x = np.zeros(n, dtype)
    res = np.zeros(o.hist_cap, dtype)
    st = Stats()
    getattr(lib(), f"oracle_gmres_{suf}")(n, _p(rp), _p(ci), _p(va), _p(b), _p(x0), _p(M), _p(N),
                                           C.byref(o), _p(x), _p(res), C.byref(st))
    return _result(st, x, res)


def minres(A, b, x0=None, M=None, dtype=np.float64, **kw):
    """minres! (src/minres.jl:164-485)."""
    suf, _ = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    b, x0, M = _vec(b, dtype), _vec(x0, dtype), _vec(M, dtype)
    o = _opts(n, kw, 1 << 22)
    x = np.zeros(n, dtype)
    res, ares, acond = (np.zeros(o.hist_cap, dtype) for _ in range(3))
    npc = np.zeros(n, dtype)
    st = Stats()
    getattr(lib(), f"oracle_minres_{suf}")(n, _p(rp), _p(ci), _p(va), _p(b), _p(x0), _p(M), C.byref(o),
                                            _p(x), _p(res), _p(ares), _p(acond), _p(npc), C.byref(st))
    k = min(st.nAres, o.hist_cap)
    return _result(st, x, res, dict(Aresiduals=ares[:k].copy(), Acond=acond[:k].copy(), npc_dir=npc))


def cgs(A, b, c=None, x0=None, M=None, N=None, dtype=np.float64, **kw):
    """cgs! (src/cgs.jl:125-282)."""
    suf, _ = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    b, c, x0, M, N = (_vec(v, dtype) for v in (b, c, x0, M, N))
    o = _opts(n, kw, 1 << 22)
    x = np.zeros(n, dtype)
    res = np.zeros(o.hist_cap, dtype)
    st = Stats()
    getattr(lib(), f"oracle_cgs_{suf}")(n, _p(rp), _p(ci), _p(va), _p(b), _p(c), _p(x0), _p(M), _p(N),
                                         C.byref(o), _p(x), _p(res), C.byref(st))
    return _result(st, x, res)


def cg_lanczos(A, b, x0=None, M=None, check_curvature=False, dtype=np.float64, **kw):
    """cg_lanczos! (src/cg_lanczos.jl:110-264).  Extra stats key: Anorm (LanczosStats)."""
    suf, ct = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    b, x0, M = _vec(b, dtype), _vec(x0, dtype), _vec(M, dtype)
    o = _opts(n, kw, 1 << 22)
    x = np.zeros(n, dtype)
    res = np.zeros(o.hist_cap, dtype)
    anorm = ct(0)
    st = Stats()
    getattr(lib(), f"oracle_cg_lanczos_{suf}")(n, _p(rp), _p(ci), _p(va), _p(b), _p(x0), _p(M), int(check_curvature),
                                                C.byref(o), _p(x), _p(res), C.byref(anorm), C.byref(st))
    return _result(st, x, res, dict(Anorm=float(anorm.value)))


def _arnoldi_family(name, A, b, x0, M, N, dtype, kw):
    suf, _ = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    b, x0, M, N = (_vec(v, dtype) for v in (b, x0, M, N))
    o = _opts(n, kw, 1 << 22)
    x = np.zeros(n, dtype)
    res = np.zeros(o.hist_cap, dtype)
    st = Stats()
    getattr(lib(), f"oracle_{name}_{suf}")(n, _p(rp), _p(ci), _p(va), _p(b), _p(x0), _p(M), _p(N),
                                            C.byref(o), _p(x), _p(res), C.byref(st))
    return _result(st, x, res)


def fom(A, b, x0=None, M=None, N=None, dtype=np.float64, **kw):
    """fom! (src/fom.jl:121-368)."""
    return _arnoldi_family("fom", A, b, x0, M, N, dtype, kw)


def fgmres(A, b, x0=None, M=None, N=None, dtype=np.float64, **kw):
    """fgmres! (src/fgmres.jl:128-388); N: None or the diagonal of a fixed right preconditioner."""
    return _arnoldi_family("fgmres", A, b, x0, M, N, dtype, kw)


def dqgmres(A, b, x0=None, M=None, N=None, dtype=np.float64, **kw):
    """dqgmres! (src/dqgmres.jl:121-335)."""
    return _arnoldi_family("dqgmres", A, b, x0, M, N, dtype, kw)


def diom(A, b, x0=None, M=None, N=None, dtype=np.float64, **kw):
    """diom! (src/diom.jl:121-332)."""
    x, st = _arnoldi_family("diom", A, b, x0, M, N, dtype, kw)
    if st["error"]:
        raise ArithmeticError(st["status"])
    return x, st


def cr(A, b, x0=None, M=None, gamma=math.nan, dtype=np.float64, **kw):
    """cr! (src/cr.jl:128-478).  Extra stats keys: Aresiduals, npc_dir."""
    suf, _ = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    b, x0, M = _vec(b, dtype), _vec(x0, dtype), _vec(M, dtype)
    o = _opts(n, kw, 1 << 22)
    x = np.zeros(n, dtype)
    res, ares = np.zeros(o.hist_cap, dtype), np.zeros(o.hist_cap, dtype)
    npc = np.zeros(n, dtype)
    st = Stats()
    f = getattr(lib(), f"oracle_cr_{suf}")
    f.argtypes = [C.c_int] + [C.c_void_p] * 6 + [C.c_double] + [C.c_void_p] * 6
    rc = f(n, _p(rp), _p(ci), _p(va), _p(b), _p(x0), _p(M), float(gamma), C.cast(C.byref(o), C.c_void_p), _p(x), _p(res), _p(ares),
           _p(npc), C.cast(C.byref(st), C.c_void_p))
    if rc:
        raise ArithmeticError({1: "'linesearch' set to 'true' but radius > 0", 2: "warm_start and linesearch cannot be used together",
                               5: "Indefinite system and no trust region"}.get(rc, f"to_boundary error {rc - 10}"))
    k = min(st.nAres, o.hist_cap)
    return _result(st, x, res, dict(Aresiduals=ares[:k].copy(), npc_dir=npc))


def block_gmres(A, B, X0=None, M=None, N=None, dtype=np.float64, **kw):
    """block_gmres! (src/block_gmres.jl:110-359).  B, X0, X: n x p (any layout; converted to column-major)."""
    suf, _ = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    B = np.asfortranarray(B, dtype=dtype)
    p = B.shape[1]
    X0f = None if X0 is None else np.asfortranarray(X0, dtype=dtype)
    M, N = _vec(M, dtype), _vec(N, dtype)
    o = _opts(n, kw, 1 << 22)
    X = np.zeros((n, p), dtype, order="F")
    res = np.zeros(o.hist_cap, dtype)
    st = Stats()
    getattr(lib(), f"oracle_block_gmres_{suf}")(n, p, _p(rp), _p(ci), _p(va), _p(B), _p(X0f), _p(M), _p(N),
                                                 C.byref(o), _p(X), _p(res), C.byref(st))
    return _result(st, X, res)


def householder(Q, compact=False, dtype=np.float64):
    """householder!(Q, R, tau; compact) (src/block_krylov_utils.jl:201-208) -> (Q or reflectors, R, tau)."""
    suf, _ = _suf(dtype)
    Q = np.array(Q, dtype=dtype, order="F")
    m, k = Q.shape
    R = np.zeros((k, k), dtype, order="F")
    tau = np.zeros(k, dtype)
    getattr(lib(), f"oracle_householder_{suf}")(m, k, _p(Q), _p(R), _p(tau), int(compact))
    return Q, R, tau


def cg_timed(rowptr, colind, val, b, iters, threads=1, history=False):
    """Fixed-iteration CG loop on the host (bench.py CPU legs).  Returns (seconds, x, rNorm) and, with
    history=True, a fourth item: the residual norms of iterations 0..iters (bench.py's parity block)."""
    L = lib()
    L.oracle_cg_timed_f64.restype = C.c_double
    n = len(rowptr) - 1
    rowptr = np.ascontiguousarray(rowptr, dtype=np.int32)
    colind = np.ascontiguousarray(colind, dtype=np.int32)
    val = np.ascontiguousarray(val, dtype=np.float64)
    b = np.ascontiguousarray(b, dtype=np.float64)
    x = np.zeros(n)
    rn = C.c_double()
    hist = np.zeros(int(iters) + 1) if history else None
    t = L.oracle_cg_timed_f64(n, _p(rowptr), _p(colind), _p(val), _p(b), int(iters), int(threads), _p(x), C.byref(rn),
                              _p(hist) if history else None)
    if history:
        return float(t), x, rn.value, hist
    return float(t), x, rn.value


def spmv(A, x, dtype=np.float64):
    suf, _ = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    x = _vec(x, dtype)
    y = np.zeros(n, dtype)
    getattr(lib(), f"oracle_spmv_{suf}")(n, _p(rp), _p(ci), _p(va), _p(x), _p(y))
    return y


def dot(x, y, dtype=np.float64):
    suf, _ = _suf(dtype)
    x, y = _vec(x, dtype), _vec(y, dtype)
    return float(getattr(lib(), f"oracle_dot_{suf}")(len(x), _p(x), _p(y)))


def sym_givens(a, b, dtype=np.float64):
    suf, ct = _suf(dtype)
    c, s, r = ct(), ct(), ct()
    getattr(lib(), f"oracle_sym_givens_{suf}")(ct(a), ct(b), C.byref(c), C.byref(s), C.byref(r))
    return c.value, s.value, r.value


def roots_quadratic(q2, q1, q0, nitref=1, dtype=np.float64):
    suf, ct = _suf(dtype)
    r1, r2 = ct(), ct()
    rc = getattr(lib(), f"oracle_roots_quadratic_{suf}")(ct(q2), ct(q1), ct(q0), nitref, C.byref(r1), C.byref(r2))
    if rc:
        raise ArithmeticError("The quadratic `q` doesn't have real roots.")
    return r1.value, r2.value


def to_boundary(x, d, radius, flip=False, xNorm2=0.0, dNorm2=0.0, M=None, ldiv=False, dtype=np.float64):
    suf, ct = _suf(dtype)
    x, d, M = _vec(x, dtype), _vec(d, dtype), _vec(M, dtype)
    z = np.zeros_like(x)
    s1, s2 = ct(), ct()
    rc = getattr(lib(), f"oracle_to_boundary_{suf}")(len(x), _p(x), _p(d), _p(z), ct(radius), int(flip),
                                                     ct(xNorm2), ct(dNorm2), _p(M), int(ldiv),
                                                     C.byref(s1), C.byref(s2))
    if rc:
        raise ArithmeticError({1: "radius must be positive", 2: "zero direction",
                               3: "outside of the trust region"}.get(rc, "no real roots"))
    return s1.value, s2.value


# --------------------------------------------------------------------------
# Problem generators: literal transcriptions of the reference's test helpers.
# --------------------------------------------------------------------------

def eye(n):
    """eye(n) = sparse(I, n, n)  (test/get_div_grad.jl:2)."""
    return sp.identity(n, format="csc")


def ddx(n):
    """1-D staggered-grid difference, n x (n+1)  (test/get_div_grad.jl:21-25)."""
    e = np.ones(n)
    rows = np.concatenate([np.arange(n), np.arange(n)])
    cols = np.concatenate([np.arange(n), np.arange(1, n + 1)])
    return sp.csc_matrix((np.concatenate([-e, e]), (rows, cols)), shape=(n, n + 1))


def get_div_grad(n1, n2, n3):
    """Div * Div'  (test/get_div_grad.jl:8-19) -- literal Kronecker construction."""
    D1 = sp.kron(eye(n3), sp.kron(eye(n2), ddx(n1), format="csc"), format="csc")
    D2 = sp.kron(eye(n3), sp.kron(ddx(n2), eye(n1), format="csc"), format="csc")
    D3 = sp.kron(ddx(n3), sp.kron(eye(n2), eye(n1), format="csc"), format="csc")
    Div = sp.hstack([D1, D2, D3], format="csc")
    A = sp.csr_matrix(Div @ Div.T)
    A.sort_indices()
    return A


def sparse_laplacian(n=16):
    """test/test_utils.jl:153-157"""
    return get_div_grad(n, n, n), np.ones(n ** 3)


def symmetric_definite(n=10):
    """test/test_utils.jl:18-23"""
    A = sp.diags([np.ones(n - 1), 4 * np.ones(n), np.ones(n - 1)], [-1, 0, 1], format="csr")
    return A, A @ np.arange(1, n + 1, dtype=float)


def symmetric_indefinite(n=10, shift=0):
    """test/test_utils.jl:26-31"""
    A = sp.diags([np.ones(n - 1), np.ones(n), np.ones(n - 1)], [-1, 0, 1], format="csr") - shift * sp.identity(n)
    A = sp.csr_matrix(A)
    return A, A @ np.arange(1, n + 1, dtype=float)


def kron_unsymmetric(n=64):
    """test/test_utils.jl:160-169"""
    T = sp.diags([-np.ones(n - 1), 3.0 * np.ones(n), -2.0 * np.ones(n - 1)], [-1, 0, 1], format="csr")
    Id = sp.identity(n, format="csr")
    A = sp.kron(T, Id, format="csr") + sp.kron(Id, T, format="csr")
    Id2 = Id  # the reference re-uses the same n x n identity in the second step
    A = sp.kron(A, Id2, format="csr") + sp.kron(Id2, A, format="csr")
    A = sp.csr_matrix(A)
    A.sort_indices()
    return A, A @ np.ones(A.shape[0])


def almost_singular(n=16):
    """test/test_utils.jl:172-177"""
    A = sp.csr_matrix(get_div_grad(n, n, n) - 5 * sp.identity(n ** 3))
    return A, A @ np.ones(n ** 3)


def cartesian_poisson(n=50, m=50):
    """test/test_utils.jl:294-299 + test/get_div_grad.jl:179-222"""
    dx, dy = 1.0 / (n + 1), 1.0 / (m + 1)
    xs = np.array([i * dx for i in range(1, n + 1)])
    ys = np.array([j * dy for j in range(1, m + 1)])
    A = sp.lil_matrix((n * m, n * m))
    for i in range(n):
        for j in range(m):
            k = i + j * n
            A[k, k] = -2.0 / (dx * dx) - 2.0 / (dy * dy)
            if i >= 1:
                A[k, k - 1] = 1.0 / (dx * dx)
            if i <= n - 2:
                A[k, k + 1] = 1.0 / (dx * dx)
            if j >= 1:
                A[k, k - n] = 1.0 / (dy * dy)
            if j <= m - 2:
                A[k, k + n] = 1.0 / (dy * dy)
    b = np.zeros(n * m)
    for i in range(n):
        for j in range(m):
            b[i + j * n] = -2.0 * math.pi * math.pi * math.sin(math.pi * xs[i]) * math.sin(math.pi * ys[j])
    return sp.csr_matrix(A), b


def square_preconditioned(n=10):
    """test/test_utils.jl:302-307; returns (A, b, diag(M^-1))."""
    A = sp.csr_matrix(np.ones((n, n)) + (n - 1) * np.eye(n))
    return A, 10.0 * np.arange(1, n + 1, dtype=float), np.full(n, 1.0 / n)


def zero_rhs(n=10, seed=0):
    """test/test_utils.jl:319-323 (rand matrix, b = 0)."""
    return sp.csr_matrix(np.random.default_rng(seed).random((n, n))), np.zeros(n)


def square_inconsistent(n=10):
    """test/test_utils.jl (Diagonal(ones) with A[1,1]=0, b=ones)."""
    d = np.ones(n)
    d[0] = 0.0
    A = sp.csr_matrix(sp.diags(d))
    return A, np.ones(n)


def singular_consistent(n=10):
    """test/test_utils.jl:181-186"""
    A = np.array([[float(i * j) for j in range(1, n + 1)] for i in range(1, n + 1)]) + 5 * np.eye(n)
    A[:, 0] = 1.0  # chained broadcast assignment: every target gets one(FC)
    A[:, 1] = 1.0
    A[1, :] = 1.0
    A[0, :] = 1.0
    return sp.csr_matrix(A), A @ np.ones(n)


# ---- more generators of test/test_utils.jl and test/get_div_grad.jl (restated; dense ones returned as CSR) ------
def nonsymmetric_definite(n=10):
    """test/test_utils.jl:72-80 (real case): n on the diagonal, +1 above, -1 below; b = A [1..n]."""
    A = np.where(np.eye(n, dtype=bool), float(n), np.where(np.triu(np.ones((n, n), bool), 1), 1.0, -1.0))
    return sp.csr_matrix(A), A @ np.arange(1.0, n + 1)


def nonsymmetric_indefinite(n=10):
    """test/test_utils.jl:83-91 (real case): diagonal n (-1)^(i j) with 1-based i = j."""
    A = np.where(np.triu(np.ones((n, n), bool), 1), 1.0, -1.0)
    for i in range(1, n + 1):
        A[i - 1, i - 1] = n * (-1.0) ** (i * i)
    return sp.csr_matrix(A), A @ np.arange(1.0, n + 1)


def two_preconditioners(n=10, m=20):
    """test/test_utils.jl:310-316: A = ones + (n-1) I, b = ones, M = I/sqrt(n), N = I/sqrt(m) (as diagonals)."""
    A = np.ones((n, n)) + (n - 1) * np.eye(n)
    return sp.csr_matrix(A), np.ones(n), np.full(n, 1 / math.sqrt(n)), np.full(n, 1 / math.sqrt(m))


def system_zero_quad(n=2):
    """test/test_utils.jl:57-69: diag(1, -1, 0, ...), b = e1 + e2, so that b'Ab = 0."""
    A = np.zeros((n, n)); A[0, 0] = 1.0; A[1, 1] = -1.0
    b = np.zeros(n); b[0] = b[1] = 1.0
    return sp.csr_matrix(A), b


def bc_breakdown():
    """test/test_utils.jl:204-209: b'c = 0."""
    A = sp.csr_matrix(np.array([[1.0, 2.0], [3.0, 4.0]]))
    return A, np.array([0.0, 1.0]), np.array([1.0, 0.0])


def polar_poisson(n=50, m=50):
    """test/get_div_grad.jl:141-176 with f = -3 cos(theta), g = 0 (test/test_utils.jl:286-291), R = 1."""
    R = 1.0
    dr = 2 * R / (2 * n + 1)
    r = [(i - 0.5) * dr for i in range(1, n + 2)]
    dth = 2 * math.pi / m
    th = [(j - 1) * dth for j in range(1, m + 2)]
    lam = np.array([1 / (2 * (k - 0.5)) for k in range(1, n + 1)])
    beta = np.array([1 / ((k - 0.5) ** 2 * dth ** 2) for k in range(1, n + 1)])
    D = sp.diags(beta)
    T = sp.diags([1.0 - lam[1:], -2.0 * np.ones(n), 1.0 + lam[:-1]], [-1, 0, 1])
    A = sp.lil_matrix((n * m, n * m))
    for k in range(m):
        A[k * n:(k + 1) * n, k * n:(k + 1) * n] = (T - 2 * D).toarray()
        if k <= m - 2:
            A[(k + 1) * n:(k + 2) * n, k * n:(k + 1) * n] = D.toarray()
            A[k * n:(k + 1) * n, (k + 1) * n:(k + 2) * n] = D.toarray()
    A[(m - 1) * n:m * n, 0:n] = D.toarray()
    A[0:n, (m - 1) * n:m * n] = D.toarray()
    b = np.zeros(n * m)
    for i in range(n):
        for j in range(m):
            b[i + n * j] = dr * dr * (-3.0 * math.cos(th[j]))
    return sp.csr_matrix(A), b
