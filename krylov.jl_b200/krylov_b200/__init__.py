"""krylov_b200 -- host-side mirror of Krylov.jl's workspace/solver API for the
H100 path, over the C ABI of libkrylov_b200.so.

Names and argument meanings follow the reference (src/interface.jl:67-246,
src/krylov_workspaces.jl, src/workspace_accessors.jl:140-204):

    ws = CgWorkspace(A, b)            # or krylov_workspace("cg", A, b)
    cg_(ws, A, b; atol, rtol, ...)    # Julia's cg!(ws, A, b; ...)
    x, stats = cg(A, b, ...)          # out-of-place
    solution(ws), statistics(ws), issolved(ws), iteration_count(ws), warm_start_(ws, x0)

`A` is a scipy.sparse matrix (or anything scipy can turn into CSR) that is
uploaded once into HBM as int32/0-based CSR, or a Python callable
`A(x_host) -> y_host` (matrix-free, staged through pinned memory like the
reference's C callback operator).  `b`, `x0`, `c` are NumPy arrays (host) or
torch CUDA tensors (device; zero-copy).  All arithmetic runs in the CUDA
library; this module contains no numerical code.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from . import _lib
from ._lib import (KRYLOV_CPU, KRYLOV_CUDA, KRYLOV_FLOAT32, KRYLOV_FLOAT64, SOLVER_IDS, KrylovB200Options,
                   KrylovB200Stats, KrylovOptions, KrylovWorkspaceOptions, lib)

__all__ = ["KrylovWorkspace", "SimpleStats", "AdjointStats", "B200Error", "CsrOperator", "BlockGmresWorkspace",
           "block_gmres", "block_gmres_", "krylov_workspace", "krylov_solve", "krylov_solve_", "solution", "statistics",
           "results", "issolved", "iteration_count", "elapsed_time", "Aprod_count", "warm_start_", "device_count"]
# the workspace class, solver! and solver of every row of _SOLVERS are added where they are made


class B200Error(RuntimeError):
    """Raised where the reference raises ErrorException (status -1 from the C ABI)."""


@dataclass
class SimpleStats:
    """src/krylov_stats.jl:24-36"""
    niter: int = 0
    solved: bool = False
    inconsistent: bool = False
    indefinite: bool = False
    npcCount: int = 0
    residuals: list = field(default_factory=list)
    Aresiduals: list = field(default_factory=list)
    Acond: list = field(default_factory=list)
    allocation_timer: float = 0.0
    timer: float = 0.0
    status: str = "unknown"
    Anorm: float = math.nan          # LanczosStats (src/krylov_stats.jl), cg_lanczos! only


@dataclass
class AdjointStats:
    """src/krylov_stats.jl:263-280: the statistics of bilqr! / trilqr!; `solved` is solved_primal and solved_dual."""
    niter: int = 0
    solved_primal: bool = False
    solved_dual: bool = False
    residuals_primal: list = field(default_factory=list)
    residuals_dual: list = field(default_factory=list)
    timer: float = 0.0
    status: str = "unknown"

    @property
    def solved(self) -> bool:
        return self.solved_primal and self.solved_dual


def device_count() -> int:
    return lib().krylov_b200_device_count()


def _dtype_id(dtype) -> int:
    dtype = np.dtype(dtype)
    if dtype == np.float64:
        return KRYLOV_FLOAT64
    if dtype == np.float32:
        return KRYLOV_FLOAT32
    raise B200Error(f"unsupported element type {dtype} (Float32/Float64 only on this path)")


def _is_torch(x) -> bool:
    return type(x).__module__.startswith("torch")


def _ptr(a):
    """(pointer, keepalive) of a NumPy array or torch tensor; None -> NULL."""
    if a is None:
        return None, None
    if _is_torch(a):
        a = a.contiguous()
        return C.c_void_p(a.data_ptr()), a
    return a.ctypes.data_as(C.c_void_p), a


_KEYWORDS = {   # solve keyword -> (the option struct it travels in, its field there, conversion)
    **{k: (KrylovOptions, k, float) for k in ("atol", "rtol", "lambda_", "radius")},
    **{k: (KrylovOptions, k, int) for k in ("itmax", "verbose", "restart", "reorthogonalization", "linesearch")},
    "timemax": (KrylovOptions, "timemax", lambda t: math.nan if math.isinf(t) else float(t)),
    **{k: (KrylovB200Options, k, float) for k in ("etol", "conlim", "axtol", "btol", "sigma", "utol")},
    **{k: (KrylovB200Options, k, int) for k in ("history", "ldiv", "fused", "batch", "time_kernels", "check_curvature",
                                                "transfer_to_lsqr", "transfer_to_bicg")},
    "gamma": (KrylovB200Options, "cr_gamma", float),
    "artol": (KrylovB200Options, "axtol", float),                  # MINARES's Artol
    "utolx": (KrylovB200Options, "utol", float),                   # LNLQ's tolerances on its error bounds
    "utoly": (KrylovB200Options, "etol", float),
    "transfer_to_craig": (KrylovB200Options, "transfer_to_bicg", int),     # LNLQ
    "transfer_to_usymcg": (KrylovB200Options, "transfer_to_bicg", int),    # TriLQR
}


def _options(kw, defaults):
    """The KrylovOptions / KrylovB200Options pair of one solve from its option keywords.  None keeps the library's
    default for atol, rtol and the keywords whose default is None."""
    o, e = lib().krylov_default_options(), lib().krylov_b200_default_options()
    for name, val in kw.items():
        if val is None and (name in ("atol", "rtol") or defaults.get(name) is None):
            continue
        struct, field_, conv = _KEYWORDS[name]
        setattr(o if struct is KrylovOptions else e, field_, conv(val))
    return o, e


class CsrOperator:
    """A CSR operator resident in HBM, independent of any workspace (SURVEY.md 8f-4):

        A = CsrOperator.read_mtx("bcsstk01.mtx")     # Matrix Market ingestion (benchmark/benchmarks.jl:23-33)
        At = A.transpose()                           # A^T = A^H for the real types of this path
        kb.cg(A, b)                                  # solvers accept it like a SciPy matrix
        G = CsrOperator.from_scipy(G_mn)             # rectangular (m, n): kb.lsqr(G, b), kb.lsmr(G, b)
    """

    def __init__(self, csr_handle, ctx, dtype, owns_ctx=True):
        self._csr, self._ctx, self.dtype, self._owns_ctx = csr_handle, ctx, np.dtype(dtype), owns_ctx
        m, n, nnz = C.c_int(), C.c_int(), C.c_longlong()
        lib().kb200_csr_shape(self._csr, C.byref(m), C.byref(n), C.byref(nnz))
        self.shape, self.nnz = (m.value, n.value), nnz.value

    @classmethod
    def read_mtx(cls, path, dtype=np.float64, device: int = -1):
        ctx = lib().kb200_ctx_create(device)
        if not ctx:
            raise B200Error(_lib.last_error())
        h = lib().kb200_csr_read_mtx(ctx, os.fsencode(path), _dtype_id(dtype))
        if not h:
            lib().kb200_ctx_destroy(ctx)
            raise B200Error(_lib.last_error())
        return cls(h, ctx, dtype)

    @classmethod
    def from_scipy(cls, A, dtype=None, device: int = -1):
        import scipy.sparse as sp
        M = sp.csr_matrix(A)
        M.sort_indices()
        dtype = np.dtype(dtype or M.dtype)
        ctx = lib().kb200_ctx_create(device)
        rp, ci, va = np.ascontiguousarray(M.indptr), np.ascontiguousarray(M.indices), np.ascontiguousarray(M.data, dtype=dtype)
        ci = ci.astype(rp.dtype)
        args = (int(M.nnz), rp.ctypes.data_as(C.c_void_p), ci.ctypes.data_as(C.c_void_p), va.ctypes.data_as(C.c_void_p), 0,
                rp.dtype.itemsize, 0)
        if M.shape[0] == M.shape[1]:
            h = lib().kb200_csr_create(ctx, _dtype_id(dtype), M.shape[0], *args)
        else:
            h = lib().kb200_csr_create_rect(ctx, _dtype_id(dtype), M.shape[0], M.shape[1], *args)
        if not h:
            lib().kb200_ctx_destroy(ctx)
            raise B200Error(_lib.last_error())
        return cls(h, ctx, dtype)

    def transpose(self):
        h = lib().kb200_csr_transpose(self._ctx, self._csr)
        if not h:
            raise B200Error(_lib.last_error())
        out = CsrOperator(h, self._ctx, self.dtype, owns_ctx=False)
        out._parent = self                       # shares (and keeps alive) the context
        return out

    T = property(transpose)

    def to_scipy(self):
        import scipy.sparse as sp
        n = self.shape[0]
        rp, ci, va = np.empty(n + 1, np.int32), np.empty(self.nnz, np.int32), np.empty(self.nnz, self.dtype)
        if lib().kb200_csr_download(self._ctx, self._csr, rp.ctypes.data_as(C.c_void_p), ci.ctypes.data_as(C.c_void_p),
                                    va.ctypes.data_as(C.c_void_p)) != 0:
            raise B200Error(_lib.last_error())
        return sp.csr_matrix((va, ci, rp), shape=self.shape)

    def matvec(self, x):
        """y = A x on the GPU (host arrays in and out)."""
        x = np.ascontiguousarray(x, dtype=self.dtype)
        if x.shape[0] != self.shape[1]:
            raise B200Error(f"x has {x.shape[0]} entries, the operator {self.shape[1]} columns")
        n = self.shape[0]
        L = lib()
        dx, dy = L.kb200_alloc(x.nbytes), L.kb200_alloc(n * self.dtype.itemsize)
        try:
            L.kb200_h2d(dx, x.ctypes.data_as(C.c_void_p), x.nbytes)
            if L.kb200_spmv_csr(self._ctx, self._csr, dx, dy, 0) != 0 or L.kb200_sync(self._ctx) != 0:
                raise B200Error(_lib.last_error())
            y = np.empty(n, self.dtype)
            L.kb200_d2h(y.ctypes.data_as(C.c_void_p), dy, y.nbytes)
            return y
        finally:
            L.kb200_free(dx)
            L.kb200_free(dy)

    def free(self):
        if getattr(self, "_csr", None):
            lib().kb200_csr_destroy(self._csr)
            self._csr = None
            if self._owns_ctx and self._ctx:
                lib().kb200_ctx_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class KrylovWorkspace:
    """One workspace = all device vectors of one solver (krylov_workspaces.jl)."""

    solver = ""
    nA = 1  # operator products per iteration (workspace_accessors.jl:101-139)

    def __init__(self, m_or_A, n_or_b=None, dtype=None, *, memory: int = 0, window: int = 0, device: str = "host",
                 solver: Optional[str] = None):
        if solver:
            self.solver = solver
        A = None
        if hasattr(m_or_A, "shape") and not isinstance(m_or_A, (int, np.integer)):   # (A, b) constructor
            A, b = m_or_A, n_or_b
            m, n = A.shape
            if dtype is None:
                dtype = (b.cpu().numpy().dtype if _is_torch(b) else np.asarray(b).dtype) if b is not None else A.dtype
            if b is not None and _is_torch(b):
                device = "cuda"
        else:
            m, n = int(m_or_A), int(n_or_b)
            dtype = dtype or np.float64
        self.m, self.n = int(m), int(n)
        self.dtype = np.dtype(dtype)
        self.device = device
        self._keep = []
        self._cb = None
        self._h = C.c_void_p()
        w = KrylovWorkspaceOptions(memory, window)
        rc = lib().krylov_workspace_create(SOLVER_IDS[self.solver], self.m, self.n, _dtype_id(self.dtype),
                                           KRYLOV_CUDA if device == "cuda" else KRYLOV_CPU, C.byref(w), C.byref(self._h))
        if rc != 0:
            raise B200Error(f"krylov_workspace_create({self.solver}) -> {rc}: {_lib.last_error()}")
        self._ext = lib().krylov_b200_default_options()
        self._op_id = None
        if A is not None and not callable(A):
            self.set_operator(A)

    # -- lifetime -----------------------------------------------------------
    def free(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            lib().krylov_workspace_free(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    def _order_after(self, *arrays):
        """Stream contract of device inputs (include/krylov_b200.h): torch tensors are produced on torch's current
        stream, the library works on its own non-blocking stream -- make the latter wait for the former."""
        for a in arrays:
            if a is not None and _is_torch(a) and a.is_cuda:
                import torch
                s = torch.cuda.current_stream(a.device)
                if lib().krylov_b200_wait_stream(self._h, C.c_void_p(s.cuda_stream)) != 0:
                    raise B200Error(_lib.last_error())
                return

    # -- operator -----------------------------------------------------------
    def set_operator(self, A):
        """Upload A as the device-resident CSR operator (krylov_b200_set_operator_csr)."""
        if id(A) == self._op_id:
            return
        if isinstance(A, CsrOperator):  # a device-resident operator (Matrix Market file, transposed operator, ...)
            if A.shape != (self.m, self.n):
                raise B200Error(f"(workspace.m, workspace.n) = ({self.m}, {self.n}) is inconsistent with size(A) = {A.shape}")
            if lib().krylov_b200_attach_csr(self._h, A._csr) != 0:
                raise B200Error(_lib.last_error())
            self._keep.append(A)
            self._op_id = id(A)
            return
        if isinstance(A, tuple):        # (rowptr, colind, values[, index_base]) NumPy or torch
            rp, ci, va = A[:3]
            base = A[3] if len(A) > 3 else 0
            loc = 1 if _is_torch(va) else 0
            if loc:
                ib = rp.element_size()
                nnz = int(va.numel())
            else:
                rp = np.ascontiguousarray(rp)
                ci = np.ascontiguousarray(ci, dtype=rp.dtype)
                va = np.ascontiguousarray(va, dtype=self.dtype)
                ib = rp.dtype.itemsize
                nnz = int(va.shape[0])
            n = int(rp.shape[0]) - 1
        else:
            import scipy.sparse as sp
            M = sp.csr_matrix(A)
            M.sort_indices()
            if M.shape != (self.m, self.n):
                raise B200Error(f"(workspace.m, workspace.n) = ({self.m}, {self.n}) is inconsistent with size(A) = {M.shape}")
            rp = np.ascontiguousarray(M.indptr)
            ci = np.ascontiguousarray(M.indices, dtype=rp.dtype)
            va = np.ascontiguousarray(M.data, dtype=self.dtype)
            ib, base, loc, nnz, n = rp.dtype.itemsize, 0, 0, int(M.nnz), M.shape[0]
        p_rp, k1 = _ptr(rp)
        p_ci, k2 = _ptr(ci)
        p_va, k3 = _ptr(va)
        self._order_after(va)
        rc = lib().krylov_b200_set_operator_csr(self._h, n, nnz, p_rp, p_ci, p_va, int(base), int(ib), loc)
        if rc != 0:
            raise B200Error(_lib.last_error())
        self._op_id = id(A)

    def share_operator(self, other: "KrylovWorkspace"):
        if lib().krylov_b200_share_operator(self._h, other._h) != 0:
            raise B200Error(_lib.last_error())
        self._op_id = other._op_id

    def _set_diag(self, which: int, d):
        attached = getattr(self, "_precond_attached", None)
        if attached is None:
            attached = self._precond_attached = [False, False]
        if d is None:
            if not attached[which]:             # nothing to detach: no library call on the per-solve path
                return
            lib().krylov_b200_set_preconditioner_diag(self._h, which, None, 0)
            if not isinstance(self, BlockGmresWorkspace):
                lib().krylov_b200_set_preconditioner_blockdiag(self._h, which, 0, None, 0)
            attached[which] = False
            return
        attached[which] = True
        if getattr(d, "ndim", 1) == 3:      # block-Jacobi: (nblocks, bs, bs) dense diagonal blocks (SURVEY.md 8f-1)
            nb, bs, bs2 = d.shape
            if bs != bs2 or nb != (self.n + bs - 1) // bs:
                raise B200Error(f"block-diagonal preconditioner: expected ({(self.n + bs - 1) // bs}, {bs}, {bs}) blocks, got {tuple(d.shape)}")
            if not _is_torch(d):
                d = np.ascontiguousarray(d, dtype=self.dtype)
            p, keep = _ptr(d)
            self._order_after(d)
            lib().krylov_b200_set_preconditioner_diag(self._h, which, None, 0)
            if lib().krylov_b200_set_preconditioner_blockdiag(self._h, which, int(bs), p, 1 if _is_torch(d) else 0) != 0:
                raise B200Error(_lib.last_error())
            return
        if not isinstance(self, BlockGmresWorkspace):
            lib().krylov_b200_set_preconditioner_blockdiag(self._h, which, 0, None, 0)
        if not _is_torch(d):
            d = np.ascontiguousarray(d, dtype=self.dtype)
        p, keep = _ptr(d)
        self._order_after(d)
        if lib().krylov_b200_set_preconditioner_diag(self._h, which, p, 1 if _is_torch(d) else 0) != 0:
            raise B200Error(_lib.last_error())

    # -- solve --------------------------------------------------------------
    def _wrap(self, f, nin, nout):
        """Host callback y = f(x) with len(x) = nin and len(y) = nout (staged through pinned memory)."""
        if self.device == "cuda":
            raise B200Error("Python callables are host operators; create the workspace with device='host'")
        dt = self.dtype

        def tramp(xp, yp, _ud):
            x = np.ctypeslib.as_array(C.cast(xp, C.POINTER(C.c_byte)), shape=(nin * dt.itemsize,)).view(dt)
            y = np.ctypeslib.as_array(C.cast(yp, C.POINTER(C.c_byte)), shape=(nout * dt.itemsize,)).view(dt)
            y[:] = f(x)
        return _lib.MATVEC(tramp)

    @property
    def _row(self) -> Optional["_Solver"]:
        return _SOLVERS.get(self.solver)

    def solve(self, A, b, *args, **kw):
        """solver!(ws, A, b; kwargs...), and bilqr! / trilqr!(ws, A, b, c; kwargs...): the keywords and defaults are
        listed in help() of the workspace class.  A: a SciPy matrix, a CsrOperator or a (rowptr, colind, values)
        tuple (uploaded as a CSR operator); or host callables: A itself for the solvers that do not apply A^T, a
        scipy.sparse.linalg.LinearOperator or a (matvec, rmatvec) pair for those that do.  M / N: None (identity), a
        1-D array (Diagonal preconditioner), a host callable, or, for the solvers that do not apply A^T, the
        (nblocks, bs, bs) diagonal blocks of a block-Jacobi preconditioner."""
        row, name = self._row, self.solver
        if args:
            if row.c != "n" or len(args) > 1 or "c" in kw:
                raise TypeError(f"{name}!: the arguments after the workspace are A, b{', c' if row.c == 'n' else ''}")
            kw["c"] = args[0]
        if kw.keys() - row.kw.keys():
            raise B200Error(f"{name}!: unsupported keyword argument(s) {', '.join(sorted(kw.keys() - row.kw.keys()))}")
        kw = {**row.kw, **row.fixed, **kw}
        c, M, N, callback = (kw.pop(k, None) for k in ("c", "M", "N", "callback"))
        if row.c == "n" and c is None:
            raise B200Error(f"{name}! solves A^T y = c as well: c must be given")
        if kw.pop("sqd", False):
            if kw["lambda_"] != 0:
                raise B200Error("sqd cannot be set to true if λ ≠ 0 !")
            kw["lambda_"] = 1.0
        o, e = _options(kw, row.kw)
        keep = [self._set_options(e, callback)]
        m, n = self.m, self.n
        fA = fAt = None
        if row.At:
            if hasattr(A, "matvec") and hasattr(A, "rmatvec") and not isinstance(A, CsrOperator):   # LinearOperator
                A = (A.matvec, A.rmatvec)
            if isinstance(A, tuple) and len(A) == 2 and all(callable(f) for f in A):
                fA, fAt = self._wrap(A[0], n, m), self._wrap(A[1], m, n)
        elif callable(A) and not hasattr(A, "shape"):
            fA = self._wrap(A, n, n)
        if fA is None and A is not None:
            self.set_operator(A)
        fP = []
        for which, (P, space) in enumerate(((M, row.M), (N, row.N))):
            if callable(P) and not hasattr(P, "shape"):
                fP.append(self._wrap(P, *[m if space == "m" else n] * 2))
                self._set_diag(which, None)
            else:
                if row.At and getattr(P, "ndim", 1) != 1:
                    raise B200Error(f"{name} takes diagonal preconditioners (1-D arrays) or host callables")
                fP.append(None)
                self._set_diag(which, P)
        keep += [fA, fAt] + fP
        return self._solve_staged(o, fA, fAt, *fP, b, c, n if row.c == "n" else m)

    def _set_options(self, e, callback):
        """Install the KrylovB200Options of one solve, `callback` behind a trampoline; returns what must outlive the
        solve."""
        if callback is not None:
            wsref = self

            def cb_tramp(_ws, _user):
                r = callback(wsref)
                if not isinstance(r, (bool, np.bool_)):
                    wsref._cb_error = TypeError(f"callback must return Bool, got {type(r).__name__}")   # cg.jl:264
                    return 1
                return int(r)
            e.callback = _lib.CALLBACK(cb_tramp)
        self._cb_error = None
        lib().krylov_b200_set_options(self._h, C.byref(e))
        return e.callback

    def _solve_staged(self, o, fA, fAt, fM, fN, b, c, c_len):
        """Stage b (m entries) and c (c_len entries), call krylov_solve and raise what it or the callback reported."""
        if not _is_torch(b):
            b = np.ascontiguousarray(b, dtype=self.dtype)
            if self.device == "cuda":
                raise B200Error("ktypeof(b) must be a device vector for a device workspace")
        elif self.device != "cuda":
            raise B200Error("ktypeof(b) must be a host vector for a host workspace")
        if b.shape[0] != self.m:
            raise B200Error("Inconsistent problem size")
        pb, kb_ = _ptr(b)
        if c is not None:
            if not _is_torch(c):
                c = np.ascontiguousarray(c, dtype=self.dtype)
            if c.shape[0] != c_len:
                raise B200Error("Inconsistent problem size")
        pc, kc = _ptr(c)
        self._order_after(kb_, kc)
        null = _lib.MATVEC()
        rc = lib().krylov_solve(self._h, fA or null, fAt or null, fM or null, fN or null, pb, pc, None, C.byref(o))
        if self._cb_error is not None:
            raise self._cb_error
        if rc != 0:
            raise B200Error(_lib.last_error())
        return self

    def warm_start(self, x0, y0=None):
        """warm_start!(workspace, x0), and warm_start!(workspace, x0, y0) for BiLQR / TriLQR: x0 has n entries, y0 m."""
        if (y0 is not None) != (self._row.c == "n"):
            raise TypeError(f"{self.solver} warm-starts from {'x0 and y0' if self._row.c == 'n' else 'x0 alone'}")
        if not _is_torch(x0):
            x0 = np.ascontiguousarray(x0, dtype=self.dtype)
        if y0 is not None:
            if not _is_torch(y0):
                y0 = np.ascontiguousarray(y0, dtype=self.dtype)
            px, kx = _ptr(x0)
            py, ky = _ptr(y0)
            self._order_after(kx, ky)
            if lib().krylov_warm_start2(self._h, px, py, int(x0.shape[0]), int(y0.shape[0])) != 0:
                raise B200Error(_lib.last_error())
            return self
        if x0.shape[0] != self.n:
            raise B200Error(f"x0 should have size {self.n}")
        p, k = _ptr(x0)
        self._order_after(k)
        rc = lib().krylov_warm_start(self._h, p, self.n)
        if rc != 0:
            raise B200Error(_lib.last_error())
        return self

    # -- accessors ------------------------------------------------------------
    @property
    def x(self):
        """solution(ws): a host copy (or a torch CUDA tensor for device workspaces)."""
        if self.device == "cuda":
            import torch
            out = torch.empty(self.n, dtype=torch.float64 if self.dtype == np.float64 else torch.float32, device="cuda")
            lib().krylov_get_x(self._h, C.c_void_p(out.data_ptr()), self.n)
            return out
        out = np.empty(self.n, dtype=self.dtype)
        if lib().krylov_get_x(self._h, out.ctypes.data_as(C.c_void_p), self.n) != 0:
            raise B200Error(_lib.last_error())
        return out

    def vector(self, name: str) -> np.ndarray:
        """Host copy of a workspace vector by its reference field name (x, r, p, Ap, npc_dir, ...)."""
        p = C.c_void_p()
        if lib().krylov_b200_get_vector(self._h, name.encode(), C.byref(p)) != 0 or not p.value:
            raise B200Error(f"workspace has no vector {name!r}")
        out = np.empty(self.n, dtype=self.dtype)
        lib().kb200_d2h(out.ctypes.data_as(C.c_void_p), p, out.nbytes)
        return out

    @property
    def y(self):
        """The second solution, m entries (x = A^T y of CRAIG, CRAIGMR and LNLQ; A^T y = c of BiLQR and TriLQR): a
        host copy (or a torch CUDA tensor for device workspaces)."""
        if not getattr(self._row, "y", False):
            raise AttributeError(f"{self.solver} has no second solution y")
        if self.device == "cuda":
            import torch
            out = torch.empty(self.m, dtype=torch.float64 if self.dtype == np.float64 else torch.float32, device="cuda")
            if lib().krylov_get_y(self._h, C.c_void_p(out.data_ptr()), self.m) != 0:
                raise B200Error(_lib.last_error())
            return out
        out = np.empty(self.m, dtype=self.dtype)
        if lib().krylov_get_y(self._h, out.ctypes.data_as(C.c_void_p), self.m) != 0:
            raise B200Error(_lib.last_error())
        return out

    @property
    def stats(self):
        """SimpleStats, with the error-bound histories of LSLQ and LNLQ; AdjointStats for BiLQR and TriLQR."""
        s = KrylovB200Stats()
        if lib().krylov_b200_get_stats(self._h, C.byref(s)) != 0:
            raise B200Error(_lib.last_error())

        def hist(which, cnt):
            buf = (C.c_double * max(cnt, 1))()
            k = lib().krylov_b200_get_history(self._h, which, buf, cnt)
            return list(buf[:max(k, 0)])
        if getattr(self._row, "c", None) == "n":
            return AdjointStats(s.niter, bool(s.solved_primal), bool(s.solved_dual), hist(0, s.nresiduals),
                                hist(6, s.nresiduals_dual), s.timer, s.status.decode("utf-8"))
        out = SimpleStats(s.niter, bool(s.solved), bool(s.inconsistent), bool(s.indefinite), s.npcCount,
                          hist(0, s.nresiduals), hist(1, s.nAresiduals), hist(2, s.nAcond), s.allocation_timer, s.timer,
                          s.status.decode("utf-8"))
        out.Anorm = s.Anorm          # LanczosStats.Anorm (cg_lanczos!), NaN otherwise
        bounds = getattr(self._row, "bounds", ())
        for attr, slot, count in bounds:
            setattr(out, attr, hist(slot, getattr(s, count)))
        if bounds:
            out.error_with_bnd = bool(s.error_with_bnd)
        return out

    @property
    def launches(self) -> int:
        return int(lib().krylov_b200_launch_count(self._h))

    @property
    def kernel_times(self):
        """(K1 ms, K2 ms, timed iterations) of the last solve run with time_kernels=True."""
        out = (C.c_double * 3)()
        lib().krylov_b200_get_kernel_times(self._h, out)
        return float(out[0]), float(out[1]), int(out[2])

    @property
    def npc_dir(self):
        return self.vector("npc_dir")


class BlockGmresWorkspace(KrylovWorkspace):
    """BlockGmresWorkspace(m, n, p, dtype; memory=5) (src/block_krylov_workspaces.jl:108-171): block_gmres! on
    n x p blocks of right-hand sides (SURVEY.md 8f-2).  B, X0 and X are n x p arrays (any layout on the Python
    side; the C ABI exchanges the reference's column-major blocks)."""

    solver = "block_gmres"

    def __init__(self, m, n, p, dtype=np.float64, *, memory: int = 0, device: str = "host"):
        self.m, self.n, self.p = int(m), int(n), int(p)
        self.dtype = np.dtype(dtype)
        self.device = device
        self._keep = []
        self._cb = None
        self._h = C.c_void_p()
        w = KrylovWorkspaceOptions(memory, 0)
        rc = lib().krylov_block_workspace_create(0, self.m, self.n, self.p, _dtype_id(self.dtype),
                                                 KRYLOV_CUDA if device == "cuda" else KRYLOV_CPU, C.byref(w), C.byref(self._h))
        if rc != 0:
            raise B200Error(f"krylov_block_workspace_create -> {rc}: {_lib.last_error()}")
        self._ext = lib().krylov_b200_default_options()
        self._op_id = None

    def free(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            lib().krylov_block_workspace_free(self._h)
            self._h = C.c_void_p()

    def _block_cb(self, f):
        if f is None:
            return _lib.BLOCK_MATVEC(), None
        n, p, dt = self.n, self.p, self.dtype
        if self.device == "cuda":
            raise B200Error("Python callables are host operators; create the workspace with device='host'")

        def tramp(xp, yp, pcols, _ud):
            X = np.ctypeslib.as_array(C.cast(xp, C.POINTER(C.c_byte)), shape=(n * pcols * dt.itemsize,)).view(dt)
            Y = np.ctypeslib.as_array(C.cast(yp, C.POINTER(C.c_byte)), shape=(n * pcols * dt.itemsize,)).view(dt)
            Y.reshape((pcols, n)).T[:] = f(X.reshape((pcols, n)).T)       # column-major n x p views
        cb = _lib.BLOCK_MATVEC(tramp)
        return cb, cb

    def _colmajor(self, B):
        if _is_torch(B):
            return B.t().contiguous()                                     # p x n row-major == n x p column-major
        return np.asfortranarray(B, dtype=self.dtype)

    def solve(self, A, B, *, M=None, N=None, atol=None, rtol=None, itmax=0, timemax=math.inf, verbose=0, history=False,
              callback=None, restart=False, reorthogonalization=False, ldiv=False):
        """block_gmres!(ws, A, B; kwargs...)  (src/block_gmres.jl:85-98)."""
        o = lib().krylov_default_options()
        if atol is not None:
            o.atol = float(atol)
        if rtol is not None:
            o.rtol = float(rtol)
        o.itmax, o.verbose = int(itmax), int(verbose)
        o.timemax = math.nan if math.isinf(timemax) else float(timemax)
        o.restart, o.reorthogonalization = int(restart), int(reorthogonalization)
        e = lib().krylov_b200_default_options()
        e.history, e.ldiv = int(history), int(ldiv)
        keep = []
        if callback is not None:
            wsref = self

            def cb_tramp(_ws, _user):
                r = callback(wsref)
                if not isinstance(r, (bool, np.bool_)):
                    wsref._cb_error = TypeError(f"callback must return Bool, got {type(r).__name__}")
                    return 1
                return int(r)
            e.callback = _lib.CALLBACK(cb_tramp)
            keep.append(e.callback)
        self._cb_error = None
        lib().krylov_b200_set_options(self._h, C.byref(e))
        fA = None
        if callable(A) and not hasattr(A, "shape"):
            fA, k = self._block_cb(A)
            keep.append(k)
        elif A is not None:
            self.set_operator(A)
        fM = fN = None
        for which, P in ((0, M), (1, N)):
            if P is None:
                self._set_diag(which, None)
            elif callable(P) and not hasattr(P, "shape"):
                f, k = self._block_cb(P)
                keep.append(k)
                if which == 0:
                    fM = f
                else:
                    fN = f
                self._set_diag(which, None)
            else:
                self._set_diag(which, P)
        if tuple(B.shape) != (self.n, self.p):
            raise B200Error("Inconsistent problem size")
        if _is_torch(B) != (self.device == "cuda"):
            raise B200Error("ktypeof(B) must match the workspace storage (host array / device tensor)")
        Bc = self._colmajor(B)
        pb, kb_ = _ptr(Bc)
        self._order_after(kb_)
        null = _lib.BLOCK_MATVEC()
        rc = lib().krylov_block_solve(self._h, fA or null, fM or null, fN or null, pb, None, C.byref(o))
        del keep
        if self._cb_error is not None:
            raise self._cb_error
        if rc != 0:
            raise B200Error(_lib.last_error())
        return self

    def warm_start(self, X0):
        if tuple(X0.shape) != (self.n, self.p):
            raise B200Error(f"X0 should have size {self.n} x {self.p}")
        Xc = self._colmajor(X0)
        p, k = _ptr(Xc)
        self._order_after(k)
        if lib().krylov_block_warm_start(self._h, p, self.n, self.p) != 0:
            raise B200Error(_lib.last_error())
        return self

    @property
    def x(self):
        """solution(ws): n x p (host array, or a torch CUDA tensor for device workspaces)."""
        if self.device == "cuda":
            import torch
            out = torch.empty((self.p, self.n), dtype=torch.float64 if self.dtype == np.float64 else torch.float32, device="cuda")
            if lib().krylov_block_get_X(self._h, C.c_void_p(out.data_ptr()), self.n, self.p) != 0:
                raise B200Error(_lib.last_error())
            return out.t()
        out = np.empty((self.n, self.p), dtype=self.dtype, order="F")
        if lib().krylov_block_get_X(self._h, out.ctypes.data_as(C.c_void_p), self.n, self.p) != 0:
            raise B200Error(_lib.last_error())
        return out

    X = x

    @property
    def qr_fallbacks(self) -> int:
        """Panel QR factorizations that took the slow Householder path (rank-deficient blocks); 0 normally."""
        return int(lib().krylov_b200_block_qr_fallbacks(self._h))


def block_gmres(A, B, X0=None, *, memory=0, **kw):
    """(X, stats) = block_gmres(A, B[, X0]; memory=5, kwargs...)  (src/block_gmres.jl:1-60)"""
    n, p = B.shape
    dt = B.cpu().numpy().dtype if _is_torch(B) else np.asarray(B).dtype
    if dt not in (np.float32, np.float64):
        dt = np.float64
    ws = BlockGmresWorkspace(n, n, p, dt, memory=memory, device="cuda" if _is_torch(B) else "host")
    try:
        if X0 is not None:
            ws.warm_start(X0)
        ws.solve(A, B if _is_torch(B) else np.asarray(B, dtype=dt), **kw)
        return ws.x, ws.stats
    finally:
        ws.free()


def block_gmres_(ws: BlockGmresWorkspace, A, B, X0=None, **kw):
    """block_gmres!(workspace, A, B[, X0]; kwargs...)"""
    if X0 is not None:
        ws.warm_start(X0)
    return ws.solve(A, B, **kw)


# ---------------------------------------------------------------------------------------------------------------------
# The shift solvers: one Lanczos process for p shifted systems, p solutions (their own handle kind in the C ABI).
# ---------------------------------------------------------------------------------------------------------------------
@dataclass
class LanczosShiftStats:
    """src/krylov_stats.jl:169-179: one residual history (`residuals`) and one `indefinite` flag per shift; Anorm and
    Acond stay NaN, as the reference leaves them."""
    niter: int = 0
    solved: bool = False
    residuals: list = field(default_factory=list)
    indefinite: list = field(default_factory=list)
    Anorm: float = math.nan
    Acond: float = math.nan
    allocation_timer: float = 0.0
    timer: float = 0.0
    status: str = "unknown"


_SHIFT_KW = dict(M=None, ldiv=False, atol=None, rtol=None, itmax=0, timemax=math.inf, verbose=0, history=False,
                 callback=None, fused=True)


class _ShiftWorkspace(KrylovWorkspace):
    """Workspace of a shift solver: X and P hold n x nshifts entries besides the Lanczos vectors."""

    solver_id = 0
    rect = False            # A is m x n and its adjoint is applied (CGLS-Lanczos-shift)
    keywords = _SHIFT_KW

    def __init__(self, m, n, nshifts, dtype=np.float64, *, device: str = "host"):
        self.m, self.n, self.nshifts = int(m), int(n), int(nshifts)
        self.dtype = np.dtype(dtype)
        self.device = device
        self._keep = []
        self._cb = None
        self._h = C.c_void_p()
        rc = lib().krylov_b200_shift_workspace_create(self.solver_id, self.m, self.n, self.nshifts, _dtype_id(self.dtype),
                                                      KRYLOV_CUDA if device == "cuda" else KRYLOV_CPU, C.byref(self._h))
        if rc != 0:
            raise B200Error(f"krylov_b200_shift_workspace_create({self.solver}) -> {rc}: {_lib.last_error()}")
        self._ext = lib().krylov_b200_default_options()
        self._op_id = None

    def free(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            lib().krylov_b200_shift_workspace_free(self._h)
            self._h = C.c_void_p()

    def solve(self, A, b, shifts, **kw):
        """solver!(ws, A, b, shifts; kwargs...): the keywords of the class's `keywords`.  A: a SciPy matrix, a
        CsrOperator or a (rowptr, colind, values) tuple; or a host callable (CG-Lanczos-shift), a LinearOperator or a
        (matvec, rmatvec) pair (CGLS-Lanczos-shift).  M: None, a 1-D diagonal, (nblocks, bs, bs) block-Jacobi blocks or
        a host callable (CG-Lanczos-shift only)."""
        name = self.solver
        if kw.keys() - self.keywords.keys():
            raise B200Error(f"{name}!: unsupported keyword argument(s) {', '.join(sorted(kw.keys() - self.keywords.keys()))}")
        kw = {**self.keywords, **kw}
        M, callback = kw.pop("M"), kw.pop("callback")
        shifts = np.ascontiguousarray(shifts.cpu().numpy() if _is_torch(shifts) else shifts, dtype=np.float64).ravel()
        if shifts.shape[0] != self.nshifts:
            raise B200Error(f"workspace.nshifts = {self.nshifts} is inconsistent with length(shifts) = {shifts.shape[0]}")
        if self.rect and M is not None:
            raise B200Error("Preconditioner `M` is not supported.")
        o, e = _options(kw, self.keywords)
        keep = [self._set_options(e, callback)]
        m, n = self.m, self.n
        fA = fAt = fM = None
        if self.rect:
            if hasattr(A, "matvec") and hasattr(A, "rmatvec") and not isinstance(A, CsrOperator):   # LinearOperator
                A = (A.matvec, A.rmatvec)
            if isinstance(A, tuple) and len(A) == 2 and all(callable(f) for f in A):
                fA, fAt = self._wrap(A[0], n, m), self._wrap(A[1], m, n)
        elif callable(A) and not hasattr(A, "shape"):
            fA = self._wrap(A, n, n)
        if fA is None and A is not None:
            self.set_operator(A)
        if callable(M) and not hasattr(M, "shape"):
            fM = self._wrap(M, n, n)
            self._set_diag(0, None)
        else:
            self._set_diag(0, M)
        keep += [fA, fAt, fM]
        if not _is_torch(b):
            b = np.ascontiguousarray(b, dtype=self.dtype)
            if self.device == "cuda":
                raise B200Error("ktypeof(b) must be a device vector for a device workspace")
        elif self.device != "cuda":
            raise B200Error("ktypeof(b) must be a host vector for a host workspace")
        if b.shape[0] != m:
            raise B200Error("Inconsistent problem size")
        pb, kb_ = _ptr(b)
        self._order_after(kb_)
        null = _lib.MATVEC()
        sh = (C.c_double * self.nshifts)(*shifts.tolist())
        rc = lib().krylov_b200_shift_solve(self._h, fA or null, fAt or null, fM or null, pb, sh, None, C.byref(o))
        del keep
        if self._cb_error is not None:
            raise self._cb_error
        if rc != 0:
            raise B200Error(_lib.last_error())
        return self

    @property
    def x(self):
        """solution(ws): the nshifts solutions, host arrays (or torch CUDA tensors for device workspaces)."""
        out = []
        for i in range(self.nshifts):
            if self.device == "cuda":
                import torch
                xi = torch.empty(self.n, dtype=torch.float64 if self.dtype == np.float64 else torch.float32, device="cuda")
                p = C.c_void_p(xi.data_ptr())
            else:
                xi = np.empty(self.n, dtype=self.dtype)
                p = xi.ctypes.data_as(C.c_void_p)
            if lib().krylov_b200_shift_get_x(self._h, i, p, self.n) != 0:
                raise B200Error(_lib.last_error())
            out.append(xi)
        return out

    @property
    def stats(self) -> LanczosShiftStats:
        p = self.nshifts
        niter, solved, timer = C.c_int(), C.c_int(), C.c_double()
        status = C.create_string_buffer(96)
        indef, hlen = (C.c_int * p)(), (C.c_int * p)()
        if lib().krylov_b200_shift_get_stats(self._h, C.byref(niter), C.byref(solved), C.byref(timer), status, 96, indef,
                                             hlen) != 0:
            raise B200Error(_lib.last_error())
        res = []
        for i in range(p):
            buf = (C.c_double * max(hlen[i], 1))()
            k = lib().krylov_b200_shift_get_history(self._h, i, buf, hlen[i])
            res.append(list(buf[:max(k, 0)]))
        s = KrylovB200Stats()
        lib().krylov_b200_get_stats(self._h, C.byref(s))
        return LanczosShiftStats(niter.value, bool(solved.value), res, [bool(v) for v in indef], math.nan, math.nan,
                                 s.allocation_timer, timer.value, status.value.decode("utf-8"))


class CgLanczosShiftWorkspace(_ShiftWorkspace):
    """CgLanczosShiftWorkspace(m, n, nshifts, dtype) (src/krylov_workspaces.jl:604-660): cg_lanczos_shift! solves
    (A + σᵢ I) xᵢ = b for every shift σᵢ with one Lanczos process; m == n."""
    solver, solver_id = "cg_lanczos_shift", _lib.KRYLOV_B200_CG_LANCZOS_SHIFT
    keywords = dict(_SHIFT_KW, check_curvature=False)


class CglsLanczosShiftWorkspace(_ShiftWorkspace):
    """CglsLanczosShiftWorkspace(m, n, nshifts, dtype): cgls_lanczos_shift! solves (AᵀA + σᵢ I) xᵢ = Aᵀb for every
    shift σᵢ, A m x n (b: m entries, xᵢ: n); no preconditioner."""
    solver, solver_id, rect = "cgls_lanczos_shift", _lib.KRYLOV_B200_CGLS_LANCZOS_SHIFT, True


def _make_shift(name, cls):
    def inplace(ws, A, b, shifts, **kw):
        if ws.solver != name:
            raise B200Error(f"{name}! needs a {cls.__name__}")
        return ws.solve(A, b, shifts, **kw)

    def outofplace(A, b, shifts, **kw):
        n = _columns(name, A, kw.pop("n", None)) if cls.rect else b.shape[0]
        if _is_torch(b):
            import torch
            dt = {torch.float32: np.float32, torch.float64: np.float64}.get(b.dtype, np.float64)
        else:
            dt = np.asarray(b).dtype
        if dt not in (np.float32, np.float64):
            dt = np.float64
        ws = cls(b.shape[0], int(n), len(shifts), dt, device="cuda" if _is_torch(b) else "host")
        try:
            ws.solve(A, b, shifts, **kw)
            return ws.x, ws.stats
        finally:
            ws.free()
    inplace.__name__, outofplace.__name__ = name + "_", name
    inplace.__doc__ = f"{name}!(workspace, A, b, shifts; kwargs...)"
    outofplace.__doc__ = f"(xs, stats) = {name}(A, b, shifts; kwargs...): xs holds one solution per shift"
    return inplace, outofplace


cg_lanczos_shift_, cg_lanczos_shift = _make_shift("cg_lanczos_shift", CgLanczosShiftWorkspace)
cgls_lanczos_shift_, cgls_lanczos_shift = _make_shift("cgls_lanczos_shift", CglsLanczosShiftWorkspace)
__all__ += ["LanczosShiftStats", "CgLanczosShiftWorkspace", "CglsLanczosShiftWorkspace", "cg_lanczos_shift",
            "cg_lanczos_shift_", "cgls_lanczos_shift", "cgls_lanczos_shift_"]


# ---------------------------------------------------------------------------------------------------------------------
# The solvers: one row each.  The workspace class, solver! and solver of every row are made from it below.
# ---------------------------------------------------------------------------------------------------------------------
_COMMON = dict(atol=None, rtol=None, itmax=0, timemax=math.inf, verbose=0, history=False, callback=None, fused=True,
               ldiv=False)


@dataclass
class _Solver:
    """What the binding needs to know of one solver; the library checks the rest.

    cls, cite: the workspace class's name and where the reference documents the solver's keywords.
    kw: the keywords it takes besides _COMMON, M, N and c, with their defaults (None keeps the library's default).
    fixed: option keywords it does not take but sets to these values.
    nA: operator products per iteration (workspace_accessors.jl:101-139).
    M, N: the space a host-callable preconditioner acts on, "m" or "n"; None where the solver takes none.
    c: None; "m": optional, m entries; "n": required, n entries, for the adjoint system A^T y = c solved along with
       A x = b (the third positional argument, then x0 and y0 for a warm start; AdjointStats).
    rect: A is m x n, so the out-of-place form takes n= with a tuple operator, and (unless c is "n") no x0.
    At: A^T is applied: A is a CSR operator, a LinearOperator or a (matvec, rmatvec) pair, and M, N are 1-D.
    y: there is a second solution y, m entries.
    bounds: (stats attribute, history slot, count field) of the error-bound histories in its statistics: LSLQStats
      (src/krylov_stats.jl:352-365), and LNLQStats, whose two bounds travel in LSLQ's slots 3 and 4.
    ws_kw: the workspace options the out-of-place form takes."""
    cls: str
    cite: str
    kw: dict = field(default_factory=dict)
    fixed: dict = field(default_factory=dict)
    nA: int = 1
    M: Optional[str] = None
    N: Optional[str] = None
    c: Optional[str] = None
    rect: bool = False
    At: bool = False
    y: bool = False
    bounds: tuple = ()
    ws_kw: tuple = ()

    def __post_init__(self):
        taken = [k for k in ("M", "N", "c") if getattr(self, k)]
        self.kw = {k: v for k, v in {**_COMMON, **dict.fromkeys(taken), **self.kw}.items() if k not in self.fixed}


_SQUARE = dict(kw=dict(radius=0.0, linesearch=False, lambda_=0.0, etol=None, conlim=None, restart=False,
                       reorthogonalization=False, batch=0, time_kernels=False, check_curvature=False, gamma=None,
                       artol=None), M="n", N="n", c="m", ws_kw=("memory", "window"))
_LSQ = dict(M="m", N="n", rect=True, At=True, ws_kw=("window",))
_LN = dict(nA=2, M="m", N="n", rect=True, At=True, y=True)
_SQD = dict(sqd=False, lambda_=0.0)
_SOLVERS = {
    "cg": _Solver("CgWorkspace", "cg.jl:100-111", **_SQUARE),
    "cr": _Solver("CrWorkspace", "cr.jl", **_SQUARE),
    "minres": _Solver("MinresWorkspace", "minres.jl:138-151", **_SQUARE),
    "diom": _Solver("DiomWorkspace", "diom.jl", **_SQUARE),
    "fom": _Solver("FomWorkspace", "fom.jl", **_SQUARE),
    "dqgmres": _Solver("DqgmresWorkspace", "dqgmres.jl", **_SQUARE),
    "gmres": _Solver("GmresWorkspace", "gmres.jl:96-108", **_SQUARE),
    "fgmres": _Solver("FgmresWorkspace", "fgmres.jl", **_SQUARE),
    "bicgstab": _Solver("BicgstabWorkspace", "bicgstab.jl:105-116", nA=2, **_SQUARE),
    "cgs": _Solver("CgsWorkspace", "cgs.jl", nA=2, **_SQUARE),
    "cg_lanczos": _Solver("CgLanczosWorkspace", "cg_lanczos.jl", **_SQUARE),
    "car": _Solver("CarWorkspace", "car.jl:90-99", M="n", ws_kw=("memory", "window")),
    "minares": _Solver("MinaresWorkspace", "minares.jl:93-104", dict(lambda_=0.0, artol=None), M="n",
                       ws_kw=("memory", "window")),
    "lsqr": _Solver("LsqrWorkspace", "lsqr.jl:145-162", dict(_SQD, radius=0.0, etol=None, axtol=None, btol=None,
                                                              conlim=None, atol=0.0, rtol=0.0), **_LSQ),
    "lsmr": _Solver("LsmrWorkspace", "lsmr.jl", dict(_SQD, radius=0.0, etol=None, axtol=None, btol=None, conlim=None,
                                                     atol=0.0, rtol=0.0), **_LSQ),
    "lslq": _Solver("LslqWorkspace", "lslq.jl:178-196", dict(_SQD, transfer_to_lsqr=False, sigma=0.0, etol=None,
                                                              utol=None, btol=None, conlim=None),
                    bounds=(("err_lbnds", 3, "nerr_lbnds"), ("err_ubnds_lq", 4, "nerr_ubnds_lq"),
                            ("err_ubnds_cg", 5, "nerr_ubnds_cg")), **_LSQ),
    "cgls": _Solver("CglsWorkspace", "cgls.jl:110-121", dict(radius=0.0, lambda_=0.0), **dict(_LSQ, N=None)),
    "crls": _Solver("CrlsWorkspace", "crls.jl:101-112", dict(radius=0.0, lambda_=0.0), **dict(_LSQ, N=None)),
    "bilq": _Solver("BilqWorkspace", "bilq.jl:97-109", dict(transfer_to_bicg=True), nA=2, M="m", N="n", c="m", At=True,
                    ws_kw=("memory", "window")),
    "qmr": _Solver("QmrWorkspace", "qmr.jl:104-115", fixed=dict(transfer_to_bicg=True), nA=2, M="m", N="n", c="m",
                   At=True, ws_kw=("memory", "window")),
    "bilqr": _Solver("BilqrWorkspace", "bilqr.jl:99-107", dict(transfer_to_bicg=True), dict(ldiv=False), nA=2, c="n",
                     At=True, y=True),
    "trilqr": _Solver("TrilqrWorkspace", "trilqr.jl", dict(transfer_to_usymcg=True), dict(ldiv=False), nA=2, c="n",
                      rect=True, At=True, y=True),
    "craig": _Solver("CraigWorkspace", "craig.jl:151-166", dict(_SQD, transfer_to_lsqr=False, btol=None, conlim=None),
                     **_LN),
    "craigmr": _Solver("CraigmrWorkspace", "craigmr.jl:141-153", _SQD, **_LN),
    "lnlq": _Solver("LnlqWorkspace", "lnlq.jl:144-160", dict(_SQD, transfer_to_craig=True, sigma=0.0, utolx=None,
                                                              utoly=None),
                    bounds=(("error_bnd_x", 3, "nerr_lbnds"), ("error_bnd_y", 4, "nerr_ubnds_lq")), **_LN),
    "cgne": _Solver("CgneWorkspace", "cgne.jl:116-126", dict(lambda_=0.0), **dict(_LN, M=None, N="m", y=False)),
    "crmr": _Solver("CrmrWorkspace", "crmr.jl:114-124", dict(lambda_=0.0), **dict(_LN, M=None, N="m", y=False)),
}


def _columns(name, A, n):
    if n is None:
        if not hasattr(A, "shape"):
            raise B200Error(f"{name}: pass n= (number of columns) with a tuple operator")
        n = A.shape[1]
    return n


def _positional(who, row, args, kw):
    """Move the arguments after b into kw -- c, x0 and y0 for the solvers that require c, x0 for the others -- and
    return the warm start (x0, y0)."""
    names = ("c", "x0", "y0") if row.c == "n" else ("x0",)
    if len(args) > len(names):
        raise TypeError(f"{who}: the arguments after b are {', '.join(names)}")
    for k, v in zip(names, args):
        if k in kw:
            raise TypeError(f"{who}: {k} is given twice")
        kw[k] = v
    return kw.pop("x0", None), kw.pop("y0", None) if row.c == "n" else None


def _warm_start(who, row, ws, x0, y0):
    if row.c == "n":
        if (x0 is None) != (y0 is None):
            raise B200Error(f"{who}: pass both x0 and y0, or neither")
        if x0 is not None:
            ws.warm_start(x0, y0)
    elif x0 is not None:
        ws.warm_start(x0)


def _make_inplace(name, row):
    def f(ws, A, b, *args, **kw):
        if ws.solver != name:
            raise B200Error(f"{name}! needs a {row.cls}")
        _warm_start(name + "!", row, ws, *_positional(name + "!", row, args, kw))
        return ws.solve(A, b, **kw)
    f.__name__ = name + "_"
    f.__doc__ = f"{name}!(workspace, A, b{', c[, x0, y0]' if row.c == 'n' else '[, x0]'}; kwargs...)"
    return f


def _make_outofplace(name, row):
    def f(A, b, *args, **kw):
        x0, y0 = _positional(name, row, args, kw)
        if row.c == "n":
            if kw.get("c") is None:
                raise B200Error(f"{name}! solves A^T y = c as well: c must be given")
            n = kw["c"].shape[0]
        elif row.rect:
            if x0 is not None:
                raise B200Error(f"{name} does not support warm-start (it takes no x0)")
            n = _columns(name, A, kw.pop("n", None))
        else:
            n = b.shape[0]
        if _is_torch(b):       # the element type of a torch b is read without copying it to the host
            import torch
            dt = {torch.float32: np.float32, torch.float64: np.float64}.get(b.dtype, np.float64)
        else:
            dt = np.asarray(b).dtype
        if dt not in (np.float32, np.float64):
            dt = np.float64
        ws_kw = {k: kw.pop(k) for k in row.ws_kw if k in kw}
        ws = globals()[row.cls](b.shape[0], int(n), dt, device="cuda" if _is_torch(b) else "host", **ws_kw)
        try:
            _warm_start(name, row, ws, x0, y0)
            ws.solve(A, b, **kw)
            return (ws.x, ws.y, ws.stats) if row.y else (ws.x, ws.stats)
        finally:
            ws.free()
    f.__name__ = name
    f.__doc__ = (f"({'x, y' if row.y else 'x'}, stats) = {name}(A, b{', c[, x0, y0]' if row.c == 'n' else '' if row.rect else '[, x0]'}; "
                 f"kwargs...)  (src/{row.cite})")
    return f


for _name, _row in _SOLVERS.items():
    globals()[_row.cls] = type(_row.cls, (KrylovWorkspace,), dict(
        solver=_name, nA=_row.nA, __doc__=f"Workspace of {_name}! (src/{_row.cite}); solve keywords and defaults: "
                                          + ", ".join(f"{k}={v!r}" for k, v in _row.kw.items()) + "."))
    globals()[_name + "_"], globals()[_name] = _make_inplace(_name, _row), _make_outofplace(_name, _row)
    __all__ += [_row.cls, _name, _name + "_"]


def krylov_workspace(method: str, *args, **kw) -> KrylovWorkspace:
    """krylov_workspace(Val(method), ...)  (src/interface.jl:248-348)"""
    if method not in _SOLVERS:
        raise B200Error(f"method {method!r} is outside the GPU path ({', '.join(sorted(_SOLVERS))})")
    return globals()[_SOLVERS[method].cls](*args, **kw)


def krylov_solve_(ws: KrylovWorkspace, A, b, x0=None, **kw) -> KrylovWorkspace:
    """krylov_solve!(ws, A, b[, x0]; kw...)"""
    if x0 is not None:
        ws.warm_start(x0)
    return ws.solve(A, b, **kw)


def krylov_solve(method: str, A, b, x0=None, **kw):
    """krylov_solve(method, A, b[, x0]; kwargs...): the out-of-place form of `method`.  BiLQR and TriLQR, which
    take c as well, raise KeyError like a method outside the GPU path."""
    if _SOLVERS[method].c == "n":
        raise KeyError(method)
    return globals()[method](A, b, x0, **kw)


# workspace_accessors.jl:140-152
def solution(ws): return ws.x
def statistics(ws): return ws.stats
def results(ws): return (ws.x, ws.stats)
def issolved(ws): return bool(lib().krylov_is_solved(ws._h) == 1)
def iteration_count(ws): return int(lib().krylov_niter(ws._h))
def elapsed_time(ws): return float(lib().krylov_elapsed_time(ws._h))
def Aprod_count(ws): return ws.nA * iteration_count(ws)
def warm_start_(ws, x0): return ws.warm_start(x0)


# ---------------------------------------------------------------------------------------------------------------------
# Krylov processes (src/krylov_processes.jl): the basis and the projected matrix of k steps, on the GPU
# ---------------------------------------------------------------------------------------------------------------------
def _tridiag_structure(k):
    """colptr / rowval (0-based) of the reference's (k+1) x k tridiagonal T: 3k-1 stored entries."""
    colptr = np.zeros(k + 1, np.int64)
    rowval = np.zeros(3 * k - 1, np.int64)
    for i in range(1, k + 1):
        pos = colptr[i - 1]
        colptr[i] = 3 * i - 1
        rows = (i, i + 1) if i == 1 else (i - 1, i, i + 1)
        rowval[pos:pos + len(rows)] = np.array(rows) - 1
    return colptr, rowval


def _bidiag_structure(k):
    """colptr / rowval (0-based) of golub_kahan's (k+1) x (k+1) lower bidiagonal L: 2k+1 stored entries."""
    colptr = np.zeros(k + 2, np.int64)
    rowval = np.zeros(2 * k + 1, np.int64)
    for i in range(1, k + 2):
        pos = colptr[i - 1]
        rows = (i, i + 1) if i <= k else (i,)
        colptr[i] = pos + len(rows)
        rowval[pos:pos + len(rows)] = np.array(rows) - 1
    return colptr, rowval


def _csc(nzval, structure, shape):
    import scipy.sparse as sp
    colptr, rowval = structure
    return sp.csc_matrix((nzval, rowval, colptr), shape=shape)


class _ProcessCall:
    """Operators and device vectors of one process call: A (and Aᵀ) as CSR objects, b / c and the outputs V / U on the
    device, NumPy inputs staged in and out, torch inputs used in place."""

    def __init__(self, name, A, vecs, At, adjoint):
        import scipy.sparse as sp
        self.name, self._free = name, []
        self.torch = any(_is_torch(v) for v in vecs)
        first = vecs[0]
        if self.torch:
            if not all(_is_torch(v) and v.is_cuda for v in vecs):
                raise B200Error(f"{name}: pass b and c both as torch CUDA tensors or both as NumPy arrays")
            self.dtype = np.dtype(str(first.dtype).replace("torch.", ""))
        else:
            self.dtype = np.asarray(first).dtype
            if self.dtype.kind in "iub":
                self.dtype = np.dtype(np.float64)
        self.dt = _dtype_id(self.dtype)                 # complex and other types are refused here
        if isinstance(A, CsrOperator):
            self.A = A
        elif sp.issparse(A):
            self.A = CsrOperator.from_scipy(A, dtype=self.dtype)
            self._free.append(self.A)
        else:
            raise B200Error(f"{name} needs a CSR operator (a SciPy sparse matrix or a CsrOperator); matrix-free operators "
                            "and callbacks are not supported")
        if self.A.dtype != self.dtype:
            raise B200Error(f"{name}: the operator is {self.A.dtype}, b is {self.dtype}")
        self.m, self.n = self.A.shape
        self.At = None
        if adjoint:
            if At is None:                               # formed once per call
                At = A.T if sp.issparse(A) else None
            if isinstance(At, CsrOperator):
                self.At = At
            elif At is not None:
                if not sp.issparse(At):
                    raise B200Error(f"{name}: At must be a SciPy sparse matrix or a CsrOperator")
                if At.shape != (self.n, self.m):
                    raise B200Error(f"{name}: At must be {self.n} x {self.m}, got {At.shape[0]} x {At.shape[1]}")
                self.At = CsrOperator.from_scipy(At, dtype=self.dtype)
                self._free.append(self.At)

    def vec_in(self, v, length, label):
        if int(v.shape[0]) != length or len(v.shape) != 1:
            raise B200Error(f"{self.name}: {label} must have {length} entries, got shape {tuple(v.shape)}")
        if self.torch:
            import torch
            if v.dtype != getattr(torch, self.dtype.name):
                raise B200Error(f"{self.name}: {label} must be {self.dtype}")
            v = v.contiguous()
            self._free.append(v)
            return C.c_void_p(v.data_ptr())
        v = np.ascontiguousarray(v, dtype=self.dtype)
        d = lib().kb200_alloc(max(v.nbytes, 1))
        self._free.append(d)
        if lib().kb200_h2d(d, v.ctypes.data_as(C.c_void_p), v.nbytes) != 0:
            raise B200Error(_lib.last_error())
        return C.c_void_p(d)

    def basis(self, rows, k):
        """Device storage of an output basis, rows x (k+1) column-major."""
        if self.torch:
            import torch
            V = torch.empty((k + 1, rows), dtype=getattr(torch, self.dtype.name), device="cuda").t()
            return V, C.c_void_p(V.data_ptr())
        d = lib().kb200_alloc(rows * (k + 1) * self.dtype.itemsize)
        self._free.append(d)
        return d, C.c_void_p(d)

    def out(self, V, rows, k):
        if self.torch:
            return V
        h = np.empty((rows, k + 1), self.dtype, order="F")
        if lib().kb200_d2h(h.ctypes.data_as(C.c_void_p), C.c_void_p(V), h.nbytes) != 0:
            raise B200Error(_lib.last_error())
        return h

    def run(self, *args):
        if self.torch:
            import torch
            torch.cuda.current_stream().synchronize()    # b / c complete before the library's stream reads them
        rc = getattr(lib(), f"kb200_{self.name}")(self.A._ctx, self.A._csr, *args)
        if rc != 0:
            msg = _lib.last_error() if rc == -1 else f"{self.name}: unsupported element type"
            raise B200Error(msg.split(f"kb200_{self.name}: ", 1)[-1])

    def close(self):
        for f in self._free:
            if isinstance(f, CsrOperator):
                f.free()
            elif isinstance(f, int):
                lib().kb200_free(C.c_void_p(f))
        self._free = []


def _flags(allow_breakdown, reorthogonalization=False):
    return int(bool(allow_breakdown)) | (2 if reorthogonalization else 0)


def hermitian_lanczos(A, b, k: int, *, allow_breakdown: bool = False, reorthogonalization: bool = False):
    """V, β, T = hermitian_lanczos(A, b, k) (src/krylov_processes.jl:28-103): V is n x (k+1), βv₁ = b and T the
    (k+1) x k tridiagonal matrix with A V[:, :k] = V T, as a scipy.sparse.csc_matrix with the reference's structure.
    A: a symmetric SciPy sparse matrix or CsrOperator; b: NumPy array or torch CUDA tensor (then V is a torch tensor with
    column-major strides and nothing is copied to the host but the coefficients)."""
    P = _ProcessCall("hermitian_lanczos", A, [b], None, False)
    try:
        pb = P.vec_in(b, P.n, "b")
        V, pV = P.basis(P.n, k)
        beta, nz = C.c_double(), np.zeros(max(3 * k - 1, 0), np.float64)
        P.run(int(k), P.dt, pb, pV, C.byref(beta), nz.ctypes.data_as(C.POINTER(C.c_double)),
              _flags(allow_breakdown, reorthogonalization))
        return P.out(V, P.n, k), beta.value, _csc(nz.astype(P.dtype), _tridiag_structure(k), (k + 1, k))
    finally:
        P.close()


def arnoldi(A, b, k: int, *, allow_breakdown: bool = False, reorthogonalization: bool = False):
    """V, β, H = arnoldi(A, b, k) (src/krylov_processes.jl:250-296): V is n x (k+1), βv₁ = b and H the dense
    (k+1) x k upper Hessenberg matrix with A V[:, :k] = V H (modified Gram-Schmidt; reorthogonalization: a second pass
    against every previous vector)."""
    P = _ProcessCall("arnoldi", A, [b], None, False)
    try:
        pb = P.vec_in(b, P.n, "b")
        V, pV = P.basis(P.n, k)
        beta, H = C.c_double(), np.zeros((max(k, 0) + 1, max(k, 0)), np.float64, order="F")
        P.run(int(k), P.dt, pb, pV, C.byref(beta), H.ctypes.data_as(C.POINTER(C.c_double)),
              _flags(allow_breakdown, reorthogonalization))
        return P.out(V, P.n, k), beta.value, np.asfortranarray(H.astype(P.dtype))
    finally:
        P.close()


def golub_kahan(A, b, k: int, *, allow_breakdown: bool = False, At=None):
    """V, U, β, L = golub_kahan(A, b, k) (src/krylov_processes.jl:323-402): A is m x n, V n x (k+1), U m x (k+1),
    βu₁ = b and L the (k+1) x (k+1) lower bidiagonal matrix with A V[:, :k] = U L[:, :k] and Aᵀ U = V Lᵀ.
    At: Aᵀ (SciPy or CsrOperator); by default it is formed once for the call."""
    P = _ProcessCall("golub_kahan", A, [b], At, True)
    try:
        pb = P.vec_in(b, P.m, "b")
        V, pV = P.basis(P.n, k)
        U, pU = P.basis(P.m, k)
        beta, nz = C.c_double(), np.zeros(max(2 * k + 1, 0), np.float64)
        P.run(P.At._csr if P.At else None, int(k), P.dt, pb, pV, pU, C.byref(beta),
              nz.ctypes.data_as(C.POINTER(C.c_double)), _flags(allow_breakdown))
        return (P.out(V, P.n, k), P.out(U, P.m, k), beta.value,
                _csc(nz.astype(P.dtype), _bidiag_structure(k), (k + 1, k + 1)))
    finally:
        P.close()


def _two_sided(name, A, b, c, k, allow_breakdown, At, lb, lc):
    P = _ProcessCall(name, A, [b, c], At, True)
    try:
        rows_v, rows_u = (P.n, P.n) if name == "nonhermitian_lanczos" else (P.m, P.n)
        pb, pc = P.vec_in(b, lb(P), "b"), P.vec_in(c, lc(P), "c")
        V, pV = P.basis(rows_v, k)
        U, pU = P.basis(rows_u, k)
        beta, gamma = C.c_double(), C.c_double()
        nzT, nzH = np.zeros(max(3 * k - 1, 0), np.float64), np.zeros(max(3 * k - 1, 0), np.float64)
        P.run(P.At._csr if P.At else None, int(k), P.dt, pb, pc, pV, pU, C.byref(beta), C.byref(gamma),
              nzT.ctypes.data_as(C.POINTER(C.c_double)), nzH.ctypes.data_as(C.POINTER(C.c_double)), _flags(allow_breakdown))
        s = _tridiag_structure(k)
        return (P.out(V, rows_v, k), beta.value, _csc(nzT.astype(P.dtype), s, (k + 1, k)), P.out(U, rows_u, k), gamma.value,
                _csc(nzH.astype(P.dtype), s, (k + 1, k)))
    finally:
        P.close()


def nonhermitian_lanczos(A, b, c, k: int, *, allow_breakdown: bool = False, At=None):
    """V, β, T, U, γᴴ, Tᴴ = nonhermitian_lanczos(A, b, c, k) (src/krylov_processes.jl:133-224): square A, βv₁ = b,
    γᴴu₁ = c, A V[:, :k] = V T and Aᵀ U[:, :k] = U Tᴴ with Uᵀ V = I.  When cᵀb == 0 (allow_breakdown) V[:, 0] and U[:, 0]
    are zero, where the reference leaves them undefined."""
    return _two_sided("nonhermitian_lanczos", A, b, c, k, allow_breakdown, At, lambda P: P.n, lambda P: P.n)


def saunders_simon_yip(A, b, c, k: int, *, allow_breakdown: bool = False, At=None):
    """V, β, T, U, γᴴ, Tᴴ = saunders_simon_yip(A, b, c, k) (src/krylov_processes.jl:431-524): A is m x n, V m x (k+1),
    U n x (k+1), βv₁ = b, γᴴu₁ = c, A U[:, :k] = V T and Aᵀ V[:, :k] = U Tᴴ."""
    return _two_sided("saunders_simon_yip", A, b, c, k, allow_breakdown, At, lambda P: P.m, lambda P: P.n)


__all__ += ["hermitian_lanczos", "arnoldi", "golub_kahan", "nonhermitian_lanczos", "saunders_simon_yip"]
