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
from typing import Callable, Optional

import numpy as np

from . import _lib
from ._lib import (KRYLOV_CPU, KRYLOV_CUDA, KRYLOV_FLOAT32, KRYLOV_FLOAT64, SOLVER_IDS, KrylovB200Options,
                   KrylovB200Stats, KrylovOptions, KrylovWorkspaceOptions, lib)

__all__ = ["CgWorkspace", "GmresWorkspace", "BicgstabWorkspace", "MinresWorkspace", "KrylovWorkspace", "SimpleStats",
           "cg", "cg_", "gmres", "gmres_", "bicgstab", "bicgstab_", "minres", "minres_", "krylov_workspace",
           "krylov_solve", "krylov_solve_", "solution", "statistics", "results", "issolved", "iteration_count",
           "elapsed_time", "Aprod_count", "warm_start_", "device_count", "B200Error",
           "FomWorkspace", "FgmresWorkspace", "CgsWorkspace", "CgLanczosWorkspace", "fom", "fom_", "fgmres", "fgmres_",
           "cgs", "cgs_", "cg_lanczos", "cg_lanczos_", "CrWorkspace", "DiomWorkspace", "DqgmresWorkspace", "cr", "cr_", "diom",
           "diom_", "dqgmres", "dqgmres_", "BlockGmresWorkspace", "block_gmres", "block_gmres_", "CsrOperator",
           "LsqrWorkspace", "LsmrWorkspace", "lsqr", "lsqr_", "lsmr", "lsmr_",
           "CglsWorkspace", "CrlsWorkspace", "cgls", "cgls_", "crls", "crls_", "LslqWorkspace", "lslq", "lslq_",
           "BilqWorkspace", "QmrWorkspace", "bilq", "bilq_", "qmr", "qmr_",
           "CarWorkspace", "MinaresWorkspace", "car", "car_", "minares", "minares_",
           "AdjointStats", "BilqrWorkspace", "TrilqrWorkspace", "bilqr", "bilqr_", "trilqr", "trilqr_",
           "CraigWorkspace", "CraigmrWorkspace", "craig", "craig_", "craigmr", "craigmr_", "LnlqWorkspace", "lnlq", "lnlq_",
           "CgneWorkspace", "CrmrWorkspace", "cgne", "cgne_", "crmr", "crmr_"]


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


def _float(v):
    return None if v is None else float(v)


def _options(atol, rtol, itmax, timemax, verbose, history, ldiv, fused, opts=(), ext=()):
    """The KrylovOptions / KrylovB200Options pair of one solve: the keywords every solver takes, then the solver's own
    fields (`opts` into KrylovOptions, `ext` into KrylovB200Options; a None value keeps the default)."""
    o = lib().krylov_default_options()
    if atol is not None:
        o.atol = float(atol)
    if rtol is not None:
        o.rtol = float(rtol)
    o.itmax, o.verbose = int(itmax), int(verbose)
    o.timemax = math.nan if math.isinf(timemax) else float(timemax)
    e = lib().krylov_b200_default_options()
    e.history, e.ldiv, e.fused = int(history), int(ldiv), int(fused)
    for struct, fields in ((o, opts), (e, ext)):
        for name, val in dict(fields).items():
            if val is not None:
                setattr(struct, name, val)
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
    def _wrap_matvec(self, f: Optional[Callable]):
        if f is None:
            return _lib.MATVEC(), None
        n, dt = self.n, self.dtype
        if self.device == "cuda":
            raise B200Error("Python callables are host operators; create the workspace with device='host'")

        def tramp(xp, yp, _ud):
            x = np.ctypeslib.as_array(C.cast(xp, C.POINTER(C.c_byte)), shape=(n * dt.itemsize,)).view(dt)
            y = np.ctypeslib.as_array(C.cast(yp, C.POINTER(C.c_byte)), shape=(n * dt.itemsize,)).view(dt)
            y[:] = f(x)
        cb = _lib.MATVEC(tramp)
        return cb, cb

    def solve(self, A, b, *, c=None, M=None, N=None, atol=None, rtol=None, itmax=0, timemax=math.inf, verbose=0,
              history=False, callback=None, radius=0.0, linesearch=False, lambda_=0.0, etol=None, conlim=None,
              restart=False, reorthogonalization=False, ldiv=False, fused=True, batch=0, time_kernels=False,
              check_curvature=False, gamma=None, artol=None):
        """solver!(ws, A, b; kwargs...)  -- kwargs as in cg.jl:100-111, gmres.jl:96-108,
        bicgstab.jl:105-116, minres.jl:138-151.  M / N: None (identity), a 1-D array
        (Diagonal preconditioner) or a host callable."""
        o, e = _options(atol, rtol, itmax, timemax, verbose, history, ldiv, fused,
                        opts=dict(radius=float(radius), linesearch=int(linesearch), lambda_=float(lambda_),
                                  restart=int(restart), reorthogonalization=int(reorthogonalization)),
                        ext=dict(batch=int(batch), time_kernels=int(time_kernels), check_curvature=int(check_curvature),
                                 cr_gamma=_float(gamma), etol=_float(etol), conlim=_float(conlim),
                                 axtol=_float(artol)))   # MINARES's Artol travels in the axtol field
        keep = [self._set_options(e, callback)]
        fA = None
        if callable(A) and not hasattr(A, "shape"):
            fA, k = self._wrap_matvec(A)
            keep.append(k)
        elif A is not None:
            self.set_operator(A)
        fM = fN = None
        for which, P in ((0, M), (1, N)):
            if P is None:
                self._set_diag(which, None)
            elif callable(P) and not hasattr(P, "shape"):
                f, k = self._wrap_matvec(P)
                keep.append(k)
                if which == 0:
                    fM = f
                else:
                    fN = f
                self._set_diag(which, None)
            else:
                self._set_diag(which, P)
        return self._solve_staged(o, fA, None, fM, fN, b, c, self.m)

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

    def warm_start(self, x0):
        if not _is_torch(x0):
            x0 = np.ascontiguousarray(x0, dtype=self.dtype)
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
    def stats(self) -> SimpleStats:
        s = KrylovB200Stats()
        if lib().krylov_b200_get_stats(self._h, C.byref(s)) != 0:
            raise B200Error(_lib.last_error())

        def hist(which, cnt):
            buf = (C.c_double * max(cnt, 1))()
            k = lib().krylov_b200_get_history(self._h, which, buf, cnt)
            return list(buf[:max(k, 0)])
        out = SimpleStats(s.niter, bool(s.solved), bool(s.inconsistent), bool(s.indefinite), s.npcCount,
                          hist(0, s.nresiduals), hist(1, s.nAresiduals), hist(2, s.nAcond), s.allocation_timer, s.timer,
                          s.status.decode("utf-8"))
        out.Anorm = s.Anorm          # LanczosStats.Anorm (cg_lanczos!), NaN otherwise
        if self.solver == "lslq":    # LSLQStats (src/krylov_stats.jl:352-365)
            out.err_lbnds, out.err_ubnds_lq = hist(3, s.nerr_lbnds), hist(4, s.nerr_ubnds_lq)
            out.err_ubnds_cg, out.error_with_bnd = hist(5, s.nerr_ubnds_cg), bool(s.error_with_bnd)
        elif self.solver == "lnlq":  # LNLQStats (src/krylov_stats.jl): the bounds travel in LSLQ's history slots 3 and 4
            out.error_bnd_x, out.error_bnd_y = hist(3, s.nerr_lbnds), hist(4, s.nerr_ubnds_lq)
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


class CgWorkspace(KrylovWorkspace):
    solver = "cg"


class MinresWorkspace(KrylovWorkspace):
    solver = "minres"


class GmresWorkspace(KrylovWorkspace):
    solver = "gmres"


class BicgstabWorkspace(KrylovWorkspace):
    solver = "bicgstab"
    nA = 2


# sibling solvers on the same kernels (SURVEY.md 8f-3)
class FomWorkspace(KrylovWorkspace):
    solver = "fom"


class FgmresWorkspace(KrylovWorkspace):
    solver = "fgmres"


class CgsWorkspace(KrylovWorkspace):
    solver = "cgs"
    nA = 2


class CgLanczosWorkspace(KrylovWorkspace):
    solver = "cg_lanczos"


class CrWorkspace(KrylovWorkspace):
    solver = "cr"


class DiomWorkspace(KrylovWorkspace):
    solver = "diom"


class DqgmresWorkspace(KrylovWorkspace):
    solver = "dqgmres"


class CarWorkspace(KrylovWorkspace):
    solver = "car"

    def solve(self, A, b, *, M=None, ldiv=False, atol=None, rtol=None, itmax=0, timemax=math.inf, verbose=0,
              history=False, callback=None, fused=True, **unknown):
        """car!(ws, A, b; kwargs...)  -- kwargs as in car.jl:90-99: atol and rtol default to sqrt(eps), itmax = 0
        means 2n.  M: None, the diagonal of a Diagonal preconditioner, or a host callable."""
        if unknown:
            raise B200Error(f"car!: unsupported keyword argument(s) {', '.join(sorted(unknown))}")
        return super().solve(A, b, M=M, ldiv=ldiv, atol=atol, rtol=rtol, itmax=itmax, timemax=timemax, verbose=verbose,
                             history=history, callback=callback, fused=fused)


class MinaresWorkspace(KrylovWorkspace):
    solver = "minares"

    def solve(self, A, b, *, M=None, ldiv=False, lambda_=0.0, atol=None, rtol=None, artol=None, itmax=0,
              timemax=math.inf, verbose=0, history=False, callback=None, fused=True, **unknown):
        """minares!(ws, A, b; kwargs...)  -- kwargs as in minares.jl:93-104 (λ is lambda_, Artol is artol; atol, rtol
        and artol default to sqrt(eps)).  M must be None: the reference does not support preconditioners yet."""
        if unknown:
            raise B200Error(f"minares!: unsupported keyword argument(s) {', '.join(sorted(unknown))}")
        return super().solve(A, b, M=M, ldiv=ldiv, lambda_=lambda_, atol=atol, rtol=rtol, artol=artol, itmax=itmax,
                             timemax=timemax, verbose=verbose, history=history, callback=callback, fused=fused)


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


class _LeastSquaresWorkspace(KrylovWorkspace):
    """Workspace of lsqr! / lsmr! on an m x n operator (src/krylov_workspaces.jl LsqrWorkspace / LsmrWorkspace):
    b has m entries, x has n.  `window` (default 5) sizes the forward-error window."""
    _N_on_residual_space = False    # CGNE / CRMR: N acts on the m-dimensional residual space

    def _wrap_rect(self, f, nin, nout):
        """Host callback y = f(x) with len(x) = nin and len(y) = nout (staged through pinned memory)."""
        if self.device == "cuda":
            raise B200Error("Python callables are host operators; create the workspace with device='host'")
        dt = self.dtype

        def tramp(xp, yp, _ud):
            x = np.ctypeslib.as_array(C.cast(xp, C.POINTER(C.c_byte)), shape=(nin * dt.itemsize,)).view(dt)
            y = np.ctypeslib.as_array(C.cast(yp, C.POINTER(C.c_byte)), shape=(nout * dt.itemsize,)).view(dt)
            y[:] = f(x)
        return _lib.MATVEC(tramp)

    def solve(self, A, b, *, M=None, N=None, ldiv=False, sqd=False, lambda_=0.0, radius=0.0, etol=None, axtol=None,
              btol=None, conlim=None, atol=0.0, rtol=0.0, itmax=0, timemax=math.inf, verbose=0, history=False,
              callback=None, fused=True):
        """lsqr!(ws, A, b; kwargs...) / lsmr!(ws, A, b; kwargs...)  -- kwargs as in lsqr.jl:145-162 (atol and rtol
        default to 0 as in Julia; etol, axtol, btol default to sqrt(eps), conlim to 1/sqrt(eps)).

        A: a SciPy matrix, a CsrOperator or a (rowptr, colind, values) tuple (uploaded as a CSR operator), or a
        scipy.sparse.linalg.LinearOperator / (matvec, rmatvec) pair of host callables.  M (m entries) and N (n entries):
        None, the diagonal of a Diagonal preconditioner, or a host callable."""
        if sqd and lambda_ != 0:
            raise B200Error("sqd cannot be set to true if λ ≠ 0 !")
        if sqd:
            lambda_ = 1.0
        o, e = _options(atol, rtol, itmax, timemax, verbose, history, ldiv, fused,
                        opts=dict(radius=float(radius), lambda_=float(lambda_)),
                        ext=dict(etol=_float(etol), axtol=_float(axtol), btol=_float(btol), conlim=_float(conlim)))
        return self._run(A, b, M, N, o, e, callback)

    def _run(self, A, b, M, N, o, e, callback, c=None, c_len=None):
        """Set the options, the operator pair and the preconditioners, stage b (and c, of c_len entries, default m) and
        call krylov_solve."""
        m, n = self.m, self.n
        keep = [self._set_options(e, callback)]
        fA = fAt = None
        if hasattr(A, "matvec") and hasattr(A, "rmatvec") and not isinstance(A, CsrOperator):   # LinearOperator
            fA, fAt = self._wrap_rect(A.matvec, n, m), self._wrap_rect(A.rmatvec, m, n)
        elif isinstance(A, tuple) and len(A) == 2 and all(callable(f) for f in A):
            fA, fAt = self._wrap_rect(A[0], n, m), self._wrap_rect(A[1], m, n)
        elif A is not None:
            self.set_operator(A)
        keep += [fA, fAt]
        fP = [None, None]
        for which, (P, ln) in enumerate(((M, m), (N, m if self._N_on_residual_space else n))):
            if P is not None and callable(P) and not hasattr(P, "shape"):
                fP[which] = self._wrap_rect(P, ln, ln)
                keep.append(fP[which])
                self._set_diag(which, None)
            else:
                if P is not None and getattr(P, "ndim", 1) != 1:
                    raise B200Error(f"{self.solver} takes diagonal preconditioners (1-D arrays) or host callables")
                self._set_diag(which, P)
        return self._solve_staged(o, fA, fAt, fP[0], fP[1], b, c, m if c_len is None else c_len)


class LsqrWorkspace(_LeastSquaresWorkspace):
    solver = "lsqr"


class LsmrWorkspace(_LeastSquaresWorkspace):
    solver = "lsmr"


class LslqWorkspace(_LeastSquaresWorkspace):
    """Workspace of lslq! on an m x n operator (src/krylov_workspaces.jl LslqWorkspace): b has m entries, x has n;
    `window` (default 5) sizes the forward-error window."""
    solver = "lslq"

    def solve(self, A, b, *, M=None, N=None, ldiv=False, transfer_to_lsqr=False, sqd=False, lambda_=0.0, sigma=0.0,
              etol=None, utol=None, btol=None, conlim=None, atol=None, rtol=None, itmax=0, timemax=math.inf, verbose=0,
              history=False, callback=None, fused=True, **unknown):
        """lslq!(ws, A, b; kwargs...)  -- kwargs as in lslq.jl:178-196: etol, utol, btol, atol and rtol default to
        sqrt(eps), conlim to 1/sqrt(eps); σ (`sigma`) > 0 turns on the Gauss-Radau error bounds.  M (m entries) and N
        (n entries): None, the diagonal of a Diagonal preconditioner, or a host callable."""
        if unknown:
            raise B200Error(f"lslq!: unsupported keyword argument(s) {', '.join(sorted(unknown))}")
        if sqd and lambda_ != 0:
            raise B200Error("sqd cannot be set to true if λ ≠ 0 !")
        if sqd:
            lambda_ = 1.0
        o, e = _options(atol, rtol, itmax, timemax, verbose, history, ldiv, fused, opts=dict(lambda_=float(lambda_)),
                        ext=dict(sigma=float(sigma), transfer_to_lsqr=int(transfer_to_lsqr), etol=_float(etol),
                                 utol=_float(utol), btol=_float(btol), conlim=_float(conlim)))
        return self._run(A, b, M, N, o, e, callback)


class _NormalEquationsWorkspace(_LeastSquaresWorkspace):
    """Workspace of cgls! / crls! on an m x n operator (src/krylov_workspaces.jl CglsWorkspace / CrlsWorkspace):
    b has m entries, x has n."""

    def solve(self, A, b, *, M=None, ldiv=False, radius=0.0, lambda_=0.0, atol=None, rtol=None, itmax=0,
              timemax=math.inf, verbose=0, history=False, callback=None, fused=True, **unknown):
        """cgls!(ws, A, b; kwargs...) / crls!(ws, A, b; kwargs...)  -- kwargs as in cgls.jl:110-121 and
        crls.jl:101-112: atol and rtol default to sqrt(eps), itmax = 0 means m + n.  M (m entries) acts on the residual
        space: None, the diagonal of a Diagonal preconditioner, or a host callable.  There is no N."""
        if unknown:
            raise B200Error(f"{self.solver}!: unsupported keyword argument(s) {', '.join(sorted(unknown))}")
        o, e = _options(atol, rtol, itmax, timemax, verbose, history, ldiv, fused,
                        opts=dict(radius=float(radius), lambda_=float(lambda_)))
        return self._run(A, b, M, None, o, e, callback)


class CglsWorkspace(_NormalEquationsWorkspace):
    solver = "cgls"


class CrlsWorkspace(_NormalEquationsWorkspace):
    solver = "crls"


class _BiorthWorkspace(_LeastSquaresWorkspace):
    """Workspace of bilq! / qmr! on a square operator (src/krylov_workspaces.jl BilqWorkspace / QmrWorkspace).  Both
    apply A and its adjoint: a CSR operator (its transpose is formed once and cached), or a
    scipy.sparse.linalg.LinearOperator / (matvec, rmatvec) pair of host callables."""
    nA = 2

    def _solve(self, A, b, c, M, N, ldiv, atol, rtol, itmax, timemax, verbose, history, callback, fused, unknown,
               transfer_to_bicg=True):
        if unknown:
            raise B200Error(f"{self.solver}!: unsupported keyword argument(s) {', '.join(sorted(unknown))}")
        o, e = _options(atol, rtol, itmax, timemax, verbose, history, ldiv, fused,
                        ext=dict(transfer_to_bicg=int(transfer_to_bicg)))
        return self._run(A, b, M, N, o, e, callback, c)


class BilqWorkspace(_BiorthWorkspace):
    solver = "bilq"

    def solve(self, A, b, *, c=None, transfer_to_bicg=True, M=None, N=None, ldiv=False, atol=None, rtol=None, itmax=0,
              timemax=math.inf, verbose=0, history=False, callback=None, fused=True, **unknown):
        """bilq!(ws, A, b; kwargs...)  -- kwargs as in bilq.jl:97-109: c defaults to b, atol and rtol to sqrt(eps),
        itmax = 0 means 2n.  M, N: None, the diagonal of a Diagonal preconditioner, or a self-adjoint host callable."""
        return self._solve(A, b, c, M, N, ldiv, atol, rtol, itmax, timemax, verbose, history, callback, fused, unknown,
                           transfer_to_bicg)


class QmrWorkspace(_BiorthWorkspace):
    solver = "qmr"

    def solve(self, A, b, *, c=None, M=None, N=None, ldiv=False, atol=None, rtol=None, itmax=0, timemax=math.inf,
              verbose=0, history=False, callback=None, fused=True, **unknown):
        """qmr!(ws, A, b; kwargs...)  -- kwargs as in qmr.jl:104-115 (defaults as for bilq!)."""
        return self._solve(A, b, c, M, N, ldiv, atol, rtol, itmax, timemax, verbose, history, callback, fused, unknown)


class _AdjointWorkspace(_LeastSquaresWorkspace):
    """Workspace of bilqr! / trilqr! (src/krylov_workspaces.jl BilqrWorkspace / TrilqrWorkspace): the primal system
    A x = b and the adjoint system A^T y = c, solved together.  A is m x n (square for BiLQR): b and y have m entries,
    c and x have n.  Both apply A and its adjoint: a CSR operator (its transpose is formed once and cached), or a
    scipy.sparse.linalg.LinearOperator / (matvec, rmatvec) pair of host callables.  Neither takes a preconditioner."""
    nA = 2

    def _solve(self, A, b, c, transfer, atol, rtol, itmax, timemax, verbose, history, callback, fused, unknown):
        if unknown:
            raise B200Error(f"{self.solver}!: unsupported keyword argument(s) {', '.join(sorted(unknown))}")
        if c is None:
            raise B200Error(f"{self.solver}! solves A^T y = c as well: c must be given")
        # TriLQR's transfer_to_usymcg travels in the transfer_to_bicg field
        o, e = _options(atol, rtol, itmax, timemax, verbose, history, False, fused, ext=dict(transfer_to_bicg=int(transfer)))
        return self._run(A, b, None, None, o, e, callback, c, c_len=self.n)

    def warm_start(self, x0, y0):
        """warm_start!(workspace, x0, y0): x0 has n entries, y0 m."""
        if not _is_torch(x0):
            x0 = np.ascontiguousarray(x0, dtype=self.dtype)
        if not _is_torch(y0):
            y0 = np.ascontiguousarray(y0, dtype=self.dtype)
        px, kx = _ptr(x0)
        py, ky = _ptr(y0)
        self._order_after(kx, ky)
        if lib().krylov_warm_start2(self._h, px, py, int(x0.shape[0]), int(y0.shape[0])) != 0:
            raise B200Error(_lib.last_error())
        return self

    @property
    def y(self):
        """The solution of A^T y = c: a host copy (or a torch CUDA tensor for device workspaces)."""
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
    def stats(self) -> AdjointStats:
        s = KrylovB200Stats()
        if lib().krylov_b200_get_stats(self._h, C.byref(s)) != 0:
            raise B200Error(_lib.last_error())

        def hist(which, cnt):
            buf = (C.c_double * max(cnt, 1))()
            k = lib().krylov_b200_get_history(self._h, which, buf, cnt)
            return list(buf[:max(k, 0)])
        return AdjointStats(s.niter, bool(s.solved_primal), bool(s.solved_dual), hist(0, s.nresiduals),
                            hist(6, s.nresiduals_dual), s.timer, s.status.decode("utf-8"))


class BilqrWorkspace(_AdjointWorkspace):
    solver = "bilqr"

    def solve(self, A, b, c, *, transfer_to_bicg=True, atol=None, rtol=None, itmax=0, timemax=math.inf, verbose=0,
              history=False, callback=None, fused=True, **unknown):
        """bilqr!(ws, A, b, c; kwargs...)  -- kwargs as in bilqr.jl:99-107: atol and rtol default to sqrt(eps),
        itmax = 0 means 2n."""
        return self._solve(A, b, c, transfer_to_bicg, atol, rtol, itmax, timemax, verbose, history, callback, fused,
                           unknown)


class TrilqrWorkspace(_AdjointWorkspace):
    solver = "trilqr"

    def solve(self, A, b, c, *, transfer_to_usymcg=True, atol=None, rtol=None, itmax=0, timemax=math.inf, verbose=0,
              history=False, callback=None, fused=True, **unknown):
        """trilqr!(ws, A, b, c; kwargs...)  -- kwargs as in trilqr.jl: atol and rtol default to sqrt(eps), itmax = 0
        means m + n.  A is m x n, b has m entries and c n."""
        return self._solve(A, b, c, transfer_to_usymcg, atol, rtol, itmax, timemax, verbose, history, callback, fused,
                           unknown)


class _LeastNormWorkspace(_LeastSquaresWorkspace):
    """Workspace of craig! / craigmr! on an m x n operator (src/krylov_workspaces.jl CraigWorkspace / CraigmrWorkspace):
    the least-norm solution of A x = b, x = A^T y.  b and y have m entries, x has n.  A and its adjoint: a CSR operator
    (its transpose is formed once and cached), or a scipy.sparse.linalg.LinearOperator / (matvec, rmatvec) pair of host
    callables.  M (m entries) and N (n entries): None, the diagonal of a Diagonal preconditioner, or a host callable."""
    nA = 2

    def _solve(self, A, b, M, N, ldiv, sqd, lambda_, atol, rtol, itmax, timemax, verbose, history, callback, fused,
               unknown, transfer_to_lsqr=False, btol=None, conlim=None, ext=None):
        if unknown:
            raise B200Error(f"{self.solver}!: unsupported keyword argument(s) {', '.join(sorted(unknown))}")
        if sqd and lambda_ != 0:
            raise B200Error("sqd cannot be set to true if λ ≠ 0 !")
        if sqd:
            lambda_ = 1.0
        o, e = _options(atol, rtol, itmax, timemax, verbose, history, ldiv, fused, opts=dict(lambda_=float(lambda_)),
                        ext=dict(dict(transfer_to_lsqr=int(transfer_to_lsqr), btol=_float(btol), conlim=_float(conlim)),
                                 **(ext or {})))
        return self._run(A, b, M, N, o, e, callback)

    y = _AdjointWorkspace.y


class CraigWorkspace(_LeastNormWorkspace):
    solver = "craig"

    def solve(self, A, b, *, M=None, N=None, ldiv=False, transfer_to_lsqr=False, sqd=False, lambda_=0.0, btol=None,
              conlim=None, atol=None, rtol=None, itmax=0, timemax=math.inf, verbose=0, history=False, callback=None,
              fused=True, **unknown):
        """craig!(ws, A, b; kwargs...)  -- kwargs as in craig.jl:151-166: btol, atol and rtol default to sqrt(eps),
        conlim to 1/sqrt(eps), itmax = 0 means m + n; transfer_to_lsqr acts when λ > 0."""
        return self._solve(A, b, M, N, ldiv, sqd, lambda_, atol, rtol, itmax, timemax, verbose, history, callback, fused,
                           unknown, transfer_to_lsqr, btol, conlim)


class CraigmrWorkspace(_LeastNormWorkspace):
    solver = "craigmr"

    def solve(self, A, b, *, M=None, N=None, ldiv=False, sqd=False, lambda_=0.0, atol=None, rtol=None, itmax=0,
              timemax=math.inf, verbose=0, history=False, callback=None, fused=True, **unknown):
        """craigmr!(ws, A, b; kwargs...)  -- kwargs as in craigmr.jl:141-153: atol and rtol default to sqrt(eps),
        itmax = 0 means m + n."""
        return self._solve(A, b, M, N, ldiv, sqd, lambda_, atol, rtol, itmax, timemax, verbose, history, callback, fused,
                           unknown)


class LnlqWorkspace(_LeastNormWorkspace):
    solver = "lnlq"

    def solve(self, A, b, *, M=None, N=None, ldiv=False, transfer_to_craig=True, sqd=False, lambda_=0.0, sigma=0.0,
              utolx=None, utoly=None, atol=None, rtol=None, itmax=0, timemax=math.inf, verbose=0, history=False,
              callback=None, fused=True, **unknown):
        """lnlq!(ws, A, b; kwargs...)  -- kwargs as in lnlq.jl:144-160: utolx, utoly, atol and rtol default to sqrt(eps),
        itmax = 0 means m + n; σ (`sigma`) > 0, or λ > 0, turns on the upper bounds on ‖x - x*‖ and ‖y - y*‖
        (stats.error_bnd_x / error_bnd_y)."""
        ext = {"sigma": float(sigma), "transfer_to_bicg": int(transfer_to_craig)}
        for name, val in (("utol", utolx), ("etol", utoly)):          # the C ABI carries utolx in utol, utoly in etol
            if val is not None:
                ext[name] = float(val)
        return self._solve(A, b, M, N, ldiv, sqd, lambda_, atol, rtol, itmax, timemax, verbose, history, callback, fused,
                           unknown, ext=ext)


class _NormalLeastNormWorkspace(_LeastSquaresWorkspace):
    """Workspace of cgne! / crmr! on an m x n operator (src/krylov_workspaces.jl CgneWorkspace / CrmrWorkspace): the
    least-norm solution of A x = b by CG / CR on A A^T y = b, x = A^T y.  b has m entries, x has n; only x is returned.
    A and its adjoint: a CSR operator (its transpose is formed once and cached), or a scipy.sparse.linalg.LinearOperator
    / (matvec, rmatvec) pair of host callables.  N (m entries) acts on the residual space: None, the diagonal of a
    Diagonal preconditioner, or a host callable.  There is no M."""
    nA = 2
    _N_on_residual_space = True

    def solve(self, A, b, *, N=None, ldiv=False, lambda_=0.0, atol=None, rtol=None, itmax=0, timemax=math.inf,
              verbose=0, history=False, callback=None, fused=True, **unknown):
        """cgne!(ws, A, b; kwargs...) / crmr!(ws, A, b; kwargs...)  -- kwargs as in cgne.jl:116-126 and
        crmr.jl:114-124: atol and rtol default to sqrt(eps), itmax = 0 means m + n, λ (`lambda_`) >= 0."""
        if unknown:
            raise B200Error(f"{self.solver}!: unsupported keyword argument(s) {', '.join(sorted(unknown))}")
        o, e = _options(atol, rtol, itmax, timemax, verbose, history, ldiv, fused, opts=dict(lambda_=float(lambda_)))
        return self._run(A, b, None, N, o, e, callback)


class CgneWorkspace(_NormalLeastNormWorkspace):
    solver = "cgne"


class CrmrWorkspace(_NormalLeastNormWorkspace):
    solver = "crmr"


def _one_shot(name, b, n, run, **ws_kw):
    """Create the workspace of `name` (m = len(b) rows, n columns) for b's element type and place, return run(ws) and
    free it.  The element type of a torch b is read without copying it to the host."""
    if _is_torch(b):
        import torch
        dt = {torch.float32: np.float32, torch.float64: np.float64}.get(b.dtype, np.float64)
    else:
        dt = np.asarray(b).dtype
    if dt not in (np.float32, np.float64):
        dt = np.float64
    ws = _WS[name](b.shape[0], int(n), dt, device="cuda" if _is_torch(b) else "host", **ws_kw)
    try:
        return run(ws)
    finally:
        ws.free()


def _columns(name, A, n):
    if n is None:
        if not hasattr(A, "shape"):
            raise B200Error(f"{name}: pass n= (number of columns) with a tuple operator")
        n = A.shape[1]
    return n


def _make_least_norm(name):
    def f(A, b, x0=None, *, n=None, **kw):
        if x0 is not None:
            raise B200Error(f"{name} does not support warm-start (it takes no x0)")

        def run(ws):
            ws.solve(A, b, **kw)
            return ws.x, ws.y, ws.stats
        return _one_shot(name, b, _columns(name, A, n), run)
    f.__name__ = name
    f.__doc__ = f"(x, y, stats) = {name}(A, b; kwargs...)  (src/{name}.jl); A is m x n, b has m entries, x = A^T y"
    return f


def _make_normal_least_norm(name):
    def f(A, b, x0=None, *, n=None, **kw):
        if x0 is not None:
            raise B200Error(f"{name} does not support warm-start (it takes no x0)")

        def run(ws):
            ws.solve(A, b, **kw)
            return ws.x, ws.stats
        return _one_shot(name, b, _columns(name, A, n), run)
    f.__name__ = name
    f.__doc__ = f"(x, stats) = {name}(A, b; kwargs...)  (src/{name}.jl); A is m x n, b has m entries, x = A^T y"
    return f


def _make_adjoint(name):
    def f(A, b, c, x0=None, y0=None, **kw):
        def run(ws):
            if (x0 is None) != (y0 is None):
                raise B200Error(f"{name}: pass both x0 and y0, or neither")
            if x0 is not None:
                ws.warm_start(x0, y0)
            ws.solve(A, b, c, **kw)
            return ws.x, ws.y, ws.stats
        return _one_shot(name, b, c.shape[0], run)
    f.__name__ = name
    f.__doc__ = f"(x, y, stats) = {name}(A, b, c[, x0, y0]; kwargs...)  (src/{name}.jl); A is m x n, b has m entries, c n"
    return f


def _make_adjoint_inplace(name):
    def f(ws, A, b, c, x0=None, y0=None, **kw):
        if ws.solver != name:
            raise B200Error(f"{name}! needs a {_WS[name].__name__}")
        if (x0 is None) != (y0 is None):
            raise B200Error(f"{name}!: pass both x0 and y0, or neither")
        if x0 is not None:
            ws.warm_start(x0, y0)
        return ws.solve(A, b, c, **kw)
    f.__name__ = name + "_"
    f.__doc__ = f"{name}!(workspace, A, b, c[, x0, y0]; kwargs...)"
    return f


def _make_least_squares(name):
    def f(A, b, *, n=None, window=0, **kw):
        def run(ws):
            ws.solve(A, b, **kw)
            return ws.x, ws.stats
        return _one_shot(name, b, _columns(name, A, n), run, window=window)
    f.__name__ = name
    f.__doc__ = f"(x, stats) = {name}(A, b; window=5, kwargs...)  (src/{name}.jl); A is m x n, b has m entries"
    return f


_WS = {"cg": CgWorkspace, "minres": MinresWorkspace, "gmres": GmresWorkspace, "bicgstab": BicgstabWorkspace,
       "fom": FomWorkspace, "fgmres": FgmresWorkspace, "cgs": CgsWorkspace, "cg_lanczos": CgLanczosWorkspace,
       "cr": CrWorkspace, "diom": DiomWorkspace, "dqgmres": DqgmresWorkspace, "lsqr": LsqrWorkspace,
       "lsmr": LsmrWorkspace, "cgls": CglsWorkspace, "crls": CrlsWorkspace,
       "lslq": LslqWorkspace, "bilq": BilqWorkspace, "qmr": QmrWorkspace, "car": CarWorkspace,
       "minares": MinaresWorkspace, "bilqr": BilqrWorkspace, "trilqr": TrilqrWorkspace, "craig": CraigWorkspace,
       "craigmr": CraigmrWorkspace, "lnlq": LnlqWorkspace, "cgne": CgneWorkspace, "crmr": CrmrWorkspace}


def krylov_workspace(method: str, *args, **kw) -> KrylovWorkspace:
    """krylov_workspace(Val(method), ...)  (src/interface.jl:248-348)"""
    if method not in _WS:
        raise B200Error(f"method {method!r} is outside the GPU path ({', '.join(sorted(_WS))})")
    return _WS[method](*args, **kw)


def krylov_solve_(ws: KrylovWorkspace, A, b, x0=None, **kw) -> KrylovWorkspace:
    """krylov_solve!(ws, A, b[, x0]; kw...)"""
    if x0 is not None:
        ws.warm_start(x0)
    return ws.solve(A, b, **kw)


def _make_inplace(name):
    def f(ws, A, b, x0=None, **kw):
        if ws.solver != name:
            raise B200Error(f"{name}! needs a {_WS[name].__name__}")
        return krylov_solve_(ws, A, b, x0, **kw)
    f.__name__ = name + "_"
    f.__doc__ = f"{name}!(workspace, A, b[, x0]; kwargs...)"
    return f


def _make_outofplace(name):
    def f(A, b, x0=None, *, memory=0, window=0, **kw):
        def run(ws):
            krylov_solve_(ws, A, b, x0, **kw)
            return ws.x, ws.stats
        return _one_shot(name, b, b.shape[0], run, memory=memory, window=window)
    f.__name__ = name
    f.__doc__ = f"(x, stats) = {name}(A, b[, x0]; kwargs...)"
    return f


cg_, gmres_, bicgstab_, minres_ = (_make_inplace(s) for s in ("cg", "gmres", "bicgstab", "minres"))
cg, gmres, bicgstab, minres = (_make_outofplace(s) for s in ("cg", "gmres", "bicgstab", "minres"))
fom_, fgmres_, cgs_, cg_lanczos_ = (_make_inplace(s) for s in ("fom", "fgmres", "cgs", "cg_lanczos"))
fom, fgmres, cgs, cg_lanczos = (_make_outofplace(s) for s in ("fom", "fgmres", "cgs", "cg_lanczos"))
cr_, diom_, dqgmres_ = (_make_inplace(s) for s in ("cr", "diom", "dqgmres"))
cr, diom, dqgmres = (_make_outofplace(s) for s in ("cr", "diom", "dqgmres"))
lsqr_, lsmr_ = (_make_inplace(s) for s in ("lsqr", "lsmr"))
lsqr, lsmr = (_make_least_squares(s) for s in ("lsqr", "lsmr"))
cgls_, crls_, lslq_ = (_make_inplace(s) for s in ("cgls", "crls", "lslq"))
cgls, crls, lslq = (_make_least_squares(s) for s in ("cgls", "crls", "lslq"))
bilq_, qmr_ = (_make_inplace(s) for s in ("bilq", "qmr"))
bilq, qmr = (_make_outofplace(s) for s in ("bilq", "qmr"))
car_, minares_ = (_make_inplace(s) for s in ("car", "minares"))
car, minares = (_make_outofplace(s) for s in ("car", "minares"))
bilqr_, trilqr_ = (_make_adjoint_inplace(s) for s in ("bilqr", "trilqr"))
bilqr, trilqr = (_make_adjoint(s) for s in ("bilqr", "trilqr"))
craig_, craigmr_ = (_make_inplace(s) for s in ("craig", "craigmr"))
craig, craigmr = (_make_least_norm(s) for s in ("craig", "craigmr"))
lnlq_, lnlq = _make_inplace("lnlq"), _make_least_norm("lnlq")
cgne_, crmr_ = (_make_inplace(s) for s in ("cgne", "crmr"))
cgne, crmr = (_make_normal_least_norm(s) for s in ("cgne", "crmr"))


def krylov_solve(method: str, A, b, x0=None, **kw):
    return {"cg": cg, "gmres": gmres, "bicgstab": bicgstab, "minres": minres, "fom": fom, "fgmres": fgmres, "cgs": cgs,
            "cg_lanczos": cg_lanczos, "cr": cr, "diom": diom, "dqgmres": dqgmres, "bilq": bilq,
            "qmr": qmr, "car": car, "minares": minares, "craig": craig, "craigmr": craigmr,
            "lnlq": lnlq, "cgne": cgne, "crmr": crmr}[method](A, b, x0, **kw)


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
