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
import inspect
import math
import os
import subprocess
from typing import NamedTuple

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


_TOLERANCES = ("atol", "rtol", "etol", "axtol", "btol", "utol", "utolx", "utoly", "conlim", "artol")


class Options(C.Structure):
    """oracle_options (krylov_oracle_impl.h): the keyword arguments of every solver."""
    _fields_ = ([(f, C.c_double) for f in _TOLERANCES + ("lambda_", "sigma", "radius", "gamma")]
                + [(f, C.c_int) for f in ("itmax", "history", "window", "memory", "restart", "reorthogonalization",
                                          "linesearch", "ldiv", "check_curvature", "transfer_to_lsqr",
                                          "transfer_to_craig", "transfer")]
                + [("timemax", C.c_double), ("callback", _ITER_CB), ("cb_user", C.c_void_p), ("hist_cap", C.c_int)])

    def __init__(self):
        super().__init__(**{f: math.nan for f in _TOLERANCES + ("gamma",)}, timemax=-1.0)


class Problem(C.Structure):
    """problem_f32 / problem_f64: A (m x n) and Aᵀ as CSR, and the vectors; NULL where not given."""
    _fields_ = [("m", C.c_int), ("n", C.c_int)] + [(f, C.c_void_p) for f in (
        "rowptr", "colind", "val", "trowptr", "tcolind", "tval", "b", "c", "x0", "y0", "M", "N")]


_HISTORIES = ("residuals", "Aresiduals", "Acond", "err_lbnds", "err_ubnds_lq", "err_ubnds_cg", "error_bnd_x",
              "error_bnd_y", "residuals_dual")


def _outputs_type(ct):
    """outputs_f32 / outputs_f64: the solutions, the histories (residuals counted in Stats.nres, Aresiduals and Acond
    in Stats.nAres, the others in n_<name>), the npc direction and the scalar results."""
    class Outputs(C.Structure):
        _fields_ = ([(f, C.c_void_p) for f in ("x", "y") + _HISTORIES]
                    + [("n_" + h, C.c_int) for h in _HISTORIES[3:]]
                    + [("npc_dir", C.c_void_p), ("Anorm", ct), ("error_with_bnd", C.c_int),
                       ("solved_primal", C.c_int), ("solved_dual", C.c_int)])
    return Outputs


_OUTPUTS = {C.c_double: _outputs_type(C.c_double), C.c_float: _outputs_type(C.c_float)}


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


# ---- the solvers: one row per solver, one solve path ----------------------------------------------------------------
_REQUIRED = inspect.Parameter.empty
_VECTORS = ("c", "x0", "y0", "M", "N")
# The keyword arguments every square solver accepts (each reads those its reference signature has), hist_cap included.
_SQUARE_KW = dict(atol=math.nan, rtol=math.nan, itmax=0, history=True, radius=0.0, linesearch=False, lambda_=0.0,
                  etol=math.nan, conlim=math.nan, window=0, memory=0, restart=False, reorthogonalization=False,
                  ldiv=False, hist_cap=None)
_STOP = (("timemax", math.inf), ("callback", None))
_SIMPLE = ("niter", "solved", "inconsistent", "indefinite", "npcCount", "error", "status", "residuals")  # SimpleStats
_LEASTNORM = ("niter", "solved", "inconsistent", "status", "residuals")
_ADJOINT = ("niter", "solved", "solved_primal", "solved_dual", "status", "residuals_primal", "residuals_dual")


def _trust_region_error(rc, st):
    return rc and {12: "zero direction", 13: "outside of the trust region"}.get(rc, "no real roots")


def _cr_error(rc, st):
    return rc and {1: "'linesearch' set to 'true' but radius > 0", 2: "warm_start and linesearch cannot be used together",
                   5: "Indefinite system and no trust region"}.get(rc, f"to_boundary error {rc - 10}")


def _status_error(rc, st):
    return st["error"] and st["status"]


class _Solver(NamedTuple):
    doc: str
    params: tuple                # positional parameters after (A, b), in order, with their defaults
    keywords: dict               # the further keyword arguments and their defaults; hist_cap=None: accepted
    stats: tuple = _SIMPLE       # the stats keys, in order
    rect: bool = False           # itmax defaults to m + n (else 2n) where the history capacity is sized
    transpose: bool = False      # the body applies Aᵀ, passed as its own CSR
    two: bool = False            # returns (x, y, stats)
    hist_extra: int = 2          # hist_cap = min(itmax + hist_extra, 2^22)
    fixed_cap: bool = False      # a hist_cap keyword is accepted and ignored
    error: object = None         # (return code, stats) -> the ArithmeticError message, or a false value


_LSQ_KW = dict(sqd=False, lambda_=0.0, atol=0.0, rtol=0.0, etol=math.nan, axtol=math.nan, btol=math.nan,   # lsqr.jl:155
               conlim=math.nan, radius=0.0, itmax=0, history=True, window=0, ldiv=False, hist_cap=None)
_CGLS_KW = dict(atol=math.nan, rtol=math.nan, lambda_=0.0, radius=0.0, itmax=0, history=True, ldiv=False, hist_cap=None)
_CRAIG_KW = dict(lambda_=0.0, sqd=False, atol=math.nan, rtol=math.nan, btol=math.nan, conlim=math.nan, itmax=0,
                 history=True, ldiv=False, transfer_to_lsqr=False)
_CGNE_KW = dict(lambda_=0.0, atol=math.nan, rtol=math.nan, itmax=0, history=True, ldiv=False)
_XMN = (("x0", None), ("M", None), ("N", None))

_SOLVERS = {
    "cg": _Solver("cg! (src/cg.jl:120-291).  M: None or the diagonal of a Diagonal preconditioner.",
                  (("x0", None), ("M", None)), _SQUARE_KW, _SIMPLE + ("npc_dir",)),
    "bicgstab": _Solver("bicgstab! (src/bicgstab.jl:125-277).", (("c", None),) + _XMN, _SQUARE_KW),
    "gmres": _Solver("gmres! (src/gmres.jl:121-384).", _XMN, _SQUARE_KW),
    "minres": _Solver("minres! (src/minres.jl:164-485).", (("x0", None), ("M", None)), _SQUARE_KW,
                      _SIMPLE + ("Aresiduals", "Acond", "npc_dir")),
    "cgs": _Solver("cgs! (src/cgs.jl:125-282).", (("c", None),) + _XMN, _SQUARE_KW),
    "cg_lanczos": _Solver("cg_lanczos! (src/cg_lanczos.jl:110-264).  Extra stats key: Anorm (LanczosStats).",
                          (("x0", None), ("M", None), ("check_curvature", False)), _SQUARE_KW, _SIMPLE + ("Anorm",)),
    "fom": _Solver("fom! (src/fom.jl:121-368).", _XMN, _SQUARE_KW),
    "fgmres": _Solver("fgmres! (src/fgmres.jl:128-388); N: None or the diagonal of a fixed right preconditioner.",
                      _XMN, _SQUARE_KW),
    "dqgmres": _Solver("dqgmres! (src/dqgmres.jl:121-335).", _XMN, _SQUARE_KW),
    "diom": _Solver("diom! (src/diom.jl:121-332).", _XMN, _SQUARE_KW, error=_status_error),
    "cr": _Solver("cr! (src/cr.jl:128-478).  Extra stats keys: Aresiduals, npc_dir.",
                  (("x0", None), ("M", None), ("gamma", math.nan)), _SQUARE_KW, _SIMPLE + ("Aresiduals", "npc_dir"),
                  error=_cr_error),
    "car": _Solver("car! (src/car.jl:108-256).  M: None or the diagonal of a Diagonal preconditioner (ldiv=True applies "
                   "its inverse); callback(iter) -> bool stops the solve when true; timemax in seconds.  Extra stats key: "
                   "Aresiduals.", (("x0", None), ("M", None)) + _STOP, _SQUARE_KW, _SIMPLE + ("Aresiduals",)),
    "minares": _Solver("minares! (src/minares.jl:113-595), M = I.  lambda_: the shift λ; artol: the kwarg Artol (None -> "
                       "sqrt(eps)).  Extra stats key: Aresiduals.",
                       (("x0", None), ("lambda_", 0.0), ("artol", None)) + _STOP, _SQUARE_KW, _SIMPLE + ("Aresiduals",)),
    "bilq": _Solver("bilq! (src/bilq.jl:118-407).  c: None (= b) or the shadow vector; M, N: None or the diagonal of a "
                    "Diagonal preconditioner; callback(iter) -> bool stops the solve when true; timemax in seconds.",
                    (("c", None),) + _XMN + (("transfer_to_bicg", True),) + _STOP, _SQUARE_KW, transpose=True),
    "qmr": _Solver("qmr! (src/qmr.jl:124-405); arguments as for bilq.", (("c", None),) + _XMN + _STOP, _SQUARE_KW,
                   transpose=True),
    "bilqr": _Solver("bilqr! (src/bilqr.jl:115-484) -> (x, y, stats).  callback(iter) -> bool stops the solve when true.",
                     (("c", _REQUIRED), ("x0", None), ("y0", None), ("transfer_to_bicg", True)) + _STOP, _SQUARE_KW,
                     _ADJOINT, transpose=True, two=True, fixed_cap=True),
    "trilqr": _Solver("trilqr! (src/trilqr.jl:114-461) -> (x, y, stats); A is m x n, b has m entries, c n.",
                      (("c", _REQUIRED), ("x0", None), ("y0", None), ("transfer_to_usymcg", True)) + _STOP, _SQUARE_KW,
                      _ADJOINT, rect=True, transpose=True, two=True, fixed_cap=True),
    "lsqr": _Solver("lsqr! (src/lsqr.jl:174-440) on an m x n matrix.  M (m) / N (n): None or the diagonal of a Diagonal "
                    "operator.\n    kwargs: lambda_, sqd, radius, etol, axtol, btol, conlim, atol, rtol (default 0), itmax, "
                    "window, ldiv, history.\n    Extra stats key: Aresiduals.",
                    (("M", None), ("N", None)), _LSQ_KW, _SIMPLE + ("Aresiduals", "Anorm"), rect=True,
                    error=_trust_region_error),
    "lsmr": _Solver("lsmr! (src/lsmr.jl:178-455); same arguments as lsqr.  Extra stats keys: Aresiduals, Anorm "
                    "(LsmrStats).", (("M", None), ("N", None)), _LSQ_KW, _SIMPLE + ("Aresiduals", "Anorm"), rect=True,
                    error=_trust_region_error),
    "cgls": _Solver("cgls! (src/cgls.jl:129-243) on an m x n matrix.  M (m entries): None or the diagonal of a Diagonal "
                    "operator.\n    kwargs: lambda_, radius, atol, rtol (default sqrt(eps)), itmax, ldiv, history.  Extra "
                    "stats key: Aresiduals.", (("M", None),), _CGLS_KW, _SIMPLE + ("Aresiduals",), rect=True,
                    error=_trust_region_error),
    "crls": _Solver("crls! (src/crls.jl:120-268); same arguments as cgls.", (("M", None),), _CGLS_KW,
                    _SIMPLE + ("Aresiduals",), rect=True, error=_trust_region_error),
    "lslq": _Solver("lslq! (src/lslq.jl:201-520) on an m x n matrix.  M (m) / N (n): None or the diagonal of a Diagonal "
                    "operator.\n    kwargs: lambda_, sqd, sigma, etol, utol, btol, conlim, atol, rtol (default "
                    "sqrt(eps)), itmax, window, ldiv,\n    transfer_to_lsqr, history.  Extra stats keys: Aresiduals, "
                    "err_lbnds, err_ubnds_lq, err_ubnds_cg, error_with_bnd.", (("M", None), ("N", None)),
                    dict(lambda_=0.0, sqd=False, sigma=0.0, atol=math.nan, rtol=math.nan, etol=math.nan, utol=math.nan,
                         btol=math.nan, conlim=math.nan, itmax=0, history=True, window=0, ldiv=False,
                         transfer_to_lsqr=False, hist_cap=None),
                    _SIMPLE + ("Aresiduals", "err_lbnds", "err_ubnds_lq", "err_ubnds_cg", "error_with_bnd"), rect=True),
    "craig": _Solver("craig! (src/craig.jl:174-405) -> (x, y, stats).  M (m) / N (n): None or the diagonal of a Diagonal "
                     "operator.\n    kwargs: lambda_, sqd, transfer_to_lsqr, btol, conlim, atol, rtol, itmax, ldiv, "
                     "history.  callback(iter) -> bool.", (("M", None), ("N", None)) + _STOP, _CRAIG_KW, _LEASTNORM,
                     rect=True, transpose=True, two=True),
    "craigmr": _Solver("craigmr! (src/craigmr.jl:161-396) -> (x, y, stats); stats also has Aresiduals.  Same arguments as "
                       "craig, without\n    transfer_to_lsqr, btol and conlim.", (("M", None), ("N", None)) + _STOP,
                       _CRAIG_KW, _LEASTNORM + ("Aresiduals",), rect=True, transpose=True, two=True),
    "lnlq": _Solver("lnlq! (src/lnlq.jl:168-568) -> (x, y, stats); stats also has error_bnd_x, error_bnd_y and "
                    "error_with_bnd.\n    M (m) / N (n): None or the diagonal of a Diagonal operator.  kwargs: lambda_, "
                    "sqd, sigma, transfer_to_craig\n    (default True), utolx, utoly, atol, rtol, itmax, ldiv, history.  "
                    "callback(iter) -> bool.", (("M", None), ("N", None)) + _STOP,
                    dict(lambda_=0.0, sqd=False, sigma=0.0, atol=math.nan, rtol=math.nan, utolx=math.nan,
                         utoly=math.nan, itmax=0, history=True, ldiv=False, transfer_to_craig=True),
                    _LEASTNORM + ("error_bnd_x", "error_bnd_y", "error_with_bnd"), rect=True, transpose=True, two=True,
                    hist_extra=3),
    "cgne": _Solver("cgne! (src/cgne.jl:134-252) -> (x, stats).  N (m entries): None or the diagonal of a Diagonal "
                    "operator on the\n    residual space.  kwargs: lambda_, atol, rtol, itmax, ldiv, history.  "
                    "callback(iter) -> bool.", (("N", None),) + _STOP, _CGNE_KW, _LEASTNORM, rect=True, transpose=True),
    "crmr": _Solver("crmr! (src/crmr.jl:132-244) -> (x, stats); stats also has Aresiduals.  Same arguments as cgne.",
                    (("N", None),) + _STOP, _CGNE_KW, _LEASTNORM + ("Aresiduals",), rect=True, transpose=True),
}


def _callback(f):
    return _ITER_CB() if f is None else _ITER_CB(lambda it, _u: int(bool(f(it))))


_CONVERT = dict({k: int for k in ("history", "linesearch", "restart", "reorthogonalization", "ldiv", "check_curvature",
                                  "transfer_to_lsqr", "transfer_to_craig", "transfer_to_bicg", "transfer_to_usymcg")},
                gamma=float, artol=lambda a: math.nan if a is None else float(a),
                timemax=lambda t: -1.0 if math.isinf(t) else float(t), callback=_callback)
_FIELD = {"transfer_to_bicg": "transfer", "transfer_to_usymcg": "transfer"}


def _options(keywords, kw, default_itmax, hist_extra=2, fixed_cap=False):
    """Pops the accepted keywords into an Options; whatever is left in kw raises TypeError."""
    o = Options()
    sqd = kw.pop("sqd", False) if "sqd" in keywords else False
    for key, default in keywords.items():
        if key not in ("sqd", "hist_cap"):
            v = kw.pop(key, default)
            setattr(o, _FIELD.get(key, key), _CONVERT[key](v) if key in _CONVERT else v)
    if sqd:
        if o.lambda_ != 0:
            raise ValueError("sqd cannot be set to true if λ ≠ 0 !")
        o.lambda_ = 1.0
    itmax = o.itmax if o.itmax > 0 else default_itmax
    o.hist_cap = min(itmax + hist_extra, 1 << 22)
    if "hist_cap" in keywords:
        cap = kw.pop("hist_cap", o.hist_cap)
        if not fixed_cap:
            o.hist_cap = cap
    if kw:
        raise TypeError(f"unknown options {sorted(kw)}")
    return o


def _stat(key, st, out, hist, cap):
    if key in ("niter", "npcCount", "error"):
        return getattr(st, key)
    if key in ("solved", "inconsistent", "indefinite"):
        return bool(getattr(st, key))
    if key == "status":
        return st.status.decode("utf-8")
    if key in ("error_with_bnd", "solved_primal", "solved_dual"):
        return bool(getattr(out, key))
    if key == "Anorm":
        return float(out.Anorm)
    if key == "npc_dir":
        return hist[key]
    h = "residuals" if key == "residuals_primal" else key
    k = st.nres if h == "residuals" else st.nAres if h in ("Aresiduals", "Acond") else getattr(out, "n_" + h)
    return hist[h][:min(k, cap)].copy()


def _solve(name, A, b, dtype, kw):
    row = _SOLVERS[name]
    suf, ct = _suf(dtype)
    A = sp.csr_matrix(A)
    m, n = A.shape
    P = Problem(m, n)
    _, rp, ci, va = _csr(A, dtype)
    P.rowptr, P.colind, P.val = _p(rp), _p(ci), _p(va)
    if row.transpose:
        _, trp, tci, tva = _csr(A.T, dtype)
        P.trowptr, P.tcolind, P.tval = _p(trp), _p(tci), _p(tva)
    params = dict(row.params)
    vecs = dict(b=_vec(b, dtype))
    for v in _VECTORS:
        if v in params:
            vecs[v] = _vec(kw.pop(v, None), dtype)
            if vecs[v] is None and params[v] is _REQUIRED:
                raise TypeError(f"{name}() missing required argument: '{v}'")
            setattr(P, v, _p(vecs[v]))
    P.b = _p(vecs["b"])
    if "y0" in params and (vecs["x0"] is None) != (vecs["y0"] is None):
        raise ValueError("pass both x0 and y0, or neither")
    keywords = {**row.keywords, **{k: d for k, d in row.params if k not in _VECTORS}}
    o = _options(keywords, kw, m + n if row.rect else 2 * n, row.hist_extra, row.fixed_cap)
    out = _OUTPUTS[ct]()
    x, y = np.zeros(n, dtype), (np.zeros(m, dtype) if row.two else None)
    hist = {h: np.zeros(o.hist_cap, dtype) for h in _HISTORIES
            if h in row.stats or (h == "residuals" and "residuals_primal" in row.stats)}
    if "npc_dir" in row.stats:
        hist["npc_dir"] = np.zeros(n, dtype)
    out.x, out.y = _p(x), _p(y)
    for h, buf in hist.items():
        setattr(out, h, _p(buf))
    st = Stats()
    rc = getattr(lib(), f"oracle_solve_{suf}")(name.encode(), C.byref(P), C.byref(o), C.byref(out), C.byref(st))
    stats = {k: _stat(k, st, out, hist, o.hist_cap) for k in row.stats}
    msg = row.error and row.error(rc, stats)
    if msg:
        raise ArithmeticError(msg)
    return x, y, stats


def solve(name, A, b, *, c=None, x0=None, y0=None, M=None, N=None, dtype=np.float64, **kw):
    """Runs the oracle solver `name` (a key of _SOLVERS) -> (x, y, stats), y None for the single-solution solvers.
    The vectors a solver does not take must be None; kw are its keyword arguments (an unknown one raises TypeError)."""
    given = {k: v for k, v in dict(c=c, x0=x0, y0=y0, M=M, N=N).items() if v is not None}
    return _solve(name, A, b, dtype, {**given, **kw})


def _named(name):
    """The solver function `name`, with its reference signature and return shape."""
    row = _SOLVERS[name]
    K = inspect.Parameter.POSITIONAL_OR_KEYWORD
    sig = inspect.Signature([inspect.Parameter("A", K), inspect.Parameter("b", K)]
                            + [inspect.Parameter(k, K, default=d) for k, d in row.params]
                            + [inspect.Parameter("dtype", K, default=np.float64),
                               inspect.Parameter("kw", inspect.Parameter.VAR_KEYWORD)])

    def f(*args, **kwargs):
        bound = sig.bind(*args, **kwargs)
        bound.apply_defaults()
        a = bound.arguments
        x, y, stats = _solve(name, a.pop("A"), a.pop("b"), a.pop("dtype"), {**a.pop("kw"), **a})
        return (x, y, stats) if row.two else (x, stats)

    f.__name__ = f.__qualname__ = name
    f.__doc__, f.__signature__ = row.doc, sig
    return f


for _name in _SOLVERS:
    globals()[_name] = _named(_name)


def block_gmres(A, B, X0=None, M=None, N=None, dtype=np.float64, **kw):
    """block_gmres! (src/block_gmres.jl:110-359).  B, X0, X: n x p (any layout; converted to column-major)."""
    suf, _ = _suf(dtype)
    n, rp, ci, va = _csr(A, dtype)
    B = np.asfortranarray(B, dtype=dtype)
    p = B.shape[1]
    X0f = None if X0 is None else np.asfortranarray(X0, dtype=dtype)
    M, N = _vec(M, dtype), _vec(N, dtype)
    o = _options(_SQUARE_KW, kw, 2 * n)
    X = np.zeros((n, p), dtype, order="F")
    hist = dict(residuals=np.zeros(o.hist_cap, dtype))
    st = Stats()
    getattr(lib(), f"oracle_block_gmres_{suf}")(n, p, _p(rp), _p(ci), _p(va), _p(B), _p(X0f), _p(M), _p(N),
                                                 C.byref(o), _p(X), _p(hist["residuals"]), C.byref(st))
    return X, {k: _stat(k, st, None, hist, o.hist_cap) for k in _SIMPLE}


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
