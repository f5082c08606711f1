"""GPU: every served solver and Krylov process against the CPU oracle, bit for bit, on operators of at most 256 rows and
columns.

There every streaming kernel and every staged operator runs one CTA (stream_grid gives 1 CTA for n <= 256, a staged
operator of <= 256 rows has one tile), and each reduction holds term i on thread i of 256: its order is a fixed fold
that the oracle copies in dot mode 2 (krylov_oracle_impl.h: kdot).  Everything else -- vector updates, SpMV, the scalar
recurrences -- is meant to be the same operation for operation on both sides.  So with the oracle in mode 2 the GPU
must return the same bytes: x (and y), every history, niter, status and every flag, on the fused, two-launch and
primitive paths, staged and untiled, with and without preconditioners.  A difference of one ulp is a defect that the
tolerance-based parity tests cannot see: an FMA contracted into a scalar update, a reciprocal where the reference
divides, another association.  The one departure DESIGN.md documents that these runs would reach is in EXCEPTIONS.

The premise is tested first, on its own: kb200_dot / kb200_nrm2 equal the NumPy fold at every size up to 256, and a
staged operator of <= 256 rows plans one tile on one CTA."""
import ctypes as C
import functools

import numpy as np
import pytest
import scipy.sparse as sp

from krylov_b200 import _lib
from oracle import processes_oracle
from oracle import oracle as O
from test_oracle_dot_tree import device_tree, operands

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]
SIZES = [1, 2, 31, 32, 33, 255, 256]

# The one departure DESIGN.md documents that these runs would reach, with the heading of its section there.  knorm of
# the primitive path (blas1.cu: k_nrm2) is BLAS nrm2 and rescales once 0 < Σ xᵢ² < n·realmin, where the oracle keeps
# sqrt(Σ).  A run with every tolerance 0 gets there when a residual recurrence keeps shrinking, so every run stops
# before its first history entry in (0, sqrt(n·realmin)) (normal_range_run); exact zeros are inside the range.
EXCEPTIONS = {"norms below the normal range": "DESIGN.md, 'knorm is BLAS nrm2 at the range ends'"}


# ----------------------------------------------------------------------------------------------------------------------
# The premise: one CTA, and the oracle's mode 2 is its order
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", DTYPES)
def test_premise_dot_and_nrm2_are_the_one_cta_fold(dt):
    L = _lib.lib()
    ctx = L.kb200_ctx_create(-1)
    kdt = _lib.KRYLOV_FLOAT64 if dt == np.float64 else _lib.KRYLOV_FLOAT32
    try:
        for n in sorted(set(SIZES) | {3, 63, 64, 65, 128, 200}):
            x, y = operands(n, dt, 1)
            px, py = L.kb200_alloc(x.nbytes), L.kb200_alloc(y.nbytes)
            try:
                L.kb200_h2d(px, x.ctypes.data_as(C.c_void_p), x.nbytes)
                L.kb200_h2d(py, y.ctypes.data_as(C.c_void_p), y.nbytes)
                r = C.c_double()
                assert L.kb200_dot(ctx, kdt, n, px, py, C.byref(r)) == 0, _lib.last_error()
                assert dt(r.value).tobytes() == device_tree(x, y, dt).tobytes(), ("dot", n)
                assert L.kb200_nrm2(ctx, kdt, n, px, C.byref(r)) == 0, _lib.last_error()
                assert dt(r.value).tobytes() == np.sqrt(device_tree(x, x, dt)).tobytes(), ("nrm2", n)
            finally:
                L.kb200_free(px)
                L.kb200_free(py)
    finally:
        L.kb200_ctx_destroy(ctx)


@pytest.mark.parametrize("dt", DTYPES)
def test_premise_staged_small_operators_run_one_cta(dt):
    from krylov_b200 import CsrOperator
    for A in (lap(256), lap(33), div_grad(6, 6, 6), rect(256, 96), rect(96, 256)):
        op = CsrOperator.from_scipy(A, dtype=dt)
        out = (C.c_longlong * 7)()
        assert _lib.lib().kb200_csr_plan(op._csr, out) == 0, _lib.last_error()
        op.free()
        assert out[3] and out[0] == 1 and out[5] == 1, (A.shape, list(out))      # tma_ok, ntiles, grid
    op = CsrOperator.from_scipy(dense(256, True), dtype=dt)
    out = (C.c_longlong * 7)()
    assert _lib.lib().kb200_csr_plan(op._csr, out) == 0
    op.free()
    assert not out[3], list(out)                                                  # the dense twin is untiled


# ----------------------------------------------------------------------------------------------------------------------
# Operators, all with m, n <= 256
# ----------------------------------------------------------------------------------------------------------------------
def lap(n, shift=0.0):
    """The 1-D Laplacian tridiag(-1, 2, -1), minus shift I."""
    return sp.csr_matrix(sp.diags([-np.ones(n - 1), (2.0 - shift) * np.ones(n), -np.ones(n - 1)], [-1, 0, 1]))


@functools.cache
def div_grad(a, b, c):
    return O.get_div_grad(a, b, c)


@functools.cache
def kron6():
    return O.kron_unsymmetric(6)[0]


@functools.cache
def dense(n, sym):
    """A dense n x n matrix: 65 536 nonzeros at n = 256, above the untiled threshold of both types.  sym: symmetric
    positive definite; otherwise nonsymmetric with a dominant diagonal."""
    R = np.random.default_rng(n).random((n, n)) / n
    return sp.csr_matrix(R @ R.T + np.eye(n) if sym else R - R.T / 2 + np.eye(n))


@functools.cache
def rect(m, n):
    """m x n with empty rows and columns where the shape has room for them, otherwise a dense line."""
    if min(m, n) == 1:
        return sp.csr_matrix(1.0 + np.random.default_rng(m + n).random((m, n)))
    A = sp.lil_matrix(sp.random(m, n, density=0.06, random_state=m * n, format="csr") + sp.eye(m, n))
    A[3, :] = 0
    A[m - 1, :] = 0
    A[:, 1] = 0
    A[:, n - 2] = 0
    A = sp.csr_matrix(A)
    A.eliminate_zeros()
    return A


SYM_OPS = {**{f"lap{n}": functools.partial(lap, n) for n in SIZES}, "div_grad666": lambda: div_grad(6, 6, 6),
           "div_grad753": lambda: div_grad(7, 5, 3), "indefinite": lambda: lap(120, 1.0),
           "dense256": lambda: dense(256, True)}
UNSYM_OPS = {**{f"lap{n}": functools.partial(lap, n) for n in SIZES}, "div_grad753": lambda: div_grad(7, 5, 3),
             "kron6": kron6, "indefinite": lambda: lap(120, 1.0), "dense256": lambda: dense(256, False)}
RECT_OPS = {**{f"rect{m}x{n}": functools.partial(rect, m, n) for m, n in ((256, 96), (96, 256), (1, 256), (256, 1))},
            "kron6": kron6, "lap33": functools.partial(lap, 33), "dense256": lambda: dense(256, False)}


def rhs(m, zero=False):
    return np.zeros(m) if zero else np.cos(np.arange(m)) + 0.5


# ----------------------------------------------------------------------------------------------------------------------
# The solvers: the oracle of each, its operators and the options it takes
# ----------------------------------------------------------------------------------------------------------------------
SYM = ["cg", "cr", "minres", "cg_lanczos", "car", "minares"]
UNSYM = ["gmres", "fom", "fgmres", "dqgmres", "diom", "cgs", "bicgstab", "bilq", "qmr", "bilqr"]
LSQ = ["lsqr", "lsmr", "lslq", "cgls", "crls"]
LN = ["craig", "craigmr", "lnlq", "cgne", "crmr"]
# the preconditioners each takes, and in which space (m or n)
TAKES_M = {**{s: "n" for s in SYM if s != "minares"}, **{s: "n" for s in UNSYM if s != "bilqr"},
           **{s: "m" for s in LSQ + ["craig", "craigmr", "lnlq"]}}
TAKES_N = {**{s: "n" for s in ["gmres", "fom", "fgmres", "dqgmres", "diom", "cgs", "bicgstab", "bilq", "qmr"]},
           **{s: "n" for s in ["lsqr", "lsmr", "lslq", "craig", "craigmr", "lnlq"]}, "cgne": "m", "crmr": "m"}
BLOCK_JACOBI = ["cg", "cr", "minres", "cg_lanczos", "gmres", "fom", "fgmres", "dqgmres", "diom", "cgs", "bicgstab", "car"]
WARM = SYM + UNSYM
LAMBDA = LSQ + LN
ZERO_TOL = {"lsqr": dict(etol=0.0, axtol=0.0, btol=0.0, conlim=0.0), "lsmr": dict(etol=0.0, axtol=0.0, btol=0.0, conlim=0.0),
            "lslq": dict(etol=0.0, utol=0.0, btol=0.0, conlim=0.0), "craig": dict(btol=0.0, conlim=0.0),
            "minares": dict(artol=0.0)}
ALL = SYM + UNSYM + LSQ + LN + ["trilqr"]


def operators(solver):
    return SYM_OPS if solver in SYM else UNSYM_OPS if solver in UNSYM else RECT_OPS


def canon(v, dt):
    """Bytes of v in the working type; every NaN as one pattern (the CPU's and the GPU's default NaNs differ)."""
    a = np.array(v, dtype=dt).reshape(-1)
    a[np.isnan(a)] = np.nan
    return a.tobytes()


def outcome(x, y, st, keys, dt):
    """x, y and the stats named in `keys` (stats attributes or oracle stats-dict keys), in comparable form."""
    get = st.get if isinstance(st, dict) else functools.partial(getattr, st)
    out = {"x": canon(x, dt)}
    if y is not None:
        out["y"] = canon(y, dt)
    for k in keys:
        v = get(k)
        out[k] = canon(v, dt) if isinstance(v, (list, np.ndarray, float)) else v
    return out


def first_below_normal(A, so, dt):
    """The first history entry of an oracle run in (0, sqrt(n·realmin)), where squares leave the normal range and the
    primitive path's knorm starts to rescale (EXCEPTIONS), or None."""
    floor = np.sqrt(max(A.shape) * np.finfo(dt).tiny)
    hits = []
    for h in (np.abs(np.asarray(v, float)) for k, v in so.items() if isinstance(v, np.ndarray) and k != "npc_dir"):
        low = (h > 0) & (h < floor)
        if low.any():
            hits.append(int(np.argmax(low)))
    return min(hits) if hits else None


def normal_range_run(solver, A, b, c, dt, kw):
    """(kw, the oracle's outcome in dot mode 2) for a run that stays in the normal range: where the oracle's history
    gets below it at entry k, the run is capped at k - 2 iterations and repeated."""
    while True:
        with O.dot_mode(2):
            if oracle_blocks(kw) is not None:
                with O.precond_block(oracle_blocks(kw)):
                    xo, yo, so = O.solve(solver, A, b, c=c, dtype=dt, **dict(kw, M=kw["M"].reshape(-1)))
            else:
                xo, yo, so = O.solve(solver, A, b, c=c, dtype=dt, **kw)
        k = first_below_normal(A, so, dt)
        if k is None:
            return kw, (xo, yo, so)
        cap = max(1, k - 2)
        assert cap < so["niter"], (solver, k, so["niter"])
        kw = dict(kw, itmax=cap)


def oracle_blocks(kw):
    """The block size of a block-Jacobi M given as (ceil(n / bs), bs, bs) blocks, or None."""
    M = kw.get("M")
    return M.shape[1] if M is not None and M.ndim == 3 else None


def oracle_keys(solver, so):
    """The stats both sides report: every key of the oracle's stats dict but its error code and the CG/MINRES npc
    direction (a workspace vector, not a statistic)."""
    return [k for k in so if k not in ("error", "npc_dir") and not (k == "Anorm" and solver != "cg_lanczos")]


def run_gpu(kb, solver, A, b, c, dt, kw):
    kw = dict(kw, history=True)
    args = (A, b.astype(dt)) + ((c.astype(dt),) if solver in ("bilqr", "trilqr") else ())
    if c is not None and solver not in ("bilqr", "trilqr"):
        kw["c"] = c.astype(dt)
    out = getattr(kb, solver)(*args, **kw)
    return (out[0], None, out[1]) if len(out) == 2 else out


def diff(a, b):
    """The first key where two outcomes differ, with the first differing history index."""
    for k in a:
        if a[k] != b.get(k):
            if isinstance(a[k], bytes) and isinstance(b.get(k), bytes):
                u, v = np.frombuffer(a[k], np.uint8), np.frombuffer(b[k], np.uint8)
                n = min(len(u), len(v))
                first = int(np.argmax(u[:n] != v[:n])) if np.any(u[:n] != v[:n]) else n
                return f"{k} (byte {first}, lengths {len(u)}/{len(v)})"
            return f"{k}: {a[k]!r} != {b.get(k)!r}"
    return None


def check(kb, solver, A, b, dt, kw, fused_paths=(True, False), c=None, gpu_kw=None):
    """Run the oracle in dot mode 2 and the GPU on each path; return the differences as strings.  Where the oracle
    raises (CR on an indefinite operator without a trust region, DIOM with memory 1), the GPU must raise too."""
    try:
        kw, (xo, yo, so) = normal_range_run(solver, A, b, c, dt, kw)
    except ArithmeticError as e:
        errs = []
        for fused in fused_paths:
            try:
                run_gpu(kb, solver, A, b, c, dt, dict(kw, fused=fused, **(gpu_kw or {})))
                errs.append(f"fused={fused}: the oracle raises {e}, the GPU does not")
            except kb.B200Error:
                pass
        return errs
    keys = oracle_keys(solver, so)
    assert len(so.get("residuals", so.get("residuals_primal", [1]))) > 0
    want, got, errs = outcome(xo, yo, so, keys, dt), {}, []
    for fused in fused_paths:
        gkw = dict(kw, fused=fused, **(gpu_kw or {}))
        if oracle_blocks(kw) is not None:
            gkw["M"] = kw["M"].astype(dt)
        x, y, st = run_gpu(kb, solver, A, b, c, dt, gkw)
        got[fused] = outcome(x, y, st, keys, dt)
        d = diff(want, got[fused])
        if d:
            errs.append(f"fused={fused}: {d}")
    if len({tuple(sorted(g.items())) for g in got.values()}) > 1:
        errs.append("the GPU paths differ from each other: " + str(diff(*got.values())))
    return errs


def runs(solver, A):
    """Default tolerances, then 2 min(m, n) iterations with every tolerance 0 (into the rounding regime)."""
    zero = dict(atol=0.0, rtol=0.0, **ZERO_TOL.get(solver, {}), itmax=2 * min(A.shape))
    return {"default": {}, "fixed": zero}


def adj_c(solver, A):
    return np.sin(np.arange(A.shape[1])) + 0.25 if solver in ("bilqr", "trilqr") else None


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("solver", ALL)
def test_exact_on_every_operator(kb, solver, dt):
    fails = []
    for name, make in operators(solver).items():
        A = make()
        b = rhs(A.shape[0])
        for run, kw in runs(solver, A).items():
            for e in check(kb, solver, A, b, dt, kw, c=adj_c(solver, A)):
                fails.append(f"{name} {run}: {e}")
    assert not fails, f"{solver} {np.dtype(dt).name}: {len(fails)} cases differ\n" + "\n".join(fails[:30])


def option_operator(solver):
    if solver in SYM:
        return div_grad(7, 5, 3)
    if solver in UNSYM:
        return kron6()
    return rect(96, 256) if solver in LN else rect(256, 96)


def diag(k, seed):
    return 0.5 + np.random.default_rng(seed).random(k)


def blocks(n, bs, seed):
    """ceil(n / bs) symmetric positive definite bs x bs blocks."""
    R = np.random.default_rng(seed).random(((n + bs - 1) // bs, bs, bs))
    return 2.0 * np.eye(bs) + 0.15 * (R + R.transpose(0, 2, 1))


def option_cases(solver, A):
    """name -> (oracle and GPU keywords, extra GPU-only keywords, oracle context, rhs-is-zero)."""
    m, n = A.shape
    sp_ = {"m": m, "n": n}
    out = {}
    if solver in TAKES_M:
        out["M"] = dict(M=diag(sp_[TAKES_M[solver]], 1))
        out["M_ldiv"] = dict(M=diag(sp_[TAKES_M[solver]], 1), ldiv=True)
    if solver in TAKES_N:
        out["N"] = dict(N=diag(sp_[TAKES_N[solver]], 2))
        if solver in TAKES_M:
            out["MN"] = dict(M=diag(sp_[TAKES_M[solver]], 3), N=diag(sp_[TAKES_N[solver]], 4))
    if solver in WARM:
        out["warm"] = dict(x0=np.sin(np.arange(n)) / 4)
        if solver == "bilqr":
            out["warm"]["y0"] = np.cos(np.arange(m)) / 4
    if solver in LAMBDA:
        out["lambda"] = dict(lambda_=0.3)
    if solver == "minres":
        out["shift"] = dict(lambda_=0.7)
    if solver in ("cg", "cr"):
        out["radius"] = dict(radius=2.0)
    out["zero_rhs"] = dict()
    return out


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("solver", ALL)
def test_exact_with_options(kb, solver, dt):
    A = option_operator(solver)
    fails = []
    for name, kw in option_cases(solver, A).items():
        b = rhs(A.shape[0], zero=name == "zero_rhs")
        for run, base in runs(solver, A).items():
            for e in check(kb, solver, A, b, dt, dict(base, **kw), c=adj_c(solver, A)):
                fails.append(f"{name} {run}: {e}")
    if solver in BLOCK_JACOBI:
        A = lap(100)                                                   # 34 blocks of 3, the last one ragged
        for run, base in runs(solver, A).items():
            errs = check_block(kb, solver, A, rhs(100), dt, base, blocks(100, 3, 5))
            fails += [f"block-Jacobi {run}: {e}" for e in errs]
    assert not fails, f"{solver} {np.dtype(dt).name}: {len(fails)} cases differ\n" + "\n".join(fails[:30])


def check_block(kb, solver, A, b, dt, kw, B):
    """check() with a block-Jacobi M given as its (ceil(n / bs), bs, bs) blocks B (the oracle reads them flattened)."""
    return check(kb, solver, A, b, dt, dict(kw, M=B))


# ----------------------------------------------------------------------------------------------------------------------
# Fused CG: the persistent kernel on CSR and on the constant-coefficient encoding, the two-launch kernels, batches
# ----------------------------------------------------------------------------------------------------------------------
CG_OPS = {"lap33": lambda: lap(33), "lap256": lambda: lap(256), "div_grad666": lambda: div_grad(6, 6, 6),
          "div_grad753": lambda: div_grad(7, 5, 3), "dense256": lambda: dense(256, True)}


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("path", ["persist_dict", "persist_csr", "two_launch", "two_launch_xup0"])
def test_exact_cg_fused_paths(kb, monkeypatch, path, dt):
    monkeypatch.setenv("KB200_CSR_DICT", "1" if path == "persist_dict" else "0")
    if path == "two_launch_xup0":
        monkeypatch.setenv("KB200_XUP", "0")
    fused = True if path.startswith("persist") else 2
    fails = []
    for name, make in CG_OPS.items():
        A = make()
        n = A.shape[0]
        cases = {"plain": {}, "jacobi": dict(M=diag(n, 1)), "warm": dict(x0=np.sin(np.arange(n)) / 4)}
        for cname, kw in cases.items():
            for run, base in runs("cg", A).items():
                for batch in (1, 32):
                    for e in check(kb, "cg", A, rhs(n), dt, dict(base, **kw), fused_paths=(fused, False),
                                   gpu_kw=dict(batch=batch)):
                        fails.append(f"{name} {cname} {run} batch={batch}: {e}")
        if path.startswith("persist"):
            for run, base in runs("cg", A).items():
                fails += [f"{name} block-Jacobi {run}: {e}"
                          for e in check_block(kb, "cg", A, rhs(n), dt, base, blocks(n, 3, 6))]
    assert not fails, f"cg {path} {np.dtype(dt).name}: {len(fails)} cases differ\n" + "\n".join(fails[:30])


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("solver", ["cg", "cr"])
def test_exact_linesearch(kb, solver, dt):
    """CG / CR with linesearch on an indefinite operator: a nonpositive curvature exit with its flags."""
    A = lap(120, 1.0)
    fails = []
    for run, base in runs(solver, A).items():
        fails += [f"{run}: {e}" for e in check(kb, solver, A, rhs(120), dt, dict(base, linesearch=True))]
    assert not fails, "\n".join(fails)


# ----------------------------------------------------------------------------------------------------------------------
# The Krylov processes
# ----------------------------------------------------------------------------------------------------------------------
PROCESSES = {"hermitian_lanczos": [("lap33", lambda: lap(33)), ("div_grad666", lambda: div_grad(6, 6, 6)),
                                   ("dense256", lambda: dense(256, True)), ("lap2", lambda: lap(2))],
             "arnoldi": [("kron6", kron6), ("dense256", lambda: dense(256, False)), ("lap31", lambda: lap(31))],
             "golub_kahan": [(f"rect{m}x{n}", functools.partial(rect, m, n)) for m, n in ((256, 96), (96, 256))]
             + [("kron6", kron6)],
             "nonhermitian_lanczos": [("kron6", kron6), ("dense256", lambda: dense(256, False))],
             "saunders_simon_yip": [(f"rect{m}x{n}", functools.partial(rect, m, n)) for m, n in ((256, 96), (96, 256))]
             + [("kron6", kron6)]}


def process_parts(out):
    """Every output of a process, in the order it returns them, flattened: the bases and a dense H column-major, the
    nonzeros of a sparse T or L in their stored order (the oracle returns those nzval arrays), β and γ."""
    parts = []
    for v in out:
        if sp.issparse(v):
            parts.append(np.asarray(v.data))
        else:
            parts.append(np.ravel(np.asarray(v), order="F"))
    return parts


def call_process(mod, name, A, b, c, k, dt, **kw):
    f = getattr(mod, name)
    args = (A.astype(dt) if mod is not processes_oracle else A, b.astype(dt)) + ((c.astype(dt),) if c is not None else ())
    if mod is processes_oracle:
        kw["dtype"] = dt
    return f(*args, k, **kw)


@pytest.mark.parametrize("dt", DTYPES)
@pytest.mark.parametrize("name", list(PROCESSES))
def test_exact_processes(kb, name, dt):
    fails = []
    for opname, make in PROCESSES[name]:
        A = make()
        m, n = A.shape
        b = rhs(m)
        c = np.sin(np.arange(n)) + 0.25 if name in ("nonhermitian_lanczos", "saunders_simon_yip") else None
        variants = [dict(), dict(allow_breakdown=True)]
        if name in ("hermitian_lanczos", "arnoldi"):
            variants.append(dict(reorthogonalization=True))
        for kw in variants:
            for k in sorted({1, min(20, min(m, n)), min(m, n)}):
                try:
                    with O.dot_mode(2):
                        want = call_process(processes_oracle, name, A, b, c, k, dt, **kw)
                except processes_oracle.ProcessBreakdown as e:
                    with pytest.raises(kb.B200Error) as g:
                        call_process(kb, name, A, b, c, k, dt, **kw)
                    if str(g.value) != str(e):
                        fails.append(f"{opname} k={k} {kw}: breakdown {g.value} != {e}")
                    continue
                got = call_process(kb, name, A, b, c, k, dt, **kw)
                pw, pg = process_parts(want), process_parts(got)
                assert len(pg) == len(pw), (name, len(pg), len(pw))
                for i, (u, v) in enumerate(zip(pg, pw)):
                    if canon(u, dt) != canon(v, dt):
                        fails.append(f"{opname} k={k} {kw}: output {i} differs")
                        break
    assert not fails, f"{name} {np.dtype(dt).name}:\n" + "\n".join(fails[:30])


def test_processes_with_an_exact_breakdown(kb):
    """The path graph closes its Krylov space exactly at iteration 3 (Golub-Kahan at 1): allow_breakdown continues
    with the reference's zero columns, bit for bit in both types."""
    from process_cases import path3
    A, e1 = path3()
    fails = []
    for dt in DTYPES:
        for name in PROCESSES:
            c = e1 if name in ("nonhermitian_lanczos", "saunders_simon_yip") else None
            with O.dot_mode(2):
                want = call_process(processes_oracle, name, A, e1, c, 5, dt, allow_breakdown=True)
            got = call_process(kb, name, A, e1, c, 5, dt, allow_breakdown=True)
            pg, pw = process_parts(got), process_parts(want)
            assert len(pg) == len(pw), (name, len(pg), len(pw))
            for i, (u, v) in enumerate(zip(pg, pw)):
                if canon(u, dt) != canon(v, dt):
                    fails.append(f"{name} {np.dtype(dt).name}: output {i}")
    assert not fails, fails
