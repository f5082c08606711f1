"""GPU: every fused pass on both sides of the tile plan (csrc/spmv.cu: csr_plan), and the TMA ring at every depth.

An operator whose widest tile of 256 rows does not fit the shared-memory ring runs its passes one row per thread
(spmv_epi_rows, cg_k1_rows); one long row is enough to get there, and a dense column does the same to the transpose.
Those operators are held to the CPU oracle here, solver by solver, with the fused path shown to have run (its launches
per iteration equal those on a staged operator).  Every case pins the plan it is meant to exercise.

The ring's depth S changes no arithmetic: tile t goes to CTA t mod grid whatever S is, and every sum runs in a fixed
order, so for a fixed number of CTAs per SM every iterate and history must be byte-identical at S = 1, 2, 3, ...
A stage read before it lands, a slot refilled while live or a parity off by one phase would change bits."""
import functools

import numpy as np
import pytest
import scipy.sparse as sp

import parity
from krylov_b200 import _lib
from krylov_b200 import problems as P
from parity import TOL

pytestmark = pytest.mark.gpu

# ----------------------------------------------------------------------------------------------------------------------
# The plan: kb200_csr_plan, and the planner's default rule restated from TileLayout (csrc/spmv_tiles.cuh)
# ----------------------------------------------------------------------------------------------------------------------
TILE_ROWS = 256
KB = 1024


def ring_bytes(cap, stages, itemsize):
    """TileLayout<T>{cap}.total_bytes(stages)."""
    def up(v):
        return (v + 127) & ~127
    stage = up((TILE_ROWS + 4) * 4) + up((cap + 16 // itemsize) * itemsize) + up((cap + 8) * 4)
    return 128 + stages * stage


def per_cta_ceiling(cps):
    """Shared memory one CTA's ring may take when `cps` CTAs share an SM (the default rules of csr_plan)."""
    return 220 * KB if cps == 1 else 110 * KB if cps == 2 else 226 * KB // cps


def default_plan(cap, itemsize):
    """(CTAs per SM, stages) the planner picks for tile capacity `cap`, or None: untiled."""
    if ring_bytes(cap, 2, itemsize) * 3 <= 226 * KB:
        return 3, 2
    for cps in (2, 1):
        for s in (4, 3, 2):
            if ring_bytes(cap, s, itemsize) <= per_cta_ceiling(cps):
                return cps, s
    return None


def band_top(plan, itemsize):
    """The largest tile capacity that the default rule gives `plan`."""
    return max(c for c in range(20000) if default_plan(c, itemsize) == plan)


def untiled_from(itemsize):
    """The smallest tile capacity that the default rule leaves untiled."""
    return next(c for c in range(20000) if default_plan(c, itemsize) is None)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def plan_of(A, dtype):
    """kb200_csr_plan of A uploaded under the current environment, as a dict."""
    import ctypes as C
    from krylov_b200 import CsrOperator
    op = CsrOperator.from_scipy(A, dtype=dtype)
    out = (C.c_longlong * 7)()
    assert _lib.lib().kb200_csr_plan(op._csr, out) == 0, _lib.last_error()
    op.free()
    return dict(ntiles=out[0], tile_cap=out[1], max_row=out[2], tma_ok=bool(out[3]), stages=out[4], grid=out[5],
                smem=out[6])


def assert_plan(A, dtype, want):
    """A's plan is `want`: "untiled" or (CTAs per SM, stages), with the grid and ring size that go with it."""
    itemsize = np.dtype(dtype).itemsize
    p = plan_of(A, dtype)
    if want == "untiled":
        assert not p["tma_ok"] and default_plan(p["tile_cap"], itemsize) is None, p
        return p
    cps, s = want
    assert p["tma_ok"] and (p["stages"], p["smem"]) == (s, ring_bytes(p["tile_cap"], s, itemsize)), (want, p)
    assert p["grid"] == min(sm_count() * cps, p["ntiles"]), (want, p)
    return p


# ----------------------------------------------------------------------------------------------------------------------
# The operator catalogue
# ----------------------------------------------------------------------------------------------------------------------
def _mat(csr, shape=None):
    rp, ci, va = csr
    n = len(rp) - 1
    return sp.csr_matrix((va, ci, rp), shape=shape or (n, n))


def _line(n, seed):
    """A dense line of n small entries, between 1/n and 2/n: long enough to make a tile untiled, with a sum of order 1
    (a larger one makes the histories of the large arrow below hypersensitive to rounding)."""
    return (1.0 + np.random.default_rng(seed).random(n)) / n


def arrow(N):
    """div_grad(N) with a dense first row and column; the corner is raised above its row's sum: symmetric positive
    definite and diagonally dominant in that row."""
    A = _mat(P.div_grad_csr(N))
    n = A.shape[0]
    w = _line(n, 1)
    w[0] = w[1:].sum() + 1.0                                             # corner: 6 + the row's added entries + 1
    R = sp.csr_matrix((w, (np.zeros(n, np.int64), np.arange(n))), shape=(n, n))
    A = sp.csr_matrix(A + R + sp.csr_matrix(R.T) - sp.csr_matrix(([w[0]], ([0], [0])), shape=(n, n)))
    A.sort_indices()
    return A


def with_row(A, i, seed=2):
    """A plus a dense row i."""
    e = sp.csr_matrix(([1.0], ([i], [0])), shape=(A.shape[0], 1))
    return sp.csr_matrix(A + e @ sp.csr_matrix(_line(A.shape[1], seed)[None, :]))


def with_col(A, j, seed=3):
    """A plus a dense column j."""
    e = sp.csr_matrix(([1.0], ([0], [j])), shape=(1, A.shape[1]))
    return sp.csr_matrix(A + sp.csr_matrix(_line(A.shape[0], seed)[:, None]) @ e)


def grad(N):
    rp, ci, va = P.grad_csr(N)
    return _mat((rp, ci, va), (len(rp) - 1, N ** 3))


@functools.cache
def catalogue():
    """name -> (A, its plan in Float64 and Float32, the plan of Aᵀ in both).  The dense lines are longer than twice the
    Float32 threshold (13.9k nonzeros per tile), so every untiled case is untiled in both types."""
    K = _mat(P.kron_unsymmetric_csr(31))                                     # n = 29 791
    G31, G22 = grad(31), grad(22)                                            # 86 490 x 29 791, 30 492 x 10 648
    U = "untiled"
    out = {"arrow": arrow(31),                                               # A and Aᵀ untiled
           "kron_row": with_row(K, K.shape[0] // 2),                         # A untiled, Aᵀ staged
           "kron_col": with_col(K, K.shape[1] // 3),                         # A staged, Aᵀ untiled
           "grad_row": sp.csr_matrix(sp.vstack([G31, _line(G31.shape[1], 4)[None, :]])),
           "grad_col": sp.csr_matrix(sp.hstack([G22, _line(G22.shape[0], 5)[:, None]])),   # m > n, Aᵀ untiled
           }
    out["grad_col_t"] = sp.csr_matrix(out["grad_col"].T)                    # m < n, A untiled
    plans = {"arrow": (U, U), "kron_row": (U, (3, 2)), "kron_col": ((3, 2), U), "grad_row": (U, (3, 2)),
             "grad_col": ((3, 2), U), "grad_col_t": (U, (3, 2))}
    return {k: (A, plans[k]) for k, A in out.items()}


def _rhs(A, kind):
    m, n = A.shape
    if kind == "sym":
        return np.ones(n)
    if kind == "unsym":
        return A @ np.ones(n)
    return np.random.default_rng(11).standard_normal(m)


# ----------------------------------------------------------------------------------------------------------------------
# Oracles and the parity bars of the families' own tests
# ----------------------------------------------------------------------------------------------------------------------
SYM = ["cg", "cr", "cg_lanczos", "minres", "car", "minares"]
UNSYM = ["bicgstab", "cgs", "gmres", "gmres_restart", "fom", "fgmres", "dqgmres", "diom", "bilq", "qmr", "bilqr"]
RECT = ["lsqr", "lsmr", "lslq", "cgls", "crls", "trilqr"]
ALL = SYM + UNSYM + RECT
CORE = {"cg", "cr", "cg_lanczos", "minres", "bicgstab", "cgs", "gmres", "fom", "fgmres", "dqgmres", "diom"}
OPTS = {"gmres": dict(memory=20), "gmres_restart": dict(memory=20, restart=True), "fom": dict(memory=20),
        "fgmres": dict(memory=20), "dqgmres": dict(memory=6), "diom": dict(memory=6)}
ZERO = {"lsqr": dict(etol=0.0, axtol=0.0, btol=0.0, conlim=0.0), "lsmr": dict(etol=0.0, axtol=0.0, btol=0.0, conlim=0.0),
        "lslq": dict(etol=0.0, utol=0.0, btol=0.0, conlim=0.0), "minares": dict(artol=0.0)}


def zero_tol(solver):
    return dict(atol=0.0, rtol=0.0, **ZERO.get(solver, {}))


@pytest.fixture(scope="module")
def oracles(O):
    from oracle import adjoint_oracle, ares_oracle, biorth_oracle, cgls_oracle, lsq_oracle
    for mod in (adjoint_oracle, ares_oracle, biorth_oracle, cgls_oracle, lsq_oracle):
        mod.lib()
    return dict(core=O, lsq=lsq_oracle, cgls=cgls_oracle, biorth=biorth_oracle, ares=ares_oracle, adjoint=adjoint_oracle)


def base(solver):
    return solver.split("_restart")[0]


def compare(oracles, kb, solver, A, b, **kw):
    """parity.compare with the keys, flags, floor and count policy of the solver family's own GPU tests."""
    name = base(solver)
    kw = dict(OPTS.get(solver, {}), **kw)
    if name in CORE:
        if name == "cgs":                     # CGS squares the BiCG polynomial: x within 10x the oracle's own change
            kw.setdefault("xtol", None)
        return parity.compare(getattr(oracles["core"], name), getattr(kb, name), A, b, keys=("residuals",),
                              flags=("solved", "inconsistent"), floor=1e-9, **kw)
    if name in ("lsqr", "lsmr", "lslq", "cgls", "crls"):
        mod = oracles["lsq"] if name in ("lsqr", "lsmr") else oracles["cgls"]
        return parity.compare(getattr(mod, name), functools.partial(getattr(kb, name), n=A.shape[1]), A, b,
                              keys=("residuals", "Aresiduals"), flags=("inconsistent",), floor=1e-9, **kw)
    if name in ("bilq", "qmr"):
        return parity.compare(getattr(oracles["biorth"], name), getattr(kb, name), A, b, keys=("residuals",),
                              flags=("solved",), floor=1e-12, unsteady="range", check_length=False, xtol=None, **kw)
    if name in ("car", "minares"):
        return parity.compare(getattr(oracles["ares"], name), getattr(kb, name), A, b, keys=("residuals", "Aresiduals"),
                              flags=("solved",), floor=1e-12, unsteady="widened", scaled_resid=name == "minares",
                              xtol=None, **kw)
    return compare_adjoint(oracles["adjoint"], kb, name, A, b, np.cos(np.arange(A.shape[1])), **kw)


def compare_adjoint(AO, kb, solver, A, b, c, xtol=None, **kw):
    """tests/test_gpu_adjoint.py's bar: the pair as one block system diag(A, Aᵀ) with right-hand side [b; c]."""
    m = A.shape[0]
    K = sp.block_diag((A, sp.csr_matrix(A.T)), format="csr")

    def oracle(K_, bc, **kw_):
        x, y, st = getattr(AO, solver)(A, bc[:m], bc[m:], **kw_)
        return np.concatenate([x, y]), st

    def gpu(op, bc, **kw_):
        x, y, st = getattr(kb, solver)(op, bc[:m], bc[m:], **kw_)
        return np.concatenate([x, y]), st

    return parity.compare(oracle, gpu, K, np.concatenate([b, c]), keys=("residuals_primal", "residuals_dual"),
                          flags=("solved_primal", "solved_dual"), floor=1e-9, unsteady="widened", xtol=xtol, gpu_A=A, **kw)


def solver_kwargs(solver, converge):
    """Default tolerances with an iteration cap (square systems), or a fixed number of iterations (least squares and
    TriLQR, whose default tolerances stop where rounding decides)."""
    if converge and solver not in RECT:
        # the BiCG-type counts move with rounding near convergence (their own tests cap them at 60 iterations too)
        return dict(itmax=60 if solver in ("cgs", "bilq", "qmr", "bilqr") else 150)
    return dict(zero_tol(base(solver)), itmax=40)


# ----------------------------------------------------------------------------------------------------------------------
# 1. The catalogue pins its plans
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_catalogue_pins_its_plans(dt):
    isz = np.dtype(dt).itemsize
    assert untiled_from(isz) == (9273 if isz == 8 else 13913)
    for name, (A, (pa, pt)) in catalogue().items():
        a = assert_plan(A, dt, pa)
        t = assert_plan(sp.csr_matrix(A.T), dt, pt)
        for p, want in ((a, pa), (t, pt)):
            if want == "untiled":
                assert p["tile_cap"] >= 2 * untiled_from(4), (name, p)
    # TriLQR pads Aᵀ to max(m, n) rows with empty rows: more tiles, the same capacity
    A = catalogue()["grad_col"][0]
    m, n = A.shape
    pad = sp.csr_matrix(sp.vstack([A.T, sp.csr_matrix((m - n, m))]))
    p, q = plan_of(pad, dt), plan_of(sp.csr_matrix(A.T), dt)
    assert p["tile_cap"] == q["tile_cap"] and p["ntiles"] > q["ntiles"] and not p["tma_ok"]


# Float64 bands (tile capacity): 3 x 2 <= 3096 < 2 x 2 <= 4574 < 1 x 3 <= 6142 < 1 x 2 <= 9272 < untiled; the 2-CTA
# 3- and 4-stage rings and the 1-CTA 4-stage ring are never the default.  Float32: 4636, 6872, 9212, 13912.
STAGED = [("stencil", None, (3, 2), (3, 2)), ("random14", 14, (2, 2), (3, 2)), ("random20", 20, (1, 3), (2, 2)),
          ("random30", 30, (1, 2), (1, 3))]


def test_default_bands():
    for isz, tops in ((8, (3096, 4574, 6142, 9272)), (4, (4636, 6872, 9212, 13912))):
        for plan, top in zip([(3, 2), (2, 2), (1, 3), (1, 2)], tops):
            assert band_top(plan, isz) == top and default_plan(top + 1, isz) != plan, (isz, plan)


@pytest.mark.parametrize("name,per_row,p64,p32", STAGED)
def test_staged_plans_match_the_oracle(kb, oracles, name, per_row, p64, p32):
    """Each default staged plan, pinned in both types, with a fused solver of each kind on it.  The random operators
    take a diagonal shift of 6 (their spectra fill a disc of radius about √(per_row / 3))."""
    A = _mat(P.div_grad_csr(30) if per_row is None else P.random_csr(4000, per_row, seed=7, dtype=np.float64, shift=6.0))
    assert_plan(A, np.float64, p64)
    assert_plan(A, np.float32, p32)
    for solver in (["cg", "minres"] if per_row is None else ["bicgstab", "gmres", "bilq", "lsqr"]):
        for fused in (True, False):
            b = _rhs(A, "sym" if per_row is None else "unsym")
            compare(oracles, kb, solver, A, b, fused=fused, **solver_kwargs(solver, True))


# ----------------------------------------------------------------------------------------------------------------------
# 2. Untiled parity against the oracle
# ----------------------------------------------------------------------------------------------------------------------
ADJ = ["bilq", "qmr", "bilqr"]                                              # the square solvers that apply Aᵀ
CASES = ([(s, "arrow") for s in SYM] + [(s, "kron_row") for s in UNSYM] + [(s, "kron_col") for s in ADJ]
         + [(s, op) for s in RECT if s != "trilqr" for op in ("grad_row", "grad_col")]
         + [("trilqr", "grad_col"), ("trilqr", "grad_col_t")])


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("solver,op", CASES)
def test_untiled_matches_oracle(kb, oracles, solver, op, fused):
    A, _ = catalogue()[op]
    kind = "sym" if op == "arrow" else "unsym" if op.startswith("kron") else "rect"
    compare(oracles, kb, solver, A, _rhs(A, kind), fused=fused, **solver_kwargs(solver, True))


def launches_per_iteration(kb, solver, A, fused):
    """(launches of a 30-iteration solve - those of a 10-iteration one) / 20, all tolerances 0."""
    name = base(solver)
    m, n = A.shape
    opts = dict(OPTS.get(solver, {}))
    mem = opts.pop("memory", 0)
    b = np.cos(np.arange(m))
    args = (A, b, np.cos(np.arange(n))) if name in ("bilqr", "trilqr") else (A, b)
    ws = kb.krylov_workspace(name, m, n, np.float64, memory=mem)
    ws.solve(*args, itmax=3, fused=fused, **opts)                     # forms and caches Aᵀ outside the count
    counts = []
    for itmax in (10, 30):
        l0 = ws.launches
        ws.solve(*args, itmax=itmax, fused=fused, **zero_tol(name), **opts)
        assert ws.stats.niter == itmax + (name == "lslq"), (solver, ws.stats.status)   # lslq! runs itmax + 1
        counts.append(ws.launches - l0)
    ws.free()
    return (counts[1] - counts[0]) / 20


# the staged twin of each untiled operator: the same stencil without its dense line
TWIN = {"arrow": lambda: _mat(P.div_grad_csr(31)), "kron_row": lambda: _mat(P.kron_unsymmetric_csr(31)),
        "kron_col": lambda: _mat(P.kron_unsymmetric_csr(31)), "grad_row": lambda: grad(31),
        "grad_col": lambda: grad(22), "grad_col_t": lambda: sp.csr_matrix(grad(22).T)}


@pytest.mark.parametrize("solver,op", [c for c in CASES if c[1] in ("arrow", "kron_row", "grad_row", "grad_col_t")])
def test_untiled_runs_the_fused_passes(kb, solver, op):
    """The untiled operator launches as many kernels per iteration as its staged twin (CG: against fused = 2, the
    two-launch kernels; the persistent kernel needs a staged plan), and far fewer than the primitive path."""
    A, _ = catalogue()[op]
    T = TWIN[op]()
    assert_plan(T, np.float64, (3, 2))
    got = launches_per_iteration(kb, solver, A, True)
    want = launches_per_iteration(kb, solver, T, 2 if solver == "cg" else True)
    assert got == want, (got, want)
    assert got < launches_per_iteration(kb, solver, A, False), got


def test_cg_untiled_options_match_oracle(kb, oracles):
    """Fused CG on the arrow: M = I, a Jacobi M (cg_k1_rows<kJacobi>) and a callback (x is updated in K2)."""
    O = oracles["core"]
    A, _ = catalogue()["arrow"]
    b = np.ones(A.shape[0])
    d = 1.0 / A.diagonal()
    for fused in (True, 2, False):
        compare(oracles, kb, "cg", A, b, fused=fused)
        compare(oracles, kb, "cg", A, b, M=d, fused=fused)
    xo, so = O.cg(A, b)
    seen = []
    x, st = kb.cg(A, b, history=True, callback=lambda w: (seen.append(1), False)[1])
    assert (st.niter, st.status) == (so["niter"], so["status"]) and len(seen) >= st.niter - 1
    parity.assert_history("residuals", np.asarray(st.residuals), so["residuals"], lambda: np.zeros(len(so["residuals"])),
                          1e-9 * so["residuals"][0])
    assert np.linalg.norm(x - xo) <= TOL * np.linalg.norm(xo)


LARGE = ["cg", "minres", "cgs", "bicgstab", "gmres", "dqgmres", "bilq", "car", "bilqr", "lsqr", "cgls", "lslq", "trilqr"]


@pytest.fixture(scope="module")
def large():
    """An arrow on the 70³ grid: 343 000 rows, more than 1056 x 256, so the row loops of the untiled and stream passes
    take more than one trip."""
    A = arrow(70)
    assert A.shape[0] > 1056 * 256
    assert_plan(A, np.float64, "untiled")
    return A


@pytest.mark.parametrize("solver", LARGE)
def test_large_untiled_matches_oracle(kb, oracles, large, solver):
    kind = "sym" if solver in SYM else "unsym" if solver in UNSYM else "rect"
    compare(oracles, kb, solver, large, _rhs(large, kind), fused=True, **zero_tol(solver), itmax=15)


@pytest.fixture(scope="module")
def ragged():
    """Staged (3 x 2) with ntiles = grid + 1: exactly one CTA gets a second tile (and it is a partial tile).  A
    nonsymmetric five-point operator (upper neighbours -1.5) and the symmetric one, on a 250 x k grid."""
    grid = 3 * sm_count()
    k = grid * TILE_ROWS // 250 + 1
    S = _mat(P.div_grad_csr(250, k, 1))
    U = sp.csr_matrix(S + 0.5 * sp.triu(S, 1))
    for A in (S, U):
        p = assert_plan(A, np.float64, (3, 2))
        assert p["ntiles"] == grid + 1 and A.shape[0] % TILE_ROWS, p
    return S, U


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("solver", ALL)
def test_ragged_grid_matches_oracle(kb, oracles, ragged, solver, fused):
    S, U = ragged
    A = S if solver in SYM else U
    compare(oracles, kb, solver, A, _rhs(A, "sym" if solver in SYM else "rect"), fused=fused, **zero_tol(base(solver)),
            itmax=30)


# Float32 on untiled operators, at the bars of the families' Float32 tests
def _f32_envelope(mod, fn, *args, **kw):
    """The oracle's Float32 run and the running-max gap to the same run with double-accumulated dot products."""
    out = getattr(mod, fn)(*args, dtype=np.float32, **kw)
    with mod.dot_mode(1):
        out1 = getattr(mod, fn)(*args, dtype=np.float32, **kw)
    return out[-1], out1[-1]


def _within_envelope(res, r0, r1, cnt=None):
    r0, r1, res = np.asarray(r0, float), np.asarray(r1, float), np.asarray(res, float)
    k = min(len(res), len(r0), len(r1)) if cnt is None else cnt
    env = np.maximum.accumulate(np.abs(r0[:k] - r1[:k]) / np.maximum(r0[:k], 1e-300))
    tol = np.maximum(4 * 1.2e-7, 10 * env)
    return np.all(np.abs(res[:k] - r0[:k]) <= tol * r0[:k] + 1e-6 * r0[0])


@pytest.mark.parametrize("solver,op", [("cg", "arrow"), ("bicgstab", "kron_row")])
def test_float32_untiled_cg_bicgstab(kb, oracles, solver, op):
    O = oracles["core"]
    A, _ = catalogue()[op]
    assert_plan(A, np.float32, "untiled")
    b = _rhs(A, "sym" if op == "arrow" else "unsym").astype(np.float32)
    # stop before Float32 rounding decides the history (BiCGSTAB's oracle runs part ways after about 15 iterations)
    kw = dict(atol=0.0, rtol=0.0, itmax=30 if solver == "cg" else 12)
    so, s1 = _f32_envelope(O, solver, A, b, **kw)
    x, st = getattr(kb, solver)(A, b, history=True, **kw)
    assert st.niter == so["niter"] == kw["itmax"], (st.niter, so["niter"])
    assert _within_envelope(st.residuals, so["residuals"], s1["residuals"])


@pytest.mark.parametrize("op", ["kron_row", "kron_col"])
def test_float32_untiled_lsqr(kb, oracles, op):
    A, _ = catalogue()[op]
    b = (A @ np.ones(A.shape[1])).astype(np.float32)
    xo, so = oracles["lsq"].lsqr(A.astype(np.float32), b, dtype=np.float32)
    x, st = kb.lsqr(A.astype(np.float32), b)
    assert st.solved == so["solved"] and abs(st.niter - so["niter"]) <= 1, (st.niter, so["niter"])
    # as good a least-squares solution as the oracle's own Float32 one
    nr = [np.linalg.norm(A.T @ (b - A @ v.astype(np.float64))) for v in (x, xo)]
    assert nr[0] <= 2 * nr[1] + 1e-4 * np.linalg.norm(A.T @ b), nr


@pytest.mark.parametrize("op", ["kron_row", "kron_col"])
def test_float32_untiled_bilqr(kb, oracles, op):
    AO = oracles["adjoint"]
    A, _ = catalogue()[op]
    b, c = A @ np.ones(A.shape[1]), np.cos(np.arange(A.shape[0]))
    kw = dict(itmax=40)
    _, _, so = AO.bilqr(A, b, c, dtype=np.float32, **kw)
    with AO.dot_mode(1):
        _, _, s1 = AO.bilqr(A, b, c, dtype=np.float32, **kw)
    x, y, st = kb.bilqr(A, b.astype(np.float32), c.astype(np.float32), history=True, **kw)
    assert st.niter == so["niter"]
    for key in ("residuals_primal", "residuals_dual"):
        assert len(getattr(st, key)) == len(so[key]) and _within_envelope(getattr(st, key), so[key], s1[key]), key


# ----------------------------------------------------------------------------------------------------------------------
# 3. Ring depth must not change a bit
# ----------------------------------------------------------------------------------------------------------------------
RING = {"div_grad": SYM + ["cg_2"], "kron": UNSYM, "grad": RECT}


@functools.cache
def ring_operator(name):
    """About 10⁶ rows and 4146 tiles or more (grad: 3.44 x 10⁶ rows, Aᵀ 105³ = 1 157 625): at least 2 S + 1 tiles per
    CTA of every ring below."""
    if name == "div_grad":
        return _mat(P.div_grad_csr(102))
    if name == "kron":
        return _mat(P.kron_unsymmetric_csr(102))
    return grad(105)


@functools.cache
def ring_cap(name):
    """The larger tile capacity of the operator and its transpose."""
    A = ring_operator(name)
    return max(tile_cap(A), tile_cap(sp.csr_matrix(A.T)))


def tile_cap(A):
    rp = A.indptr
    starts = np.arange(0, A.shape[0], TILE_ROWS)
    return int(np.max(rp[np.minimum(starts + TILE_ROWS, A.shape[0])] - rp[starts]))


def ring_depths(op, cps, itemsize):
    """Every depth whose ring, for A and for Aᵀ, keeps cps CTAs well inside an SM's 228 KB (2 KB per CTA spare for
    static shared memory and the CTA's reserve), so the occupancy and the grid do not move with S."""
    A = ring_operator(op)
    cap = ring_cap(op)
    ntiles = (min(A.shape) + TILE_ROWS - 1) // TILE_ROWS
    out = []
    for s in range(1, 9):
        rb = ring_bytes(cap, s, itemsize)
        if rb <= per_cta_ceiling(cps) and cps * (rb + 2 * KB) <= 224 * KB:
            assert ntiles >= (2 * s + 1) * sm_count() * cps, (s, cps, ntiles)
            out.append(s)
    return out


def ring_run(kb, solver, A_op, m, n, dt):
    """20 iterations, all tolerances 0: x (and y), every history, niter and status, as bytes."""
    fused = True
    if solver == "cg_2":
        solver, fused = "cg", 2
    out = {}
    for fz in ((fused, False) if fused is True else (fused,)):
        name = base(solver)
        opts = dict(OPTS.get(solver, {}))
        mem = opts.pop("memory", 0)
        ws = kb.krylov_workspace(name, m, n, dt, memory=mem)
        b = np.cos(np.arange(m)).astype(dt)
        args = (A_op, b, np.sin(np.arange(n)).astype(dt)) if name in ("bilqr", "trilqr") else (A_op, b)
        ws.solve(*args, itmax=20, history=True, fused=fz, **zero_tol(name), **opts)
        st = ws.stats
        vecs = (ws.x, ws.y) if name in ("bilqr", "trilqr") else (ws.x,)
        out[fz] = tuple(v.tobytes() for v in vecs) + tuple(
            (k, np.asarray(v, dtype=np.float64).tobytes() if isinstance(v, (list, float)) else v)
            for k, v in sorted(vars(st).items()) if "timer" not in k)
        ws.free()
    return out


def ring_pass(kb, monkeypatch, op, dt, plan):
    """Every solver of the operator's group under a forced (CTAs per SM, stages), or the default plan (None)."""
    from krylov_b200 import CsrOperator
    A = ring_operator(op)
    monkeypatch.setenv("KB200_CSR_DICT", "0")
    if plan is None:
        monkeypatch.delenv("KB200_STAGES", raising=False)
        monkeypatch.delenv("KB200_CTAS_PER_SM", raising=False)
    else:
        monkeypatch.setenv("KB200_CTAS_PER_SM", str(plan[0]))
        monkeypatch.setenv("KB200_STAGES", str(plan[1]))
        assert_plan(A, dt, plan)
    A_op = CsrOperator.from_scipy(A, dtype=dt)
    m, n = A.shape
    out = {s: ring_run(kb, s, A_op, m, n, dt) for s in RING[op]}       # Aᵀ is formed and planned at the first solve
    A_op.free()
    return out


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("op", sorted(RING))
def test_ring_depth_is_bit_identical(kb, monkeypatch, op, dt):
    isz = np.dtype(dt).itemsize
    default = default_plan(ring_cap(op), isz)
    assert default == (3, 2)
    ref = ring_pass(kb, monkeypatch, op, dt, None)
    for cps in (3, 2, 1):
        depths = ring_depths(op, cps, isz)
        assert len(depths) >= (3 if cps == 3 else 4), (cps, depths)
        first = None
        for s in depths:
            got = ring_pass(kb, monkeypatch, op, dt, (cps, s))
            if first is None:
                first = got
            for solver in got:
                assert got[solver] == first[solver], (solver, cps, s)
            if (cps, s) == default:
                for solver in got:
                    assert got[solver] == ref[solver], (solver, "default plan vs forced twin")


# ----------------------------------------------------------------------------------------------------------------------
# 4. A forced ring that does not fit falls back to the default plan
# ----------------------------------------------------------------------------------------------------------------------
def test_forced_ring_beyond_the_launch_ceiling_falls_back(kb, oracles, monkeypatch):
    """KB200_CTAS_PER_SM=1 with a ring between the 220 KB every staged launcher opts in to and the planner's old 226 KB
    bound: the plan must be the default one (not a ring no launch can take), and the solve must match the oracle."""
    isz = 8
    cap = next(c for c in range(4000, 9000) if 220 * KB < ring_bytes(c, 3, isz) <= 226 * KB)
    A = sp.lil_matrix(_mat(P.div_grad_csr(20)))
    n = A.shape[0]
    extra = cap - (A[:TILE_ROWS].nnz)                                  # widen row 1 until tile 0 holds `cap` nonzeros
    cols = [j for j in range(n) if A[1, j] == 0][:extra]
    A[1, cols] = 1e-4
    A = sp.csr_matrix(A)
    assert tile_cap(A) == cap and 220 * KB < ring_bytes(cap, 3, isz) <= 226 * KB
    monkeypatch.setenv("KB200_CTAS_PER_SM", "1")
    monkeypatch.setenv("KB200_STAGES", "3")
    assert_plan(A, np.float64, default_plan(cap, isz))
    b = A @ np.ones(n)
    for fused in (True, False):
        for solver in ("bicgstab", "gmres"):
            compare(oracles, kb, solver, A, b, fused=fused, **zero_tol(solver), itmax=30)
