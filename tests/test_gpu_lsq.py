"""GPU parity of lsqr! and lsmr! on rectangular operators against the CPU oracle (oracle/krylov_oracle_lsq.h), Float64:
same iteration count, status and `inconsistent`; residual and Aᴴ-residual histories within 1e-6 relative at every
iteration (or 10x the oracle's own sensitivity to a few-ulp change of b, where that is larger); x within 1e-6."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from krylov_b200 import _lib
from krylov_b200 import problems as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-6


@pytest.fixture(scope="module")
def LO():
    """The CPU restatement of lsqr! / lsmr! and its problem generators (oracle/lsq_oracle.py; test infrastructure)."""
    from oracle import lsq_oracle
    lsq_oracle.lib()
    return lsq_oracle


def _sens(LO, solver, A, b, kw):
    """Running max of the oracle's relative history change under small relative perturbations of b (three random sign
    patterns of 1 and 8 ulps: the device's tree-ordered dot products differ from the oracle's sequential sums by a few
    roundings, not one)."""
    _, s0 = getattr(LO, solver)(A, b, **kw)
    out = [np.zeros(len(s0["residuals"])), np.zeros(len(s0["Aresiduals"]))]
    for seed in range(3):
        for ulps in (1, 8):
            sign = np.random.default_rng(seed).choice([-1.0, 1.0], size=len(b))
            _, s1 = getattr(LO, solver)(A, b * (1 + ulps * 2.2e-16 * sign), **kw)
            for i, key in enumerate(("residuals", "Aresiduals")):
                r0, r1 = np.asarray(s0[key]), np.asarray(s1[key])
                k = min(len(r0), len(r1))
                s = np.full(len(r0), np.inf)
                s[:k] = np.abs(r0[:k] - r1[:k]) / np.maximum(np.abs(r0[:k]), 1e-300)
                out[i] = np.maximum(out[i], np.maximum.accumulate(s))
    return out


def _compare(LO, kb, solver, A, b, gpu_A=None, xtol=TOL, **kw):
    """Solve on the GPU (operator gpu_A, default A) and with the oracle; assert the parity bar."""
    okw = {k: v for k, v in kw.items() if k not in ("fused",)}
    xo, so = getattr(LO, solver)(A, b, **okw)
    x, st = getattr(kb, solver)(A if gpu_A is None else gpu_A, b, history=True, n=A.shape[1], **kw)
    x = x.cpu().numpy() if hasattr(x, "cpu") else x
    assert (st.niter, st.status, st.inconsistent) == (so["niter"], so["status"], so["inconsistent"]), \
        ((st.niter, st.status, st.inconsistent), (so["niter"], so["status"], so["inconsistent"]))
    sens = None
    for i, key in enumerate(("residuals", "Aresiduals")):
        r, ro = np.asarray(getattr(st, key)), np.asarray(so[key])
        assert len(r) == len(ro), key
        tol = np.full(len(ro), TOL)
        ok = np.abs(r - ro) <= tol * np.abs(ro) + 1e-9 * abs(ro[0])
        if not ok.all():
            sens = sens or _sens(LO, solver, A, b, okw)
            tol = np.maximum(TOL, 10 * sens[i][:len(ro)])
            ok = np.abs(r - ro) <= tol * np.abs(ro) + 1e-9 * abs(ro[0])
        assert ok.all(), f"{key}: max rel deviation {np.max(np.abs(r - ro) / np.maximum(np.abs(ro), 1e-300)):.3e}"
    assert np.linalg.norm(x - xo) <= xtol * max(np.linalg.norm(xo), 1e-300), np.linalg.norm(x - xo) / np.linalg.norm(xo)
    return x, st, so


def _rect_with_gaps(m, n, seed, density=0.08):
    """Random m x n matrix with empty rows and empty columns."""
    A = sp.random(m, n, density=density, random_state=seed, format="lil")
    A[3, :] = 0
    A[m - 1, :] = 0
    A[:, 1] = 0
    A[:, n - 2] = 0
    A = sp.csr_matrix(A)
    A.eliminate_zeros()
    return A


def _shapes(LO):
    rng = np.random.default_rng(5)
    b40, A40, *_ = LO.lsq_test(40, 40, 4, 2, 0)
    b60, A60, *_ = LO.lsq_test(60, 30, 3, 3, 0)
    Aw = sp.csr_matrix(A60.T)                                   # 30 x 60: m < n
    D = sp.csr_matrix(LO.ddx(50))                                # 50 x 51
    rp, ci, va = P.grad_csr(7)
    G = sp.csr_matrix((va, ci, rp), shape=(len(rp) - 1, 7 ** 3))
    R1, R2 = _rect_with_gaps(300, 120, 1), _rect_with_gaps(90, 200, 2)
    Sq = sp.csr_matrix(sp.random(200, 200, density=0.05, random_state=3) + 4 * sp.identity(200))
    return {"square": (Sq, rng.standard_normal(200)), "tall_lstp": (A60, b60), "wide_lstp": (Aw, rng.standard_normal(30)),
            "ddx": (D, rng.standard_normal(50)), "grad7": (G, rng.standard_normal(G.shape[0])),
            "tall_gaps": (R1, rng.standard_normal(300)), "wide_gaps": (R2, rng.standard_normal(90))}


@pytest.mark.parametrize("solver", ["lsqr", "lsmr"])
@pytest.mark.parametrize("shape", ["square", "tall_lstp", "wide_lstp", "ddx", "grad7", "tall_gaps", "wide_gaps"])
@pytest.mark.parametrize("fused", [True, False])
def test_shapes_match_oracle(kb, LO, solver, shape, fused):
    A, b = _shapes(LO)[shape]
    _compare(LO, kb, solver, A, b, fused=fused, itmax=200)


@pytest.mark.parametrize("solver", ["lsqr", "lsmr"])
def test_square_lstp_before_exhaustion(kb, LO, solver):
    """test(40, 40, 4, 2, 0) has 10 distinct singular values: iteration 10 exhausts the Krylov space and its residual is
    rounding noise, so the comparison stops at 9 iterations."""
    b, A, *_ = LO.lsq_test(40, 40, 4, 2, 0)
    _, st, _ = _compare(LO, kb, solver, A, b, itmax=9)
    assert st.status == "maximum number of iterations exceeded"


@pytest.mark.parametrize("solver", ["lsqr", "lsmr"])
def test_options_match_oracle(kb, LO, solver):
    A, b = _shapes(LO)["tall_gaps"]
    m, n = A.shape
    dm = np.linspace(0.5, 2.0, m)
    dn = np.linspace(1.0, 3.0, n)
    _compare(LO, kb, solver, A, b, lambda_=1e-2, itmax=300)                       # lambda > 0 stays fused
    _compare(LO, kb, solver, A, b, M=dm, N=dn, itmax=300)
    _compare(LO, kb, solver, A, b, M=dm, N=dn, ldiv=True, itmax=300)
    _compare(LO, kb, solver, A, b, M=dm, itmax=300)
    xs, _, _ = _compare(LO, kb, solver, A, b, itmax=300)
    _compare(LO, kb, solver, A, b, radius=0.5 * np.linalg.norm(xs), itmax=300)   # trust region: primitive path
    As, bs, Ms, Ns = LO.sqd()
    _compare(LO, kb, solver, As, bs, M=1 / Ms, N=1 / Ns, sqd=True)
    Ar, br, lam = LO.regularization()
    _compare(LO, kb, solver, Ar, br, lambda_=lam)


@pytest.mark.parametrize("solver", ["lsqr", "lsmr"])
def test_host_callbacks_and_device_b(kb, LO, solver):
    import torch
    from scipy.sparse.linalg import aslinearoperator
    A, b = _shapes(LO)["grad7"]
    _compare(LO, kb, solver, A, b, gpu_A=aslinearoperator(A), itmax=100)
    _compare(LO, kb, solver, A, b, gpu_A=(lambda x: A @ x, lambda y: A.T @ y), itmax=100)
    xo, so = getattr(LO, solver)(A, b, itmax=100)
    x, st = getattr(kb, solver)(A, torch.tensor(b, device="cuda"), itmax=100, history=True)
    assert x.is_cuda and st.niter == so["niter"] and st.status == so["status"]
    assert np.linalg.norm(x.cpu().numpy() - xo) <= TOL * np.linalg.norm(xo)


@pytest.mark.parametrize("solver", ["lsqr", "lsmr"])
@pytest.mark.parametrize("fused", [True, False])
def test_exact_breakdowns(kb, LO, solver, fused):
    n = 20
    _, st, _ = _compare(LO, kb, solver, sp.identity(n, format="csr"), np.linspace(1, 2, n), fused=fused)   # beta = 0 at iteration 1
    assert st.niter == 1
    A = sp.csr_matrix(sp.vstack([sp.identity(n), sp.csr_matrix((3, n))]))
    b = np.zeros(n + 3)
    b[n + 1] = 1.0                                              # b orthogonal to range(A): alpha = 0
    _, st, _ = _compare(LO, kb, solver, A, b, fused=fused)
    assert st.status == "x is a minimum least-squares solution" and st.niter == 0
    _, st, _ = _compare(LO, kb, solver, A, np.zeros(n + 3), fused=fused)
    assert st.status == "x is a zero-residual solution"


@pytest.mark.parametrize("solver", ["lsqr", "lsmr"])
def test_callback_user_exit(kb, LO, solver):
    A, b = _shapes(LO)["grad7"]
    seen = []

    def cb(ws):
        seen.append(1)
        return len(seen) >= 3
    x, st = getattr(kb, solver)(A, b, callback=cb)
    assert st.status == "user-requested exit" and st.niter == 3


@pytest.mark.parametrize("solver", ["lsqr", "lsmr"])
def test_fused_against_primitives(kb, LO, solver):
    rp, ci, va = P.grad_csr(24)
    m, n = len(rp) - 1, 24 ** 3
    b = np.random.default_rng(1).standard_normal(m)
    kw = dict(atol=0.0, rtol=0.0, axtol=0.0, btol=0.0, etol=0.0, conlim=0.0, history=True)
    out, launches = {}, {}
    for fused in (True, False):
        ws = kb.krylov_workspace(solver, m, n, np.float64)
        ws.set_operator((rp, ci, va))
        counts = []
        for itmax in (10, 30):
            l0 = ws.launches
            ws.solve(None, b, itmax=itmax, fused=fused, **kw)
            counts.append(ws.launches - l0)
        launches[fused] = (counts[1] - counts[0]) / 20
        out[fused] = (ws.x, ws.stats)
        ws.free()
    (xf, sf), (xp, spr) = out[True], out[False]
    assert (sf.niter, sf.status) == (spr.niter, spr.status)
    for key in ("residuals", "Aresiduals"):
        a, c = np.asarray(getattr(sf, key)), np.asarray(getattr(spr, key))
        assert np.all(np.abs(a - c) <= 1e-12 * np.abs(c) + 1e-14 * c[0]), key
    assert np.linalg.norm(xf - xp) <= 1e-8 * np.linalg.norm(xp)
    assert launches[True] <= 3 and launches[False] >= 11, launches


@pytest.mark.parametrize("solver", ["lsqr", "lsmr"])
def test_bench_size_parity(kb, LO, solver):
    """The benchmark workload (gradient of the 215^3 grid, m = 29 676 450, n = 9 938 375) over 4 iterations."""
    N = 215
    rp, ci, va = P.grad_csr(N)
    m, n = len(rp) - 1, N ** 3
    A = sp.csr_matrix((va, ci, rp), shape=(m, n))
    b = np.random.default_rng(0).standard_normal(m)
    kw = dict(atol=0.0, rtol=0.0, axtol=0.0, btol=0.0, etol=0.0, conlim=0.0, itmax=4)
    _compare(LO, kb, solver, A, b, gpu_A=(rp, ci, va), **kw)


@pytest.mark.parametrize("solver", ["lsqr", "lsmr"])
def test_float32(kb, LO, solver):
    A, _ = _shapes(LO)["square"]
    b = A @ np.ones(A.shape[1])
    A32, b32 = A.astype(np.float32), b.astype(np.float32)
    xo, so = getattr(LO, solver)(A32, b32, dtype=np.float32)
    x, st = getattr(kb, solver)(A32, b32)
    assert st.solved and abs(st.niter - so["niter"]) <= 1, (st.niter, so["niter"])
    r = b - A @ x.astype(np.float64)
    assert np.linalg.norm(A.T @ r) <= 1e-3 * np.linalg.norm(A.T @ b)


def _flat_spmv(dev_ctx, L, csr, x, ylen):
    px, py = L.kb200_alloc(x.nbytes), L.kb200_alloc(8 * ylen)
    try:
        L.kb200_h2d(px, x.ctypes.data_as(C.c_void_p), x.nbytes)
        out = {}
        for variant in (1, 2):
            assert L.kb200_spmv_csr(dev_ctx, csr, px, py, variant) == 0, _lib.last_error()
            L.kb200_sync(dev_ctx)
            y = np.empty(ylen)
            L.kb200_d2h(y.ctypes.data_as(C.c_void_p), py, y.nbytes)
            out[variant] = y
        return out
    finally:
        L.kb200_free(px)
        L.kb200_free(py)


@pytest.mark.parametrize("shape", [(3000, 700), (700, 3000)])
def test_rectangular_spmv_and_transpose_bit_exact(shape):
    L = _lib.lib()
    m, n = shape
    rng = np.random.default_rng(4)
    A = _rect_with_gaps(m, n, 9, density=0.01)
    A.data = rng.integers(-4, 5, size=A.nnz).astype(np.float64)
    A.eliminate_zeros()
    A.sort_indices()
    ctx = L.kb200_ctx_create(0)
    rp, ci = A.indptr.astype(np.int32), A.indices.astype(np.int32)
    csr = L.kb200_csr_create_rect(ctx, _lib.KRYLOV_FLOAT64, m, n, A.nnz, rp.ctypes.data_as(C.c_void_p),
                                  ci.ctypes.data_as(C.c_void_p), A.data.ctypes.data_as(C.c_void_p), 0, 4, 0)
    assert csr, _lib.last_error()
    mm, nn, nz = C.c_int(), C.c_int(), C.c_longlong()
    L.kb200_csr_shape(csr, C.byref(mm), C.byref(nn), C.byref(nz))
    assert (mm.value, nn.value, nz.value) == (m, n, A.nnz)
    csrT = L.kb200_csr_transpose(ctx, csr)
    assert csrT, _lib.last_error()
    L.kb200_csr_shape(csrT, C.byref(mm), C.byref(nn), C.byref(nz))
    assert (mm.value, nn.value) == (n, m)
    for M_, op, xlen, ylen in ((A, csr, n, m), (sp.csr_matrix(A.T), csrT, m, n)):
        x = rng.integers(-3, 4, size=xlen).astype(np.float64)
        referenced = np.zeros(xlen, bool)
        referenced[M_.indices] = True
        x[~referenced] = np.nan                                  # unreferenced entries must never reach y
        xr = np.where(referenced, x, 0.0)
        plan = (C.c_longlong * 7)()
        L.kb200_csr_plan(op, plan)
        assert plan[3], "the tile plan should fit: the staged kernel is the one under test"
        for variant, y in _flat_spmv(ctx, L, op, x, ylen).items():
            assert np.array_equal(y, M_ @ xr), variant
    # a column index beyond the declared columns is refused
    bad = ci.copy()
    bad[np.argmax(np.diff(rp) > 0)] = n
    assert not L.kb200_csr_create_rect(ctx, _lib.KRYLOV_FLOAT64, m, n, A.nnz, rp.ctypes.data_as(C.c_void_p),
                                       bad.ctypes.data_as(C.c_void_p), A.data.ctypes.data_as(C.c_void_p), 0, 4, 0)
    L.kb200_csr_destroy(csrT)
    L.kb200_csr_destroy(csr)
    L.kb200_ctx_destroy(ctx)


def test_c_abi_rules(kb):
    L = _lib.lib()
    ws = C.c_void_p()
    assert L.krylov_workspace_create(_lib.KRYLOV_LSQR, 5, 3, _lib.KRYLOV_FLOAT64, 0, None, C.byref(ws)) == 0
    assert L.krylov_workspace_create(_lib.KRYLOV_CG, 5, 3, _lib.KRYLOV_FLOAT64, 0, None, C.byref(C.c_void_p())) == -1
    f = _lib.MATVEC(lambda x, y, u: None)
    b = np.ones(5)
    assert L.krylov_solve(ws, f, _lib.MATVEC(), _lib.MATVEC(), _lib.MATVEC(), b.ctypes.data_as(C.c_void_p), None, None, None) == -1
    assert "matvec_At" in _lib.last_error()
    assert L.krylov_get_y(ws, None, 5) == -2
    assert L.krylov_warm_start(ws, np.zeros(3).ctypes.data_as(C.c_void_p), 3) == -1
    assert L.krylov_b200_dist_init(ws, 0, 1, 0, None, None) == -1
    assert L.krylov_workspace_free(ws) == 0


def _ref_prog(name):
    path = os.path.join(ROOT, "oracle", "_ref", name)
    if not os.path.exists(path):
        pytest.skip(f"oracle/_ref/{name} was not built (reference tree absent at build time)")
    return subprocess.run([path], capture_output=True, text=True, timeout=600)


def test_reference_least_squares_example():
    out = _ref_prog("least_squares")
    assert out.returncode == 0, out.stderr
    assert "Solved: yes" in out.stdout and "x = [ 1.00 2.00 3.00 ]" in " ".join(out.stdout.split()), out.stdout


def test_reference_test_all_solvers_lsqr_lsmr_rows():
    out = _ref_prog("test_all_solvers")
    rows = [l for l in out.stdout.splitlines() if l.split() and l.split()[0].lower() in ("lsqr", "lsmr")]
    assert len(rows) >= 2, out.stdout[-2000:]
    for l in rows:
        assert "PASS" in l, l
