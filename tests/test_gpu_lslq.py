"""GPU parity of lslq! on rectangular operators against the CPU oracle (oracle/krylov_oracle_lslq.h), Float64, at the bar
of tests/test_gpu_cgls.py: same iteration count, status and `inconsistent`; residual, Aᴴ-residual and error-bound
histories within 1e-6 relative (or 10x the oracle's own sensitivity to a few-ulp change of b); x within 1e-6."""
import ctypes as C
import functools
import os

import numpy as np
import pytest
import scipy.sparse as sp

import parity
from krylov_b200 import _lib
from krylov_b200 import problems as P
from parity import TOL

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
G = parity.golden_module("lslq")
BOUNDS = ("err_lbnds", "err_ubnds_lq", "err_ubnds_cg")


@pytest.fixture(scope="module")
def CO():
    from oracle import cgls_oracle
    cgls_oracle.lib()
    return cgls_oracle


def _compare(CO, kb, A, b, **kw):
    """The bar of tests/test_gpu_cgls.py, and the error-bound histories against the oracle's with the same perturbations
    of b (the bounds are built from the LQ iterates ζ, far more sensitive than the residuals)."""
    x, st, so = parity.compare(CO.lslq, functools.partial(kb.lslq, n=A.shape[1]), A, b,
                               keys=("residuals", "Aresiduals"), flags=("inconsistent",), floor=1e-9, **kw)
    assert st.error_with_bnd == so["error_with_bnd"]
    okw = {k: v for k, v in kw.items() if k not in ("fused", "gpu_A", "xtol")}
    runs = functools.cache(lambda: parity.perturbed_runs(CO.lslq, A, b, **okw))
    for key in BOUNDS:
        r, ro = np.asarray(getattr(st, key)), np.asarray(so[key])
        assert len(r) == len(ro), key
        parity.assert_history(key, r, ro, lambda: parity.sens(ro, runs(), key), 1e-300)
    return x, st, so


def _compare_early(CO, kb, A, b, fused, **kw):
    """LSLQ's default √eps tolerances stop most runs where rounding noise decides the last iterations: the oracle's own
    iteration count moves under a few-ulp change of b.  Histories and x are compared up to two iterations before the
    earliest stop among the oracle's perturbed runs (lslq! tests `iter ≥ itmax` before its increment, so itmax = k runs
    k + 1 iterations), x against 10x the oracle's own change under the same perturbations; the full solve must stop
    within two iterations of the range of the perturbed runs."""
    _, so = CO.lslq(A, b, **kw)
    stops = [so["niter"]] + [s["niter"] for _, s in parity.perturbed_runs(CO.lslq, A, b, **kw)]
    if min(stops) > 3:
        kk = dict(kw, itmax=min(stops) - 3)
        _compare(CO, kb, A, b, fused=fused, xtol=None, **kk)
    else:
        _compare(CO, kb, A, b, fused=fused, **kw)
    _, st = kb.lslq(A, b, fused=fused, **kw)
    assert st.solved == so["solved"] and min(stops) - 2 <= st.niter <= max(stops) + 2, (st.niter, stops)


@pytest.mark.parametrize("shape", ["square", "tall_lstp", "wide_lstp", "ddx", "grad7", "tall_gaps", "wide_gaps"])
@pytest.mark.parametrize("fused", [True, False])
def test_shapes_match_oracle(kb, CO, shape, fused):
    A, b = parity.shapes()[shape]
    _compare_early(CO, kb, A, b, fused, itmax=200)


@pytest.mark.parametrize("fused", [True, False])
def test_options_match_oracle(kb, CO, fused):
    A, b = parity.shapes()["tall_gaps"]
    m, n = A.shape
    dm, dn = np.linspace(0.5, 2.0, m), np.linspace(1.0, 3.0, n)
    _compare_early(CO, kb, A, b, fused, lambda_=1e-2, itmax=300)                  # λ > 0 stays fused
    _compare_early(CO, kb, A, b, fused, M=dm, N=dn, itmax=300)
    _compare_early(CO, kb, A, b, fused, M=dm, N=dn, ldiv=True, itmax=300)
    _compare_early(CO, kb, A, b, fused, N=dn, itmax=300)
    for t in (False, True):
        _compare_early(CO, kb, A, b, fused, sigma=1e-3, utol=1e-4, transfer_to_lsqr=t, itmax=300)
        _compare_early(CO, kb, A, b, fused, sigma=5.0, transfer_to_lsqr=t, itmax=300)
    _compare_early(CO, kb, A, b, fused, etol=1e-3, btol=1e-3, conlim=1e3, atol=1e-10, rtol=1e-10, itmax=300)
    for key in sorted(G.cases()):                               # the reference's known-answer problems
        Ak, bk, kw = G.cases()[key]
        _compare_early(CO, kb, Ak, bk, fused, **kw)


def test_error_bounds_of_the_reference(kb, CO):
    b, A, *_ = CO.lsq_test(40, 40, 4, 4, 0)
    _, st = kb.lslq(A, b, sigma=1.0)
    assert st.error_with_bnd
    rng = np.random.default_rng(0)                              # test/test_lslq.jl, fixed orthogonal factors
    U, _ = np.linalg.qr(rng.random((6, 6)))
    V, _ = np.linalg.qr(rng.random((4, 4)))
    A = sp.csr_matrix(U @ np.vstack([np.diag([1.0, 2.0, 3.0, 4.0]), np.zeros((2, 4))]) @ V.T)
    b = np.ones(6)
    x_exact = np.linalg.lstsq(A.toarray(), b, rcond=None)[0]
    for t in (False, True):
        for fused in (True, False):
            x, st = kb.lslq(A, b, sigma=1.0 - 1.0e-10, history=True, transfer_to_lsqr=t, fused=fused)
            assert abs(st.err_ubnds_lq[-1]) <= np.sqrt(2.2e-16) and abs(st.err_ubnds_cg[-1]) <= np.sqrt(2.2e-16)
            assert np.linalg.norm(x - x_exact) <= np.sqrt(2.2e-16) * np.linalg.norm(x_exact)


def test_host_callbacks_and_device_b(kb, CO):
    import torch
    from scipy.sparse.linalg import aslinearoperator
    A, b = parity.shapes()["grad7"]
    _compare(CO, kb, A, b, gpu_A=aslinearoperator(A), itmax=100)
    _compare(CO, kb, A, b, gpu_A=(lambda x: A @ x, lambda y: A.T @ y), itmax=100, sigma=1e-2)
    xo, so = CO.lslq(A, b, itmax=100)
    x, st = kb.lslq(A, torch.tensor(b, device="cuda"), itmax=100, history=True)
    assert x.is_cuda and st.niter == so["niter"] and st.status == so["status"]
    assert np.linalg.norm(x.cpu().numpy() - xo) <= TOL * np.linalg.norm(xo)


@pytest.mark.parametrize("fused", [True, False])
def test_zero_rhs_and_zero_adjoint_residual(kb, CO, fused):
    n = 20
    A = sp.csr_matrix(sp.vstack([sp.identity(n), sp.csr_matrix((3, n))]))
    b = np.zeros(n + 3)
    _, st, _ = _compare(CO, kb, A, b, fused=fused)
    assert st.status == "x is a zero-residual solution" and st.niter == 0
    b[n + 1] = 1.0
    x, st, _ = _compare(CO, kb, A, b, fused=fused)
    assert st.status == "x is a minimum least-squares solution" and st.niter == 0 and not x.any()


def test_callback_unsupported_kwargs_and_abi(kb, CO):
    A, b = parity.shapes()["grad7"]
    seen = []

    def cb(ws):
        seen.append(1)
        return len(seen) >= 3
    _, st = kb.lslq(A, b, callback=cb, history=True)
    assert st.status == "user-requested exit" and st.niter == 3 and len(st.residuals) == 4
    with pytest.raises(TypeError):
        kb.lslq(A, b, callback=lambda ws: "string")
    for kw in (dict(radius=1.0), dict(axtol=1e-3), dict(gamma=1.0)):
        with pytest.raises(kb.B200Error):
            kb.lslq(A, b, **kw)
    L = _lib.lib()
    ws = C.c_void_p()
    assert L.krylov_workspace_create(_lib.KRYLOV_LSLQ, 5, 3, _lib.KRYLOV_FLOAT64, 0, None, C.byref(ws)) == 0
    f = _lib.MATVEC(lambda x, y, u: None)
    bb = np.ones(5)
    assert L.krylov_solve(ws, f, _lib.MATVEC(), _lib.MATVEC(), _lib.MATVEC(), bb.ctypes.data_as(C.c_void_p), None, None, None) == -1
    assert "matvec_At" in _lib.last_error()
    assert L.krylov_get_y(ws, None, 5) == -2
    assert L.krylov_warm_start(ws, np.zeros(3).ctypes.data_as(C.c_void_p), 3) == -1
    assert L.krylov_b200_dist_init(ws, 0, 1, 0, None, None) == -1
    assert L.krylov_workspace_free(ws) == 0


def test_fused_against_primitives(kb):
    rp, ci, va = P.grad_csr(24)
    m, n = len(rp) - 1, 24 ** 3
    b = np.random.default_rng(1).standard_normal(m)
    for lam, sig in ((0.0, 0.0), (1e-2, 1e-3)):
        kw = dict(atol=0.0, rtol=0.0, etol=0.0, utol=0.0, btol=0.0, conlim=0.0, lambda_=lam, sigma=sig, history=True)
        out, launches = {}, {}
        for fused in (True, False):
            ws = kb.krylov_workspace("lslq", m, n, np.float64)
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
        for key in ("residuals", "Aresiduals") + BOUNDS:
            a, c = np.asarray(getattr(sf, key)), np.asarray(getattr(spr, key))
            assert len(a) == len(c) and np.all(np.abs(a - c) <= 1e-12 * np.abs(c) + 1e-14 * max(np.max(np.abs(c), initial=0), 1e-300)), key
        assert np.linalg.norm(xf - xp) <= 1e-10 * np.linalg.norm(xp)
        assert launches[True] == 3 and launches[False] >= 10, launches


def test_bench_size_parity(kb, CO):
    N = 215
    rp, ci, va = P.grad_csr(N)
    m, n = len(rp) - 1, N ** 3
    A = sp.csr_matrix((va, ci, rp), shape=(m, n))
    b = np.random.default_rng(0).standard_normal(m)
    _compare(CO, kb, A, b, gpu_A=(rp, ci, va), atol=0.0, rtol=0.0, etol=0.0, btol=0.0, conlim=0.0, itmax=4)


def test_float32(kb, CO):
    A, _ = parity.shapes()["square"]
    b = A @ np.ones(A.shape[1])
    A32, b32 = A.astype(np.float32), b.astype(np.float32)
    _, so = CO.lslq(A32, b32, dtype=np.float32)
    x, st = kb.lslq(A32, b32)
    assert st.solved and abs(st.niter - so["niter"]) <= 3, (st.niter, so["niter"])
    r = b - A @ x.astype(np.float64)
    assert np.linalg.norm(A.T @ r) <= 1e-3 * np.linalg.norm(A.T @ b)
