"""GPU parity of lnlq! against the CPU oracle (oracle/krylov_oracle_lnlq.h), Float64: same iteration count,
status, solved flag and error_with_bnd; the residual history and the σ-based bounds within parity.TOL relative at every
iteration (or 10x the oracle's own sensitivity to a few-ulp change of b, where that is larger); x and y within 1e-6
relative where the counts are steady.  Both paths: the fused one (2 launches per pass) and fused = 0."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.sparse as sp

import parity
from krylov_b200 import _lib
from parity import TOL

pytestmark = pytest.mark.gpu
FLAGS = ("solved", "error_with_bnd")


@pytest.fixture(scope="module")
def O():
    from oracle import lnlq_oracle
    lnlq_oracle.lib()
    return lnlq_oracle


@pytest.fixture(scope="module")
def kb():
    import krylov_b200
    if krylov_b200.device_count() < 1:
        pytest.skip("no CUDA device")
    return krylov_b200


def compare(O, kb, A, b, *, bounds=False, xtol=TOL, **kw):
    """parity.compare on x and the residual history (and error_bnd_x / error_bnd_y with bounds), then y against the
    oracle's y where the counts match."""
    ys = {}

    def oracle(A_, b_, **kw_):
        x, y, st = O.lnlq(A_, b_, **kw_)
        ys.setdefault("oracle", y)
        return x, st

    def gpu(A_, b_, **kw_):
        x, y, st = kb.lnlq(A_, b_, **kw_)
        ys["gpu"] = y.cpu().numpy() if hasattr(y, "cpu") else y
        return x, st

    keys = ("residuals", "error_bnd_x", "error_bnd_y") if bounds else ("residuals",)
    x, st, so = parity.compare(oracle, gpu, A, b, keys=keys, flags=FLAGS, floor=1e-9, xtol=xtol, **kw)
    if st.niter == so["niter"] and xtol is not None:
        yo = ys["oracle"]
        assert np.linalg.norm(ys["gpu"] - yo) <= TOL * max(np.linalg.norm(yo), 1e-300)
    return x, ys["gpu"], st, so


def oracle_cases(O):
    """name -> (A, b, kwargs, has bounds): the problems of the reference's test_lnlq.jl (tests/golden/gen_golden_lnlq.py,
    without the NaN-producing small_ln LNLQ point)."""
    out = {}
    for name, (A, b, kw) in parity.golden_module("lnlq").cases().items():
        if name == "small_ln_lq":
            continue
        bounds = kw.get("sigma", 0.0) > 0 or kw.get("lambda_", 0.0) > 0 or kw.get("sqd", False)
        out[name] = (A, b, kw, bounds)
    return out


CASES = sorted(n for n in __import__("json").load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                                                     "oracle_lnlq.json"))) if n != "small_ln_lq")


def compare_unsteady(O, kb, A, b, *, fused, bounds, **kw):
    """Where the oracle's own outcome moves under a few-ulp change of b (these small systems terminate exactly, and the
    last residual or bound discriminant is rounding noise), the GPU's (niter, status, error_with_bnd) must be one of
    the oracle's outcomes, the histories must follow up to where the oracle's own move by 1e-3, and x and y must lie
    within 10x the oracle's own change."""
    def run(A_, b_, **kw_):
        x, y, st = O.lnlq(A_, b_, **kw_)
        return np.concatenate([x, y]), st
    xyo, so = run(A, b, **kw)
    runs = parity.perturbed_runs(run, A, b, **kw)
    outcomes = {(s["niter"], s["status"], s["error_with_bnd"]) for _, s in runs} | {(so["niter"], so["status"],
                                                                                       so["error_with_bnd"])}
    x, y, st = kb.lnlq(A, b, history=True, fused=fused, **kw)
    assert (st.niter, st.status, st.error_with_bnd) in outcomes, ((st.niter, st.status, st.error_with_bnd), outcomes)
    for key in ("residuals", "error_bnd_x", "error_bnd_y") if bounds else ("residuals",):
        rg, ro = np.asarray(getattr(st, key)), np.asarray(so[key])
        k = min(len(rg), len(ro))
        sn = parity.sens(ro, runs, key)
        k = min(k, int(np.argmax(sn > 1e-3)) if np.any(sn > 1e-3) else k)
        parity.assert_history(key, rg[:k], ro[:k], lambda: sn, 1e-9 * (abs(ro[0]) if len(ro) else 0.0))
    bar = max(TOL, 10 * parity.xsens(xyo, runs))
    assert np.linalg.norm(np.concatenate([x, y]) - xyo) <= bar * np.linalg.norm(xyo)


def oracle_is_steady(O, A, b, kw):
    def run(A_, b_, **kw_):
        x, _, st = O.lnlq(A_, b_, **kw_)
        return x, st
    _, so = run(A, b, **kw)
    return all((s["niter"], s["status"], s["error_with_bnd"]) == (so["niter"], so["status"], so["error_with_bnd"])
               for _, s in parity.perturbed_runs(run, A, b, **kw))


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("case", CASES)
def test_oracle_cases(O, kb, case, fused):
    A, b, kw, bounds = oracle_cases(O)[case]
    if not oracle_is_steady(O, A, b, kw):
        compare_unsteady(O, kb, A, b, fused=fused, bounds=bounds, **kw)
        return
    # small_sp_1 runs to itmax on an inconsistent system: its last steps work on rounding noise
    compare(O, kb, A, b, fused=fused, bounds=bounds, xtol=None if case.startswith("small_sp_1") else TOL, **kw)


def consistent_shapes():
    """parity.shapes() with b = A z: consistent systems on m > n, m < n, m = n and operators with empty rows and
    columns."""
    rng = np.random.default_rng(11)
    return {k: (A, A @ rng.standard_normal(A.shape[1])) for k, (A, _) in parity.shapes().items()}


ZERO_TOL = dict(atol=0.0, rtol=0.0, utolx=0.0, utoly=0.0)


@pytest.mark.parametrize("transfer", [False, True])
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("shape", sorted(parity.shapes()))
def test_shapes(O, kb, shape, fused, transfer):
    A, b = consistent_shapes()[shape]
    compare(O, kb, A, b, fused=fused, itmax=10, transfer_to_craig=transfer, xtol=None if "lstp" in shape else TOL,
            **ZERO_TOL)


@pytest.mark.parametrize("fused", [True, False])
def test_shapes_with_bounds(O, kb, fused):
    """σ > 0 on the fused path: the bounds are host scalars, the passes are the same."""
    A, b = consistent_shapes()["tall_gaps"]
    compare(O, kb, A, b, fused=fused, itmax=10, sigma=1e-3, bounds=True, atol=0.0, rtol=0.0)


def test_fused_path_runs_and_untiled_twin_matches(O, kb):
    """2 launches per pass on a staged operator, and as many on its untiled twins (the gradient with a dense row: A
    untiled; with a dense column: Aᵀ untiled), whose results match the oracle."""
    G = parity.grad(24)
    rng = np.random.default_rng(3)
    b = G @ rng.standard_normal(G.shape[1])
    assert parity.launches_per_iteration(kb, "lnlq", G, b, extra_iter=1, **ZERO_TOL) == 2
    assert parity.launches_per_iteration(kb, "lnlq", G, b, fused=False, extra_iter=1, **ZERO_TOL) > 2
    for row in (True, False):
        U = parity.dense_line(parity.grad(24), row)
        bu = U @ rng.standard_normal(U.shape[1])
        assert parity.launches_per_iteration(kb, "lnlq", U, bu, extra_iter=1, **ZERO_TOL) == 2
        compare(O, kb, U, bu, fused=True, itmax=40, xtol=None, **ZERO_TOL)


def test_ring_depth_changes_no_bit(kb, monkeypatch):
    """On an operator of about 10⁶ rows, at 3, 2 and 1 CTAs per SM, every ring depth gives byte-identical x, y,
    histories, niter and status (parity.assert_ring_depth_changes_no_bit)."""
    A = parity.grad(72)                                         # 1 119 744 rows, 373 248 columns
    b = A @ np.cos(np.arange(A.shape[1], dtype=np.float64))
    kw = dict(itmax=20, history=True, **ZERO_TOL)

    def run():
        x, y, st = kb.lnlq(A, b, **kw)
        return x.tobytes(), y.tobytes(), np.asarray(st.residuals).tobytes(), st.niter, st.status
    parity.assert_ring_depth_changes_no_bit(monkeypatch, run)


def test_options_against_oracle(O, kb):
    A, b = O.over_consistent()
    Au, bu = O.under_consistent()
    compare(O, kb, A, b, itmax=1)                                                  # itmax: niter = 2
    compare(O, kb, Au, bu, lambda_=1e-2, fused=True, bounds=True)                 # λ > 0 (primitive path)
    compare(O, kb, Au, bu, M=np.linspace(1, 2, Au.shape[0]), N=np.linspace(1, 3, Au.shape[1]))   # diagonal M / N
    compare(O, kb, Au, bu, sigma=0.5, utolx=1e-3, utoly=1e-3, bounds=True)        # bounds stop the solve
    compare(O, kb, A, b, sigma=0.5, utolx=1e10, utoly=1e10, bounds=True)          # ... before the loop: niter = 1
    x, y, st = kb.lnlq(Au, bu, timemax=0.0)
    assert st.status == "time limit exceeded" and st.niter == 2


@pytest.mark.parametrize("fused", [True, False])
def test_callback_reads_current_x_and_y(O, kb, fused):
    """The callback sees the x and y of the pass it is called after (the fused y update is flushed before it)."""
    A, b = O.over_consistent()
    seen = []
    ws = kb.LnlqWorkspace(A.shape[0], A.shape[1], np.float64)
    try:
        ws.solve(A, b, fused=fused, atol=0.0, rtol=0.0, utolx=0.0, utoly=0.0,
                 callback=lambda w: seen.append((w.x.copy(), w.y.copy())) or len(seen) >= 2)
        assert ws.stats.status == "user-requested exit" and ws.stats.niter == 3
        for k in (1, 2):
            xs, ys = seen[k - 1]
            # y: the oracle's after k passes (a tired LNLQ-point exit leaves y as the last pass made it)
            _, yo, so = O.lnlq(A, b, itmax=k, transfer_to_craig=False, **ZERO_TOL)
            assert so["niter"] == k + 1
            assert np.linalg.norm(ys - yo) <= TOL * np.linalg.norm(yo)
            # x: (xᵃᵘˣ)ₖ, which the terminal step moves on; restated densely
            xo = _xaux_after(A, b, k)
            assert np.linalg.norm(xs - xo) <= TOL * np.linalg.norm(xo)
    finally:
        ws.free()


def _xaux_after(A, b, k):
    """(xᵃᵘˣ)ₖ = Vₖtₖ, the x the reference's callback sees after pass k (λ = 0, M = N = I), restated densely."""
    A = A.toarray()
    beta = np.linalg.norm(b)
    u = b / beta
    v = A.T @ u
    alpha = np.linalg.norm(v)
    v = v / alpha
    x, tau = np.zeros(A.shape[1]), beta / alpha
    for _ in range(k):
        x = x + tau * v
        u = A @ v - alpha * u
        beta = np.linalg.norm(u)
        u = u / beta
        v = A.T @ u - beta * v
        alpha_n = np.linalg.norm(v)
        v = v / alpha_n
        tau, alpha = -beta * tau / alpha_n, alpha_n
    return x


def test_float32_within_dot_rounding_envelope(O, kb):
    A, b = consistent_shapes()["tall_gaps"]
    kw = dict(itmax=15, **ZERO_TOL)
    _, _, s0 = O.lnlq(A, b, dtype=np.float32, **kw)
    with O.dot_mode(1):
        _, _, s1 = O.lnlq(A, b, dtype=np.float32, **kw)
    for fused in (True, False):
        _, _, st = kb.lnlq(A, b.astype(np.float32), history=True, fused=fused, **kw)
        r0, r1, rg = (np.asarray(v, dtype=np.float64) for v in (s0["residuals"], s1["residuals"], st.residuals))
        k = min(len(r0), len(r1), len(rg))
        env = np.maximum(np.abs(r1[:k] - r0[:k]), 1e-5 * np.abs(r0[:k]))
        assert np.all(np.abs(rg[:k] - r0[:k]) <= 10 * np.maximum.accumulate(env / np.abs(r0[:k])) * np.abs(r0[:k]))


def test_torch_device_inputs(O, kb):
    import torch
    A, b = O.under_consistent()
    x, y, st = kb.lnlq(A, torch.tensor(b, device="cuda"))
    xo, yo, so = O.lnlq(A, b)
    assert st.niter == so["niter"] and st.status == so["status"]
    assert np.linalg.norm(x.cpu().numpy() - xo) <= TOL * np.linalg.norm(xo)
    assert np.linalg.norm(y.cpu().numpy() - yo) <= TOL * np.linalg.norm(yo)


def test_c_abi_contract(O, kb):
    L = _lib.lib()
    sid = _lib.SOLVER_IDS["lnlq"]
    assert sid == 30
    h = C.c_void_p()
    assert L.krylov_workspace_create(sid, 3, 4, 2, _lib.KRYLOV_CPU, None, C.byref(h)) == -2        # Complex
    assert L.krylov_workspace_create(sid, 3, 4, 3, _lib.KRYLOV_CPU, None, C.byref(h)) == -2
    ws = kb.LnlqWorkspace(3, 4, np.float64)
    try:
        A = sp.csr_matrix(np.array([[1.0, 0, 2, 0], [0, 1.0, 0, 3], [1.0, 1, 0, 0]]))
        null = _lib.MATVEC()
        f = _lib.MATVEC(lambda x, y, u: None)
        b = np.array([1.0, 2.0, 3.0])
        rc = L.krylov_solve(ws._h, f, null, null, null, b.ctypes.data_as(C.c_void_p), None, None, None)
        assert rc == -1 and "lnlq applies the adjoint of A" in _lib.last_error()
        ws.solve(A, b, utolx=0.0, utoly=0.0)
        y = np.empty(3)
        assert L.krylov_get_y(ws._h, y.ctypes.data_as(C.c_void_p), 3) == 0
        np.testing.assert_allclose(ws.x, A.T @ y, rtol=1e-10)
        x0 = np.zeros(4)
        assert L.krylov_warm_start(ws._h, x0.ctypes.data_as(C.c_void_p), 4) == -1
        assert "does not support warm-start" in _lib.last_error()
        assert L.krylov_warm_start2(ws._h, x0.ctypes.data_as(C.c_void_p), y.ctypes.data_as(C.c_void_p), 4, 3) == -2
        assert L.krylov_b200_dist_init(ws._h, 0, 2, 0, None, None) == -1
        blocks = np.ones((2, 2, 2))
        assert L.krylov_b200_set_preconditioner_blockdiag(ws._h, 0, 2, blocks.ctypes.data_as(C.c_void_p), 0) == -1
        for name in ("x", "Nv", "y", "w̄", "wbar", "Mu"):
            p = C.c_void_p()
            assert L.krylov_b200_get_vector(ws._h, name.encode(), C.byref(p)) == 0 and p.value, name
        # the reused fields: σ in sigma, utolx in utol, utoly in etol, transfer_to_craig in transfer_to_bicg; the bounds
        # in history slots 3 and 4 with their lengths in nerr_lbnds / nerr_ubnds_lq
        Ao, bo = O.over_consistent()
        for transfer in (False, True):
            ws2 = kb.LnlqWorkspace(Ao.shape[0], Ao.shape[1], np.float64)
            try:
                ws2.solve(Ao, bo, sigma=0.5, utolx=1e-4, utoly=1e-5, atol=0.0, rtol=0.0, transfer_to_craig=transfer,
                          history=True)
                _, _, so = O.lnlq(Ao, bo, sigma=0.5, utolx=1e-4, utoly=1e-5, atol=0.0, rtol=0.0,
                                  transfer_to_craig=transfer)
                st = ws2.stats
                assert (st.niter, st.status, st.error_with_bnd) == (so["niter"], so["status"], so["error_with_bnd"])
                s = _lib.KrylovB200Stats()
                assert L.krylov_b200_get_stats(ws2._h, C.byref(s)) == 0
                assert s.nerr_lbnds == len(so["error_bnd_x"]) and s.nerr_ubnds_lq == len(so["error_bnd_y"])
                for key in ("error_bnd_x", "error_bnd_y"):            # the last bounds are rounding noise near 0
                    want = np.asarray(so[key])
                    np.testing.assert_allclose(getattr(st, key), want, rtol=TOL, atol=1e-9 * want[0])
            finally:
                ws2.free()
    finally:
        ws.free()


def test_sqd_with_lambda_raises(kb):
    with pytest.raises(kb.B200Error, match="sqd cannot be set to true if λ ≠ 0 !"):
        kb.lnlq(sp.csr_matrix(np.eye(2)), np.ones(2), sqd=True, lambda_=1.0)
