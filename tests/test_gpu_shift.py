"""GPU: CG-Lanczos-shift and CGLS-Lanczos-shift through the C ABI against the CPU restatement (oracle/shift_oracle.py).

At <= 256 rows every pass runs one CTA and the oracle's dot mode 2 is the device's reduction order, so the GPU must
return the oracle's bytes: every x_i, every per-shift history, niter, status and the indefinite flags, on the fused
path (the shift-update pass, and CG-Lanczos's grouped passes or CGLS-Lanczos-shift's SpMV epilogues) and the primitive
path (fused = False), with a diagonal and a block-Jacobi M, and with more active shifts than one pass takes.  Beyond
one CTA: tolerance parity, agreement between paths and inputs, the launch count per iteration, and the refusals."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

from krylov_b200 import _lib
from oracle import oracle as O
from oracle import shift_oracle as S
from oracle.lsq_oracle import lsq_test

pytestmark = pytest.mark.gpu

DTYPES = [np.float64, np.float32]
PASS = 16                                   # kShiftPass (kb_internal.h): active shifts per shift-update launch


def _lap1d(n):
    return sp.diags([-np.ones(n - 1), 2.5 * np.ones(n), -np.ones(n - 1)], [-1, 0, 1], format="csr")


def _same(kb, xs, st, xo, so, where):
    assert st.niter == so["niter"] and st.status == so["status"], (where, st.niter, so["niter"], st.status, so["status"])
    assert st.indefinite == so["indefinite"], where
    assert len(xs) == len(xo)
    for i, (x, y) in enumerate(zip(xs, xo)):
        assert x.tobytes() == y.tobytes(), (where, "x", i, np.max(np.abs(x - y)))
    for i, (r, ro) in enumerate(zip(st.residuals, so["residuals"])):
        assert np.asarray(r, dtype=ro.dtype).tobytes() == ro.tobytes(), (where, "residuals", i)


def _bit_cases():
    Ad = O.get_div_grad(6, 6, 6)                                   # 216 rows
    bd = np.linspace(1.0, 2.0, Ad.shape[0])
    d = 1.0 / Ad.diagonal()
    yield "spread", Ad, bd, [0.5, 5.0, 50.0], {}
    yield "one_shift", Ad, bd, [2.0], {}
    yield "many_shifts", Ad, bd, list(np.logspace(-2, 3, 37)), {}
    yield "diag_M", Ad, bd, [0.5, 5.0, 50.0], dict(M=d)
    yield "diag_M_ldiv", Ad, bd, [1.0, 10.0], dict(M=Ad.diagonal().copy(), ldiv=True)
    A, b = O.symmetric_definite()
    yield "negcurv", A, b, [-4.0, -3.0, 2.0], dict(check_curvature=True, itmax=10)
    yield "negcurv_off", A, b, [-4.0, -3.0, 2.0], dict(itmax=10)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("dt", DTYPES)
def test_cg_lanczos_shift_bit_for_bit(kb, dt, fused):
    for name, A, b, shifts, kw in _bit_cases():
        with S.dot_mode(2):
            xo, so = S.cg_lanczos_shift(A, b, shifts, dtype=dt, **kw)
        xs, st = kb.cg_lanczos_shift(A.astype(dt), b.astype(dt), shifts, history=True, fused=fused,
                                     **{k: (v.astype(dt) if k == "M" else v) for k, v in kw.items()})
        _same(kb, xs, st, xo, so, (name, dt.__name__, fused))


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("dt", DTYPES)
def test_block_jacobi_M_bit_for_bit(kb, dt, fused):
    A = O.get_div_grad(6, 6, 6)
    n, bs = A.shape[0], 4
    Ad = A.toarray()
    blocks = np.stack([np.linalg.inv(Ad[i:i + bs, i:i + bs]) for i in range(0, n, bs)])
    b = np.linspace(1.0, 2.0, n)
    with S.dot_mode(2), S.precond_block(bs):
        xo, so = S.cg_lanczos_shift(A, b, [0.5, 5.0], M=blocks.reshape(-1), dtype=dt)
    xs, st = kb.cg_lanczos_shift(A.astype(dt), b.astype(dt), [0.5, 5.0], M=blocks.astype(dt), history=True, fused=fused)
    _same(kb, xs, st, xo, so, ("block-Jacobi", dt.__name__, fused))


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("dt", DTYPES)
def test_cgls_lanczos_shift_bit_for_bit(kb, dt, fused):
    b, A = lsq_test(40, 40, 4, 2, 0)[:2]                           # 160 x 40 (four duplicated blocks)
    for shifts in ([1.0, 2.0, 3.0, 4.0, 5.0, 6.0], list(np.logspace(-3, 2, 37))):
        with S.dot_mode(2):
            xo, so = S.cgls_lanczos_shift(A, b, shifts, dtype=dt)
        xs, st = kb.cgls_lanczos_shift(A.astype(dt), b.astype(dt), shifts, history=True, fused=fused)
        _same(kb, xs, st, xo, so, ("cgls", len(shifts), dt.__name__, fused))


@pytest.mark.parametrize("name", ["divgrad16", "ragged"])
def test_tolerance_parity_beyond_one_cta(kb, name):
    if name == "divgrad16":
        A = O.get_div_grad(16, 16, 16)
        b = np.ones(A.shape[0])
    else:
        A = _lap1d(1001)
        b = np.sin(np.arange(1001.0))
    shifts = [0.01, 0.1, 1.0, 10.0]
    xo, so = S.cg_lanczos_shift(A, b, shifts)
    xs, st = kb.cg_lanczos_shift(A, b, shifts, history=True)
    assert st.niter == so["niter"] and st.status == so["status"]
    for r, ro in zip(st.residuals, so["residuals"]):
        assert len(r) == len(ro) and np.all(np.abs(np.asarray(r) - ro) <= 1e-6 * np.abs(ro))
    for x, y in zip(xs, xo):
        assert np.linalg.norm(x - y) <= 1e-8 * np.linalg.norm(y)
    # CGLS-Lanczos-shift on a well-conditioned tall operator (AᵀA = 4 I + a sparse low-rank part): its histories keep
    # their digits to the end, which those of the ill-conditioned lsq_test problems do not beyond one CTA
    A2 = sp.vstack([2.0 * sp.eye(300), sp.random(200, 300, density=0.02, random_state=3)]).tocsr()
    b2 = np.cos(np.arange(500.0))
    xo, so = S.cgls_lanczos_shift(A2, b2, shifts)
    xs, st = kb.cgls_lanczos_shift(A2, b2, shifts, history=True)
    assert st.niter == so["niter"]
    for r, ro in zip(st.residuals, so["residuals"]):
        assert len(r) == len(ro) and np.all(np.abs(np.asarray(r) - ro) <= 1e-6 * np.abs(ro))


def test_paths_and_inputs_agree(kb):
    import torch
    A = O.get_div_grad(16, 16, 16)
    n = A.shape[0]
    b = np.ones(n)
    shifts = [0.0, 0.5, 5.0, 50.0]
    xf, sf = kb.cg_lanczos_shift(A, b, shifts, history=True, fused=True)
    xp, spp = kb.cg_lanczos_shift(A, b, shifts, history=True, fused=False)
    assert sf.niter == spp.niter and sf.status == spp.status
    for r1, r0 in zip(sf.residuals, spp.residuals):
        assert np.allclose(r1, r0, rtol=1e-7, atol=1e-12 * r0[0])
    for x1, x0 in zip(xf, xp):
        assert np.linalg.norm(x1 - x0) <= 1e-8 * np.linalg.norm(x0)
    # sigma = 0 is cg_lanczos!'s iteration on the same passes: byte for byte
    xs, st = kb.cg_lanczos_shift(A, b, shifts, atol=0.0, rtol=0.0, itmax=12, history=True)
    x0, s0 = kb.cg_lanczos(A, b, atol=0.0, rtol=0.0, itmax=12, history=True)
    assert st.niter == s0.niter == 12
    assert xs[0].tobytes() == x0.tobytes() and st.residuals[0] == s0.residuals
    # a host callable operator runs the primitive Lanczos half and the same shift-update pass
    xc, sc = kb.cg_lanczos_shift(lambda v: A @ v, b, shifts, history=True)
    assert sc.niter == sf.niter
    for x1, x0 in zip(xc, xf):
        assert np.linalg.norm(x1 - x0) <= 1e-8 * np.linalg.norm(x0)
    # torch inputs: same bytes as host inputs
    xt, stt = kb.cg_lanczos_shift(A, torch.tensor(b, device="cuda"), shifts, history=True)
    assert all(torch.is_tensor(x) for x in xt) and stt.residuals == sf.residuals
    for x1, x0 in zip(xt, xf):
        assert x1.cpu().numpy().tobytes() == x0.tobytes()
    # CGLS: CSR against a (matvec, rmatvec) pair
    b2, A2 = lsq_test(400, 300, 3, 2, 0)[:2]
    x1, s1 = kb.cgls_lanczos_shift(A2, b2, shifts)
    x2, s2 = kb.cgls_lanczos_shift((lambda v: A2 @ v, lambda u: A2.T @ u), b2, shifts, n=A2.shape[1])
    assert s1.niter == s2.niter
    for u, w in zip(x1, x2):
        assert np.linalg.norm(u - w) <= 1e-8 * np.linalg.norm(w)


def _per_iteration(kb, ws, A, b, shifts, k1, k2):
    counts = []
    for k in (k1, k2):
        l0 = ws.launches
        ws.solve(A, b, shifts, atol=0.0, rtol=0.0, itmax=k)
        assert ws.stats.niter == k
        counts.append(ws.launches - l0)
    return (counts[1] - counts[0]) / (k2 - k1)


def test_launches_per_iteration(kb):
    A = O.get_div_grad(16, 16, 16)
    n = A.shape[0]
    b = np.ones(n)
    ws = kb.CgLanczosShiftWorkspace(n, n, PASS)
    assert _per_iteration(kb, ws, A, b, list(np.logspace(-1, 2, PASS)), 5, 25) <= 3
    ws.free()
    ws = kb.CgLanczosShiftWorkspace(n, n, PASS + 1)           # one more pass per iteration past kShiftPass shifts
    assert _per_iteration(kb, ws, A, b, list(np.logspace(-1, 2, PASS + 1)), 5, 25) <= 4
    ws.free()
    b2, A2 = lsq_test(400, 300, 3, 2, 0)[:2]
    ws = kb.CglsLanczosShiftWorkspace(A2.shape[0], A2.shape[1], 8)
    assert _per_iteration(kb, ws, A2, b2, list(np.logspace(-1, 2, 8)), 3, 13) <= 4
    ws.free()


def test_edge_cases(kb):
    A, b = O.symmetric_definite()
    shifts = [1.0, 2.0, 3.0]
    for f in (kb.cg_lanczos_shift, kb.cgls_lanczos_shift):
        xs, st = f(A, np.zeros(A.shape[0]), shifts)
        assert st.status == "x is a zero-residual solution" and st.niter == 0 and all(np.all(x == 0) for x in xs)
        seen = []
        _, st = f(A, b, shifts, atol=0.0, rtol=0.0, callback=lambda ws: seen.append(ws.stats.niter) or len(seen) >= 2)
        assert st.status == "user-requested exit" and st.niter == 2
        with pytest.raises(TypeError):
            f(A, b, shifts, callback=lambda ws: "string")
        with pytest.raises(kb.B200Error, match="unsupported keyword"):
            f(A, b, shifts, radius=1.0)
    assert np.isnan(st.Anorm) and np.isnan(st.Acond)


def test_refusals(kb):
    L = _lib.lib()
    h = C.c_void_p()
    assert L.krylov_b200_shift_workspace_create(101, 5, 5, 2, 3, 0, C.byref(h)) == -2          # complex
    assert L.krylov_b200_shift_workspace_create(7, 5, 5, 2, 1, 0, C.byref(h)) == -2            # not a shift solver
    assert L.krylov_b200_shift_workspace_create(101, 5, 5, 0, 1, 0, C.byref(h)) == -1          # nshifts <= 0
    assert L.krylov_b200_shift_workspace_create(101, 5, 6, 2, 1, 0, C.byref(h)) == -1          # CG: rectangular
    assert "square" in _lib.last_error()
    ws = kb.CgLanczosShiftWorkspace(10, 10, 2)
    x = np.zeros(10)
    null = _lib.MATVEC()
    assert L.krylov_solve(ws._h, null, null, null, null, x.ctypes.data_as(C.c_void_p), None, None, None) == -1
    assert "krylov_b200_shift_solve" in _lib.last_error()
    assert L.krylov_get_x(ws._h, x.ctypes.data_as(C.c_void_p), 10) == -1
    assert L.krylov_warm_start(ws._h, x.ctypes.data_as(C.c_void_p), 10) == -1
    assert L.krylov_b200_dist_init(ws._h, 0, 2, 0, None, None) == -1
    assert L.krylov_b200_shift_get_x(ws._h, 2, x.ctypes.data_as(C.c_void_p), 10) == -1      # shift out of range
    d = np.ones(10)
    assert L.krylov_b200_set_preconditioner_diag(ws._h, 1, d.ctypes.data_as(C.c_void_p), 0) == -1   # no N
    assert "no right preconditioner N" in _lib.last_error()
    assert L.krylov_b200_set_preconditioner_blockdiag(ws._h, 1, 2, np.ones(20).ctypes.data_as(C.c_void_p), 0) == -1
    ws.free()
    b2, A2 = lsq_test(40, 40, 4, 1, 0)[:2]
    with pytest.raises(kb.B200Error, match="Preconditioner `M` is not supported."):
        kb.cgls_lanczos_shift(A2, b2, [1.0], M=np.ones(A2.shape[0]))
    ws = kb.CglsLanczosShiftWorkspace(A2.shape[0], A2.shape[1], 1)        # an M reaching the library is refused there
    ws.set_operator(A2)
    Mf = _lib.MATVEC(lambda xp, yp, u: None)
    bb = np.ascontiguousarray(b2)
    sh = (C.c_double * 1)(1.0)
    assert L.krylov_b200_shift_solve(ws._h, null, null, Mf, bb.ctypes.data_as(C.c_void_p), sh, None, None) == -1
    assert "Preconditioner `M` is not supported." in _lib.last_error()
    ws.free()
