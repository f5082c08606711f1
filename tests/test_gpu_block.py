"""GPU parity of block_gmres! (SURVEY.md 8f-2) through the C ABI against the CPU oracle (oracle/krylov_oracle_block.h):
identical iteration count, residual (Frobenius) history within 1e-6 relative, same X.  The device panel QR (CholQR2 +
Householder sign reconstruction) must reproduce LAPACK's factors, so the comparison is not only up to column signs."""
import os
import re
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rhs(n, p, seed=0):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, p))


def _check(st, X, so, Xo, tol=1e-6):
    assert st.status == so["status"], (st.status, so["status"])
    assert st.niter == so["niter"], (st.niter, so["niter"])
    r, ro = np.asarray(st.residuals), np.asarray(so["residuals"])
    assert len(r) == len(ro)
    assert np.all(np.abs(r - ro) <= tol * np.abs(ro) + 1e-9 * ro[0]), np.max(np.abs(r - ro) / ro)
    assert np.linalg.norm(X - Xo) <= 1e-6 * np.linalg.norm(Xo)


def _with_n729(cases):
    """kron_unsymmetric(8) (n = 512) under the case's own id, kron_unsymmetric(9) (n = 729) under id + "-729"."""
    out = []
    for N in (8, 9):
        for c in cases:
            vals = c if isinstance(c, tuple) else (c,)
            ident = "-".join(str(v) for v in vals) + ("-729" if N == 9 else "")
            out.append(pytest.param(*vals, N, id=ident))
    return out


@pytest.mark.parametrize("p,generic,N", _with_n729([(p, g) for g in (False, True, "prefetch", "simt", "mma8")
                                                     for p in (1, 2, 3, 4, 5, 8, 16, 32)]))
def test_block_gmres_block_sizes(kb, O, p, generic, N, monkeypatch):
    """Float64 p = 8, 16, 32 run the tensor-core panel kernels (mma.sync m8n8k4.f64; "simt" = KB200_BLOCK_MMA=0 keeps
    every p on the register-resident SIMT kernels, "mma8" = KB200_BLOCK_MMA=16 only p = 8); p = 2, 4 the SIMT ones (with
    or without software-pipelined row loads); every other p (and KB200_BLOCK_GENERIC=1) the tiled any-p kernels.
    All against the oracle, at n = 512 (a multiple of every tile and pass width) and n = 729 (ragged last tiles)."""
    if generic in ("simt", "mma8") and p not in (8, 16, 32):
        pytest.skip("variant only changes p = 8 / 16 / 32")
    env = {True: dict(KB200_BLOCK_GENERIC="1"), "prefetch": dict(KB200_FAST_PREFETCH="1"), "simt": dict(KB200_BLOCK_MMA="0"),
           "mma8": dict(KB200_BLOCK_MMA="16")}.get(generic, {})
    for k, v in env.items():                    # read when the workspace is created
        monkeypatch.setenv(k, v)
    A, _ = O.kron_unsymmetric(N)
    A = sp.csr_matrix(A)
    B = A @ _rhs(A.shape[0], p)
    X, st = kb.block_gmres(A, B, memory=6, history=True)
    Xo, so = O.block_gmres(A, B, memory=6)
    _check(st, X, so, Xo)


@pytest.mark.parametrize("kw", [dict(), dict(restart=True), dict(M=True), dict(N=True), dict(M=True, N=True, restart=True),
                                dict(reorthogonalization=True), dict(x0=True), dict(x0=True, restart=True),
                                dict(atol=1e-12, rtol=1e-12)])
def test_block_gmres_options_match_oracle(kb, O, kw):
    A, _ = O.kron_unsymmetric(9)
    A = sp.csr_matrix(A + sp.diags(np.linspace(0.0, 3.0, A.shape[0])))
    n, p = A.shape[0], 4
    B = _rhs(n, p, 1)
    d = 1.0 / A.diagonal()
    args = {k: v for k, v in kw.items() if k in ("restart", "reorthogonalization", "atol", "rtol")}
    if kw.get("M"):
        args["M"] = d
    if kw.get("N"):
        args["N"] = 1.0 / np.sqrt(A.diagonal()) if kw.get("M") else d
    X0 = 0.25 * np.ones((n, p)) if kw.get("x0") else None
    X, st = kb.block_gmres(A, B, X0, memory=5, history=True, **args)
    Xo, so = O.block_gmres(A, B, X0=X0, memory=5, **args)
    _check(st, X, so, Xo)


def test_block_gmres_float32_callbacks_and_torch(kb, O):
    import torch
    A, _ = O.kron_unsymmetric(8)
    A = sp.csr_matrix(A)
    n, p = A.shape[0], 4
    B = A @ _rhs(n, p, 2)
    X, st = kb.block_gmres(A, B.astype(np.float32), memory=8, history=True)
    Xo, so = O.block_gmres(A, B, memory=8, dtype=np.float32)
    assert st.solved and abs(st.niter - so["niter"]) <= 1
    assert np.linalg.norm(B - A @ X.astype(np.float64)) / np.linalg.norm(B) <= 5e-3
    # host block callbacks see the reference's column-major blocks (krylov.h:105-107)
    X, st = kb.block_gmres(lambda Xb: A @ Xb, B, memory=8, history=True)
    Xo, so = O.block_gmres(A, B, memory=8)
    _check(st, X, so, Xo)
    X, st = kb.block_gmres(A, B, M=lambda Yb: Yb / A.diagonal()[:, None], memory=8, history=True)
    Xo, so = O.block_gmres(A, B, M=1.0 / A.diagonal(), memory=8)
    _check(st, X, so, Xo)
    # device-resident blocks (torch), user exit, type error of a non-Bool callback
    Bt = torch.from_numpy(B).cuda()
    Xt, st = kb.block_gmres(A, Bt, memory=8, history=True)
    _check(st, Xt.cpu().numpy(), so if False else O.block_gmres(A, B, memory=8)[1], O.block_gmres(A, B, memory=8)[0])
    cnt = []
    X, st = kb.block_gmres(A, B, atol=0.0, rtol=0.0, callback=lambda w: (cnt.append(1), len(cnt) >= 2)[1])
    assert st.status == "user-requested exit" and st.niter == 2
    with pytest.raises(TypeError):
        kb.block_gmres(A, B, callback=lambda w: "string")


@pytest.mark.parametrize("p,N", _with_n729([3, 4, 8, 16, 32]))
def test_device_householder_path_matches_oracle_on_full_rank_blocks(kb, O, p, N, monkeypatch):
    """KB200_QR_FORCE_HOUSEHOLDER=1 sends EVERY panel QR through the slow path (LAPACK's dgeqr2 + dorg2r run as column
    operations on row ranges of the device panel, at odd row offsets; the DMMA kernels for p = 8 / 16 / 32).  On
    full-rank blocks that path must give LAPACK's factors, so the whole solve matches the oracle at the usual 1e-6."""
    monkeypatch.setenv("KB200_QR_FORCE_HOUSEHOLDER", "1")
    A, _ = O.kron_unsymmetric(N)
    A = sp.csr_matrix(A)
    B = A @ _rhs(A.shape[0], p, 3)
    ws = kb.BlockGmresWorkspace(A.shape[0], A.shape[0], p, memory=6)
    ws.solve(A, B, history=True)
    X, st, nfall = ws.x, ws.stats, ws.qr_fallbacks
    ws.free()
    Xo, so = O.block_gmres(A, B, memory=6)
    assert nfall >= st.niter
    _check(st, X, so, Xo)


@pytest.mark.parametrize("N", [8, 9])
@pytest.mark.parametrize("p", [8, 16, 32])
def test_block_gmres_float32_wide_blocks(kb, O, p, N):
    """Float32 panels at p = 8, 16, 32 (SIMT kernels: the DMMA path is Float64 only), with the checks of the p = 4
    Float32 case above: solved within one iteration of the Float32 oracle, true residual small."""
    A, _ = O.kron_unsymmetric(N)
    A = sp.csr_matrix(A)
    B = A @ _rhs(A.shape[0], p, 2)
    X, st = kb.block_gmres(A, B.astype(np.float32), memory=8, history=True)
    Xo, so = O.block_gmres(A, B, memory=8, dtype=np.float32)
    assert st.solved and abs(st.niter - so["niter"]) <= 1, (st.niter, so["niter"])
    assert np.linalg.norm(B - A @ X.astype(np.float64)) / np.linalg.norm(B) <= 5e-3


@pytest.mark.parametrize("p", [3, 4])
def test_block_gmres_rank_deficient_block_falls_back(kb, O, p):
    """Two identical right-hand sides: the Gram matrix of the block is singular and the panel QR takes the Householder
    path, which completes the basis with a direction that only rounding determines (LAPACK's does too) -- so the
    iterates are not comparable with the oracle's beyond the first residual; what must hold is that the fallback is
    counted, the recurrence residual is the true one, it never increases, and it ends near the oracle's."""
    A, b = O.sparse_laplacian(6)
    cols = [b, b, np.arange(len(b), dtype=float), np.cos(np.arange(len(b)))][:p]
    B = np.stack(cols, axis=1)
    ws = kb.BlockGmresWorkspace(A.shape[0], A.shape[0], p, memory=12)
    ws.solve(A, B, itmax=12, history=True)
    X, st = ws.x, ws.stats
    assert ws.qr_fallbacks >= 1                       # counted, never silent
    ws.free()
    Xo, so = O.block_gmres(A, B, memory=12, itmax=12)
    r = np.asarray(st.residuals)
    assert np.isfinite(r).all() and np.isfinite(X).all()
    assert r[0] == pytest.approx(so["residuals"][0], rel=1e-12)
    assert np.all(np.diff(r) <= 1e-9 * r[0])          # GMRES residuals are monotone
    assert np.linalg.norm(B - A @ X) == pytest.approx(r[-1], rel=1e-6, abs=1e-9 * r[0])
    assert r[-1] <= 10 * so["residuals"][-1] + 1e-9 * r[0]
    # well-posed blocks stay on the fast path while the Krylov blocks keep full rank (close to convergence of a small
    # problem the new block legitimately loses rank -- happy breakdown -- and the slow path takes over)
    Ak, _ = O.kron_unsymmetric(8)
    Ak = sp.csr_matrix(Ak)
    ws = kb.BlockGmresWorkspace(Ak.shape[0], Ak.shape[0], p, memory=6)
    ws.solve(Ak, Ak @ _rhs(Ak.shape[0], p, 5), itmax=5, history=True)
    assert ws.stats.niter == 5 and ws.qr_fallbacks == 0
    ws.free()


def test_reference_test_block_program():
    """interfaces/test/C/test_block.c, unmodified, linked to libkrylov_b200.so.  Its block_minres section is outside
    this library's path (create answers -2); every other check must pass."""
    exe = os.path.join(ROOT, "oracle", "_ref", "test_block")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/test_block was not built (reference tree absent at build time)")
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    section, bad = None, []
    for line in out.stdout.splitlines():
        m = re.match(r"^(\S.*) \.\.\.$", line)
        if m:
            section = m.group(1)
        elif "FAIL" in line and section != "block_minres":
            bad.append((section, line))
    assert not bad, out.stdout + out.stderr
    m = re.search(r"(\d+) checks passed, (\d+) failed", out.stdout)
    assert m and int(m.group(1)) >= 15, out.stdout
