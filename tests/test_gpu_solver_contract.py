"""GPU: the C ABI's interface facts of every single right-hand-side solver, through the raw entry points, against an
explicit table: which ids and types a workspace accepts, which solvers return y and how they warm-start, the adjoint
they need, the spaces and refusals of M and N (as callbacks and as attached diagonals), block-Jacobi, row partitioning
and whether c is required.  The per-family checks in the other test_gpu_*.py files stay with their families."""
import ctypes as C

import numpy as np
import pytest

from krylov_b200 import _lib

pytestmark = pytest.mark.gpu

SQ, LS, LN = (6, 6), (6, 4), (4, 6)        # square, overdetermined (least squares), underdetermined (least norm)
X0, XY, NO = "x0", "x0 and y0", None
ATTACH, SOLVE = "refused at attach", "refused at solve"


def refused(text):
    return ("refused", text)


CG_N = refused("right preconditioner N")      # CGLS / CRLS, CAR / MINARES
NO_M = refused("takes no preconditioner M")   # CGNE / CRMR
NO_P = refused("takes no preconditioner")     # BiLQR / TriLQR
# name: (shape, applies A^T, M, N, block-Jacobi M, c required, solutions, warm start, refuses row partitioning)
EXPECTED = {
    "cg":         (SQ, False, "n", "ignored", "ok", False, 1, X0, False),
    "cr":         (SQ, False, "n", "ignored", "ok", False, 1, X0, False),
    "minres":     (SQ, False, "n", "ignored", "ok", False, 1, X0, False),
    "cg_lanczos": (SQ, False, "n", "ignored", "ok", False, 1, X0, False),
    "gmres":      (SQ, False, "n", "n", "ok", False, 1, X0, False),
    "fom":        (SQ, False, "n", "n", "ok", False, 1, X0, False),
    "fgmres":     (SQ, False, "n", "n", "ok", False, 1, X0, False),
    "dqgmres":    (SQ, False, "n", "n", "ok", False, 1, X0, False),
    "diom":       (SQ, False, "n", "n", "ok", False, 1, X0, False),
    "cgs":        (SQ, False, "n", "n", "ok", False, 1, X0, False),
    "bicgstab":   (SQ, False, "n", "n", "ok", False, 1, X0, False),
    "bilq":       (SQ, True, "n", "n", SOLVE, False, 1, X0, True),
    "qmr":        (SQ, True, "n", "n", SOLVE, False, 1, X0, True),
    "car":        (SQ, False, "n", CG_N, "ok", False, 1, X0, True),
    # MINARES takes M at the ABI; its driver refuses it
    "minares":    (SQ, False, refused("not yet supported"), CG_N, SOLVE, False, 1, X0, True),
    "lsqr":       (LS, True, "m", "n", ATTACH, False, 1, NO, True),
    "lsmr":       (LS, True, "m", "n", ATTACH, False, 1, NO, True),
    "lslq":       (LS, True, "m", "n", ATTACH, False, 1, NO, True),
    "cgls":       (LS, True, "m", CG_N, ATTACH, False, 1, NO, True),
    "crls":       (LS, True, "m", CG_N, ATTACH, False, 1, NO, True),
    "craig":      (LN, True, "m", "n", ATTACH, False, 2, NO, True),
    "craigmr":    (LN, True, "m", "n", ATTACH, False, 2, NO, True),
    "lnlq":       (LN, True, "m", "n", ATTACH, False, 2, NO, True),
    "cgne":       (LN, True, NO_M, "m", ATTACH, False, 1, NO, True),
    "crmr":       (LN, True, NO_M, "m", ATTACH, False, 1, NO, True),
    "bilqr":      (SQ, True, NO_P, NO_P, SOLVE, True, 2, XY, True),
    "trilqr":     (LS, True, NO_P, NO_P, SOLVE, True, 2, XY, True),
}
UNSERVED = (2, 4, 14, 15, 16, 17, 23, 31, 34, -1)     # SYMMLQ, MINRES-QLP, USYMLQ, USYMQR, TriCG, TriMR, USYMLQR, GPMR


def test_table_covers_every_solver():
    assert set(EXPECTED) == set(_lib.SOLVER_IDS)


def test_unserved_ids_and_complex_types():
    L = _lib.lib()
    for sid in UNSERVED:
        for dt in (_lib.KRYLOV_FLOAT32, _lib.KRYLOV_FLOAT64):
            assert L.krylov_workspace_create(sid, 4, 4, dt, _lib.KRYLOV_CPU, None, C.byref(C.c_void_p())) == -2, sid
    for name, sid in _lib.SOLVER_IDS.items():
        m, n = EXPECTED[name][0]
        for dt in (2, 3):                                        # ComplexF32, ComplexF64
            assert L.krylov_workspace_create(sid, m, n, dt, _lib.KRYLOV_CPU, None, C.byref(C.c_void_p())) == -2, name


def operator(shape):
    if shape == SQ:
        return 4.0 * np.eye(6) - np.eye(6, k=1) - np.eye(6, k=-1)
    A = np.array([[2.0, 1, 0, 0], [1, 3, 1, 0], [0, 1, 4, 1], [0, 0, 1, 5], [1, 0, 0, 1], [0, 1, 1, 0]])
    return A if shape == LS else A.T.copy()


def ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_solver_contract(name, dtype):
    L = _lib.lib()
    shape, adjoint, M, N, bdiag, c_required, nsol, warm, no_dist = EXPECTED[name]
    m, n = shape
    A = operator(shape)
    nz = np.nonzero(A)
    rowptr = np.concatenate([[0], np.cumsum(np.count_nonzero(A, axis=1))]).astype(np.int32)
    colind = nz[1].astype(np.int32)
    vals = A[nz].astype(dtype)
    b = (A @ np.ones(n)).astype(dtype)
    c = (A.T @ np.ones(m)).astype(dtype) if c_required else None
    pad = max(m, n) + 4
    f64 = dtype == np.float64
    tol = 1e-6 if f64 else 1e-2
    dt = _lib.KRYLOV_FLOAT64 if f64 else _lib.KRYLOV_FLOAT32
    null = _lib.MATVEC()
    noop = _lib.MATVEC(lambda x, y, u: None)
    opts = L.krylov_default_options()
    if f64:
        opts.atol = opts.rtol = 1e-12

    ws = C.c_void_p()
    assert L.krylov_workspace_create(_lib.SOLVER_IDS[name], m, n, dt, _lib.KRYLOV_CPU, None, C.byref(ws)) == 0
    try:
        assert L.krylov_b200_set_operator_csr(ws, m, len(colind), ptr(rowptr), ptr(colind), ptr(vals), 0, 4, 0) == 0

        def solve(fM=null, fN=null, cc=c):
            return L.krylov_solve(ws, null, null, fM, fN, ptr(b), ptr(cc), None, C.byref(opts))

        def get_x():
            x = np.empty(n, dtype)
            assert L.krylov_get_x(ws, ptr(x), n) == 0
            return x

        def refusal(rc, text):
            err = _lib.last_error()
            assert rc == -1 and text.lower() in err.lower(), err

        assert solve() == 0, _lib.last_error()
        x_plain = get_x()
        assert np.all(np.isfinite(x_plain))

        def same_x():
            x = get_x()
            assert np.linalg.norm(x - x_plain) <= tol * np.linalg.norm(x_plain), (x, x_plain)

        if c_required:
            refusal(solve(cc=None), "c must be given")
        y = np.empty(m, dtype)
        assert L.krylov_get_y(ws, ptr(y), m) == (0 if nsol == 2 else -2)
        if adjoint:
            rc = L.krylov_solve(ws, noop, null, null, null, ptr(b), ptr(c), None, C.byref(opts))
            err = _lib.last_error()
            assert rc == -1 and name in err and "matvec_At" in err, err

        for which, slot in ((0, M), (1, N)):
            cb = dict(fM=noop) if which == 0 else dict(fN=noop)
            if isinstance(slot, tuple):
                refusal(solve(**cb), slot[1])
                assert L.krylov_b200_set_preconditioner_diag(ws, which, ptr(np.ones(pad, dtype)), 0) == 0
                refusal(solve(), slot[1])
            elif slot == "ignored":
                assert solve(**cb) == 0, _lib.last_error()
                assert L.krylov_b200_set_preconditioner_diag(ws, which, ptr(np.full(pad, np.nan, dtype)), 0) == 0
                assert solve() == 0, _lib.last_error()
                same_x()
            else:
                # the slot's length: an identity diagonal of that many entries, NaN past them, changes nothing
                ln = m if slot == "m" else n
                d = np.concatenate([np.ones(ln), np.full(pad - ln, np.nan)]).astype(dtype)
                assert L.krylov_b200_set_preconditioner_diag(ws, which, ptr(d), 0) == 0
                assert solve() == 0, _lib.last_error()
                same_x()
            assert L.krylov_b200_set_preconditioner_diag(ws, which, None, 0) == 0

        blocks = np.tile(np.eye(2, dtype=dtype), (pad // 2, 1, 1))
        rc = L.krylov_b200_set_preconditioner_blockdiag(ws, 0, 2, ptr(blocks), 0)
        if bdiag == ATTACH:
            refusal(rc, "not available on")
        else:
            assert rc == 0, _lib.last_error()
            if bdiag == SOLVE:
                refusal(solve(), "preconditioner")
            else:
                assert solve() == 0, _lib.last_error()
                same_x()
        assert L.krylov_b200_set_preconditioner_blockdiag(ws, 0, 2, None, 0) == 0

        if no_dist:                                              # refused before anything is set up
            refusal(L.krylov_b200_dist_init(ws, 0, 2, 0, None, None), "row-partitioned")

        x0, y0 = np.zeros(n, dtype), np.zeros(m, dtype)
        rc = L.krylov_warm_start(ws, ptr(x0), n)
        if warm == X0:
            assert rc == 0, _lib.last_error()
        else:
            refusal(rc, "krylov_warm_start2" if warm == XY else "support warm-start")
        assert L.krylov_warm_start2(ws, ptr(x0), ptr(y0), n, m) == (0 if warm == XY else -2)
    finally:
        assert L.krylov_workspace_free(ws) == 0
