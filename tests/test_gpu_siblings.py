"""GPU parity of the sibling solvers (SURVEY.md 8f-3: cgs!, cg_lanczos!, fom!, fgmres!) through the C ABI against the
CPU oracle (oracle/krylov_oracle_siblings.h).  Same bar as the four hot-path solvers: identical iteration count and
status, residual history within 1e-6 relative (Float64)."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

pytestmark = pytest.mark.gpu


def _problems(O):
    Al, bl = O.sparse_laplacian(10)
    Al = sp.csr_matrix(Al + sp.diags(np.linspace(0.0, 4.0, Al.shape[0])))      # non-constant diagonal
    Ak, bk = O.kron_unsymmetric(9)
    Ak = sp.csr_matrix(Ak + sp.diags(np.linspace(0.0, 3.0, Ak.shape[0])))
    return (Al, bl), (Ak, bk)


def _check(st, x, so, xo, tol=1e-6, xtol=1e-6):
    assert st.status == so["status"], (st.status, so["status"])
    assert st.niter == so["niter"], (st.niter, so["niter"])
    r, ro = np.asarray(st.residuals), np.asarray(so["residuals"])
    assert len(r) == len(ro)
    assert np.all(np.abs(r - ro) <= tol * np.abs(ro) + 1e-9 * ro[0]), np.max(np.abs(r - ro) / ro)
    assert np.linalg.norm(x - xo) <= xtol * np.linalg.norm(xo)


@pytest.mark.parametrize("kw", [dict(), dict(M=True), dict(N=True), dict(M=True, N=True), dict(x0=True)])
def test_cgs_matches_oracle(kb, O, kw):
    (_, _), (A, b) = _problems(O)
    d = 1.0 / A.diagonal()
    args = {}
    if kw.get("M"):
        args["M"] = d
    if kw.get("N"):
        args["N"] = 1.0 / np.sqrt(A.diagonal()) if kw.get("M") else d
    x0 = 0.5 * np.ones(len(b)) if kw.get("x0") else None
    x, st = kb.cgs(A, b, x0, history=True, **args)
    xo, so = O.cgs(A, b, x0=x0, **args)
    _check(st, x, so, xo, tol=1e-4)          # CGS squares the BiCG polynomial: the oracle itself moves 5e-8 per ulp of b


def test_cgs_breakdown_and_zero_rhs(kb, O):
    A2 = sp.csr_matrix(np.array([[1.0, 2.0], [3.0, 4.0]]))
    x, st = kb.cgs(A2, np.array([0.0, 1.0]), c=np.array([1.0, 0.0]))
    assert st.status == "Breakdown bᴴc = 0" and not st.solved and st.niter == 0
    A, b = O.zero_rhs()
    x, st = kb.cgs(A, b)
    assert np.linalg.norm(x) == 0 and st.status == "x is a zero-residual solution"


@pytest.mark.parametrize("kw", [dict(), dict(M=True), dict(x0=True), dict(itmax=7)])
def test_cg_lanczos_matches_oracle(kb, O, kw):
    (A, b), _ = _problems(O)
    args = {}
    if kw.get("M"):
        args["M"] = 1.0 / A.diagonal()
    if kw.get("itmax"):
        args["itmax"] = kw["itmax"]
    x0 = 0.5 * np.ones(len(b)) if kw.get("x0") else None
    x, st = kb.cg_lanczos(A, b, x0, history=True, **args)
    xo, so = O.cg_lanczos(A, b, x0=x0, **args)
    _check(st, x, so, xo)
    assert st.Anorm == pytest.approx(so["Anorm"], rel=1e-10)
    assert st.indefinite == so["indefinite"]


def test_cg_lanczos_negative_curvature(kb, O):
    n = 10
    A, b = O.symmetric_definite(n)
    A = sp.lil_matrix(A)
    A[n - 2, n - 2] = -4.0                     # test/test_cg_lanczos.jl: negative curvature detection
    A = sp.csr_matrix(A)
    x, st = kb.cg_lanczos(A, b, check_curvature=True, history=True)
    xo, so = O.cg_lanczos(A, b, check_curvature=True)
    assert st.status == "negative curvature" == so["status"] and st.indefinite and st.niter == so["niter"]
    assert np.allclose(x, xo, rtol=1e-10, atol=1e-14)


@pytest.mark.parametrize("name", ["fom", "fgmres", "gmres"])
@pytest.mark.parametrize("kw", [dict(), dict(restart=True), dict(M=True), dict(N=True), dict(M=True, N=True, restart=True),
                                dict(reorthogonalization=True), dict(x0=True), dict(x0=True, restart=True)])
def test_fom_fgmres_match_oracle(kb, O, name, kw):
    _, (A, b) = _problems(O)
    d = 1.0 / A.diagonal()
    args = dict(restart=kw.get("restart", False), reorthogonalization=kw.get("reorthogonalization", False))
    if kw.get("M"):
        args["M"] = d
    if kw.get("N"):
        args["N"] = 1.0 / np.sqrt(A.diagonal()) if kw.get("M") else d
    x0 = 0.5 * np.ones(len(b)) if kw.get("x0") else None
    mem = 12
    out = {}
    for fused in (True, False):
        ws = kb.krylov_workspace(name, A.shape[0], A.shape[1], np.float64, memory=mem)
        if x0 is not None:
            ws.warm_start(x0)
        ws.solve(A, b, history=True, fused=fused, **args)
        out[fused] = (ws.x, ws.stats, ws.launches)
        ws.free()
    xo, so = getattr(O, name)(A, b, x0=x0, memory=mem, **args)
    # FOM's residual estimate divides by the LU pivots of H: its history is less well conditioned than GMRES's
    tol = 1e-5 if name == "fom" else 1e-6
    for fused in (True, False):
        _check(out[fused][1], out[fused][0], so, xo, tol=tol)
    eligible = not kw.get("reorthogonalization") and not (name in ("fom", "gmres") and kw.get("N"))
    if eligible:
        assert out[True][2] < out[False][2]


@pytest.mark.parametrize("name", ["fom", "fgmres", "gmres"])
def test_fom_fgmres_memory_growth_and_special_cases(kb, O, name):
    f, fo = getattr(kb, name), getattr(O, name)
    A, b = O.kron_unsymmetric(7)
    x, st = f(A, b, memory=5, history=True)                      # non-restarted: V, (Z), R, l/c grow past `memory`
    xo, so = fo(A, b, memory=5)
    assert st.niter == so["niter"] > 5 and st.status == so["status"]
    assert np.allclose(st.residuals, so["residuals"], rtol=1e-5, atol=1e-9 * so["residuals"][0])
    assert np.linalg.norm(x - xo) <= 1e-6 * np.linalg.norm(xo)
    A, b = O.square_inconsistent()
    x, st = f(A, b)
    xo, so = fo(A, b)
    assert st.inconsistent and so["inconsistent"] and st.status == so["status"]
    A, b = O.zero_rhs()
    x, st = f(A, b)
    assert np.linalg.norm(x) == 0 and st.status == "x is a zero-residual solution"


def test_fgmres_flexible_preconditioner(kb, O):
    """test/test_fgmres.jl: a right preconditioner that changes at every application (sign flips)."""
    A, b = O.cartesian_poisson(12, 12)
    J = 1.0 / A.diagonal()
    state = {"w": 1.0}

    def N(x):
        state["w"] = -state["w"]
        return state["w"] * (J * x)
    x, st = kb.fgmres(A, b, N=N, memory=40)
    assert st.solved and np.linalg.norm(b - A @ x) / np.linalg.norm(b) <= 1e-6


def test_sibling_float32_and_callback(kb, O):
    (Al, bl), (Ak, bk) = _problems(O)
    for name, A, b in (("cgs", Ak, bk), ("fom", Ak, bk), ("fgmres", Ak, bk), ("cg_lanczos", Al, bl)):
        x, st = getattr(kb, name)(A, b.astype(np.float32), history=True)
        xo, so = getattr(O, name)(A, b, dtype=np.float32)
        assert st.solved and abs(st.niter - so["niter"]) <= 2, name
        assert np.linalg.norm(b - A @ x.astype(np.float64)) / np.linalg.norm(b) <= 5e-3, name
        cnt = []
        x, st = getattr(kb, name)(A, b, atol=0.0, rtol=0.0, callback=lambda w: (cnt.append(1), len(cnt) >= 3)[1])
        # fom.jl:237 does not test the user exit in its inner loop: the pass runs one more step on the (zero) V[4]
        # that was never formed, breaks down there, and only then leaves -- reproduced literally
        assert st.status == "user-requested exit" and st.niter == (4 if name == "fom" else 3), name
        with pytest.raises(TypeError):
            getattr(kb, name)(A, b, callback=lambda w: "string")
    # the same extra FOM step past `memory` (no restart), where V[k] was never allocated: a zero column as within it
    cnt = []
    x, st = kb.fom(Ak, bk, memory=5, atol=0.0, rtol=0.0, callback=lambda w: (cnt.append(1), len(cnt) >= 7)[1])
    assert st.status == "user-requested exit" and st.niter == 8


def test_sibling_solvers_through_the_reference_c_abi(kb, O):
    """krylov_workspace_create accepts the reference's enum values KRYLOV_CR / DIOM / DQGMRES / FOM / FGMRES / CGS
    (interfaces/include/krylov.h:50-60) and still answers -2 for what is not built."""
    from krylov_b200 import _lib
    L = _lib.lib()
    Ak, bk = O.kron_unsymmetric(6)
    Al, bl = O.sparse_laplacian(6)                # cr! needs a symmetric operator
    n = Ak.shape[0]
    assert Al.shape[0] == n
    cur = {}

    def matvec(xp, yp, _ud):
        A = cur["A"]
        xv = np.ctypeslib.as_array(C.cast(xp, C.POINTER(C.c_double)), shape=(n,))
        yv = np.ctypeslib.as_array(C.cast(yp, C.POINTER(C.c_double)), shape=(n,))
        yv[:] = A @ xv
    cb = _lib.MATVEC(matvec)
    null = _lib.MATVEC()
    for sid, name in ((7, "fom"), (9, "fgmres"), (11, "cgs"), (1, "cr"), (5, "diom"), (6, "dqgmres")):
        A, b = (sp.csr_matrix(Al), bl) if name == "cr" else (sp.csr_matrix(Ak), bk)
        cur["A"] = A
        h = C.c_void_p()
        assert L.krylov_workspace_create(sid, n, n, 1, 0, None, C.byref(h)) == 0
        o = L.krylov_default_options()
        assert L.krylov_solve(h, cb, null, null, null, b.ctypes.data_as(C.c_void_p), None, None, C.byref(o)) == 0
        x = np.empty(n)
        assert L.krylov_get_x(h, x.ctypes.data_as(C.c_void_p), n) == 0
        xo, so = getattr(O, name)(A, b, history=False)
        assert L.krylov_is_solved(h) == 1 and L.krylov_niter(h) == so["niter"]
        assert np.linalg.norm(x - xo) <= 1e-6 * np.linalg.norm(xo)
        assert L.krylov_workspace_free(h) == 0
    h = C.c_void_p()
    assert L.krylov_workspace_create(2, n, n, 1, 0, None, C.byref(h)) == -2       # KRYLOV_SYMMLQ: not built


@pytest.mark.parametrize("name", ["dqgmres", "diom"])
@pytest.mark.parametrize("kw", [dict(), dict(M=True), dict(N=True), dict(M=True, N=True), dict(reorthogonalization=True),
                                dict(x0=True), dict(memory=40)])
def test_dqgmres_diom_match_oracle(kb, O, name, kw):
    _, (A, b) = _problems(O)
    d = 1.0 / A.diagonal()
    args = dict(reorthogonalization=kw.get("reorthogonalization", False))
    if kw.get("M"):
        args["M"] = d
    if kw.get("N"):
        args["N"] = 1.0 / np.sqrt(A.diagonal()) if kw.get("M") else d
    x0 = 0.5 * np.ones(len(b)) if kw.get("x0") else None
    mem = kw.get("memory", 6)                    # truncated: memory << niter
    x, st = getattr(kb, name)(A, b, x0, memory=mem, history=True, **args)
    xo, so = getattr(O, name)(A, b, x0=x0, memory=mem, **args)
    # incomplete orthogonalization amplifies reduction-order noise more than the full methods do
    _check(st, x, so, xo, tol=1e-5, xtol=1e-6)


def test_dqgmres_status_order_and_diom_memory(kb, O):
    _, (A, b) = _problems(O)
    x, st = kb.dqgmres(A, b, memory=4, itmax=3, history=True)            # dqgmres.jl:319-320: "tired" overrides "solved"
    xo, so = O.dqgmres(A, b, memory=4, itmax=3)
    assert st.status == so["status"] == "maximum number of iterations exceeded" and st.niter == 3
    with pytest.raises(kb.B200Error):
        kb.DiomWorkspace(10, 10, np.float64, memory=1)                   # mod(., memory - 1) in the reference


@pytest.mark.parametrize("kw", [dict(), dict(M=True), dict(x0=True), dict(linesearch=True), dict(radius=10.0), dict(radius=30.0),
                                dict(radius=0.5), dict(itmax=5)])
def test_cr_matches_oracle(kb, O, kw):
    (A, b), _ = _problems(O)
    args = {k: v for k, v in kw.items() if k in ("linesearch", "radius", "itmax")}
    if kw.get("M"):
        # with M != I cr! tracks ||r||_M through rNorm^2 -= alpha rho (cr.jl:382-384), which stagnates near 1e-7 by
        # cancellation: the reference's own test runs this case with atol = 1e-5, rtol = 0 (test_cr.jl)
        args.update(M=1.0 / A.diagonal(), atol=1e-5, rtol=0.0)
    x0 = 0.5 * np.ones(len(b)) if kw.get("x0") else None
    x, st = kb.cr(A, b, x0, history=True, **args)
    xo, so = O.cr(A, b, x0=x0, **args)
    _check(st, x, so, xo)
    assert np.allclose(st.Aresiduals, so["Aresiduals"], rtol=1e-6, atol=1e-9 * so["Aresiduals"][0])
    assert st.indefinite == so["indefinite"] and st.npcCount == so["npcCount"]


def test_cr_curvature_cases(kb, O):
    """test/test_cr.jl: linesearch / trust-region exits on indefinite and zero-curvature systems."""
    A, b = O.symmetric_indefinite(shift=10)
    ws = kb.CrWorkspace(A, b)
    kb.cr_(ws, A, b, linesearch=True)
    st, npc = ws.stats, ws.npc_dir
    assert st.status == "nonpositive curvature" and st.niter == 0 and st.solved and st.indefinite
    assert npc @ (A @ npc) <= 0 and np.array_equal(ws.x, b)
    A2 = sp.csr_matrix(np.array([[1.0, 0.0], [0.0, 0.0]]))
    ws = kb.CrWorkspace(A2, np.ones(2))
    kb.cr_(ws, A2, np.ones(2), linesearch=True)
    xo, so = O.cr(A2, np.ones(2), linesearch=True)
    assert ws.stats.npcCount == so["npcCount"] == 2 and ws.stats.status == so["status"]
    A4 = sp.csr_matrix(np.array([[0.0, 1.0], [1.0, 0.0]]))
    x, st = kb.cr(A4, np.array([1.0, 0.0]))
    assert st.status == "b is a zero-curvature direction" and np.linalg.norm(x) == 0 and st.solved and st.niter == 0
    # indefinite systems inside a trust region: the negative-curvature branches of cr.jl:268-373 (npcCount 0 and 2,
    # exits after 1, 2 and 4 iterations), same branch and same point on the boundary as the oracle
    for n, shift, radius in ((12, 0, 5.0), (12, 0, 50.0), (12, 3, 5.0), (20, 2, 50.0), (30, 1, 500.0), (12, 10, 5000.0)):
        Ai, bi = O.symmetric_indefinite(n=n, shift=shift)
        ws = kb.CrWorkspace(Ai, bi)
        kb.cr_(ws, Ai, bi, radius=radius, history=True)
        x, st = ws.x, ws.stats
        xo, so = O.cr(Ai, bi, radius=radius)
        assert st.status == so["status"] and st.niter == so["niter"] and st.npcCount == so["npcCount"], (n, shift, radius)
        assert st.indefinite == so["indefinite"]
        assert np.linalg.norm(x - xo) <= 1e-8 * max(1.0, np.linalg.norm(xo)), (n, shift, radius)
        if so["npcCount"]:
            assert np.allclose(ws.npc_dir, so["npc_dir"], rtol=1e-8, atol=1e-10)
    Ai, bi = O.symmetric_indefinite(n=12)
    with pytest.raises(kb.B200Error):
        kb.cr(Ai, bi)                            # "Indefinite system and no trust region"
    with pytest.raises(kb.B200Error):
        kb.cr(A, b, linesearch=True, radius=1.0)


@pytest.mark.parametrize("solver,kw", [("cgs", {}), ("cg_lanczos", {}), ("cr", {}), ("dqgmres", dict(memory=6)), ("diom", dict(memory=6)),
                                       ("dqgmres", dict(memory=20)), ("diom", dict(memory=3))])
def test_grouped_passes_equal_the_primitive_path(kb, O, solver, kw):
    """fused=True groups the vector operations of an iteration into a few passes (fused_phases.cu: 4 launches for
    cgs!, 3 for cg_lanczos! / cr!, window + 3 for dqgmres! / diom!); every element update repeats the k* sequence it
    replaces, so against fused=False: same iteration count and status, histories equal to dot-product rounding, and
    far fewer launches."""
    (Al, bl), (Ak, bk) = _problems(O)
    A, b = (Al, bl) if solver in ("cg_lanczos", "cr") else (Ak, bk)
    kw = dict(kw)
    mem = kw.pop("memory", 0)
    out = {}
    for fused in (True, False):
        ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64, memory=mem)
        l0 = ws.launches
        ws.solve(A, b, history=True, fused=fused, **kw)
        out[fused] = (ws.x, ws.stats, ws.launches - l0)
        ws.free()
    (x1, s1, l1), (x0, s0, l0) = out[True], out[False]
    assert s1.niter == s0.niter and s1.status == s0.status
    assert np.allclose(s1.residuals, s0.residuals, rtol=1e-7 if solver != "cgs" else 1e-4, atol=1e-12 * s0.residuals[0])
    assert np.linalg.norm(x1 - x0) <= 1e-8 * np.linalg.norm(x0)
    assert l1 < 0.7 * l0, (l1, l0)
