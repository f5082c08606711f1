"""The parity bar of the GPU solver tests against the CPU oracle, and the other helpers shared by the solver families'
tests: the golden-case generators, the gradient operators and their untiled twins, launch counting and the ring-depth
sweep.

A GPU history must follow the oracle's within TOL relative at every iteration, or within 10x the oracle's own change
under a few-ulp perturbation of b where that is larger: the device's tree-ordered dot products differ from the oracle's
sequential sums by a few roundings, so the oracle's sensitivity to such a change is the measured width of the bar."""
import functools
import importlib.util
import os

import numpy as np
import scipy.sparse as sp

from krylov_b200 import problems as P

TOL = 1e-6


def perturbed_runs(fn, A, b, **kw):
    """fn(A, b (1 + k eps s), **kw) for three random sign patterns s and k = 1 and 8 ulps: the oracle's runs under
    small relative perturbations of b."""
    out = []
    for seed in range(3):
        for ulps in (1, 8):
            sign = np.random.default_rng(seed).choice([-1.0, 1.0], size=len(b))
            out.append(fn(A, b * (1 + ulps * 2.2e-16 * sign), **kw))
    return out


def sens(r0, runs, key):
    """Running max of the relative change of history `key` (r0: the unperturbed one) over the perturbed runs."""
    out = np.zeros(len(r0))
    for _, s1 in runs:
        r1 = np.asarray(s1[key])
        k = min(len(r0), len(r1))
        s = np.full(len(r0), np.inf)
        s[:k] = np.abs(r0[:k] - r1[:k]) / np.maximum(np.abs(r0[:k]), 1e-300)
        out = np.maximum(out, np.maximum.accumulate(s))
    return out


def xsens(x0, runs):
    """The largest relative change of x (x0: the unperturbed one) over the perturbed runs."""
    return max(np.linalg.norm(x1 - x0) / max(np.linalg.norm(x0), 1e-300) for x1, _ in runs)


def assert_history(key, got, want, sens_of, floor):
    """Every entry of `got` within TOL relative of `want` plus the absolute `floor`; where that misses, within
    max(TOL, 10 sens_of()) relative instead (sens_of, the oracle's own sensitivity, is only evaluated then)."""
    ok = np.abs(got - want) <= TOL * np.abs(want) + floor
    if not ok.all():
        tol = np.maximum(TOL, 10 * sens_of()[:len(want)])
        ok = np.abs(got - want) <= tol * np.abs(want) + floor
    assert ok.all(), f"{key}: max rel deviation {np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-300)):.3e}"


def compare(oracle, gpu, A, b, *, keys, flags, floor, unsteady=None, check_length=True, scaled_resid=False, xtol=TOL,
            gpu_A=None, device_b=False, **kw):
    """Solve with oracle(A, b, **kw) and gpu(gpu_A or A, b, history=True, fused=..., **kw); assert the parity bar and
    return (x, stats, the oracle's stats).

    keys: the histories compared, with an absolute floor of `floor` |their first oracle entry|.
    flags: the stats that must match besides niter and status.
    unsteady: where the oracle's own iteration count moves under the perturbations of b -- None: that is not tolerated,
      the counts must match; "range": the GPU's count must lie in the range of the oracle's; "widened": in that range
      widened by its spread.  Status and flags must still match, the residual ‖b - (A + λI) x‖ must be within TOL ‖b‖
      (TOL ‖A‖₂ ‖x‖ ‖b‖ with scaled_resid), and the histories are compared up to where the oracle's own moves by 1e-3.
    check_length: the histories have the oracle's lengths where its iteration count is steady.
    xtol: the bar on ‖x - x_oracle‖ / ‖x_oracle‖ where the counts match; None: max(TOL, 10x the oracle's own change).
    device_b: b, and c if given, go to the GPU as CUDA tensors."""
    fused = kw.pop("fused", True)
    xo, so = oracle(A, b, **kw)
    runs = functools.cache(lambda: perturbed_runs(oracle, A, b, **kw))
    bg, gkw = b, kw
    if device_b:
        import torch
        bg = torch.tensor(b, device="cuda")
        gkw = {k: (torch.tensor(v, device="cuda") if k == "c" else v) for k, v in kw.items()}
    x, st = gpu(A if gpu_A is None else gpu_A, bg, history=True, fused=fused, **gkw)
    x = x.cpu().numpy() if hasattr(x, "cpu") else x
    got = (st.niter, st.status) + tuple(getattr(st, f) for f in flags)
    want = (so["niter"], so["status"]) + tuple(so[f] for f in flags)
    nits = [s["niter"] for _, s in runs()] if unsteady else []
    steady = all(k == so["niter"] for k in nits)
    if steady:
        assert got == want, (got, want)
    else:
        lo, hi = min(nits + [so["niter"]]), max(nits + [so["niter"]])
        w = hi - lo if unsteady == "widened" else 0
        assert lo - w <= st.niter <= hi + w, (st.niter, so["niter"], nits)
        assert got[1:] == want[1:], (got, want)
        r = b - A @ x - kw.get("lambda_", 0.0) * x
        bar = TOL * np.linalg.norm(A.toarray(), 2) * np.linalg.norm(x) if scaled_resid else TOL
        assert np.linalg.norm(r) <= bar * np.linalg.norm(b)
    for key in keys:
        rg, ro = np.asarray(getattr(st, key)), np.asarray(so[key])
        if steady and check_length:
            assert len(rg) == len(ro), (key, len(rg), len(ro))
        k = min(len(rg), len(ro))
        if not steady:
            s = sens(ro, runs(), key)
            k = min(k, int(np.argmax(s > 1e-3)) if np.any(s > 1e-3) else k)
        assert_history(key, rg[:k], ro[:k], lambda: sens(ro, runs(), key), floor * (abs(ro[0]) if len(ro) else 0.0))
    if st.niter == so["niter"]:
        bar = max(TOL, 10 * xsens(xo, runs())) if xtol is None else xtol
        assert np.linalg.norm(x - xo) <= bar * max(np.linalg.norm(xo), 1e-300), np.linalg.norm(x - xo) / np.linalg.norm(xo)
    return x, st, so


def rect_with_gaps(m, n, seed, density=0.08):
    """Random m x n matrix with empty rows and empty columns."""
    A = sp.random(m, n, density=density, random_state=seed, format="lil")
    A[3, :] = 0
    A[m - 1, :] = 0
    A[:, 1] = 0
    A[:, n - 2] = 0
    A = sp.csr_matrix(A)
    A.eliminate_zeros()
    return A


def shapes():
    """The rectangular (and one square) operators of the least-squares parity tests, each with a right-hand side."""
    from oracle import lsq_oracle
    rng = np.random.default_rng(5)
    b60, A60, *_ = lsq_oracle.lsq_test(60, 30, 3, 3, 0)
    Aw = sp.csr_matrix(A60.T)                                   # 30 x 60: m < n
    D = sp.csr_matrix(lsq_oracle.ddx(50))                       # 50 x 51
    G = grad(7)
    R1, R2 = rect_with_gaps(300, 120, 1), rect_with_gaps(90, 200, 2)
    Sq = sp.csr_matrix(sp.random(200, 200, density=0.05, random_state=3) + 4 * sp.identity(200))
    return {"square": (Sq, rng.standard_normal(200)), "tall_lstp": (A60, b60), "wide_lstp": (Aw, rng.standard_normal(30)),
            "ddx": (D, rng.standard_normal(50)), "grad7": (G, rng.standard_normal(G.shape[0])),
            "tall_gaps": (R1, rng.standard_normal(300)), "wide_gaps": (R2, rng.standard_normal(90))}


def golden_module(name):
    """tests/golden/gen_golden_<name>.py loaded as a module: the generator of a family's frozen oracle cases."""
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"gen_golden_{name}.py")
    spec = importlib.util.spec_from_file_location(f"gen_golden_{name}", path)
    module = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(module)
    return module


def grad(N):
    """The gradient of the N³ grid (problems.grad_csr) as a SciPy CSR matrix: one row per grid edge, N³ columns."""
    rp, ci, va = P.grad_csr(N)
    return sp.csr_matrix((va, ci, rp), shape=(len(rp) - 1, N ** 3))


def dense_line(A, row):
    """A plus a dense row (row=True) or column: long enough that its tile, or the tile of Aᵀ, is untiled."""
    A = sp.lil_matrix(A)
    line = 1.0 + np.arange(A.shape[1 if row else 0]) / A.shape[1 if row else 0]
    if row:
        A[0, :] = line
    else:
        A[:, 0] = line.reshape(-1, 1)
    return sp.csr_matrix(A)


def launches_per_iteration(kb, solver, A, b, fused=True, *, extra_iter=0, **solve_kw):
    """The kernel launches one more iteration costs: the difference between solves of 12 and 6 iterations, over 6.
    solve_kw must make the solve run to itmax, where it reports itmax + extra_iter iterations (LNLQ counts the
    terminal pass too)."""
    def launches(itmax):
        ws = kb.krylov_workspace(solver, A.shape[0], A.shape[1], np.float64)
        try:
            ws.solve(A, b, fused=fused, itmax=itmax, **solve_kw)
            assert ws.stats.niter == itmax + extra_iter, ws.stats.status
            return ws.launches
        finally:
            ws.free()
    return (launches(12) - launches(6)) / 6


def assert_ring_depth_changes_no_bit(monkeypatch, run):
    """run() solves and returns its outcome as a tuple of bytes and scalars.  At 3, 2 and 1 CTAs per SM, every ring
    depth from 1 to 4 must give the same tuple (KB200_CTAS_PER_SM / KB200_STAGES are read when an operator is planned).
    The CTA count sets the grid, and with it the order of the grid-wide sums, so the comparison is within one CTA
    count; the default plan must equal one of the forced ones."""
    monkeypatch.delenv("KB200_STAGES", raising=False)
    monkeypatch.delenv("KB200_CTAS_PER_SM", raising=False)
    default = run()
    ref, default_forced = {}, False
    for cps in (3, 2, 1):
        for stages in (1, 2, 3, 4):
            monkeypatch.setenv("KB200_CTAS_PER_SM", str(cps))
            monkeypatch.setenv("KB200_STAGES", str(stages))
            out = run()
            default_forced = default_forced or out == default
            assert out == ref.setdefault(cps, out), (cps, stages)
    assert default_forced
