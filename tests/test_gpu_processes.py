"""GPU: the Krylov processes (kb.hermitian_lanczos, arnoldi, golub_kahan, nonhermitian_lanczos, saunders_simon_yip)
against the CPU oracle and the reference's identities, their breakdowns, launch totals on staged and untiled operators,
bit-identity across TMA ring depths, the single device-to-host copy per call and the refusals."""
import ctypes as C
import functools

import numpy as np
import pytest
import scipy.sparse as sp

from oracle import oracle as Osh
from oracle import processes_oracle as P
from parity import TOL, perturbed_runs
from process_cases import K, check_identities, path3, problems

pytestmark = pytest.mark.gpu

NAMES = ("hermitian_lanczos", "arnoldi", "golub_kahan", "nonhermitian_lanczos", "saunders_simon_yip")
TWO_SIDED = ("nonhermitian_lanczos", "saunders_simon_yip")


def call(mod, name, A, b, c, k, **kw):
    f = getattr(mod, name)
    return f(A, b, c, k, **kw) if c is not None else f(A, b, k, **kw)


def coefs(name, out):
    """β (and γ) and the coefficients of one output tuple of the Python API, flattened in the oracle's order (sparse ->
    nzval; dense H column-major)."""
    if name == "arnoldi":
        return np.concatenate([[float(out[1])], np.ravel(np.asarray(out[2], np.float64), order="F")])
    return np.concatenate([np.asarray(x.data, np.float64) if sp.issparse(x) else [float(x)]
                           for x in out if sp.issparse(x) or np.ndim(x) == 0])


def oracle_coefs(name, out):
    if name == "arnoldi":
        return np.concatenate([[out[1]], np.ravel(out[2], order="F")])
    return np.concatenate([np.atleast_1d(np.asarray(x, np.float64)) for x in out if np.ndim(x) <= 1])


def bases(out):
    return [np.asarray(x.cpu() if hasattr(x, "cpu") else x, np.float64) for x in out if np.ndim(x) == 2 and not sp.issparse(x)
            and x.shape[1] == out[0].shape[1]]


def sensitivity(name, A, b, c, k, dtype, **kw):
    """The oracle's coefficients and bases and their largest relative change under few-ulp perturbations of b."""
    o0 = call(P, name, A, b, c, k, dtype=dtype, **kw)
    c0, v0 = oracle_coefs(name, o0), bases(o0)
    fn = (lambda A_, b_: (call(P, name, A_, b_, c, k, dtype=dtype, **kw), None))
    runs = [r for r, _ in perturbed_runs(fn, A, b)]
    sc = np.zeros(len(c0))
    sv = np.zeros(len(v0))
    for r in runs:
        c1 = oracle_coefs(name, r)
        sc = np.maximum(sc, np.maximum.accumulate(np.abs(c1 - c0) / np.maximum(np.abs(c0), 1e-300)))
        for j, (a, bb) in enumerate(zip(bases(r), v0)):
            sv[j] = max(sv[j], np.linalg.norm(a - bb) / max(np.linalg.norm(bb), 1e-300))
    return c0, v0, sc, sv


def assert_parity(name, got, A, b, c, k, dtype=np.float64, tol=TOL, **kw):
    c0, v0, sc, sv = sensitivity(name, A, b, c, k, dtype, **kw)
    cg = coefs(name, got)
    assert cg.shape == c0.shape
    floor = 1e-12 * np.max(np.abs(c0))
    bar = np.maximum(tol, 10 * sc) * np.abs(c0) + floor
    assert np.all(np.abs(cg - c0) <= bar), f"{name}: max rel {np.max(np.abs(cg - c0) / np.maximum(np.abs(c0), 1e-300)):.3e}"
    for j, (g, w) in enumerate(zip(bases(got), v0)):
        assert np.linalg.norm(g - w) <= max(tol, 10 * sv[j]) * max(np.linalg.norm(w), 1e-300), (name, j)


@pytest.mark.parametrize("name", NAMES)
def test_identities_on_the_reference_problems(kb, name):
    """rand(n, n) / rand(m, n) as test/test_processes.jl draws them: their dominant singular value separates so fast
    that the unreorthogonalized processes lose orthogonality within k = 20 steps, and from there the order of the dot
    products alone moves the late coefficients, so these problems check the identities, not the digits."""
    A, b, c = problems()[name]
    check_identities(name, A, b, c, call(kb, name, A, b, c, K))


def parity_problem(name):
    """Sparse, well-separated problems for the digit-by-digit comparison at k = 12."""
    r = np.random.default_rng(4)
    if name in ("golub_kahan", "saunders_simon_yip"):
        A = sp.random(900, 1300, density=0.01, random_state=4, format="csr") + sp.eye(900, 1300, format="csr")
        return sp.csr_matrix(A), r.random(900), r.random(1300) if name == "saunders_simon_yip" else None
    rp, ci, va = kb_problems().div_grad_csr(10) if name == "hermitian_lanczos" else kb_problems().kron_unsymmetric_csr(10)
    A = sp.csr_matrix((va, ci, rp))
    return A, r.random(A.shape[0]), r.random(A.shape[0]) if name == "nonhermitian_lanczos" else None


def kb_problems():
    from krylov_b200 import problems as KP
    return KP


@pytest.mark.parametrize("name", NAMES)
def test_parity_with_the_oracle_float64(kb, name):
    A, b, c = parity_problem(name)
    assert_parity(name, call(kb, name, A, b, c, 12), A, b, c, 12)


@pytest.mark.parametrize("name", ["hermitian_lanczos", "arnoldi"])
def test_parity_reorthogonalization(kb, name):
    A, b, c = problems()[name]
    out = call(kb, name, A, b, c, K, reorthogonalization=True)
    check_identities(name, A, b, c, out)
    assert_parity(name, out, A, b, c, K, reorthogonalization=True)


@pytest.mark.parametrize("name", NAMES)
def test_float32_within_dot_rounding_envelope(kb, name):
    """Float32 against the Float32 oracle: the bar is the gap between the oracle's sequential Float32 dots and the same
    dots accumulated in Float64 (the measured effect of dot rounding alone), times 10, with TOL as the floor."""
    A, b, c = problems(seed=3, m=120, n=200)[name]
    A32 = A.astype(np.float32)
    b32, c32 = b.astype(np.float32), None if c is None else c.astype(np.float32)
    k = 8
    out = call(kb, name, A32, b32, c32, k)
    o0 = call(P, name, A32, b32, c32, k, dtype=np.float32)
    with Osh.dot_mode(1):
        o1 = call(P, name, A32, b32, c32, k, dtype=np.float32)
    c0, c1 = oracle_coefs(name, o0), oracle_coefs(name, o1)
    env = np.maximum.accumulate(np.abs(c1 - c0) / np.maximum(np.abs(c0), 1e-30))
    cg = coefs(name, out)
    assert np.all(np.abs(cg - c0) <= np.maximum(1e-5, 10 * env) * np.abs(c0) + 1e-6 * np.max(np.abs(c0))), name
    for g, w in zip(bases(out), bases(o0)):
        assert np.linalg.norm(g - w) <= max(1e-3, 10 * env[-1]) * np.linalg.norm(w)


@pytest.mark.parametrize("shape", [(120, 200), (200, 120)])
@pytest.mark.parametrize("name", ["golub_kahan", "saunders_simon_yip"])
def test_rectangular_both_ways_and_given_At(kb, name, shape):
    m, n = shape
    A, b, c = problems(seed=5, m=m, n=n)[name]
    k = 10
    out = call(kb, name, A, b, c, k)
    check_identities(name, A, b, c, out, k=k)
    assert_parity(name, out, A, b, c, k)
    At = kb.CsrOperator.from_scipy(A.T)
    out2 = call(kb, name, A, b, c, k, At=At)
    At.free()
    for x, y in zip(out, out2):
        assert np.array_equal(kb_dense(x), kb_dense(y))


def kb_dense(x):
    return x.toarray() if sp.issparse(x) else np.asarray(x)


@pytest.mark.parametrize("name", NAMES)
def test_torch_inputs_stay_on_device(kb, name):
    import torch
    A, b, c = problems(seed=9, m=100, n=150)[name]
    k = 6
    ref = call(kb, name, A, b, c, k)
    tb = torch.tensor(b, device="cuda")
    tc = None if c is None else torch.tensor(c, device="cuda")
    out = call(kb, name, A, tb, tc, k)
    for x, y in zip(out, ref):
        if isinstance(x, torch.Tensor):
            assert x.is_cuda and x.shape == y.shape and x.stride() == (1, y.shape[0])
            assert np.array_equal(x.cpu().numpy(), y)
        else:
            assert np.array_equal(kb_dense(x), kb_dense(y))
    assert ref[0].flags.f_contiguous


BREAKDOWN = {"hermitian_lanczos": ("Exact breakdown β₁ == 0.", "Exact breakdown βᵢ₊₁ == 0 at iteration i = 3."),
             "arnoldi": ("Exact breakdown β == 0.", "Exact breakdown Hᵢ₊₁.ᵢ == 0 at iteration i = 3."),
             "golub_kahan": ("Exact breakdown β₁ == 0.", "Exact breakdown αᵢ₊₁ == 0 at iteration i = 1."),
             "nonhermitian_lanczos": ("Exact breakdown β₁γ₁ == 0.", "Exact breakdown βᵢ₊₁γᵢ₊₁ == 0 at iteration i = 3."),
             "saunders_simon_yip": ("Exact breakdown β₁ == 0.", "Exact breakdown βᵢ₊₁ == 0 at iteration i = 3.")}


@pytest.mark.parametrize("zero", [True, False])
@pytest.mark.parametrize("name", NAMES)
def test_breakdown_text_iteration_and_zero_columns(kb, name, zero):
    A, e1 = path3()
    b = np.zeros_like(e1) if zero else e1
    c = e1 if name in TWO_SIDED else None
    with pytest.raises(kb.B200Error) as e:
        call(kb, name, A, b, c, 5)
    assert str(e.value) == BREAKDOWN[name][0 if zero else 1]
    out = call(kb, name, A, b, c, 5, allow_breakdown=True)
    ref = call(P, name, A, b, c, 5, allow_breakdown=True)
    for x in out:
        assert np.all(np.isfinite(kb_dense(x)))
    for g, w in zip(bases(out), bases(ref)):
        assert np.array_equal(g, w)                    # exact arithmetic: the same zero columns as kfill!
    assert np.array_equal(coefs(name, out), oracle_coefs(name, ref))


def launches_per_call(kb, name, A_op, At_op, b, c, k, **kw):
    L = kb._lib.lib()
    before = L.kb200_ctx_launch_count(A_op._ctx)
    if name in ("golub_kahan",) + TWO_SIDED:
        kw["At"] = At_op
    call(kb, name, A_op, b, c, k, **kw)
    return L.kb200_ctx_launch_count(A_op._ctx) - before


def expected_launches(name, k, reorth=False):
    if name == "hermitian_lanczos":
        return 4 * k + 1 if reorth else 2 * k + 2       # β₁, 2 per step (reorth: 3 at step 1, 4 after), final v
    if name == "arnoldi":
        per = sum(2 * j + 1 if reorth else j + 1 for j in range(1, k + 1))
        return 2 + per
    if name == "golub_kahan":
        return 3 + 2 * k                                 # β₁, α₁, 2 per step, final u and v
    if name == "nonhermitian_lanczos":
        return 2 + 2 * k                                 # cᵀb, 2 per step, final v and u
    return 3 + 3 * k                                     # β₁, γ₁, 3 per step, final v and u


@functools.cache
def twin_problem(name, untiled):
    """A staged operator, or its untiled twin: the same matrix with one dense row (too long for any tile ring), with
    b and c.  Lanczos gets the symmetric part, so that the untiled twin is a symmetric operator too."""
    sq = name not in ("golub_kahan", "saunders_simon_yip")
    m, n = (20000, 20000) if sq else (16000, 20000)
    g = np.random.default_rng(11)
    nz = m * n // 2000                                   # density 0.0005 (duplicates summed)
    R = sp.coo_matrix((g.random(nz), (g.integers(0, m, nz), g.integers(0, n, nz))), shape=(m, n))
    A = sp.csr_matrix(R + sp.eye(m, n, format="csr"))
    A.sort_indices()
    if untiled:
        A = sp.csr_matrix(sp.vstack([sp.csr_matrix(np.linspace(1, 2, n)[None, :] / n), A[1:]]))   # scaled like the other rows
    if name == "hermitian_lanczos":
        A = sp.csr_matrix(A + A.T)
    r = np.random.default_rng(2)
    b = r.random(m)
    c = r.random(n) if name in TWO_SIDED else None
    return A, b, c


def operator_pair(kb, name, untiled):
    A, b, c = twin_problem(name, untiled)
    A_op = kb.CsrOperator.from_scipy(A)
    At_op = kb.CsrOperator.from_scipy(A.T)
    return A_op, At_op, b, c


def plan(kb, op):
    out = (C.c_longlong * 7)()
    kb._lib.lib().kb200_csr_plan(op._csr, out)
    return bool(out[3])


@pytest.mark.parametrize("untiled", [False, True])
@pytest.mark.parametrize("name", NAMES)
def test_launch_totals_on_staged_and_untiled_operators(kb, name, untiled):
    A_op, At_op, b, c = operator_pair(kb, name, untiled)
    assert plan(kb, A_op) != untiled
    for k in (1, 7):
        for reorth in ((False, True) if name in ("hermitian_lanczos", "arnoldi") else (False,)):
            kw = {"reorthogonalization": True} if reorth else {}
            assert launches_per_call(kb, name, A_op, At_op, b, c, k, **kw) == expected_launches(name, k, reorth), (name, k, reorth)
    A_op.free()
    At_op.free()


@pytest.mark.parametrize("reorth", [False, True])
@pytest.mark.parametrize("name", NAMES)
def test_untiled_operators_match_the_oracle(kb, name, reorth):
    """The untiled passes (spmv_epi_rows on the divided gather) against the oracle, with the parity bar of the staged
    ones; Aᵀ is given, and for the one-sided processes also formed by the call."""
    if reorth and name not in ("hermitian_lanczos", "arnoldi"):
        pytest.skip("reorthogonalization is a keyword of hermitian_lanczos and arnoldi only")
    A, b, c = twin_problem(name, True)
    A_op, At_op, _, _ = operator_pair(kb, name, True)
    assert not plan(kb, A_op)
    kw = {"reorthogonalization": True} if reorth else {}
    if name in ("golub_kahan",) + TWO_SIDED:
        kw["At"] = At_op
    out = call(kb, name, A_op, b, c, 6, **kw)
    assert_parity(name, out, A, b, c, 6, **{k: v for k, v in kw.items() if k != "At"})
    A_op.free()
    At_op.free()


@pytest.mark.parametrize("name", NAMES)
def test_one_device_to_host_copy_per_call(kb, name):
    import torch
    from torch.profiler import ProfilerActivity, profile
    A_op, At_op, b, c = operator_pair(kb, name, False)
    tb = torch.tensor(b, device="cuda")
    tc = None if c is None else torch.tensor(c, device="cuda")
    kw = {"At": At_op} if name in ("golub_kahan",) + TWO_SIDED else {}
    call(kb, name, A_op, tb, tc, 5, **kw)                # warm-up
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        call(kb, name, A_op, tb, tc, 5, **kw)
        torch.cuda.synchronize()
    d2h = [e for e in prof.events() if "memcpy" in e.name.lower() and "dtoh" in e.name.lower().replace(" ", "")]
    assert len(d2h) == 1, [e.name for e in d2h]
    A_op.free()
    At_op.free()


def test_ring_depth_is_bit_identical(kb, monkeypatch):
    """Every process on a staged operator with 1, 2 and 3 ring stages at 3 CTAs per SM gives the same bytes."""
    rp, ci, va = kb.problems.div_grad_csr(48)
    A = sp.csr_matrix((va, ci, rp))
    rpk, cik, vak = kb.problems.kron_unsymmetric_csr(48)
    B = sp.csr_matrix((vak, cik, rpk))
    G = sp.csr_matrix(B[:, : B.shape[1] - 1000])
    cases = {"hermitian_lanczos": (A, None), "arnoldi": (B, None), "nonhermitian_lanczos": (B, np.sin(np.arange(B.shape[0]))),
             "golub_kahan": (G, None), "saunders_simon_yip": (G, np.sin(np.arange(G.shape[1])))}
    monkeypatch.setenv("KB200_CSR_DICT", "0")
    monkeypatch.setenv("KB200_CTAS_PER_SM", "3")
    results = {}
    for stages in (1, 2, 3):
        monkeypatch.setenv("KB200_STAGES", str(stages))
        for name, (M, c) in cases.items():
            b = np.cos(np.arange(M.shape[0]))
            A_op = kb.CsrOperator.from_scipy(M)
            At_op = kb.CsrOperator.from_scipy(M.T)
            assert plan(kb, A_op) and plan(kb, At_op)
            kw = {"At": At_op} if name in ("golub_kahan",) + TWO_SIDED else {}
            out = call(kb, name, A_op, b, c, 12, **kw)
            results.setdefault(name, []).append(b"".join(kb_dense(x).tobytes() if not np.isscalar(x) else np.float64(x).tobytes()
                                                         for x in out))
            A_op.free()
            At_op.free()
    for name, r in results.items():
        assert r[0] == r[1] == r[2], name


def test_refusals(kb):
    A, b, c = problems(seed=1, m=30, n=40)["golub_kahan"]
    S = sp.csr_matrix(np.eye(30))
    with pytest.raises(kb.B200Error, match="element type"):
        kb.hermitian_lanczos(S, np.ones(30, np.complex128), 3)
    with pytest.raises(kb.B200Error, match="CSR operator"):
        kb.hermitian_lanczos(lambda x: x, np.ones(30), 3)
    with pytest.raises(kb.B200Error, match="30 entries"):
        kb.arnoldi(S, np.ones(29), 3)
    with pytest.raises(kb.B200Error, match="k must be at least 1"):
        kb.arnoldi(S, np.ones(30), 0)
    with pytest.raises(kb.B200Error, match="must be square"):
        kb.hermitian_lanczos(A, np.ones(40), 3)
    with pytest.raises(kb.B200Error, match="At must be"):
        kb.golub_kahan(A, b, 3, At=sp.csr_matrix(np.ones((30, 40))))
    with pytest.raises(kb.B200Error, match="40 entries"):
        kb.saunders_simon_yip(A, b, np.ones(39), 3)
    # the C ABI: a complex dtype is -2, a dtype other than the CSR object's -1
    L = kb._lib.lib()
    op = kb.CsrOperator.from_scipy(S)
    beta, T = C.c_double(), (C.c_double * 8)()
    assert L.kb200_hermitian_lanczos(op._ctx, op._csr, 3, 3, None, None, C.byref(beta), T, 0) == -2
    assert L.kb200_hermitian_lanczos(op._ctx, op._csr, 3, 0, None, None, C.byref(beta), T, 0) == -1
    assert "dtype differs" in kb._lib.last_error()
    op.free()
