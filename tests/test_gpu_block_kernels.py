"""GPU: the block_gmres! kernels one at a time (krylov_b200_block_panel_op, kb200_spmm_csr) against plain references.

Panel products.  Operands are small integers (|v| <= 4), S has distinct entries and is not symmetric, alpha and beta
are in {0, 1, -1, 0.5, -2}.  Every product and partial sum is then a multiple of 1/4 far below 2^53, so in Float64
the kernels must return the exact result whatever their summation order, FMA contraction or DMMA order; dropped or
duplicated rows, swapped fragments, a transposed S or G or a lost partial are exact mismatches.  The reference is
the same integer arithmetic (float64 BLAS is exact on it).  Float32 is held to the same exactness while the sum of
|products| stays below 2^22; past that it gets the rounding bound of its launch shape (see `_chain`).

Every panel carries NaN guard rows: 3 before its range (an odd row offset, as the Householder fallback's row ranges
have) and 5 after.  A kernel that reads outside its range turns G or Out into NaN; one that writes outside changes
the guard bits.  `rows` runs over {1, 7, 8, 9, p, 255, 257, B - 1, B + 1, 3B + 5}, where B is the number of rows one
full pass of the path's grid covers, computed from the SM count the way the launchers do."""
import ctypes as C
import math

import numpy as np
import pytest
import scipy.sparse as sp

from krylov_b200 import _lib
from krylov_b200 import problems as P

pytestmark = pytest.mark.gpu

KBLOCK = 256                # threads of the SIMT / tiled panel kernels
PANEL_TILE = 2048           # staged elements per tile of the tiled kernels
MMA_WARPS = 8               # warps per CTA of the DMMA kernels, one 8-row tile per warp
TPR = {2: 1, 4: 1, 8: 2, 16: 8, 32: 16}     # lanes per row of the SIMT kernels
TPR_ALT = {8: 4, 16: 4}                     # path 4
ALPHAS = (1.0, -1.0, 0.5, -2.0, 0.0)
BETAS = (0.0, 1.0, -1.0, 0.5, -2.0)
GUARD_LO, GUARD_HI = 3, 5
DMMA, SIMT, PREFETCH, ALT, TILED = 1, 2, 3, 4, 5


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tdt(torch, dt):
    return torch.float64 if dt == np.float64 else torch.float32


def _paths(dt, p):
    out = [TILED]
    if p in TPR:
        out += [SIMT, PREFETCH]
    if p in TPR_ALT:
        out.append(ALT)
    if dt == np.float64 and p in (8, 16, 32):
        out.append(DMMA)
    return out


def _full_pass(path, p, sms):
    """Rows one full pass of the path's grid covers (block.cu: launch_mma_f64, block_ws_create, panel_grid) on a
    workspace whose n is large enough for the grid to saturate."""
    if path == DMMA:
        return sms * (3 if p <= 16 else 2) * MMA_WARPS * 8
    if path in (SIMT, PREFETCH, ALT):
        return 2 * sms * (KBLOCK // (TPR_ALT if path == ALT else TPR)[p])
    return (PANEL_TILE // (p | 1)) * 4 * sms


def _rows(p, B):
    return sorted({1, 7, 8, 9, p, 255, 257, B - 1, B + 1, 3 * B + 5})


def _chain(path, p, rows, sms):
    """Longest addition chain of one entry of G on this launch shape: the rows one lane (or one DMMA accumulator)
    sums, plus the shuffle or row-group depth inside the CTA, plus the warps, plus the CTAs of the last-block sum."""
    if path == DMMA:
        tiles = -(-rows // 8)
        grid = max(1, min(sms * (3 if p <= 16 else 2), -(-tiles // MMA_WARPS)))
        per_warp = -(-tiles // (grid * MMA_WARPS))
        return 8 * per_warp + MMA_WARPS + grid
    if path in (SIMT, PREFETCH, ALT):
        tpr = (TPR_ALT if path == ALT else TPR)[p]
        grid = 2 * sms
        passes = -(-rows // (grid * (KBLOCK // tpr)))
        return passes + int(math.log2(32 // tpr)) + KBLOCK // 32 + grid
    trows = PANEL_TILE // (p | 1)
    grid = 4 * sms
    nbi = (p + 3) // 4
    ngroups = KBLOCK // (nbi * nbi)
    tiles_per_cta = -(-(-(-rows // trows)) // grid)
    return -(-trows // ngroups) * tiles_per_cta + ngroups + grid


def _gamma(k, dt):
    u = 2.0 ** -53 if dt == np.float64 else 2.0 ** -24
    return k * u / (1 - k * u)


def _check(got, ref, absbound, k, dt, what):
    """Bit-exact while every partial sum is exact in dt, else |got - ref| <= gamma_k |.|-bound."""
    assert np.isfinite(got).all(), f"{what}: non-finite entries (a read outside the row range?)"
    exact_limit = 2.0 ** (51 if dt == np.float64 else 22)
    if absbound.max() < exact_limit:
        bad = got.astype(np.float64) != ref
        assert not bad.any(), f"{what}: {bad.sum()} of {bad.size} entries differ from the exact result, first at {np.argwhere(bad)[0]}"
    else:
        err = np.abs(got.astype(np.float64) - ref)
        tol = _gamma(k, dt) * absbound
        assert np.all(err <= tol), f"{what}: error {err.max():.3e} over the rounding bound (k = {k})"


class Panels:
    """Device panels with NaN guard rows around a `rows`-row range, refilled from pristine host data per call."""

    def __init__(self, torch, dt, p):
        self.torch, self.dt, self.p = torch, dt, p
        self.tdt = _tdt(torch, dt)
        self.bufs = {}

    def make(self, name, data):
        t = self.torch
        rows = data.shape[0]
        buf = t.full((GUARD_LO + rows + GUARD_HI, self.p), float("nan"), dtype=self.tdt, device="cuda")
        buf[GUARD_LO:GUARD_LO + rows] = t.from_numpy(np.ascontiguousarray(data, dtype=self.dt)).cuda()
        self.bufs[name] = (buf, rows)
        return buf.data_ptr() + GUARD_LO * self.p * buf.element_size()

    def rows_of(self, name):
        buf, rows = self.bufs[name]
        return buf[GUARD_LO:GUARD_LO + rows].cpu().numpy()

    def guards_unchanged(self, name):
        buf, rows = self.bufs[name]
        h = buf.cpu().numpy()
        iv = np.int64 if self.dt == np.float64 else np.int32
        g = np.concatenate([h[:GUARD_LO], h[GUARD_LO + rows:]]).view(iv)
        nan = np.full(1, np.nan, self.dt).view(iv)[0]
        return bool(np.all(g == nan))


class BlockWs:
    def __init__(self, kb, n, p, dt):
        self.ws = kb.BlockGmresWorkspace(n, n, p, dt, memory=1)
        self.n, self.p, self.dt = n, p, dt

    def op(self, torch, op, path, rows, alpha=0.0, In=None, S=None, beta=0.0, Out=None, Next=None, G=None):
        torch.cuda.synchronize()
        return _lib.lib().krylov_b200_block_panel_op(self.ws._h, op, path, rows, alpha, In, S, beta, Out, Next, G)

    def free(self):
        self.ws.free()


def _smat(p, rng):
    """p x p small integers, non-symmetric; for p <= 3 all entries distinct (|v| <= 4 allows no more)."""
    if p <= 3:
        return rng.permutation(np.arange(-4, 5))[:p * p].reshape(p, p).astype(np.float64)
    S = rng.integers(-4, 5, size=(p, p)).astype(np.float64)
    S[0, 1], S[1, 0] = 3.0, -2.0
    return S


def _run_case(torch, ws, path, p, dt, rows, data, S, sms, variant):
    """One (rows) point: op 0 with and without Next, op 1 and op 2 with a rotating (alpha, beta, alias, Next) choice."""
    In_h, Out_h, Nx_h = (d[:rows] for d in data)
    pan = Panels(torch, dt, p)
    Sd = torch.from_numpy(np.asfortranarray(S).ravel(order="F").astype(dt)).cuda()
    Gd = torch.full((p * p,), float("nan"), dtype=_tdt(torch, dt), device="cuda")
    k = _chain(path, p, rows, sms)
    tag = f"path {path} p {p} {np.dtype(dt).name} rows {rows}"

    def gram(L, R):
        return L.T @ R, np.abs(L).T @ np.abs(R)

    for use_next in (False, True):                                          # op 0
        Gd.fill_(float("nan"))
        po = pan.make("out", Out_h)
        pn = pan.make("next", Nx_h) if use_next else None
        assert ws.op(torch, 0, path, rows, Out=po, Next=pn, G=Gd.data_ptr()) == 0, _lib.last_error()
        G = Gd.cpu().numpy().reshape(p, p, order="F")
        ref, bound = gram(Nx_h if use_next else Out_h, Out_h)
        _check(G, ref, bound, k, dt, f"{tag} op 0 next={use_next}")
        assert pan.guards_unchanged("out") and np.array_equal(pan.rows_of("out"), Out_h.astype(dt)), f"{tag}: op 0 wrote Out"

    for op in (1, 2):
        combos = [(b, a, nx) for b in (False, True) for a in (False, True) for nx in ((False, True) if op == 2 else (False,))]
        beta_nz, alias, use_next = combos[variant % len(combos)]
        alpha = ALPHAS[variant % len(ALPHAS)]
        beta = BETAS[1 + variant % 4] if beta_nz else 0.0
        Gd.fill_(float("nan"))
        po = pan.make("out", Out_h)
        pi = po if alias else pan.make("in", In_h)
        pn = pan.make("next", Nx_h) if use_next else None
        rc = ws.op(torch, op, path, rows, alpha=alpha, In=pi, S=Sd.data_ptr(), beta=beta, Out=po, Next=pn,
                   G=Gd.data_ptr() if op == 2 else None)
        assert rc == 0, _lib.last_error()
        src = Out_h if alias else In_h
        ref = alpha * (src @ S) + (beta * Out_h if beta_nz else 0.0)
        bound = np.abs(alpha) * (np.abs(src) @ np.abs(S)) + (abs(beta) * np.abs(Out_h) if beta_nz else 0.0)
        Out = pan.rows_of("out")
        what = f"{tag} op {op} alpha {alpha} beta {beta} alias={alias} next={use_next}"
        _check(Out, ref, bound, p + 2, dt, what + " (Out)")
        assert pan.guards_unchanged("out"), f"{what}: guard rows of Out changed"
        if op == 2:
            O64 = Out.astype(np.float64)
            G = Gd.cpu().numpy().reshape(p, p, order="F")
            gref, gbound = gram(Nx_h if use_next else O64, O64)
            _check(G, gref, gbound, k, dt, what + " (G)")
        variant += 1
    return variant


def _ws_rows(dt, p, sms):
    return max(3 * _full_pass(path, p, sms) + 5 for path in _paths(dt, p))


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("p", list(range(1, 33)))
def test_panel_ops_exact_with_guards(kb, torch, sms, dt, p):
    """Every path the dispatch can choose for (dtype, p) -- tiled for any p, SIMT / prefetch / alternative lanes per
    row for p in {2, 4, 8, 16, 32}, DMMA for Float64 p in {8, 16, 32} -- and every op, at every rows of `_rows`."""
    n = _ws_rows(dt, p, sms)
    rng = np.random.default_rng(1000 * p + (dt == np.float32))
    data = [rng.integers(-4, 5, size=(n, p)).astype(np.float64) for _ in range(3)]
    S = _smat(p, rng)
    ws = BlockWs(kb, n, p, dt)
    try:
        for path in _paths(dt, p):
            variant = path
            for rows in _rows(p, _full_pass(path, p, sms)):
                if rows <= n:
                    variant = _run_case(torch, ws, path, p, dt, rows, data, S, sms, variant)
    finally:
        ws.free()


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("p", [1, 2, 3, 4, 5, 8, 16, 31, 32])
def test_panel_ops_random_data_within_rounding_bound(kb, torch, sms, dt, p):
    """Random normal panels against an extended-precision (np.longdouble) reference.  G must lie within
    gamma_k (|L|^T |R|), k = `_chain` of the launch shape (rows per lane + shuffle / row-group depth + warps + CTAs);
    Out within gamma_{p+2} (|alpha| |In| |S| + |beta| |Out|).  Two passes over the grid (B + 1 rows): an accumulation
    at lower precision than the kernel's type fails the bound."""
    rng = np.random.default_rng(7 + p)
    ws = BlockWs(kb, _ws_rows(dt, p, sms), p, dt)         # large enough for every grid to saturate (as `_chain` assumes)
    try:
        for path in _paths(dt, p):
            rows = _full_pass(path, p, sms) + 1
            L, R, In = (rng.standard_normal((rows, p)).astype(dt) for _ in range(3))
            S = rng.standard_normal((p, p)).astype(dt)
            pan = Panels(torch, dt, p)
            Sd = torch.from_numpy(S.ravel(order="F").copy()).cuda()
            Gd = torch.zeros(p * p, dtype=_tdt(torch, dt), device="cuda")
            Lx, Rx, Ix, Sx = (a.astype(np.longdouble) for a in (L, R, In, S))
            pr, pl = pan.make("out", R), pan.make("next", L)
            assert ws.op(torch, 0, path, rows, Out=pr, Next=pl, G=Gd.data_ptr()) == 0, _lib.last_error()
            G = Gd.cpu().numpy().reshape(p, p, order="F").astype(np.longdouble)
            k = _chain(path, p, rows, sms)
            err = np.abs(G - Lx.T @ Rx)
            assert np.all(err <= _gamma(k, dt) * (np.abs(Lx).T @ np.abs(Rx))), f"path {path}: G off by {float(err.max()):.3e}"
            po, pi = pan.make("out", R), pan.make("in", In)
            assert ws.op(torch, 2, path, rows, alpha=-1.0, In=pi, S=Sd.data_ptr(), beta=1.0, Out=po, Next=pl,
                         G=Gd.data_ptr()) == 0, _lib.last_error()
            Out = pan.rows_of("out").astype(np.longdouble)
            err = np.abs(Out - (Rx - Ix @ Sx))
            assert np.all(err <= _gamma(p + 2, dt) * (np.abs(Rx) + np.abs(Ix) @ np.abs(Sx))), f"path {path}: Out off"
            G = Gd.cpu().numpy().reshape(p, p, order="F").astype(np.longdouble)
            err = np.abs(G - Lx.T @ Out)
            assert np.all(err <= _gamma(k, dt) * (np.abs(Lx).T @ np.abs(Out))), f"path {path}: fused G off"
    finally:
        ws.free()


@pytest.mark.parametrize("dt,p,path", [(np.float64, 8, DMMA), (np.float64, 32, DMMA), (np.float64, 16, SIMT),
                                       (np.float32, 8, SIMT), (np.float64, 5, TILED), (np.float32, 32, TILED),
                                       (np.float64, 8, 0), (np.float32, 4, 0)])
def test_gram_is_deterministic_across_grids(kb, torch, sms, dt, p, path):
    """Two identical Gram products are bit-identical, also with a product on a different grid in between: the
    "last block finalises" ticket (ctx.tickets + 6) re-arms after every launch, whatever the grid."""
    rows = 3 * _full_pass(path or (DMMA if dt == np.float64 and p in (8, 16, 32) else SIMT if p in TPR else TILED), p, sms) + 5
    ws = BlockWs(kb, rows, p, dt)
    try:
        rng = np.random.default_rng(p)
        pan = Panels(torch, dt, p)
        pr, pl = pan.make("out", rng.standard_normal((rows, p))), pan.make("next", rng.standard_normal((rows, p)))
        G = []
        for r in (rows, 300, rows):
            Gd = torch.zeros(p * p, dtype=_tdt(torch, dt), device="cuda")
            assert ws.op(torch, 0, path, r, Out=pr, Next=pl, G=Gd.data_ptr()) == 0, _lib.last_error()
            G.append(Gd.cpu().numpy())
        assert np.array_equal(G[0], G[2])
        assert not np.array_equal(G[0], G[1])
    finally:
        ws.free()


def test_panel_op_rejects_unavailable_combinations(kb, torch):
    ws32 = BlockWs(kb, 64, 8, np.float32)
    ws3 = BlockWs(kb, 64, 3, np.float64)
    try:
        buf = torch.zeros(64 * 8, dtype=torch.float64, device="cuda")
        G = torch.zeros(64, dtype=torch.float64, device="cuda")
        assert ws32.op(torch, 0, DMMA, 64, Out=buf.data_ptr(), G=G.data_ptr()) == -1        # DMMA is Float64 only
        for path in (DMMA, SIMT, PREFETCH, ALT):
            assert ws3.op(torch, 0, path, 64, Out=buf.data_ptr(), G=G.data_ptr()) == -1
        assert ws3.op(torch, 0, TILED, 65, Out=buf.data_ptr(), G=G.data_ptr()) == -1        # rows > n
        assert ws3.op(torch, 3, TILED, 64, Out=buf.data_ptr(), G=G.data_ptr()) == -1
    finally:
        ws32.free()
        ws3.free()


# ---------------------------------------------------------------------------------------------------------------------
# SpMM
# ---------------------------------------------------------------------------------------------------------------------
DT = {np.float64: _lib.KRYLOV_FLOAT64, np.float32: _lib.KRYLOV_FLOAT32}


def _drop_col0(A):
    d = np.ones(A.shape[1])
    d[0] = 0.0
    A = sp.csr_matrix(sp.csr_matrix(A) @ sp.diags(d))
    A.eliminate_zeros()
    return A


def _random_pattern(n, per_row, rng):
    """`per_row` uniform column draws per row (duplicates summed) plus the diagonal."""
    rows = np.repeat(np.arange(n), per_row)
    A = sp.coo_matrix((rng.standard_normal(n * per_row), (rows, rng.integers(0, n, n * per_row))), shape=(n, n))
    return sp.csr_matrix(A) + sp.eye(n)


def _spmm_matrices(sms):
    rng = np.random.default_rng(11)
    mats = {}
    for dims in ((7, 5, 3), (33, 9, 2)):
        rp, ci, va = P.div_grad_csr(*dims)
        n = len(rp) - 1
        mats[f"div_grad{dims}"] = _drop_col0(sp.csr_matrix((va, ci, rp), shape=(n, n)))
    n = 5000
    A = _random_pattern(n, 15, rng).tolil()
    for r in (0, 255, 256, n - 1):
        A[r, :] = 0
    A[512:768, :] = 0                                       # one fully empty 256-row tile
    A[300, 1::4] = rng.standard_normal(len(range(1, n, 4)))  # a row of 1250 nonzeros
    mats["random_empty_rows"] = _drop_col0(A)
    mats["n1"] = sp.csr_matrix(np.array([[3.0]]))
    for n in (255, 256 * 40 + 1, 3 * 3 * sms * 256 + 17):  # the last: several ring positions per CTA
        mats[f"n{n}"] = _drop_col0(_random_pattern(n, 9, rng))
    n = 50_000
    A = sp.lil_matrix((n, n))
    A.setdiag(2.0)
    A[7, 1:40_001] = rng.standard_normal(40_000)           # too long a tile for the shared-memory ring
    mats["dense_row"] = _drop_col0(A)
    return mats


@pytest.fixture(scope="module")
def spmm_mats(sms):
    return _spmm_matrices(sms)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("name", ["div_grad(7, 5, 3)", "div_grad(33, 9, 2)", "random_empty_rows", "n1", "n255", "n10241",
                                  "ring", "dense_row", "random_empty_rows_1based_int64"])
def test_spmm_columns_equal_oracle_spmv(O, torch, sms, spmm_mats, dt, name):
    """Y[:, c] of every variant equals oracle.spmv(A, X[:, c]) bit for bit.  Rows of X that no nonzero references
    (column 0 among them) are NaN, so the gather an empty row issues must be discarded; the NaN guard rows of Y past
    n must be left alone.  Variant 0 for p in {1, 2, 3, 4, 8, 16, 32}, variant 1 for every p, variant 2 for
    p in {2, 4, 8, 16, 32} when the tile plan fits (else it must fail and variant 0 must fall back)."""
    key = {"ring": f"n{3 * 3 * sms * 256 + 17}", "random_empty_rows_1based_int64": "random_empty_rows"}.get(name, name)
    A = sp.csr_matrix(spmm_mats[key]).astype(dt)
    A.sort_indices()
    n = A.shape[0]
    base, ibytes = (1, 8) if name.endswith("int64") else (0, 4)
    it = np.int64 if ibytes == 8 else np.int32
    rp, ci = (A.indptr + base).astype(it), (A.indices + base).astype(it)
    va = np.ascontiguousarray(A.data, dtype=dt)
    L = _lib.lib()
    ctx = L.kb200_ctx_create(-1)
    assert ctx
    csr = L.kb200_csr_create(ctx, DT[dt], n, A.nnz, rp.ctypes.data_as(C.c_void_p), ci.ctypes.data_as(C.c_void_p),
                             va.ctypes.data_as(C.c_void_p), base, ibytes, 0)
    assert csr, _lib.last_error()
    try:
        plan = (C.c_longlong * 7)()
        L.kb200_csr_plan(csr, plan)
        if name == "ring":
            assert plan[0] >= 3 * plan[5], "every CTA should walk several ring positions"
        if name == "dense_row":
            assert not plan[3]
        X = np.random.default_rng(5).standard_normal((n, 32)).astype(dt)
        referenced = np.zeros(n, bool)
        referenced[A.indices] = True
        X[~referenced] = np.nan
        if n > 1:
            assert not referenced[0]
        Yref = np.stack([O.spmv(A, X[:, c], dtype=dt) for c in range(32)], axis=1)
        Xd = torch.from_numpy(X).cuda()
        cases = [(1, p) for p in range(1, 33)] + [(0, p) for p in (1, 2, 3, 4, 8, 16, 32)] + \
                [(2, p) for p in (2, 4, 8, 16, 32)]
        iv = np.int64 if dt == np.float64 else np.int32
        for variant, p in cases:
            Xp = Xd[:, :p].contiguous()
            Y = torch.full((n + 5, p), float("nan"), dtype=_tdt(torch, dt), device="cuda")
            torch.cuda.synchronize()
            rc = L.kb200_spmm_csr(ctx, csr, p, Xp.data_ptr(), Y.data_ptr(), variant)
            if variant == 2 and not plan[3]:
                assert rc == -1 and "tile plan" in _lib.last_error()
                continue
            assert rc == 0, _lib.last_error()
            Yh = Y.cpu().numpy()
            assert np.array_equal(Yh[:n], Yref[:, :p]), \
                f"variant {variant} p {p}: {(Yh[:n] != Yref[:, :p]).sum()} entries differ from the sequential SpMV"
            assert np.all(Yh[n:].view(iv) == np.full(1, np.nan, dt).view(iv)[0]), f"variant {variant} p {p}: wrote past n"
        assert L.kb200_spmm_csr(ctx, csr, 3, Xd.data_ptr(), Xd.data_ptr(), 2) == -1      # no TMA kernel for p = 3
    finally:
        L.kb200_csr_destroy(csr)
        L.kb200_ctx_destroy(ctx)
