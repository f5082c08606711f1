"""GPU: the two block-Jacobi kernels one at a time (kb200_blockdiag_mul, kb200_blockdiag_invert) against plain
references, at every block size 2..8, in both types.

Multiply.  With random data y must equal, bit for bit, a NumPy restatement of the kernel's order (each row summed left
to right, every product rounded before the add).  With dyadic data (small integers times powers of two) every product
and partial sum is exact, so y must equal the exact product whatever the order.

Inverse.  Compared with np.linalg.inv in float64, under c bs eps(T) kappa(B).  Blocks that need a row swap (a zero
leading entry) are mixed in everywhere; exactly singular blocks (a zero row, two equal rows) must be the only ones
zeroed and must raise the flag, and their neighbours must be intact.

Every launch carries NaN guards: x past n, the padding rows and columns of a ragged last block, and the blocks past
ceil(n / bs).  A kernel that reads one turns y or the inverse into NaN.  y and the inverse are NaN on entry and carry
guard entries past their end, whose bits must not change.  n runs over 1, bs - 1, bs, bs + 1, one n for each last-block
size, and block counts B - 1, B, B + 1 and 3B + 5, where B is the number of blocks one full pass of the launch grid
covers, computed from the SM count the way the launchers do (stream_grid: 8 CTAs per SM for the multiply, 4 for the
inverse, 256 threads, one block per thread)."""
import ctypes as C

import numpy as np
import pytest

from krylov_b200 import _lib

pytestmark = pytest.mark.gpu

KBLOCK = 256
GUARD = 7                                    # entries (vectors) or blocks (block arrays) past the end
DT = {np.float64: _lib.KRYLOV_FLOAT64, np.float32: _lib.KRYLOV_FLOAT32}
EPS = {np.float64: 2.0 ** -53, np.float32: 2.0 ** -24}
SENTINEL = -1234.5


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def dev(torch):
    L = _lib.lib()
    ctx = L.kb200_ctx_create(-1)
    assert ctx, _lib.last_error()
    yield L, ctx, torch.cuda.get_device_properties(0).multi_processor_count
    L.kb200_ctx_destroy(ctx)


def full_pass(sms, ctas_per_sm):
    """Blocks one full pass of the launch grid covers (stream_grid(nb, 1, ctas_per_sm) threads, capped at 2048 CTAs)."""
    return min(sms * ctas_per_sm, 2048) * KBLOCK


def sizes(bs, B):
    """(n, what it pins): the small edges, every last-block size, and the block counts around the full pass."""
    out = {1: "n = 1", bs - 1: "n = bs - 1", bs: "n = bs", bs + 1: "n = bs + 1"}
    for r in range(1, bs):
        out.setdefault(3 * bs + r, f"last block of {r} rows")
    for nb, ragged in ((B - 1, True), (B, False), (B + 1, True), (3 * B + 5, True)):
        out[nb * bs - (bs // 2 if ragged else 0)] = f"{nb} blocks"
    return sorted(out.items())


def nblocks(n, bs):
    return (n + bs - 1) // bs


def guarded_blocks(blocks, n, bs):
    """The block array as the kernel gets it: the padding of a ragged last block and GUARD blocks past the end NaN."""
    nb = nblocks(n, bs)
    g = np.full((nb + GUARD, bs, bs), np.nan, blocks.dtype)
    g[:nb] = blocks[:nb]
    r = n - (nb - 1) * bs
    g[nb - 1, r:, :] = np.nan
    g[nb - 1, :, r:] = np.nan
    return g


def dev_array(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def ptr(t):
    return C.c_void_p(t.data_ptr())


def run_mul(torch, dev, dt, n, bs, blocks, x):
    """y = blockdiag(blocks) x through kb200_blockdiag_mul with NaN guards; returns y[:n]."""
    L, ctx, _ = dev
    Bd = dev_array(torch, guarded_blocks(blocks, n, bs))
    xd = dev_array(torch, np.concatenate([x[:n], np.full(GUARD, np.nan, dt)]))
    y0 = np.concatenate([np.full(n, np.nan, dt), SENTINEL + np.arange(GUARD, dtype=dt)])
    yd = dev_array(torch, y0)
    torch.cuda.synchronize()
    assert L.kb200_blockdiag_mul(ctx, DT[dt], n, bs, ptr(Bd), ptr(xd), ptr(yd)) == 0, _lib.last_error()
    assert L.kb200_sync(ctx) == 0
    y = yd.cpu().numpy()
    assert not np.isnan(y[:n]).any(), f"{np.isnan(y[:n]).sum()} rows of y are NaN or were not written"
    assert y[n:].tobytes() == y0[n:].tobytes(), "entries past n were written"
    return y[:n]


def mul_restated(blocks, x, n, bs):
    """The kernel's order in NumPy: per row, acc = acc + B[i, j] * x[j] for j = 0, 1, ... in the working type.  The
    zero padding of a ragged last block adds +0 to acc, which changes no bit (acc is never -0)."""
    nb = nblocks(n, bs)
    B = blocks[:nb].copy()
    r = n - (nb - 1) * bs
    B[nb - 1, r:, :] = 0
    B[nb - 1, :, r:] = 0
    xp = np.zeros(nb * bs, blocks.dtype)
    xp[:n] = x[:n]
    xp = xp.reshape(nb, bs)
    y = np.empty((nb, bs), blocks.dtype)
    for i in range(bs):
        acc = np.zeros(nb, blocks.dtype)
        for j in range(bs):
            acc = acc + B[:, i, j] * xp[:, j]
        y[:, i] = acc
    return y.reshape(-1)[:n]


def dyadic(rng, shape, dt):
    """Integers in [-7, 7] times 2^k, k in [-3, 3]: products and sums of eight of them are exact in Float32."""
    return (rng.integers(-7, 8, shape) * 2.0 ** rng.integers(-3, 4, shape)).astype(dt)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("bs", range(2, 9))
def test_blockdiag_mul(torch, dev, dt, bs):
    B = full_pass(dev[2], 8)
    cases = sizes(bs, B)
    nmax = max(n for n, _ in cases)
    rng = np.random.default_rng(bs)
    blocks = rng.standard_normal((nblocks(nmax, bs), bs, bs)).astype(dt)
    x = rng.standard_normal(nmax).astype(dt)
    iblocks, ix = dyadic(rng, blocks.shape, dt), dyadic(rng, nmax, dt)
    for n, what in cases:
        got = run_mul(torch, dev, dt, n, bs, blocks, x)
        want = mul_restated(blocks, x, n, bs)
        bad = got.view(np.uint8).reshape(n, -1) != want.view(np.uint8).reshape(n, -1)
        assert not bad.any(), f"{what} (n = {n}): {bad.any(axis=1).sum()} rows differ from the left-to-right order, " \
                              f"first at row {np.argmax(bad.any(axis=1))}"
        got = run_mul(torch, dev, dt, n, bs, iblocks, ix)
        exact = mul_restated(iblocks.astype(np.float64), ix.astype(np.float64), n, bs)
        assert np.array_equal(got.astype(np.float64), exact), f"{what} (n = {n}): dyadic product not exact"


# ----------------------------------------------------------------------------------------------------------------------
# Inverse
# ----------------------------------------------------------------------------------------------------------------------
def run_invert(torch, dev, dt, n, bs, blocks):
    """(inverses of the first ceil(n / bs) blocks, singular flag) through kb200_blockdiag_invert with NaN guards."""
    L, ctx, _ = dev
    nb = nblocks(n, bs)
    Bd = dev_array(torch, guarded_blocks(blocks, n, bs))
    inv0 = np.full((nb + GUARD, bs, bs), np.nan, dt)
    inv0[nb:] = SENTINEL
    invd = dev_array(torch, inv0)
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    assert L.kb200_blockdiag_invert(ctx, DT[dt], n, bs, ptr(Bd), ptr(invd), ptr(flag)) == 0, _lib.last_error()
    assert L.kb200_sync(ctx) == 0
    inv = invd.cpu().numpy()
    assert inv[nb:].tobytes() == inv0[nb:].tobytes(), "blocks past ceil(n / bs) were written"
    return inv[:nb], int(flag.item())


def triangular_block(rng, r, dup=None):
    """A row-permuted upper triangular r x r block with power-of-two diagonal and small integers above it, whose first
    row has a zero leading entry (r > 1): Gauss-Jordan with partial pivoting must swap rows, and runs exactly.  dup =
    (i, j): row j is a copy of row i, an exactly singular block the elimination zeroes exactly."""
    U = np.triu(rng.integers(-3, 4, (r, r)).astype(np.float64), 1)
    U[np.diag_indices(r)] = 2.0 ** rng.integers(-1, 2, r) * rng.choice([-1.0, 1.0], r)
    if dup:
        U[dup[1]] = U[dup[0]]
    perm = rng.permutation(r)
    if r > 1 and perm[0] == 0:
        perm[[0, 1]] = perm[[1, 0]]
    return U[perm]


def fill_blocks(rng, nb, bs, n, singular):
    """nb well-conditioned random blocks; every 5th needs a row swap (a zero leading entry; every 10th a permuted
    triangular one).  singular: indices of blocks made exactly singular -- alternately a zero row and two equal rows.
    Returns the blocks (float64) and the size of each block's used part."""
    rows = np.full(nb, bs)
    rows[-1] = n - (nb - 1) * bs
    D = rng.standard_normal((nb, bs, bs)) + 2.0 * bs * np.eye(bs) * rng.choice([-1.0, 1.0], (nb, 1, 1))
    for k in range(0, nb, 5):
        D[k, 0, 0] = 0.0
    for k in list(range(0, nb, 10)) + [nb - 1]:
        D[k] = 0.0
        D[k, :rows[k], :rows[k]] = triangular_block(rng, rows[k])
    for t, k in enumerate(singular):
        r = rows[k]
        if t % 2 == 0 or r < 2:                   # a zero row, with random entries elsewhere
            D[k, rng.integers(r), :] = 0.0
        else:                                     # two equal rows of an exactly eliminated block
            i, j = sorted(rng.choice(r, 2, replace=False))
            D[k] = 0.0
            D[k, :r, :r] = triangular_block(rng, r, dup=(i, j))
    return D, rows


def check_inverse(inv, D, rows, singular, dt, what):
    eps = EPS[dt]
    Dd = D.astype(dt).astype(np.float64)                 # the blocks the kernel got, exactly
    sing = set(int(k) for k in singular)
    for r in np.unique(rows):
        ks = np.flatnonzero(rows == r)
        ok = np.array([k for k in ks if k not in sing], dtype=np.int64)
        bad = np.array([k for k in ks if k in sing], dtype=np.int64)
        if len(bad):
            assert not inv[bad].any(), f"{what}: a singular block's inverse is not zero"
        if not len(ok):
            continue
        Bk = Dd[ok, :r, :r]
        ref = np.linalg.inv(Bk)
        got = inv[ok].astype(np.float64)
        assert np.isfinite(got).all(), f"{what}: non-finite inverse entries (pivoting, or a read of the padding?)"
        assert not got[:, r:, :].any() and not got[:, :, r:].any(), f"{what}: padding of the inverse not zero"
        kappa = np.linalg.cond(Bk)
        err = np.linalg.norm(got[:, :r, :r] - ref, axis=(1, 2)) / np.linalg.norm(ref, axis=(1, 2))
        bar = 10 * r * eps * kappa
        worst = int(np.argmax(err / bar))
        assert np.all(err <= bar), f"{what}: block {ok[worst]} off by {err[worst]:.2e} (bar {bar[worst]:.2e})"


@pytest.mark.parametrize("dt", [np.float64, np.float32])
@pytest.mark.parametrize("bs", range(2, 9))
def test_blockdiag_invert(torch, dev, dt, bs):
    B = full_pass(dev[2], 4)
    rng = np.random.default_rng(100 + bs)
    for n, what in sizes(bs, B):
        nb = nblocks(n, bs)
        # without singular blocks the flag stays down, pivoting blocks included
        D, rows = fill_blocks(rng, nb, bs, n, [])
        inv, flag = run_invert(torch, dev, dt, n, bs, D.astype(dt))
        assert flag == 0, f"{what}: flag raised without a singular block"
        check_inverse(inv, D, rows, [], dt, what)
        # exactly singular blocks at the start, in the middle, in the last pass of the grid and last
        sing = sorted({0, nb // 2, max(0, nb - B // 2), nb - 1} | ({1} if nb > 2 else set()))
        D, rows = fill_blocks(rng, nb, bs, n, sing)
        inv, flag = run_invert(torch, dev, dt, n, bs, D.astype(dt))
        assert flag == 1, f"{what}: singular blocks not flagged"
        check_inverse(inv, D, rows, sing, dt, what)
        zeroed = [k for k in range(nb) if not inv[k].any()]
        assert zeroed == sing, f"{what}: zeroed {zeroed[:8]}, singular {sing[:8]}"


def test_blockdiag_kernels_refuse_bad_block_sizes(dev):
    L, ctx, _ = dev
    for bs in (0, 1, 9):
        assert L.kb200_blockdiag_mul(ctx, _lib.KRYLOV_FLOAT64, 4, bs, None, None, None) == -1
        assert "2..8" in _lib.last_error()
        assert L.kb200_blockdiag_invert(ctx, _lib.KRYLOV_FLOAT64, 4, bs, None, None, None) == -1
