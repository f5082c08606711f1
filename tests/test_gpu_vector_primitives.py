"""GPU: the vector primitives of blas1.cu (kaxpy!, kaxpby!, kscal!, kcopy!, kscalcopy!, kdivcopy!, kfill!, the diagonal
preconditioner's product and solve, kdot, knorm, the fused dot pair and the CG prologue) against exact references.

Every case runs in Float64 and Float32, at the launch shapes where grid-stride loops go wrong: a few elements, one
element either side of the grid's stride S, either side of the 4-way unrolled trip (4S), where the grid saturates, and
many trips per thread.  Every operand sits at an odd element offset inside a larger allocation, between NaN guard cells:
an element update must leave the guards' bits alone, and a reduction that read one of them would come out NaN.

- Element updates are bit-exact against NumPy's non-contracted restatement (product rounded, then the add), with
  +-0, subnormals, +-Inf and NaN among the operands: IEEE propagation through every op, no BLAS zero-coefficient
  shortcut.
- Reductions of small integers are exact (every partial sum is representable), so they must equal the exact sum.
- Reductions of random data are held to the rounding-error bound of the launch's summation tree against a correctly
  rounded reference (exact products, math.fsum).
- knorm is BLAS nrm2: within a few ulps of the exact norm from the underflow to the overflow threshold."""
import ctypes as C
import math

import numpy as np
import pytest

from krylov_b200 import _lib

pytestmark = pytest.mark.gpu

DTS = [np.float64, np.float32]
DT = {np.float64: _lib.KRYLOV_FLOAT64, np.float32: _lib.KRYLOV_FLOAT32}
UINT = {np.float64: np.uint64, np.float32: np.uint32}
GUARD_NAN = {np.float64: np.uint64(0x7FF8DEAD0000BEEF), np.float32: np.uint32(0x7FC0BEEF)}
LEAD, TRAIL = 7, 5                    # guard cells before (odd: the operand sits at an odd element offset) and after
BLOCK, PER_THREAD, MAX_PARTIALS = 256, 4, 2048   # common.cuh: kBlock, stream_grid's per_thread, kMaxPartials
EW_CTAS, RED_CTAS = 8, 4              # CTAs per SM: element updates / reductions (blas1.cu)


def sm_count():
    import torch
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def cap(ctas):
    return min(sm_count() * ctas, MAX_PARTIALS)


def grid_of(n, ctas):
    """stream_grid(n, 4, ctas): whole CTAs of 4 elements per thread, capped at ctas per SM."""
    need = -(-n // (BLOCK * PER_THREAD))
    return max(1, min(need, cap(ctas)))


# Shapes by name, from the saturated stride S = cap * 256 of the kernel's grid.  need = cap CTAs is n = 4S.
SHAPES = {
    "0": lambda S: 0, "1": lambda S: 1, "2": lambda S: 2, "3": lambda S: 3, "4": lambda S: 4,
    "255": lambda S: 255, "256": lambda S: 256, "257": lambda S: 257,
    "S-1": lambda S: S - 1, "S+1": lambda S: S + 1,
    "4S-1": lambda S: 4 * S - 1, "4S": lambda S: 4 * S, "4S+1": lambda S: 4 * S + 1, "5S-1": lambda S: 5 * S - 1,
    "need=cap-1": lambda S: 4 * S - BLOCK * PER_THREAD, "need=cap+1": lambda S: 4 * S + BLOCK * PER_THREAD,
    "many-trips": lambda S: 41 * S + 123,
}


def size(name, ctas):
    return SHAPES[name](cap(ctas) * BLOCK)


class Dev:
    def __init__(self):
        self.L = _lib.lib()
        self.ctx = self.L.kb200_ctx_create(-1)
        assert self.ctx, _lib.last_error()
        self.bufs = []

    def put(self, a):
        """a inside NaN guard cells, at an odd element offset; returns the guarded host image and the operand's pointer."""
        a = np.ascontiguousarray(a)
        dt = a.dtype.type
        full = np.empty(LEAD + len(a) + TRAIL, dt)
        full.view(UINT[dt])[:] = GUARD_NAN[dt]
        full[LEAD:LEAD + len(a)] = a
        p = self.L.kb200_alloc(full.nbytes)
        assert p
        self.bufs.append(p)
        self.L.kb200_h2d(p, full.ctypes.data_as(C.c_void_p), full.nbytes)
        return Buf(self, p, full, len(a))

    def launches(self):
        return self.L.kb200_ctx_launch_count(self.ctx)

    def close(self):
        for p in self.bufs:
            self.L.kb200_free(p)
        self.L.kb200_ctx_destroy(self.ctx)


class Buf:
    def __init__(self, dev, base, full, n):
        self.dev, self.base, self.full, self.n = dev, base, full, n
        self.ptr = base + LEAD * full.itemsize

    def get(self):
        """The operand after checking that not one bit of the guard cells changed."""
        out = np.empty_like(self.full)
        assert self.dev.L.kb200_sync(self.dev.ctx) == 0
        self.dev.L.kb200_d2h(out.ctypes.data_as(C.c_void_p), self.base, out.nbytes)
        u = UINT[out.dtype.type]
        guards = np.r_[0:LEAD, LEAD + self.n:len(out)]
        assert np.array_equal(out.view(u)[guards], self.full.view(u)[guards]), "a guard cell was written"
        return out[LEAD:LEAD + self.n]


@pytest.fixture()
def dev():
    d = Dev()
    yield d
    d.close()


def same_bits(got, exp):
    """Bit for bit, except that a NaN only has to be a NaN (payloads differ between the GPU and the host)."""
    gn, en = np.isnan(got), np.isnan(exp)
    if not np.array_equal(gn, en):
        return False
    u = UINT[got.dtype.type]
    return np.array_equal(got.view(u)[~gn], exp.astype(got.dtype).view(u)[~en])


def specials(dt):
    fi = np.finfo(dt)
    sub = fi.smallest_subnormal
    return np.array([0.0, -0.0, sub, -sub, 3 * sub, fi.tiny / 3, -fi.tiny, fi.tiny, np.inf, -np.inf, np.nan, fi.max,
                     -fi.max, 1.0, -1e-30], dtype=dt)


def special_data(n, dt, seed):
    """Normal data with about a fifth of the entries replaced by special values, at different places in each call."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n).astype(dt)
    pick = rng.random(n) < 0.2
    x[pick] = rng.choice(specials(dt), int(pick.sum()))
    if n:
        x[-1] = specials(dt)[seed % len(specials(dt))]     # the last element is the one a wrong bound drops
    return x


EW_OPS = ["axpy", "axpby", "scal", "copy", "scalcopy", "divcopy", "diagmul", "diagdiv"]


def run_elementwise(dev, op, dt, n, s, t):
    x, y, d = special_data(n, dt, 1), special_data(n, dt, 2), special_data(n, dt, 3)
    L, ctx, code = dev.L, dev.ctx, DT[dt]
    bx, by, bd = dev.put(x), dev.put(y), dev.put(d)
    with np.errstate(all="ignore"):
        s, t = dt(s), dt(t)
        if op == "axpy":
            assert L.kb200_axpy(ctx, code, n, float(s), bx.ptr, by.ptr) == 0
            exp = y + s * x
        elif op == "axpby":
            assert L.kb200_axpby(ctx, code, n, float(s), bx.ptr, float(t), by.ptr) == 0
            exp = s * x + t * y
        elif op == "scal":
            assert L.kb200_scal(ctx, code, n, float(s), by.ptr) == 0
            exp = s * y
        elif op == "copy":
            assert L.kb200_copy(ctx, code, n, by.ptr, bx.ptr) == 0
            exp = x
        elif op == "scalcopy":
            assert L.kb200_scalcopy(ctx, code, n, by.ptr, float(s), bx.ptr) == 0
            exp = s * x
        elif op == "divcopy":
            assert L.kb200_divcopy(ctx, code, n, by.ptr, bx.ptr, float(s)) == 0
            exp = x / s
        elif op == "diagmul":
            assert L.kb200_diagmul(ctx, code, n, by.ptr, bd.ptr, bx.ptr, 0) == 0
            exp = d * x
        else:
            assert L.kb200_diagmul(ctx, code, n, by.ptr, bd.ptr, bx.ptr, 1) == 0
            exp = x / d
    got = by.get()
    assert got.dtype == dt and exp.dtype == dt
    if op == "copy":     # a copy moves bits, NaN payloads included
        assert np.array_equal(got.view(UINT[dt]), exp.view(UINT[dt]))
    else:
        differ = (got.view(UINT[dt]) != exp.view(UINT[dt])) & ~(np.isnan(got) & np.isnan(exp))
        assert same_bits(got, exp), f"{op}: first mismatches at {np.flatnonzero(differ)[:5]}"
    bx.get(), bd.get()   # inputs: guards intact


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("op", EW_OPS)
def test_elementwise_bit_exact(dev, op, dt, shape):
    run_elementwise(dev, op, dt, size(shape, EW_CTAS), 0.37, -1.25)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("shape", ["257", "4S+1"])
@pytest.mark.parametrize("s,t", [(0.0, -0.0), (-np.inf, np.nan), (5e-324, 1e300)])
@pytest.mark.parametrize("op", ["axpy", "axpby", "scal", "scalcopy", "divcopy"])
def test_elementwise_special_coefficients(dev, op, dt, shape, s, t):
    """A zero, infinite, NaN or subnormal coefficient propagates like IEEE arithmetic (0 * Inf = NaN, x / 0 = +-Inf):
    no BLAS shortcut for alpha = 0.  (In Float32, 5e-324 rounds to 0 and 1e300 to Inf.)"""
    run_elementwise(dev, op, dt, size(shape, EW_CTAS), s, t)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("v", [0.0, -0.0, 2.5, -np.inf, np.nan])
def test_fill(dev, dt, shape, v):
    """0.0 takes the memset path; -0.0 must keep its sign bit, so it may not."""
    n = size(shape, EW_CTAS)
    b = dev.put(special_data(n, dt, 4))
    assert dev.L.kb200_fill(dev.ctx, DT[dt], n, b.ptr, v) == 0
    assert same_bits(b.get(), np.full(n, v, dt))


# ---------------------------------------------------------------------------------------------------------------------
# Reductions
# ---------------------------------------------------------------------------------------------------------------------
def small_ints(n, dt, seed, terms=1):
    """Integers small enough that a sum of n products of `terms` of them never leaves the exact range of dt."""
    rng = np.random.default_rng(seed)
    limit = 2.0 ** (53 if dt == np.float64 else 24)
    r = int(max(1, min(16, math.floor((limit / max(n, 1)) ** (1 / terms)) - 1)))
    return rng.integers(-r, r + 1, n).astype(dt)


def exact(v):
    return int(np.sum(v.astype(np.int64)))


def dot(dev, dt, n, bx, by):
    r = C.c_double()
    assert dev.L.kb200_dot(dev.ctx, DT[dt], n, bx.ptr, by.ptr, C.byref(r)) == 0
    return r.value


def nrm2(dev, dt, n, bx):
    r = C.c_double()
    assert dev.L.kb200_nrm2(dev.ctx, DT[dt], n, bx.ptr, C.byref(r)) == 0
    return r.value


def dot2(dev, dt, n, ba, bb, bu, bv):
    r1, r2 = C.c_double(), C.c_double()
    assert dev.L.kb200_dot2(dev.ctx, DT[dt], n, ba.ptr, bb.ptr, bu.ptr, bv.ptr, C.byref(r1), C.byref(r2)) == 0
    return r1.value, r2.value


def prologue(dev, dt, n, bb, bx, br, bp):
    g = C.c_double()
    assert dev.L.kb200_cg_prologue(dev.ctx, DT[dt], n, bb.ptr, bx.ptr, br.ptr, bp.ptr, C.byref(g)) == 0
    return g.value


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_reductions_of_small_integers_are_exact(dev, dt, shape):
    """Every partial sum is an integer below 2^53 (2^24), so each result is the exact sum, bit for bit: a dropped,
    doubled or out-of-range element, or r1 and r2 swapped, fails outright."""
    n = size(shape, RED_CTAS)
    x, y = small_ints(n, dt, 10, 2), small_ints(n, dt, 11, 2)
    u, v = small_ints(n, dt, 12, 2), small_ints(n, dt, 13, 2)
    bx, by, bu, bv = dev.put(x), dev.put(y), dev.put(u), dev.put(v)
    xy, xx, uv = exact(x * y), exact(x * x), exact(u * v)
    assert dot(dev, dt, n, bx, by) == xy
    assert nrm2(dev, dt, n, bx) == float(np.sqrt(dt(xx)))
    r1, r2 = dot2(dev, dt, n, bx, by, bu, bv)
    assert (r1, r2) == (xy, uv)
    # CG prologue: x = 0, r = p = b bit for bit, gamma = <b, b>; x, r and p start out as NaN
    junk = np.full(n, np.nan, dt)
    bx0, br, bp = dev.put(junk), dev.put(junk), dev.put(junk)
    assert prologue(dev, dt, n, bu, bx0, br, bp) == exact(u * u)
    assert np.all(bx0.get().view(UINT[dt]) == 0)
    for b in (br, bp):
        assert np.array_equal(b.get().view(UINT[dt]), u.view(UINT[dt]))
    for b in (bx, by, bu, bv):
        b.get()


@pytest.mark.parametrize("dt", DTS)
def test_negative_n_is_a_no_op(dev, dt):
    """n < 0 does what n = 0 does: every call succeeds, the reductions return 0, and nothing around the operands is
    read or written (the reductions still launch one CTA to write their result)."""
    L, ctx, code = dev.L, dev.ctx, DT[dt]
    a, b, c, d = (dev.put(np.empty(0, dt)) for _ in range(4))
    for n in (-1, -(2 ** 31)):
        assert dot(dev, dt, n, a, b) == 0
        assert nrm2(dev, dt, n, a) == 0
        assert dot2(dev, dt, n, a, b, c, d) == (0.0, 0.0)
        assert prologue(dev, dt, n, a, b, c, d) == 0
        assert L.kb200_axpy(ctx, code, n, 2.0, a.ptr, b.ptr) == 0
        assert L.kb200_axpby(ctx, code, n, 2.0, a.ptr, 3.0, b.ptr) == 0
        assert L.kb200_scal(ctx, code, n, 2.0, b.ptr) == 0
        assert L.kb200_copy(ctx, code, n, b.ptr, a.ptr) == 0
        assert L.kb200_scalcopy(ctx, code, n, b.ptr, 2.0, a.ptr) == 0
        assert L.kb200_divcopy(ctx, code, n, b.ptr, a.ptr, 2.0) == 0
        assert L.kb200_fill(ctx, code, n, b.ptr, 0.0) == 0
        assert L.kb200_fill(ctx, code, n, b.ptr, 2.5) == 0
        assert L.kb200_diagmul(ctx, code, n, b.ptr, c.ptr, a.ptr, 0) == 0
        assert L.kb200_diagmul(ctx, code, n, b.ptr, c.ptr, a.ptr, 1) == 0
    for buf in (a, b, c, d):
        buf.get()


def two_product(a, b):
    """a * b = p + e exactly (Dekker), for float64 arrays without overflow or underflow."""
    def split(z):
        c = 134217729.0 * z
        hi = c - (c - z)
        return hi, z - hi
    p = a * b
    ah, al = split(a)
    bh, bl = split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def exact_dot(x, y):
    """(correctly rounded <x, y>, sum |x_i y_i|) in float64."""
    p, e = two_product(x.astype(np.float64), y.astype(np.float64))
    return math.fsum(np.concatenate([p, e]).tolist()), math.fsum(np.abs(p).tolist())


def gamma(k, dt):
    u = np.finfo(dt).eps / 2
    return k * u / (1 - k * u)


def depth(n):
    """Roundings on the way from one product to the result: the thread's own elements, the CTA's shuffle tree (8 levels
    for 256 threads), the last CTA's per-thread sum of the grid's partials, and its shuffle tree again."""
    g = grid_of(n, RED_CTAS) if n else 1
    return -(-n // (g * BLOCK)) + 8 + -(-g // BLOCK) + 8


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_reductions_of_random_data(dev, dt, shape):
    n = size(shape, RED_CTAS)
    rng = np.random.default_rng(20)
    x, y, u, v = (rng.standard_normal(n).astype(dt) for _ in range(4))
    bx, by, bu, bv = dev.put(x), dev.put(y), dev.put(u), dev.put(v)
    k, eps = depth(n), np.finfo(dt).eps / 2

    def close_dot(got, a, b):
        ref, mag = exact_dot(a, b)
        assert abs(got - ref) <= gamma(k + 1, dt) * mag, (got, ref, mag)

    close_dot(dot(dev, dt, n, bx, by), x, y)
    r1, r2 = dot2(dev, dt, n, bx, by, bu, bv)
    close_dot(r1, x, y)
    close_dot(r2, u, v)
    ref = math.sqrt(exact_dot(x, x)[0])
    assert abs(nrm2(dev, dt, n, bx) - ref) <= (gamma(k, dt) / 2 + 3 * eps) * ref
    junk = np.full(n, np.nan, dt)
    bx0, br, bp = dev.put(junk), dev.put(junk), dev.put(junk)
    close_dot(prologue(dev, dt, n, bu, bx0, br, bp), u, u)
    assert np.all(bx0.get().view(UINT[dt]) == 0)
    assert np.array_equal(br.get().view(UINT[dt]), u.view(UINT[dt]))
    assert np.array_equal(bp.get().view(UINT[dt]), u.view(UINT[dt]))


@pytest.mark.parametrize("dt", DTS)
def test_reduction_ticket_rearms_across_grids(dev, dt):
    """The reductions share one ticket and one partials buffer per context: the last CTA re-arms the ticket for the
    next launch.  Interleaved at different grid sizes (1 CTA up to the cap; knorm both with and without its rescaling
    pass), every result is bit-identical to the same call made alone."""
    S = cap(RED_CTAS) * BLOCK
    rng = np.random.default_rng(30)
    fi = np.finfo(dt)
    calls = []
    for i, n in enumerate([100, 5 * S - 1, 3000, 4 * S + 1]):
        a, b, c = (rng.standard_normal(n).astype(dt) for _ in range(3))
        tiny = (c * dt(fi.tiny) * dt(2.0 ** -10)).astype(dt)      # knorm of subnormals: two launches
        ba, bb, bc, bt = dev.put(a), dev.put(b), dev.put(c), dev.put(tiny)
        bx0, br, bp = dev.put(a), dev.put(a), dev.put(a)
        calls += [lambda n=n, ba=ba, bb=bb: dot(dev, dt, n, ba, bb),
                  lambda n=n, ba=ba, bb=bb, bc=bc: dot2(dev, dt, n, ba, bb, bc, ba),
                  lambda n=n, bc=bc: nrm2(dev, dt, n, bc),
                  lambda n=n, bt=bt: nrm2(dev, dt, n, bt),
                  lambda n=n, bb=bb, bx0=bx0, br=br, bp=bp: prologue(dev, dt, n, bb, bx0, br, bp)]
    alone = [f() for f in calls]
    for order in (range(len(calls)), reversed(range(len(calls))), rng.permutation(len(calls))):
        order = list(order)
        got = {i: calls[i]() for i in order}
        assert [got[i] for i in range(len(calls))] == alone


# ---------------------------------------------------------------------------------------------------------------------
# knorm across the range: BLAS nrm2
# ---------------------------------------------------------------------------------------------------------------------
def exact_norm(x):
    """The norm of x's stored values: scaled by the power of two that brings max|x_i| into [0.5, 1), squared exactly,
    summed with fsum, one sqrt, scaled back (Inf when it overflows the float64 range)."""
    xd = x.astype(np.float64)
    if not np.all(np.isfinite(xd)):
        return np.nan if np.isnan(xd).any() else np.inf
    m = float(np.max(np.abs(xd))) if len(xd) else 0.0
    if m == 0:
        return 0.0
    e = math.frexp(m)[1]
    y = np.ldexp(xd, -e)
    with np.errstate(under="ignore"):
        p, err = two_product(y, y)
    with np.errstate(over="ignore"):
        return float(np.ldexp(math.sqrt(math.fsum(np.concatenate([p, err]).tolist())), e))


def check_norm(dev, dt, x, launches=None):
    n = len(x)
    b = dev.put(x)
    l0 = dev.launches()
    got = nrm2(dev, dt, n, b)
    used = dev.launches() - l0
    b.get()
    ref = exact_norm(x)
    with np.errstate(over="ignore"):
        ref_t = dt(ref)
    if np.isnan(ref):
        assert np.isnan(got)
    elif np.isinf(ref_t):
        assert got == np.inf
    else:
        assert abs(got - ref) <= 4 * float(np.spacing(ref_t)), (got, ref, float(np.spacing(ref_t)))
    blas = {np.float64: "dnrm2", np.float32: "snrm2"}[dt]
    from scipy.linalg import blas as sblas
    with np.errstate(all="ignore"):
        theirs = getattr(sblas, blas)(x) if n else 0.0
    assert np.isfinite(got) == np.isfinite(theirs), (got, theirs)
    if launches is not None:
        assert used == launches
    return got, used


RANGE_EXPS = {np.float64: [-1072, -1060, -1000, -600, -540, -538, -530, -511, -500, 0, 500, 511, 512, 520, 1000, 1020],
              np.float32: [-147, -140, -120, -100, -80, -76, -75, -70, -64, -63, -50, 0, 50, 63, 64, 66, 100, 124]}


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("shape", ["1", "257", "4S+1"])
def test_nrm2_across_the_range(dev, dt, shape):
    """x = 2^e u, with e from below the subnormal range to the overflow threshold: within 4 ulps of the exact norm,
    Inf exactly when the norm overflows dt, finite exactly when BLAS nrm2's is."""
    n = size(shape, RED_CTAS)
    rng = np.random.default_rng(40)
    u = rng.uniform(0.5, 2.0, n) * rng.choice([-1.0, 1.0], n)
    for e in RANGE_EXPS[dt]:
        with np.errstate(all="ignore"):
            x = np.ldexp(u, e).astype(dt)
        check_norm(dev, dt, x)


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("shape", ["1", "257", "4S+1"])
def test_nrm2_special_vectors(dev, dt, shape):
    n = size(shape, RED_CTAS)
    rng = np.random.default_rng(41)
    fi = np.finfo(dt)
    g = rng.standard_normal(n).astype(dt)
    check_norm(dev, dt, np.zeros(n, dt), launches=1)                                  # zero: no extra launch
    check_norm(dev, dt, (rng.integers(1, 64, n) * fi.smallest_subnormal).astype(dt), launches=2)   # all subnormal
    for at in {0, n // 2, n - 1}:
        x = g.copy()
        x[at] = dt(1.5) * dt(2.0 ** (fi.maxexp - 3))                                  # one huge entry among normal ones
        check_norm(dev, dt, x)
        x[at] = np.inf
        assert check_norm(dev, dt, x, launches=1)[0] == np.inf
        x[at] = -np.inf
        assert check_norm(dev, dt, x, launches=1)[0] == np.inf
        x[at] = np.nan
        assert math.isnan(check_norm(dev, dt, x, launches=1)[0])


@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_nrm2_in_the_normal_range_is_the_root_of_the_dot(dev, dt, shape):
    """Inside the range knorm is the one-pass sqrt(<x, x>): bit for bit, and in as many launches."""
    n = size(shape, RED_CTAS)
    x = np.random.default_rng(42).standard_normal(n).astype(dt)
    b = dev.put(x)
    l0 = dev.launches()
    d = dot(dev, dt, n, b, b)
    l1 = dev.launches()
    r = nrm2(dev, dt, n, b)
    assert r == float(np.sqrt(dt(d)))
    assert dev.launches() - l1 == l1 - l0 == 1


# ---------------------------------------------------------------------------------------------------------------------
# n = 2^31 - 1 in Float32
# ---------------------------------------------------------------------------------------------------------------------
def test_float32_at_int_max(dev):
    """The largest n the flat API takes, on torch buffers, checked on the device (never copied to the host): fill, scal
    and axpy bit for bit against torch's separately rounded mul and add, dot and knorm exact on data whose partial sums
    stay below 2^24, and the guard cells after the last element untouched."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 24 << 30:
        pytest.skip("needs about 24 GiB of free device memory")
    L, ctx, f32 = dev.L, dev.ctx, _lib.KRYLOV_FLOAT32
    n, chunk = 2 ** 31 - 1, 1 << 27
    nan_bits = int(GUARD_NAN[np.float32])
    X = torch.empty(LEAD + n + TRAIL, dtype=torch.float32, device="cuda")
    Y = torch.empty_like(X)
    try:
        for B in (X, Y):
            B.view(torch.int32)[:LEAD] = nan_bits
            B.view(torch.int32)[LEAD + n:] = nan_bits
        px, py = X.data_ptr() + 4 * LEAD, Y.data_ptr() + 4 * LEAD
        xv, yv = X[LEAD:LEAD + n], Y[LEAD:LEAD + n]

        def chunks():
            for k0 in range(0, n, chunk):
                yield k0, min(n, k0 + chunk)

        def pattern(k0, k1, mul, add):      # exactly representable, up to about +-977 with 19 significant bits
            k = torch.arange(k0, k1, device="cuda", dtype=torch.int64)
            return (((k * mul + add) % 1000003).to(torch.float32) - 500001.0) * 2.0 ** -9

        def guards_intact():
            for B in (X, Y):
                assert bool((B.view(torch.int32)[:LEAD] == nan_bits).all())
                assert bool((B.view(torch.int32)[LEAD + n:] == nan_bits).all())

        def kb(call):         # torch's stream and the context's stream do not wait for each other
            torch.cuda.synchronize()
            assert call() == 0
            assert L.kb200_sync(ctx) == 0

        kb(lambda: L.kb200_fill(ctx, f32, n, px, 1.5))
        assert all(bool((xv[a:b] == 1.5).all()) for a, b in chunks())
        guards_intact()

        s, a = 0.37, -1.25
        for k0, k1 in chunks():
            yv[k0:k1] = pattern(k0, k1, 7919, 13)
            xv[k0:k1] = pattern(k0, k1, 104729, 71)
        kb(lambda: L.kb200_scal(ctx, f32, n, s, py))
        for k0, k1 in chunks():
            exp = torch.mul(pattern(k0, k1, 7919, 13), torch.tensor(s, dtype=torch.float32))
            assert torch.equal(yv[k0:k1].view(torch.int32), exp.view(torch.int32)), k0
        kb(lambda: L.kb200_axpy(ctx, f32, n, a, px, py))
        for k0, k1 in chunks():
            sy = torch.mul(pattern(k0, k1, 7919, 13), torch.tensor(s, dtype=torch.float32))
            exp = torch.add(sy, torch.mul(pattern(k0, k1, 104729, 71), torch.tensor(a, dtype=torch.float32)))
            assert torch.equal(yv[k0:k1].view(torch.int32), exp.view(torch.int32)), k0
        guards_intact()

        # x: ones on every 251st element and on the last 2^20 (the tail every bound decides about), else zero;
        # y: +-1.  |partial sums| <= count(x) < 2^24, so the sums are exact.
        count = dotxy = 0
        for k0, k1 in chunks():
            k = torch.arange(k0, k1, device="cuda", dtype=torch.int64)
            xc = ((k % 251 == 0) | (k >= n - (1 << 20))).to(torch.float32)
            yc = (1 - 2 * ((k * 7919 >> 3) & 1)).to(torch.float32)
            xv[k0:k1], yv[k0:k1] = xc, yc
            count += int(xc.sum(dtype=torch.float64).item())
            dotxy += int((xc.double() * yc.double()).sum().item())
        assert count < 2 ** 24
        torch.cuda.synchronize()
        r = C.c_double()
        assert L.kb200_dot(ctx, f32, n, px, py, C.byref(r)) == 0
        assert r.value == dotxy
        assert L.kb200_dot(ctx, f32, n, px, px, C.byref(r)) == 0
        assert r.value == count
        assert L.kb200_nrm2(ctx, f32, n, px, C.byref(r)) == 0
        assert r.value == float(np.sqrt(np.float32(count)))
        guards_intact()
    finally:
        del X, Y
        torch.cuda.empty_cache()
