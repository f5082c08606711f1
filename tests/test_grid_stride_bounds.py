"""CPU: the grid-stride loops of blas1.cu (ew_kernel, dot_kernel, cg_prologue_kernel) touch exactly the indices [0, n)
for every n up to INT_MAX at the grids they are launched with.

Each loop is restated in 32-bit arithmetic that wraps the way the hardware's does, and run for every thread of the
grid.  The loops used to count in int: for n within 4 strides of INT_MAX, i + 3 * stride and the steps passed INT_MAX,
wrapped negative and compared below n (and signed overflow is undefined behaviour besides).  The model shows that shape
failing and the unsigned one, which the source now uses, passing.  The unsigned bound is max(n, 0): a negative n,
converted as it stands, would be near 2^32, and the reductions still launch one CTA for n <= 0."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT_MAX = 2 ** 31 - 1
BLOCK, MAX_PARTIALS = 256, 2048


def wrap(v, signed):
    v = v % 2 ** 32
    return np.where(v >= 2 ** 31, v - 2 ** 32, v) if signed else v


def grid_of(n, sms, ctas):
    """stream_grid(n, 4, ctas) (common.cuh)."""
    need = -(-n // (BLOCK * 4))
    return max(1, min(need, sms * ctas, MAX_PARTIALS))


def touched(n, stride, unrolled, signed, clamp=True):
    """Every index the loop reads or writes, over all threads, from the first trip that could go wrong on; None as soon
    as one lies outside [0, n).

    Returns (first index the model starts from, touched indices).  Trips before that are skipped in closed form:
    their indices are below n - stride and cannot wrap in either arithmetic.  The unsigned loops compare with
    un = max(n, 0) (clamp) or, without the clamp, with n converted to unsigned."""
    length = max(n, 0)
    if not signed:
        n = length if clamp else n % 2 ** 32
    i0 = np.arange(stride, dtype=np.int64)
    step = 4 * stride if unrolled else stride
    skip = max(0, (length - 2 * step) // step)
    i = i0 + skip * step
    out = []
    if unrolled:     # for (; i + 3 * stride < n; i += 4 * stride) { i, i + stride, i + 2 stride, i + 3 stride }
        live = np.ones(stride, bool)
        while live.any():
            go = live & (wrap(i + 3 * stride, signed) < n)
            for q in range(4):
                out.append(wrap(i[go] + q * stride, signed))
                if out[-1].size and (out[-1].min() < 0 or out[-1].max() >= length):
                    return None
            i = np.where(go, wrap(i + 4 * stride, signed), i)
            live = go
    live = wrap(i, signed) < n  # for (; i < n; i += stride) { i }
    while live.any():
        out.append(wrap(i[live], signed))
        if out[-1].min() < 0 or out[-1].max() >= length:
            return None
        i = np.where(live, wrap(i + stride, signed), i)
        live = live & (wrap(i, signed) < n)
    return skip * step, np.concatenate(out) if out else np.empty(0, np.int64)


def covers_exactly(n, stride, unrolled, signed, clamp=True):
    seen = touched(n, stride, unrolled, signed, clamp)
    if seen is None:
        return False
    lo, idx = seen
    return np.array_equal(np.sort(idx), np.arange(lo, max(n, 0)))


LOOPS = [("ew_kernel", 8, True), ("dot_kernel", 4, True), ("cg_prologue_kernel", 4, True)]
INT_LOOPS = [("ew_kernel", 8, True), ("dot_kernel", 4, True), ("cg_prologue_kernel", 4, False)]   # the old int shapes
SMS = [132, 114, 256]          # H100 SXM, H100 PCIe, and a count at which the grid hits kMaxPartials


def sizes(sms, ctas):
    S = min(sms * ctas, MAX_PARTIALS) * BLOCK
    return sorted({INT_MAX, INT_MAX - 1, INT_MAX - S + 1, INT_MAX - 3 * S, INT_MAX - 4 * S + 1, INT_MAX - 4 * S,
                   INT_MAX - 5 * S - 7, 2 ** 30 + 3, 4 * S + 1, 1000, 1, 0, -1, -4 * S - 1, -INT_MAX - 1})


@pytest.mark.parametrize("sms", SMS)
@pytest.mark.parametrize("kernel,ctas,unrolled", LOOPS)
def test_unsigned_loops_touch_exactly_0_to_n(kernel, ctas, unrolled, sms):
    for n in sizes(sms, ctas):
        stride = grid_of(n, sms, ctas) * BLOCK
        assert covers_exactly(n, stride, unrolled, signed=False), (kernel, n, stride)


@pytest.mark.parametrize("kernel,ctas,unrolled", INT_LOOPS)
def test_int_loops_leave_the_buffer_near_int_max(kernel, ctas, unrolled):
    """The model catches the old shape: in int, some thread reaches an index outside [0, n) at n = INT_MAX."""
    stride = grid_of(INT_MAX, 132, ctas) * BLOCK
    assert not covers_exactly(INT_MAX, stride, unrolled, signed=True)
    assert covers_exactly(INT_MAX - 5 * stride, stride, unrolled, signed=True)   # ... and is right away from the edge
    assert covers_exactly(-1, BLOCK, unrolled, signed=True)                      # a negative n touched nothing


@pytest.mark.parametrize("kernel,ctas,unrolled", LOOPS)
def test_negative_n_needs_the_clamp(kernel, ctas, unrolled):
    """A reduction launches one CTA for n <= 0.  With n converted to unsigned as it stands, n = -1 would be 2^32 - 1
    and the loop would run off the buffer; clamped to 0 it touches nothing."""
    for n in (-1, -(2 ** 31)):
        assert not covers_exactly(n, BLOCK, unrolled, signed=False, clamp=False)
        assert covers_exactly(n, BLOCK, unrolled, signed=False)


def test_source_uses_the_modelled_loops():
    src = open(os.path.join(ROOT, "krylov.jl_b200", "csrc", "blas1.cu")).read()
    src = re.sub(r"\s+", " ", src)
    assert src.count("const unsigned stride = gridDim.x * blockDim.x, un = n > 0 ? n : 0;") == 3
    assert src.count("unsigned i = blockIdx.x * blockDim.x + threadIdx.x;") == 3
    assert src.count("for (; i + 3 * stride < un; i += 4 * stride)") == 3
    assert src.count("for (; i < un; i += stride)") == 3
