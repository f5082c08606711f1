"""CPU: the oracle's dot-product modes.  Mode 2 sums in the order of the device's reductions at one CTA of 256 threads
(krylov_oracle_impl.h: kdot), which is what lets tests/test_gpu_exact_small.py hold the GPU to the oracle bit for bit;
it must equal a NumPy restatement of that fold exactly, refuse n > 256 with NaN, and leave modes 0 and 1 as they were."""
import numpy as np
import pytest

from oracle import oracle as O

SIZES = sorted(set(range(1, 257, 7)) | {1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 224, 255, 256})


def fold_in_halves(v):
    """v[l] += v[l + s] for s = 16, 8, 4, 2, 1 along the last axis of 32 lanes: lane 0 of warp_sum's xor butterfly."""
    v = v.copy()
    s = 16
    while s:
        v[..., :s] = v[..., :s] + v[..., s:2 * s]
        s >>= 1
    return v[..., 0]


def device_tree(x, y, dt):
    """Thread i holds 0 + x[i] y[i] (0 past n); 8 warps of 32 fold in halves, then the 8 warp sums padded to 32."""
    lane = np.zeros(256, dt)
    lane[:len(x)] = dt(0) + x.astype(dt) * y.astype(dt)
    warps = np.zeros(32, dt)
    warps[:8] = fold_in_halves(lane.reshape(8, 32))
    return fold_in_halves(warps)


def operands(n, dt, seed):
    """Terms of mixed magnitude (2^-20 .. 2^20), with a run of exactly cancelling pairs: sums whose rounding depends
    on the order they are added in."""
    g = np.random.default_rng(seed)
    x = g.standard_normal(n) * np.exp2(g.integers(-20, 21, n))
    y = g.standard_normal(n) * np.exp2(g.integers(-20, 21, n))
    for i in range(n // 3, 2 * n // 3 - 1, 2):
        x[i], y[i] = x[i + 1], -y[i + 1]
    return x.astype(dt), y.astype(dt)


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_mode_2_is_the_device_fold(dt):
    differs = 0
    for n in SIZES:
        for seed in range(3):
            x, y = operands(n, dt, seed)
            with O.dot_mode(2):
                got = dt(O.dot(x, y, dtype=dt))
                norm = dt(O.dot(x, x, dtype=dt))
            want = device_tree(x, y, dt)
            assert got.tobytes() == want.tobytes(), (n, seed, got, want)
            assert norm.tobytes() == device_tree(x, x, dt).tobytes(), (n, seed)
            differs += got != dt(O.dot(x, y, dtype=dt))
    assert differs > len(SIZES), differs        # the inputs make the order visible: mode 2 is not mode 0


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_mode_2_refuses_more_than_one_cta(dt):
    for n in (257, 300, 1000):
        x = np.ones(n, dt)
        with O.dot_mode(2):
            assert np.isnan(O.dot(x, x, dtype=dt)), n
    assert O.dot(np.ones(257, dt), np.ones(257, dt), dtype=dt) == 257.0         # the context manager restored mode 0


@pytest.mark.parametrize("dt", [np.float64, np.float32])
def test_modes_0_and_1_are_unchanged(dt):
    """Mode 0: the sequential sum in the working precision; mode 1: the same terms accumulated in double, rounded once."""
    for n in SIZES + [257, 1000]:
        x, y = operands(n, dt, 7)
        seq = dt(0)
        for p in x * y:
            seq = dt(seq + p)
        acc = 0.0
        for a, b in zip(x.astype(np.float64), y.astype(np.float64)):
            acc = acc + a * b
        assert dt(O.dot(x, y, dtype=dt)).tobytes() == seq.tobytes(), n
        with O.dot_mode(1):
            assert dt(O.dot(x, y, dtype=dt)).tobytes() == dt(acc).tobytes(), n
