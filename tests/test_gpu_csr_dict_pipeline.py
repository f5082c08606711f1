"""GPU: the persistent CG kernel on the constant-coefficient encoding loads each thread's next row while it sums the
current one.  These shapes reach the edges of that pipeline, and the iterates must still match the CSR path bit for
bit: a stencil whose +plane offset spans more than one sweep of the grid (one sweep = grid x 256 rows, about 101 k on
an H100), with n not a multiple of 256, so the last tile is partial and the last load ahead would fall past n."""
import numpy as np
import pytest

from test_gpu_csr_dict import _cg_outputs, stencil

pytestmark = pytest.mark.gpu

CASES = {
    # plane 330 * 330 = 108 900 rows; n = 435 600 = 1701 * 256 + 144
    "plane_beyond_sweep": dict(dims=(330, 330, 4), kw=dict(itmax=40, atol=0.0, rtol=0.0)),
    "plane_beyond_sweep_jacobi": dict(dims=(330, 330, 4), kw=dict(itmax=40, atol=0.0, rtol=0.0), M=True),
    "plane_beyond_sweep_f32": dict(dims=(330, 330, 4), kw=dict(itmax=40, atol=0.0, rtol=0.0), dtype=np.float32),
    # a single row per thread at most: nothing to load ahead
    "fewer_rows_than_threads": dict(dims=(13, 7, 3), kw=dict(itmax=30, atol=0.0, rtol=0.0)),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_pipelined_dict_cg_bit_identical_to_csr(case, monkeypatch):
    c = CASES[case]
    dt = c.get("dtype", np.float64)
    A = stencil(c["dims"], dt)
    n = A.shape[0]
    b = np.random.default_rng(5).standard_normal(n).astype(dt)
    kw = dict(c["kw"])
    if c.get("M"):
        kw["M"] = (1.0 / np.linspace(5.0, 7.0, n)).astype(dt)
    on = _cg_outputs(A, b, True, monkeypatch, **kw)
    off = _cg_outputs(A, b, False, monkeypatch, **kw)
    assert on["niter"] > 0
    assert on == off
