"""Synthetic benchmark matrices, generated directly as int32 / 0-based CSR.

These are closed-form equivalents of the reference's test generators
(test/get_div_grad.jl:8-25, test/test_utils.jl:153-169) that scale to n ~ 1e8
without forming Kronecker products; tests/test_problems.py checks them entry
by entry against the literal transcriptions in oracle/oracle.py at small N.
`xp` may be numpy or torch (torch lets the bench build the matrix on the GPU).
"""
from __future__ import annotations

import numpy as np


def _stencil_csr(n1, n2, n3, diag, lo, hi, dtype, k_lo=0, k_hi=None, xp=np, device=None):
    """7-point stencil on an n1 x n2 x n3 grid, unknown (i,j,k) -> i + n1*(j + n2*k).

    lo[d] / hi[d]: coefficient of the neighbour at -1 / +1 along axis d
    (d = 0 fastest).  Rows of planes k_lo <= k < k_hi only (row slab), with
    GLOBAL column indices.  Returns (rowptr, colind, values), columns ascending.
    """
    if k_hi is None:
        k_hi = n3
    is_t = xp is not np
    kw = dict(device=device) if is_t else {}
    i64 = xp.int64
    nloc = n1 * n2 * (k_hi - k_lo)
    rows = xp.arange(n1 * n2 * k_lo, n1 * n2 * k_hi, dtype=i64, **kw)
    i = rows % n1
    j = (rows // n1) % n2
    k = rows // (n1 * n2)
    strides = (1, n1, n1 * n2)
    # candidate slots in ascending column order: -s2, -s1, -s0, 0, +s0, +s1, +s2
    offs = [-strides[2], -strides[1], -strides[0], 0, strides[0], strides[1], strides[2]]
    vals = [lo[2], lo[1], lo[0], diag, hi[0], hi[1], hi[2]]
    masks = [k > 0, j > 0, i > 0, None, i < n1 - 1, j < n2 - 1, k < n3 - 1]
    if is_t:
        import torch
        mask = torch.ones((nloc, 7), dtype=torch.bool, **kw)
        for s, m in enumerate(masks):
            if m is not None:
                mask[:, s] = m
        cols = rows[:, None] + torch.tensor(offs, dtype=i64, **kw)[None, :]
        tdt = torch.float64 if np.dtype(dtype) == np.float64 else torch.float32
        v = torch.tensor(vals, dtype=tdt, **kw)[None, :].expand(nloc, 7)
        counts = mask.sum(dim=1)
        rowptr = torch.zeros(nloc + 1, dtype=i64, **kw)
        rowptr[1:] = torch.cumsum(counts, 0)
        return rowptr.to(torch.int32), cols[mask].to(torch.int32), v[mask].contiguous()
    mask = np.ones((nloc, 7), dtype=bool)
    for s, m in enumerate(masks):
        if m is not None:
            mask[:, s] = m
    cols = rows[:, None] + np.asarray(offs, dtype=np.int64)[None, :]
    v = np.broadcast_to(np.asarray(vals, dtype=dtype)[None, :], (nloc, 7))
    rowptr = np.zeros(nloc + 1, dtype=np.int64)
    np.cumsum(mask.sum(axis=1), out=rowptr[1:])
    return rowptr.astype(np.int32), cols[mask].astype(np.int32), np.ascontiguousarray(v[mask])


def div_grad_csr(n1, n2=None, n3=None, dtype=np.float64, k_lo=0, k_hi=None, xp=np, device=None):
    """get_div_grad(n1,n2,n3) = Div*Div' (test/get_div_grad.jl:8-19): diagonal 6, neighbours -1."""
    n2 = n1 if n2 is None else n2
    n3 = n1 if n3 is None else n3
    return _stencil_csr(n1, n2, n3, 6.0, (-1.0, -1.0, -1.0), (-1.0, -1.0, -1.0), dtype, k_lo, k_hi, xp, device)


def kron_unsymmetric_csr(n, dtype=np.float64, k_lo=0, k_hi=None, xp=np, device=None):
    """kron_unsymmetric(n) (test/test_utils.jl:160-169): with T = tridiag(-1, 3, -2),
    A = T(x)I(x)I + 2 I(x)T(x)I + I(x)I(x)T; the first Kronecker factor is the slowest index."""
    return _stencil_csr(n, n, n, 12.0, (-1.0, -2.0, -1.0), (-2.0, -4.0, -2.0), dtype, k_lo, k_hi, xp, device)


def random_csr(n, per_row=20, seed=1234, dtype=np.float32, shift=3.0):
    """BASELINE config 4: per row `per_row` iid uniform columns with U(-1,1) values
    (indices drawn first, then values, numpy default_rng(seed)), duplicates summed, +shift on the diagonal."""
    import scipy.sparse as sp
    rng = np.random.default_rng(seed)
    cols = rng.integers(0, n, size=(n, per_row), dtype=np.int64)
    vals = rng.uniform(-1.0, 1.0, size=(n, per_row)).astype(dtype)
    rows = np.repeat(np.arange(n, dtype=np.int64), per_row)
    A = sp.coo_matrix((vals.ravel(), (rows, cols.ravel())), shape=(n, n)).tocsr()   # sums duplicates
    A = (A + shift * sp.identity(n, dtype=dtype, format="csr")).tocsr()
    A.sort_indices()
    return A.indptr.astype(np.int32), A.indices.astype(np.int32), A.data.astype(dtype)


def csr_matvec_ones(rowptr, colind, values):
    """b = A * ones (row sums), as the reference builds b for kron_unsymmetric."""
    if isinstance(values, np.ndarray):
        return np.add.reduceat(values, rowptr[:-1].astype(np.int64)) if len(values) else np.zeros(len(rowptr) - 1, values.dtype)
    import torch
    n = rowptr.numel() - 1
    out = torch.zeros(n, dtype=values.dtype, device=values.device)
    rows = torch.repeat_interleave(torch.arange(n, device=values.device), (rowptr[1:] - rowptr[:-1]).long())
    out.index_add_(0, rows, values)
    return out


def div_csr(N, dtype=np.float64, xp=np, device=None):
    """Divergence D = G^T of the N x N x N grid, assembled in closed form (xp=torch with device="cuda": on the GPU):
    m = N^3 rows (the points), n = 3 N^2 (N-1) columns (the rows of grad_csr(N)), at most six nonzeros per row.  Row p
    holds, in ascending column order, +1 where p is the neighbour and -1 where p is the base point of a difference
    along x, then y, then z.  Equal to grad_csr(N).T entry by entry.  Returns (rowptr, colind, values) as int32 CSR."""
    is_t = xp is not np
    kw = dict(device=device) if is_t else {}
    i64 = xp.int64
    p = xp.arange(N ** 3, dtype=i64, **kw)
    i, j, k = p % N, (p // N) % N, p // (N * N)
    mx = N * N * (N - 1)                                # rows of Dx (= of Dy, of Dz)

    def rx(q):
        return (q // N) * (N - 1) + q % N

    def ry(q):
        return mx + (q // (N * N)) * (N * (N - 1)) + q % (N * N)

    def rz(q):
        return 2 * mx + q
    cols = [rx(p - 1), rx(p), ry(p - N), ry(p), rz(p - N * N), rz(p)]
    keep = [i > 0, i < N - 1, j > 0, j < N - 1, k > 0, k < N - 1]
    cols, keep = xp.stack(cols, 1), xp.stack(keep, 1)
    sign = xp.tile(xp.asarray([1.0, -1.0], dtype=xp.float64, **kw), (3,)) if not is_t else \
        xp.tensor([1.0, -1.0] * 3, dtype=xp.float64, **kw)
    vals = (sign.reshape(1, 6) + xp.zeros((N ** 3, 6), dtype=xp.float64, **kw))[keep]
    colind = cols[keep]
    counts = keep.sum(1)
    if is_t:
        import torch
        rowptr = torch.zeros(N ** 3 + 1, dtype=torch.int64, **kw)
        rowptr[1:] = torch.cumsum(counts, 0)
        tdt = torch.float64 if np.dtype(dtype) == np.float64 else torch.float32
        return rowptr.to(torch.int32), colind.to(torch.int32), vals.to(tdt)
    rowptr = np.concatenate([[0], np.cumsum(counts)])
    return rowptr.astype(np.int32), colind.astype(np.int32), vals.astype(dtype)


def grad_csr(N, dtype=np.float64, xp=np, device=None):
    """Forward-difference gradient G = [Dx; Dy; Dz] of an N x N x N grid (unknown (i,j,k) -> i + N*(j + N*k)), the
    rectangular operator of the least-squares benchmark: m = 3 N^2 (N-1) rows, n = N^3 columns, two nonzeros per row
    (-1 at the point, +1 at its neighbour along the axis), columns ascending.  Rows of Dx come first (point order,
    i < N-1), then Dy (j < N-1), then Dz (k < N-1).  Its null space is the constant vector.  Returns
    (rowptr, colind, values) as int32 / 0-based CSR."""
    is_t = xp is not np
    kw = dict(device=device) if is_t else {}
    i64 = xp.int64
    pts = xp.arange(N ** 3, dtype=i64, **kw)
    i, j, k = pts % N, (pts // N) % N, pts // (N * N)
    cols = []
    for stride, coord in ((1, i), (N, j), (N * N, k)):
        base = pts[coord < N - 1]
        cols.append(xp.stack([base, base + stride], 1).reshape(-1))
    colind = xp.cat(cols) if is_t else np.concatenate(cols)
    m = colind.shape[0] // 2
    rowptr = xp.arange(0, 2 * m + 1, 2, dtype=i64, **kw)
    if is_t:
        import torch
        tdt = torch.float64 if np.dtype(dtype) == np.float64 else torch.float32
        values = torch.tensor([-1.0, 1.0], dtype=tdt, **kw).repeat(m)
        return rowptr.to(torch.int32), colind.to(torch.int32), values
    values = np.tile(np.asarray([-1.0, 1.0], dtype=dtype), m)
    return rowptr.astype(np.int32), colind.astype(np.int32), values
