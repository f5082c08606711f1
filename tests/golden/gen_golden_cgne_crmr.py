"""Regenerates tests/golden/oracle_cgne_crmr.json from the CPU oracle's cgne and crmr.

    python tests/golden/gen_golden_cgne_crmr.py

The cases are the problems of the reference's test/test_cgne.jl and test/test_crmr.jl (real case; restated in
tests/test_oracle_cgne_crmr.py, which also checks the reference's assertions on them), each run by both solvers.
These are outputs of the oracle, not of Krylov.jl: they freeze its residual (and, for CRMR, ‖Aᵀr‖) histories,
iteration counts, flags and status strings.
"""
import json
import os
import sys

import numpy as np
import scipy.sparse as sp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "krylov.jl_b200")):
    sys.path.insert(0, p)

from oracle import cgne_oracle as O  # noqa: E402


def mass_transfer():
    """The under-determined preconditioned problem of test_cgne.jl / test_crmr.jl: the least-norm force that moves a
    unit mass a unit distance with zero final velocity, N = Diagonal(1 ./ diag(A Aᵀ))."""
    A = 0.5 * np.array([[19.0, 17.0, 15.0, 13.0, 11.0, 9.0, 7.0, 5.0, 3.0, 1.0], [2.0] * 10])
    return sp.csr_matrix(A), np.array([1.0, 0.0]), 1.0 / np.diag(A @ A.T)


def base_cases():
    """name -> (A, b, oracle kwargs), shared by both solvers."""
    out = {}
    for name in ("under_consistent", "under_inconsistent", "square_consistent", "square_inconsistent",
                 "over_consistent", "over_inconsistent"):
        A, b = getattr(O, name)()
        out[name] = (A, b, {})
    A, b = O.over_inconsistent()
    out["regularization"] = (A, b, dict(lambda_=1e-3))
    A, b = O.zero_rhs()
    out["zero_rhs"] = (A, b, dict(lambda_=1e-3))
    A, b, N = O.square_preconditioned()
    out["square_preconditioned"] = (A, b, dict(N=N))
    A, b, N = mass_transfer()
    out["mass_transfer"] = (A, b, dict(N=N))
    for t in (False, True):
        A, b, c, D = O.small_sp(t)
        out[f"small_sp_{int(t)}"] = (A, b, dict(N=1.0 / D, lambda_=1.0))
    A, b = O.over_consistent()
    out["tired"] = (A, b, dict(itmax=1, atol=0.0, rtol=0.0))
    return out


def cases():
    """name -> (solver, A, b, oracle kwargs): every base case for cgne (prefix cgne_) and crmr (prefix crmr_)."""
    return {f"{solver}_{name}": (solver, A, b, kw) for solver in ("cgne", "crmr") for name, (A, b, kw) in base_cases().items()}


def run(solver, A, b, **kw):
    return getattr(O, solver)(A, b, history=True, **kw)


if __name__ == "__main__":
    out = {}
    for name, (solver, A, b, kw) in cases().items():
        x, st = run(solver, A, b, **kw)
        out[name] = dict(niter=st["niter"], solved=st["solved"], inconsistent=st["inconsistent"], status=st["status"],
                         x_head=[float(v) for v in x[:6]], residuals=[float(v) for v in st["residuals"]],
                         Aresiduals=[float(v) for v in st.get("Aresiduals", [])])
    with open(os.path.join(HERE, "oracle_cgne_crmr.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print(f"wrote {len(out)} cases")
