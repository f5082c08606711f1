"""Regenerates tests/golden/oracle_leastnorm.json from the CPU oracle's craig and craigmr.

    python tests/golden/gen_golden_leastnorm.py

The cases are the problems of the reference's test/test_craig.jl and test/test_craigmr.jl (real case; restated in
tests/test_oracle_leastnorm.py, which also checks the reference's assertions on them).  These are outputs of the oracle,
not of Krylov.jl: they freeze its per-iteration histories, iteration counts, flags and status strings.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "krylov.jl_b200")):
    sys.path.insert(0, p)

from oracle import leastnorm_oracle as O  # noqa: E402


def cases():
    """name -> (A, b, oracle kwargs); every case runs with both solvers."""
    out = {}
    for name in ("under_consistent", "under_inconsistent", "square_consistent", "square_inconsistent", "over_consistent",
                 "over_inconsistent", "small_ln", "zero_rhs"):
        A, b = getattr(O, name)()
        out[name] = (A, b, dict(lambda_=1.0e-3) if name == "zero_rhs" else {})
    A, b, lam = O.regularization()
    out["regularization"] = (A, b, dict(lambda_=lam))
    A, b, D = O.saddle_point()
    out["saddle_point"] = (A, b, dict(N=1.0 / D))
    A, b, Mi, Ni = O.two_preconditioners()
    out["two_preconditioners"] = (A, b, dict(M=Mi, N=Ni))
    A, b, M, N = O.sqd()
    out["sqd"] = (A, b, dict(M=1.0 / M, N=1.0 / N, sqd=True))
    out["sqd_lambda4"] = (A, b, dict(M=1.0 / M, N=1.0 / N, lambda_=4.0))
    for t in (False, True):
        A, b, c, D = O.small_sp(t)
        out[f"small_sp_{int(t)}"] = (A.T.tocsr(), c, dict(N=1.0 / D))
        A, b, c, M, N = O.small_sqd(t)
        out[f"small_sqd_{int(t)}"] = (A, b, dict(M=1.0 / M, N=1.0 / N, sqd=True))
    return out


def run(solver, A, b, **kw):
    return getattr(O, solver)(A, b, history=True, **kw)


if __name__ == "__main__":
    out = {}
    for name, (A, b, kw) in cases().items():
        for solver in ("craig", "craigmr"):
            x, y, st = run(solver, A, b, **kw)
            out[f"{solver}/{name}"] = dict(niter=st["niter"], solved=st["solved"], inconsistent=st["inconsistent"],
                                           status=st["status"], x_head=[float(v) for v in x[:6]],
                                           y_head=[float(v) for v in y[:6]],
                                           residuals=[float(v) for v in st["residuals"]],
                                           Aresiduals=[float(v) for v in st.get("Aresiduals", [])])
    with open(os.path.join(HERE, "oracle_leastnorm.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print(f"wrote {len(out)} cases")
