"""Regenerates tests/golden/oracle_adjoint.json from the CPU oracle's bilqr and trilqr.

    python tests/golden/gen_golden_adjoint.py

The cases are the reference's known-answer problems of test/test_bilqr.jl and test/test_trilqr.jl (real case; restated
in tests/test_oracle_adjoint.py, which also checks the reference's assertions on them), plus two TriLQR cases whose
halves converge far apart.  These are outputs of the oracle, not of Krylov.jl: they freeze its per-iteration primal and
dual residual histories, iteration counts, solved flags and status strings.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "krylov.jl_b200")):
    sys.path.insert(0, p)

from oracle import adjoint_oracle as O  # noqa: E402


def cases():
    """name -> (solver, A, b, c, oracle kwargs)."""
    out = {}
    for name in ("square_adjoint", "adjoint_ode", "adjoint_pde"):
        out["bilqr/" + name] = ("bilqr",) + tuple(getattr(O, name)()) + ({},)
    A, b, c = O.bc_breakdown()
    out["bilqr/bc_breakdown"] = ("bilqr", A, b, c, {})
    for name in ("underdetermined_adjoint", "square_adjoint", "overdetermined_adjoint", "adjoint_ode", "adjoint_pde",
                 "rectangular_adjoint"):
        out["trilqr/" + name] = ("trilqr",) + tuple(getattr(O, name)()) + ({},)
    # one half converges long before the other: a small right-hand side against an absolute tolerance
    A, b, c = O.adjoint_pde()
    nb, nc = float(np.linalg.norm(b)), float(np.linalg.norm(c))
    out["bilqr/primal_first"] = ("bilqr", A, (1e-4 * nc / nb) * b, c, dict(atol=1e-8 * nc, rtol=0.0))
    out["bilqr/dual_first"] = ("bilqr", A, b, (1e-4 * nb / nc) * c, dict(atol=1e-8 * nb, rtol=0.0))
    A, b, c = O.adjoint_ode()
    out["trilqr/primal_first"] = ("trilqr", A, 1e-6 * b, c, dict(atol=1e-9, rtol=0.0))
    out["trilqr/dual_first"] = ("trilqr", A, b, 1e-6 * c, dict(atol=1e-9, rtol=0.0))
    return out


def run(solver, A, b, c, **kw):
    return getattr(O, solver)(A, b, c, history=True, **kw)


if __name__ == "__main__":
    out = {}
    for name, (solver, A, b, c, kw) in cases().items():
        x, y, st = run(solver, A, b, c, **kw)
        out[name] = dict(niter=st["niter"], solved_primal=st["solved_primal"], solved_dual=st["solved_dual"],
                         status=st["status"], x_head=[float(v) for v in x[:6]], y_head=[float(v) for v in y[:6]],
                         residuals_primal=[float(v) for v in st["residuals_primal"]],
                         residuals_dual=[float(v) for v in st["residuals_dual"]])
    with open(os.path.join(HERE, "oracle_adjoint.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print(f"wrote {len(out)} cases")
