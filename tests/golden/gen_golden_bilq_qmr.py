"""Regenerates tests/golden/oracle_bilq_qmr.json from the CPU oracle's bilq and qmr.

    python tests/golden/gen_golden_bilq_qmr.py

The cases are the reference's known-answer problems of test/test_bilq.jl and test/test_qmr.jl (real case; restated in
tests/test_oracle_bilq_qmr.py, which also checks the reference's assertions on them).  These are outputs of the oracle,
not of Krylov.jl: they freeze its per-iteration residual histories, iteration counts and status strings.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "krylov.jl_b200")):
    sys.path.insert(0, p)

from oracle import biorth_oracle as O  # noqa: E402


def cases():
    """name -> (A, b, oracle kwargs shared by bilq and qmr): the problems of test/test_bilq.jl / test/test_qmr.jl."""
    out = {}
    for name in ("symmetric_definite", "symmetric_indefinite", "nonsymmetric_definite", "nonsymmetric_indefinite",
                 "sparse_laplacian", "zero_rhs", "polar_poisson"):
        A, b = getattr(O, name)()
        out[name] = (A, b, {})
    A, b, c = O.unsymmetric_breakdown()
    out["unsymmetric_breakdown"] = (A, b, dict(c=c))
    A, b, M = O.square_preconditioned()
    out["left_preconditioned"] = (A, b, dict(M=M))
    out["right_preconditioned"] = (A, b, dict(N=M))
    A, b, M, N = O.two_preconditioners()
    out["two_preconditioners"] = (A, b, dict(M=M, N=N))
    A, b, c = O.bc_breakdown()
    out["bc_breakdown"] = (A, b, dict(c=c))
    return out


if __name__ == "__main__":
    out = {}
    for solver in ("bilq", "qmr"):
        for name, (A, b, kw) in cases().items():
            x, st = getattr(O, solver)(A, b, history=True, **kw)
            out[f"{solver}/{name}"] = dict(niter=st["niter"], solved=st["solved"], status=st["status"],
                                           x_head=[float(v) for v in x[:6]], residuals=[float(v) for v in st["residuals"]])
    with open(os.path.join(HERE, "oracle_bilq_qmr.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print(f"wrote {len(out)} cases")
