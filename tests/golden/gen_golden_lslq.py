"""Regenerates tests/golden/oracle_lslq.json from the CPU oracle's lslq.

    python tests/golden/gen_golden_lslq.py

The cases are the reference's known-answer problems of test/test_lslq.jl (restated in tests/test_oracle_lslq.py, which
also checks the reference's assertions on them).  Like oracle_lsq.json these are outputs of the oracle, not of
Krylov.jl: they freeze its residual, Aᴴ-residual and error-bound histories.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "krylov.jl_b200")):
    sys.path.insert(0, p)

from oracle import cgls_oracle as O  # noqa: E402
from oracle import lsq_oracle as L  # noqa: E402


def cases():
    """name -> (A, b, oracle kwargs): the problems of test/test_lslq.jl (real case) that need no LAPACK factorization."""
    out = {}
    for npower in range(1, 5):
        b, A, *_ = O.lsq_test(40, 40, 4, npower, 0)
        out[f"lstp{npower}"] = (A, b, {})
        out[f"lstp{npower}_lambda"] = (A, b, dict(lambda_=1.0e-3))
    out["lstp4_sigma"] = (A, b, dict(sigma=1.0))              # the bounds turn complex: error_with_bnd
    for t in (False, True):
        sfx = "_lsqr" if t else ""
        A, b, M, N = L.two_preconditioners()
        out["two_preconditioners" + sfx] = (A, b, dict(M=M, N=N, transfer_to_lsqr=t))
        A, b, lam = L.regularization()
        out["regularization" + sfx] = (A, b, dict(lambda_=lam, transfer_to_lsqr=t))
        A, b, D = L.saddle_point()
        out["saddle_point" + sfx] = (A, b, dict(M=1 / D, transfer_to_lsqr=t))
        A, b, M, N = L.sqd()
        out["sqd" + sfx] = (A, b, dict(M=1 / M, N=1 / N, sqd=True, transfer_to_lsqr=t))
        out["sqd_lambda" + sfx] = (A, b, dict(M=1 / M, N=1 / N, lambda_=4.0, transfer_to_lsqr=t))
    return out


KEYS = ("residuals", "Aresiduals", "err_lbnds", "err_ubnds_lq", "err_ubnds_cg")

if __name__ == "__main__":
    out = {}
    for name, (A, b, kw) in cases().items():
        x, st = O.lslq(A, b, **kw)
        out[f"lslq/{name}"] = dict(niter=st["niter"], solved=st["solved"], inconsistent=st["inconsistent"], status=st["status"],
                                   error_with_bnd=st["error_with_bnd"], x_head=[float(v) for v in x[:6]],
                                   **{k: [float(v) for v in st[k]] for k in KEYS})
    with open(os.path.join(HERE, "oracle_lslq.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print(f"wrote {len(out)} cases")
