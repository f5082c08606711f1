"""Regenerates tests/golden/oracle_lsq.json from the CPU oracle's lsqr / lsmr.

    python tests/golden/gen_golden_lsq.py

The cases are the reference's known-answer problems of test/test_lsqr.jl and test/test_lsmr.jl (restated in
tests/test_oracle_lsq.py, which also checks the reference's assertions on them).  Like oracle_histories.json these are
outputs of the oracle, not of Krylov.jl: they freeze its residual and Aᴴ-residual histories.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "krylov.jl_b200")):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402

from oracle import lsq_oracle as O  # noqa: E402


def cases():
    """name -> (A, b, oracle kwargs): the problems of test/test_lsqr.jl / test_lsmr.jl (real case)."""
    out = {}
    for npower in range(1, 5):
        b, A, *_ = O.lsq_test(40, 40, 4, npower, 0)
        out[f"lstp{npower}"] = (A, b, {})
        out[f"lstp{npower}_lambda"] = (A, b, dict(lambda_=1.0e-3))
    import scipy.sparse as sp
    At = sp.csr_matrix(np.array([[i / j - j / i for j in range(1, 7)] for i in range(1, 11)]))
    bt = At @ np.ones(6)
    out["trust_free"] = (At, bt, {})
    A, b, M, N = O.two_preconditioners()
    out["two_preconditioners"] = (A, b, dict(M=M, N=N))
    A, b, lam = O.regularization()
    out["regularization"] = (A, b, dict(lambda_=lam))
    A, b, D = O.saddle_point()
    out["saddle_point"] = (A, b, dict(M=1 / D))
    A, b, M, N = O.sqd()
    out["sqd"] = (A, b, dict(M=1 / M, N=1 / N, sqd=True))
    out["sqd_lambda"] = (A, b, dict(M=1 / M, N=1 / N, lambda_=4.0))
    return out


def trust_radius(solver):
    A, b, _ = cases()["trust_free"]
    x, _ = getattr(O, solver)(A, b)
    return 0.75 * np.linalg.norm(x)


if __name__ == "__main__":
    out = {}
    for solver in ("lsqr", "lsmr"):
        cs = cases()
        cs["trust_region"] = (cs["trust_free"][0], cs["trust_free"][1], dict(radius=trust_radius(solver)))
        for name, (A, b, kw) in cs.items():
            x, st = getattr(O, solver)(A, b, **kw)
            out[f"{solver}/{name}"] = dict(niter=st["niter"], solved=st["solved"], inconsistent=st["inconsistent"],
                                           status=st["status"], residuals=[float(v) for v in st["residuals"]],
                                           Aresiduals=[float(v) for v in st["Aresiduals"]], x_head=[float(v) for v in x[:6]])
    with open(os.path.join(HERE, "oracle_lsq.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print(f"wrote {len(out)} cases")
