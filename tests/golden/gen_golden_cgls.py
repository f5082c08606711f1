"""Regenerates tests/golden/oracle_cgls.json from the CPU oracle's cgls / crls.

    python tests/golden/gen_golden_cgls.py

The cases are the reference's known-answer problems of test/test_cgls.jl and test/test_crls.jl (restated in
tests/test_oracle_cgls.py, which also checks the reference's assertions on them).  Like oracle_lsq.json these are
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
import scipy.sparse as sp  # noqa: E402

from oracle import cgls_oracle as O  # noqa: E402
from oracle import lsq_oracle as L  # noqa: E402


def psd_problem():
    """The positive semi-definite case of test/test_crls.jl with fixed orthogonal factors: A = U S V (10 x 7, singular
    values 0, 1e-6, 1, 4, 20, 15, 1e5), b = A' \\ V[:, 1] (least-norm), radius 10."""
    rng = np.random.default_rng(11)
    U, _ = np.linalg.qr(rng.random((10, 10)))
    V, _ = np.linalg.qr(rng.random((7, 7)))
    S = np.vstack([np.diag([0, 1.0e-6, 1, 4, 20, 15, 1.0e5]), np.zeros((3, 7))])
    A = U @ S @ V
    b = np.linalg.lstsq(A.T, V[:, 0], rcond=None)[0]
    return sp.csr_matrix(A), b


def cases():
    """name -> (A, b, oracle kwargs): the problems of test/test_cgls.jl / test_crls.jl (real case)."""
    out = {}
    for npower in range(1, 5):
        b, A, *_ = O.lsq_test(40, 40, 4, npower, 0)
        out[f"lstp{npower}"] = (A, b, {})
        out[f"lstp{npower}_lambda"] = (A, b, dict(lambda_=1.0e-3))
    A, b, D = L.saddle_point()
    out["saddle_point"] = (A, b, dict(M=1 / D))
    out["trust_free"] = (A, b, {})
    A, b, lam = O.regularization()
    out["regularization"] = (A, b, dict(lambda_=lam))
    return out


def trust_radius(solver):
    A, b, _ = cases()["trust_free"]
    x, _ = getattr(O, solver)(A, b)
    return 0.75 * np.linalg.norm(x)


if __name__ == "__main__":
    out = {}
    for solver in ("cgls", "crls"):
        cs = cases()
        cs["trust_region"] = (cs["trust_free"][0], cs["trust_free"][1], dict(radius=trust_radius(solver)))
        if solver == "crls":                        # (psd_problem depends on LAPACK's QR: not frozen)
            A, b, _ = cs["lstp1"]                   # atol >= 1 makes the zero-curvature test hold at iteration 1
            cs["zero_curvature"] = (A, b, dict(radius=1.0e3, atol=1.0, rtol=0.0))
        for name, (A, b, kw) in cs.items():
            x, st = getattr(O, solver)(A, b, **kw)
            out[f"{solver}/{name}"] = dict(niter=st["niter"], solved=st["solved"], inconsistent=st["inconsistent"],
                                           status=st["status"], residuals=[float(v) for v in st["residuals"]],
                                           Aresiduals=[float(v) for v in st["Aresiduals"]], x_head=[float(v) for v in x[:6]])
    with open(os.path.join(HERE, "oracle_cgls.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print(f"wrote {len(out)} cases")
