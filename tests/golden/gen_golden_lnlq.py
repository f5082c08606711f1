"""Regenerates tests/golden/oracle_lnlq.json from the CPU oracle's lnlq.

    python tests/golden/gen_golden_lnlq.py

The cases are the problems of the reference's test/test_lnlq.jl (real case, both values of transfer_to_craig;
restated in tests/test_oracle_lnlq.py, which also checks the reference's assertions on them).  These are outputs of
the oracle, not of Krylov.jl: they freeze its residual and error-bound histories, iteration counts, flags and status
strings.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "krylov.jl_b200")):
    sys.path.insert(0, p)

from oracle import lnlq_oracle as O  # noqa: E402

SIGMA = dict(atol=0.0, rtol=0.0, sigma=0.5)          # the σ variant of each case in test_lnlq.jl


def base_cases():
    """name -> (A, b, oracle kwargs) before transfer_to_craig is chosen."""
    out = {}
    A, b = O.zero_rhs()
    out["zero_rhs"] = (A, b, {})
    for name in ("under_consistent", "square_consistent", "over_consistent"):
        A, b = getattr(O, name)()
        out[name] = (A, b, dict(utolx=0.0, utoly=0.0))
        out[name + "_sigma"] = (A, b, SIGMA)
    A, b, lam = O.regularization()
    out["regularization"] = (A, b, dict(lambda_=lam, utolx=0.0, utoly=0.0))
    out["regularization_bounds"] = (A, b, dict(lambda_=lam, atol=0.0, rtol=0.0, utolx=1e-10, utoly=1e-10))
    A, b, D = O.saddle_point()
    out["saddle_point"] = (A, b, dict(N=1.0 / D))
    out["saddle_point_sigma"] = (A, b, dict(N=1.0 / D, atol=0.0, rtol=0.0, sigma=0.001))
    A, b, Mi, Ni = O.two_preconditioners()
    out["two_preconditioners"] = (A, b, dict(M=Mi, N=Ni))
    out["two_preconditioners_sigma"] = (A, b, dict(M=Mi, N=Ni, **SIGMA))
    A, b, M, N = O.sqd()
    out["sqd"] = (A, b, dict(M=1.0 / M, N=1.0 / N, sqd=True))
    out["sqd_sigma"] = (A, b, dict(M=1.0 / M, N=1.0 / N, sqd=True, **SIGMA))
    out["sqd_lambda4"] = (A, b, dict(M=1.0 / M, N=1.0 / N, lambda_=4.0))
    out["sqd_lambda4_sigma"] = (A, b, dict(M=1.0 / M, N=1.0 / N, lambda_=4.0, **SIGMA))
    for t in (False, True):
        A, b, c, D = O.small_sp(t)
        out[f"small_sp_{int(t)}"] = (A.T.tocsr(), c, dict(N=1.0 / D))
        A, b, c, M, N = O.small_sqd(t)
        out[f"small_sqd_{int(t)}"] = (A, b, dict(M=1.0 / M, N=1.0 / N, sqd=True))
    A, b = O.small_ln()
    out["small_ln"] = (A, b, {})
    A, b = O.over_consistent()
    out["tired"] = (A, b, dict(itmax=4, atol=0.0, rtol=0.0, utolx=0.0, utoly=0.0))
    return out


def cases():
    """name -> (A, b, oracle kwargs): every base case with transfer_to_craig = false (suffix _lq) and true (_cg)."""
    return {f"{name}_{tag}": (A, b, dict(kw, transfer_to_craig=t))
            for name, (A, b, kw) in base_cases().items() for tag, t in (("lq", False), ("cg", True))}


def run(A, b, **kw):
    return O.lnlq(A, b, history=True, **kw)


if __name__ == "__main__":
    out = {}
    for name, (A, b, kw) in cases().items():
        x, y, st = run(A, b, **kw)
        out[name] = dict(niter=st["niter"], solved=st["solved"], status=st["status"], error_with_bnd=st["error_with_bnd"],
                         x_head=[float(v) for v in x[:6]], y_head=[float(v) for v in y[:6]],
                         residuals=[float(v) for v in st["residuals"]],
                         error_bnd_x=[float(v) for v in st["error_bnd_x"]],
                         error_bnd_y=[float(v) for v in st["error_bnd_y"]])
    with open(os.path.join(HERE, "oracle_lnlq.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print(f"wrote {len(out)} cases")
