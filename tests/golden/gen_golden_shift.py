"""Regenerates tests/golden/oracle_shift.json: frozen residual histories, iteration counts and flags of the CPU
restatement of cg_lanczos_shift! and cgls_lanczos_shift! (oracle/shift_oracle.py) on fixed problems.
tests/test_oracle_shift.py checks that the oracle still reproduces them.  Run from the repository root:
    python tests/golden/gen_golden_shift.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import oracle as O  # noqa: E402
from oracle import shift_oracle as S  # noqa: E402
from oracle.lsq_oracle import lsq_test  # noqa: E402


def cases():
    A, b = O.symmetric_definite()
    yield "cg_symdef", S.cg_lanczos_shift, A, b, [1.0, 2.0, 3.0, 4.0, 5.0, 6.0], {}
    yield "cg_negcurv", S.cg_lanczos_shift, A, b, [-4.0, -3.0, 2.0], dict(check_curvature=True, itmax=10)
    Ad = O.get_div_grad(8, 8, 8)
    yield "cg_divgrad8", S.cg_lanczos_shift, Ad, [1.0] * Ad.shape[0], [0.5, 5.0, 50.0], {}
    Ap, bp, Mp = O.square_preconditioned()
    yield "cg_precond", S.cg_lanczos_shift, Ap, bp, [1.0, 2.0, 3.0], dict(M=Mp)
    b2, A2 = lsq_test(40, 40, 4, 2, 0)[:2]
    yield "cgls_lsq40", S.cgls_lanczos_shift, A2, b2, [1.0, 2.0, 3.0, 4.0, 5.0, 6.0], {}


def main():
    out = {}
    for name, f, A, b, shifts, kw in cases():
        _, st = f(A, b, shifts, **kw)
        out[name] = dict(niter=st["niter"], status=st["status"], indefinite=st["indefinite"],
                         residuals=[r.tolist() for r in st["residuals"]])
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "oracle_shift.json"), "w") as fh:
        json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
