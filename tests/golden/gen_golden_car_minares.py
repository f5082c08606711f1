"""Regenerates tests/golden/oracle_car_minares.json from the CPU oracle's car and minares.

    python tests/golden/gen_golden_car_minares.py

The cases are the reference's known-answer problems of test/test_car.jl and test/test_minares.jl (real case; restated in
tests/test_oracle_car_minares.py, which also checks the reference's assertions on them).  These are outputs of the
oracle, not of Krylov.jl: they freeze its per-iteration histories (residuals and Aresiduals), iteration counts and
status strings.
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "krylov.jl_b200")):
    sys.path.insert(0, p)

from oracle import ares_oracle as O  # noqa: E402


def cases():
    """solver -> name -> (A, b, oracle kwargs): the problems of test/test_car.jl and test/test_minares.jl."""
    car, minares = {}, {}
    for name in ("symmetric_definite", "sparse_laplacian", "zero_rhs", "singular_consistent", "cartesian_poisson"):
        A, b = getattr(O, name)()
        car[name] = (A, b, {})
    A, b, M = O.square_preconditioned()
    car["square_preconditioned"] = (A, b, dict(M=M))
    for name in ("symmetric_definite", "symmetric_indefinite", "sparse_laplacian", "almost_singular", "zero_rhs",
                 "square_inconsistent", "symmetric_inconsistent"):
        A, b = getattr(O, name)()
        minares[name] = (A, b, {})
    A, b = O.symmetric_indefinite()
    minares["shifted"] = (A, b, dict(lambda_=2.0))
    return {"car": car, "minares": minares}


if __name__ == "__main__":
    out = {}
    for solver, cs in cases().items():
        for name, (A, b, kw) in cs.items():
            x, st = getattr(O, solver)(A, b, history=True, **kw)
            out[f"{solver}/{name}"] = dict(niter=st["niter"], solved=st["solved"], status=st["status"],
                                           x_head=[float(v) for v in x[:6]], residuals=[float(v) for v in st["residuals"]],
                                           Aresiduals=[float(v) for v in st["Aresiduals"]])
    with open(os.path.join(HERE, "oracle_car_minares.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
    print(f"wrote {len(out)} cases")
