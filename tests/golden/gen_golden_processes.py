"""Freeze the CPU oracle's Krylov-process coefficients (oracle/krylov_oracle_processes.h) into oracle_processes.json:
every process in Float64 and Float32 on seeded 60 x 60 / 40 x 60 problems at k = 8 (with and without
reorthogonalization where it applies), values stored as exact hex floats.  Run from the repository root:
python tests/golden/gen_golden_processes.py"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]

from oracle import processes_oracle as P  # noqa: E402
from process_cases import problems  # noqa: E402

K = 8


def _hex(a):
    return [float(v).hex() for v in np.ravel(np.asarray(a, np.float64), order="F")]


def compute():
    out = {}
    for dtype in (np.float64, np.float32):
        probs = problems(seed=7, m=40, n=60)
        for name, (A, b, c) in probs.items():
            for reorth in ((False, True) if name in ("hermitian_lanczos", "arnoldi") else (False,)):
                kw = {"reorthogonalization": True} if reorth else {}
                f = getattr(P, name)
                res = f(A, b, c, K, dtype=dtype, **kw) if c is not None else f(A, b, K, dtype=dtype, **kw)
                coefs = [x for x in res[1:] if np.ndim(x) == 0 or np.asarray(x).ndim == 1 or name == "arnoldi" and np.ndim(x) == 2]
                key = f"{name}{'_reorth' if reorth else ''}_{np.dtype(dtype).name}"
                out[key] = [_hex(x) for x in coefs]
    return out


if __name__ == "__main__":
    json.dump(compute(), open(os.path.join(HERE, "oracle_processes.json"), "w"), indent=0)
