"""Throughput of qmr! and bilq! (Float64) on kron_unsymmetric(N) (the cfg3 matrix), fused Lanczos biorthogonalization
against the primitive path (fused = 0), alternated in the same run, with the algorithmic-byte model of DESIGN.md
section 3d.  One JSON line per (solver, path), then one line with the card it ran on.

    python profiles/bench_biorth.py [--N 215] [--itmax 100] [--reps 3] [--out FILE]

The workload: n = N^3 rows and columns, 7 nonzeros per row (N = 215: n = 9 938 375), assembled on the GPU; its
transpose is formed once by the library, outside the timed solves.  b = 1.  All tolerances are 0, so every solve runs
itmax iterations.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "krylov.jl_b200")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

import krylov_b200 as kb  # noqa: E402
from krylov_b200 import problems as P  # noqa: E402

PEAK = 3350.0   # GB/s, H100 SXM data sheet (HBM3)


def bytes_per_iteration(solver, n, nnz, v=8, i=4):
    """Algorithmic bytes of one fused iteration (DESIGN.md section 3d, SURVEY 8d counting): both products stream their
    matrix and row pointers once; every vector is counted once per read and once per write.  B1 4nv, B2 6nv, and the
    update pass 10nv (QMR) or 9nv (BiLQ)."""
    matrix = nnz * (v + i) + (n + 1) * i
    return 2 * matrix + {"qmr": 20, "bilq": 19}[solver] * n * v


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=215)
    ap.add_argument("--itmax", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    rp, ci, va = P.kron_unsymmetric_csr(a.N, xp=torch, device=dev)
    n, nnz = a.N ** 3, int(va.numel())
    b = torch.ones(n, dtype=torch.float64, device=dev)
    lines = []
    for solver in ("qmr", "bilq"):
        kw = dict(atol=0.0, rtol=0.0, itmax=a.itmax)
        ws = kb.krylov_workspace(solver, n, n, np.float64, device="cuda")
        ws.set_operator((rp, ci, va))
        st = torch.cuda.ExternalStream(kb.lib().krylov_b200_stream(ws._h), device=dev)
        times = {1: [], 0: []}
        launches = {}
        for fused in (1, 0):                     # warm-up: forms A^T, loads the modules
            ws.solve(None, b, fused=bool(fused), **kw)
        for _ in range(a.reps):
            for fused in (1, 0):                 # alternated, so both paths see the same machine state
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                l0 = ws.launches
                e0.record(st)
                ws.solve(None, b, fused=bool(fused), **kw)
                e1.record(st)
                torch.cuda.synchronize()
                times[fused].append(e0.elapsed_time(e1) * 1e-3)
                launches[fused] = ws.launches - l0
                assert ws.stats.niter == a.itmax, ws.stats
        ws.free()
        B = bytes_per_iteration(solver, n, nnz)
        for fused in (1, 0):
            sec = float(np.median(times[fused]))
            its = a.itmax / sec
            lines.append(dict(solver=solver, workload=f"kron_unsymmetric({a.N}) f64, n={n} nnz={nnz}, {a.itmax} iterations/solve",
                              fused=bool(fused), iterations_per_s=round(its, 1), us_per_iteration=round(1e6 / its, 1),
                              launches_per_iteration=round(launches[fused] / a.itmax, 2), bytes_per_iteration=int(B),
                              achieved_GBs=round(B * its / 1e9, 1), frac_of_byte_model_at_datasheet_hbm=round(B * its / 1e9 / PEAK, 4),
                              spread_s=[round(t, 5) for t in times[fused]]))
    lines.append(dict(card=card(), torch=torch.__version__))
    for l in lines:
        print(json.dumps(l), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            for l in lines:
                f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
