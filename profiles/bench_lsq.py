"""Throughput of lsqr!, lsmr!, lslq!, cgls! and crls! (Float64) on the forward-difference gradient G = [Dx; Dy; Dz] of an N^3 grid, fused
phases against the primitive path (fused = 0), alternated in the same run, with the algorithmic-byte model of
DESIGN.md section 3c.  One JSON line per (solver, path), then one line with the card it ran on.

    python profiles/bench_lsq.py [--N 215] [--itmax 100] [--reps 3] [--solvers lsqr,lsmr] [--out FILE]

The workload: m = 3 N^2 (N-1) rows, n = N^3 columns, 2 nonzeros per row (N = 215: m = 29 676 450, n = 9 938 375,
nnz = 59 352 900), assembled on the GPU.  b is seeded random, so the problem is inconsistent, and G has the constant
vector as its null space.  All tolerances are 0 (atol, rtol, axtol, btol, etol, conlim; cgls! / crls! have only
atol and rtol; lslq! also has etol, btol and conlim), so every solve runs itmax iterations (lslq!: itmax + 1, it tests
`iter ≥ itmax` before counting the iteration).
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


def bytes_per_iteration(solver, m, n, nnz, v=8, i=4):
    """Algorithmic bytes of one iteration (DESIGN.md section 3c, SURVEY 8d counting): both products stream their matrix
    and row pointers once; every vector is counted once per read and once per write."""
    B = 2 * nnz * (v + i) + (m + n + 2) * i
    vecs = {"lsqr": (3, 10), "lsmr": (3, 11), "lslq": (3, 9), "cgls": (5, 8), "crls": (8, 11)}[solver]   # (m-vector, n-vector) passes
    return B + vecs[0] * m * v + vecs[1] * n * v


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=215)
    ap.add_argument("--itmax", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--solvers", default="lsqr,lsmr", help="comma-separated subset of lsqr,lsmr,lslq,cgls,crls")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    rp, ci, va = P.grad_csr(a.N, xp=torch, device=dev)
    m, n, nnz = rp.numel() - 1, a.N ** 3, int(va.numel())
    g = torch.Generator(device=dev).manual_seed(0)
    b = torch.randn(m, dtype=torch.float64, device=dev, generator=g)
    lines = []
    for solver in a.solvers.split(","):
        kw = dict(atol=0.0, rtol=0.0, itmax=a.itmax)
        if solver == "lslq":
            kw.update(etol=0.0, btol=0.0, conlim=0.0)
        its_run = a.itmax + (1 if solver == "lslq" else 0)       # iterations one solve runs
        if solver in ("lsqr", "lsmr"):
            kw.update(axtol=0.0, btol=0.0, etol=0.0, conlim=0.0)
        ws = kb.krylov_workspace(solver, m, n, np.float64, device="cuda")
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
                assert ws.stats.niter == its_run, ws.stats
        ws.free()
        B = bytes_per_iteration(solver, m, n, nnz)
        for fused in (1, 0):
            sec = float(np.median(times[fused]))
            its = its_run / sec
            lines.append(dict(solver=solver, workload=f"grad_csr({a.N}) f64, m={m} n={n} nnz={nnz}, {its_run} iterations/solve",
                              fused=bool(fused), iterations_per_s=round(its, 1), us_per_iteration=round(1e6 / its, 1),
                              launches_per_iteration=round(launches[fused] / its_run, 2), bytes_per_iteration=int(B),
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
