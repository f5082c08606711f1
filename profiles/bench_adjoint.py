"""Throughput of bilqr! and trilqr! (Float64), the fused passes against the primitive path (fused = 0), alternated in the
same run, with the algorithmic-byte model of DESIGN.md section 3e.  One JSON line per (solver, path), then one line with
the card it ran on.

    python profiles/bench_adjoint.py [--N 215] [--itmax 100] [--reps 3] [--out FILE]

Workloads, assembled on the GPU (A^T is formed once by the library, outside the timed solves), all tolerances 0 so that
every solve runs itmax iterations:
  BiLQR on kron_unsymmetric(N) (n = N^3, 7 nonzeros per row), b = c = 1;
  TriLQR on the forward-difference gradient of an N^3 grid (m = 3 N^2 (N - 1) rows, n = N^3 columns, 2 nonzeros per
  row; N = 215: m = 29 676 450, n = 9 938 375), b = 1 (m entries), c = cos(0, 1, ..., n - 1) (n entries).  The gradient
  maps constant vectors to zero, so c must not be constant: with c = 1, q = A u_1 = 0 and the dual half would be
  declared solved at iteration 1.
A warm-up solve with history checks that both halves stay active through all itmax iterations, so every timed
iteration runs the update pass with both halves, as the byte model counts.
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


def matrix_bytes(rows, nnz, v=8, i=4):
    return nnz * (v + i) + (rows + 1) * i


def bytes_per_iteration(solver, m, n, nnz, v=8):
    """Algorithmic bytes of one fused iteration with both halves active (DESIGN.md section 3e, SURVEY 8d counting): each
    product streams its matrix and row pointers once; every vector is counted once per read and once per write.
    BiLQR: B1 4nv and B2 6nv (BiLQ's), U 15nv.  TriLQR: T1 (n + 3m)v, T2 on the max(m, n) rows of A^T (3n + 4m)v,
    U (7n + 8m)v."""
    if solver == "bilqr":
        return 2 * matrix_bytes(n, nnz) + 25 * n * v
    return matrix_bytes(m, nnz) + matrix_bytes(max(m, n), nnz) + (11 * n + 15 * m) * v


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
    lines = []
    for solver in ("bilqr", "trilqr"):
        if solver == "bilqr":
            rp, ci, va = P.kron_unsymmetric_csr(a.N, xp=torch, device=dev)
            m = n = a.N ** 3
            work = f"kron_unsymmetric({a.N}) f64, n={n}"
        else:
            rp, ci, va = P.grad_csr(a.N, xp=torch, device=dev)
            m, n = int(rp.numel()) - 1, a.N ** 3
            work = f"grad({a.N}) f64, m={m} n={n}"
        nnz = int(va.numel())
        b = torch.ones(m, dtype=torch.float64, device=dev)
        c = (torch.ones(n, dtype=torch.float64, device=dev) if solver == "bilqr"
             else torch.cos(torch.arange(n, dtype=torch.float64, device=dev)))
        kw = dict(atol=0.0, rtol=0.0, itmax=a.itmax)
        ws = kb.krylov_workspace(solver, m, n, np.float64, device="cuda")
        ws.set_operator((rp, ci, va))
        st = torch.cuda.ExternalStream(kb.lib().krylov_b200_stream(ws._h), device=dev)
        times = {1: [], 0: []}
        launches = {}
        for fused in (1, 0):                     # warm-up: forms A^T, loads the modules
            ws.solve(None, b, c, fused=bool(fused), history=True, **kw)
            s = ws.stats                         # both halves active in every iteration
            assert len(s.residuals_primal) == len(s.residuals_dual) == a.itmax + 1, (solver, fused, s.status)
        for _ in range(a.reps):
            for fused in (1, 0):                 # alternated, so both paths see the same machine state
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                l0 = ws.launches
                e0.record(st)
                ws.solve(None, b, c, fused=bool(fused), **kw)
                e1.record(st)
                torch.cuda.synchronize()
                times[fused].append(e0.elapsed_time(e1) * 1e-3)
                launches[fused] = ws.launches - l0
                assert ws.stats.niter == a.itmax, ws.stats
        ws.free()
        del rp, ci, va, b, c
        torch.cuda.empty_cache()
        B = bytes_per_iteration(solver, m, n, nnz)
        for fused in (1, 0):
            sec = float(np.median(times[fused]))
            its = a.itmax / sec
            lines.append(dict(solver=solver, workload=f"{work} nnz={nnz}, {a.itmax} iterations/solve",
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
