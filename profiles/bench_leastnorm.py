"""Throughput of craig!, craigmr!, lnlq!, cgne! and crmr! (Float64), the fused passes against the primitive path
(fused = 0), alternated in the same run, with the algorithmic-byte models of DESIGN.md sections 3f, 3g and 3h.  One JSON
line per (solver, path), then one line with the card it ran on.

    python profiles/bench_leastnorm.py [--N 215] [--itmax 100] [--reps 3] [--solvers craig,craigmr,lnlq,cgne,crmr]
                                       [--out FILE]

Workload, assembled on the GPU (A^T is formed once by the library, outside the timed solves): the divergence D = G^T of
the N^3 grid (problems.div_csr; N = 215: m = 9 938 375 rows, n = 29 676 450 columns, 59 352 900 nonzeros) and
b = D cos(0, 1, ..., n - 1), a consistent system whose least-norm solution is the Helmholtz projection of the cosine
field.  All tolerances are 0 (CRAIG: btol = 0 and conlim = 0, so ctol = 0; LNLQ: σ = 0 and utolx = utoly = 0) so that
every solve runs itmax iterations; a warm-up solve with history checks that it does.  An LNLQ iteration is one pass of
its loop (lnlq! reports niter = passes + 1).  CGNE and CRMR take no tolerance of their own.
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
    """Algorithmic bytes of one fused iteration (DESIGN.md section 3f, SURVEY 8d counting): each product streams its
    matrix and row pointers once; every vector is counted once per read and once per write.
    CRAIG: C1 on A^T (m + 4n)v, C2 on A (n + 6m)v.  CRAIGMR: R1 on A (n + 2m)v, R2 on A^T (m + 6n)v, R3 7m v.
    LNLQ: L1 on A (n + 6m)v, L2 on A^T (m + 4n)v: the same total as CRAIG.
    CGNE (section 3h): E1 on A (n + 2m)v, E2 on A^T (m + 4n)v.  CRMR: R1 on A (n + m)v, R2 3m v, R3 on A^T (m + 4n)v,
    R4 3n v: CGLS's model."""
    mats = matrix_bytes(m, nnz) + matrix_bytes(n, nnz)
    if solver in ("craig", "lnlq"):
        return mats + (5 * n + 7 * m) * v
    if solver == "cgne":
        return mats + (5 * n + 3 * m) * v
    if solver == "crmr":
        return mats + (8 * n + 5 * m) * v
    return mats + (7 * n + 10 * m) * v


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=215)
    ap.add_argument("--itmax", type=int, default=100)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--solvers", default="craig,craigmr,lnlq,cgne,crmr")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_leastnorm.py measures the GPU path: no CUDA device")
    dev = torch.device("cuda", 0)
    rp, ci, va = P.div_csr(a.N, xp=torch, device=dev)
    m, n, nnz = int(rp.numel()) - 1, 3 * a.N * a.N * (a.N - 1), int(va.numel())
    z = torch.cos(torch.arange(n, dtype=torch.float64, device=dev))
    rows = torch.repeat_interleave(torch.arange(m, device=dev), (rp[1:] - rp[:-1]).long())
    b = torch.zeros(m, dtype=torch.float64, device=dev).index_add_(0, rows, va * z[ci.long()])
    del z, rows
    work = f"div({a.N}) = grad({a.N})^T f64, m={m} n={n} nnz={nnz}, b = D cos(0:n-1), {a.itmax} iterations/solve"
    lines = []
    for solver in a.solvers.split(","):
        extra = {"craig": {"btol": 0.0, "conlim": 0.0}, "lnlq": {"utolx": 0.0, "utoly": 0.0}}.get(solver, {})
        kw = dict(atol=0.0, rtol=0.0, itmax=a.itmax, **extra)
        niter = a.itmax + (solver == "lnlq")     # lnlq! counts one more than its passes
        ws = kb.krylov_workspace(solver, m, n, np.float64, device="cuda")
        ws.set_operator((rp, ci, va))
        st = torch.cuda.ExternalStream(kb.lib().krylov_b200_stream(ws._h), device=dev)
        times = {1: [], 0: []}
        launches = {}
        for fused in (1, 0):                     # warm-up: forms A^T, loads the modules
            ws.solve(None, b, fused=bool(fused), history=True, **kw)
            assert ws.stats.niter == niter and len(ws.stats.residuals) == a.itmax + 1, (solver, fused, ws.stats.status)
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
                assert ws.stats.niter == niter, ws.stats
        ws.free()
        torch.cuda.empty_cache()
        B = bytes_per_iteration(solver, m, n, nnz)
        for fused in (1, 0):
            sec = float(np.median(times[fused]))
            its = a.itmax / sec
            lines.append(dict(solver=solver, workload=work, fused=bool(fused), iterations_per_s=round(its, 1),
                              us_per_iteration=round(1e6 / its, 1),
                              launches_per_iteration=round(launches[fused] / a.itmax, 2), bytes_per_iteration=int(B),
                              achieved_GBs=round(B * its / 1e9, 1), frac_of_byte_model_at_datasheet_hbm=round(B * its / 1e9 / PEAK, 4),
                              spread_s=[round(t, 5) for t in times[fused]]))
    lines.append(dict(card=card(), torch=torch.__version__))
    for ln in lines:
        print(json.dumps(ln), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            for ln in lines:
                f.write(json.dumps(ln) + "\n")


if __name__ == "__main__":
    main()
