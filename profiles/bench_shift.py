"""Time to solve a family of shifted systems with one shift solver, against one solve per shift (Float64).

    python profiles/bench_shift.py [--N 215] [--p 1,4,16,32] [--cgls-p 4] [--reps 2] [--out FILE]

Workloads, as a user would size them (a regularization sweep over log-spaced shifts in [0.1, 10]):
  * cg_lanczos_shift on get_div_grad(N) (N = 215: 9 938 375 rows, 69.3 M nonzeros) with p in --p shifts, against
    cg on A + σᵢ I for every shift (the library's fastest single solver: the persistent fused CG kernel);
  * cgls_lanczos_shift on grad_csr(N) (m = 3 N^2 (N - 1), n = N^3) with --cgls-p shifts, against cgls with λ = σᵢ.
For each: fused against fused = False, alternated in one run (min over --reps); launches and device-to-host copies per
iteration (the difference between two solves of fixed length, atol = rtol = 0; copies from a torch.profiler run of
their own); the fraction of the byte model of DESIGN.md section 3j at 3.35 TB/s; the time of the p separate solves.
One JSON line per record; the first names the card and its power limit, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "krylov.jl_b200")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

import krylov_b200 as kb  # noqa: E402
from krylov_b200 import problems as P  # noqa: E402

PEAK = 3350.0e9   # B/s, H100 SXM data sheet (HBM3)
PASS = 16         # kShiftPass (csrc/kb_internal.h)


def mat_bytes(rows, nnz, v=8):
    return nnz * (v + 4) + (rows + 1) * 4


def bytes_per_iter(solver, m, n, nnz, p, v=8):
    """DESIGN.md section 3j, with p active shifts.  CG-Lanczos-shift: the SpMV on v with <v, A v> (M + 3n vector
    words: the gather, the epilogue's read of v, the store of Mv_next) and the three-term recurrence (6n), then the
    shift update (2 + 4p)n.  CGLS-Lanczos-shift: A v with ||u_next||^2 (M_A + n + m), the u pass (5m), A^T u_next
    with ||v||^2 (M_Aᵀ + m + n), then the shift update (2 + 4p)n."""
    upd = (2 + 4 * p) * n * v
    if solver == "cg_lanczos_shift":
        return mat_bytes(n, nnz, v) + 9 * n * v + upd
    return mat_bytes(m, nnz, v) + mat_bytes(n, nnz, v) + (2 * n + 7 * m) * v + upd


def bytes_of_solve(solver, m, n, nnz, st, v=8):
    """The model over a whole solve: a converged shift leaves the update, so shift i costs its 4n words only in the
    iterations it was active in, len(residuals[i]) - 1 of them (history=True)."""
    active = sum(len(r) - 1 for r in st.residuals)
    return st.niter * bytes_per_iter(solver, m, n, nnz, 0, v) + 4 * active * n * v


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(f):
    torch.cuda.synchronize()
    t = time.perf_counter()
    f()
    torch.cuda.synchronize()
    return time.perf_counter() - t


def per_iteration(ws, A, b, shifts, fused):
    """(launches, device-to-host copies) per iteration: two fixed-length solves, the difference over 10 iterations."""
    from torch.profiler import ProfilerActivity, profile
    out = []
    for k in (5, 15):
        l0 = ws.launches
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ws.solve(A, b, shifts, atol=0.0, rtol=0.0, itmax=k, fused=fused)
            torch.cuda.synchronize()
        d2h = sum(1 for e in prof.events() if "memcpy" in e.name.lower() and "dtoh" in e.name.lower().replace(" ", ""))
        out.append((ws.launches - l0, d2h))
    return (out[1][0] - out[0][0]) / 10, (out[1][1] - out[0][1]) / 10


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=215)
    ap.add_argument("--p", default="1,4,16,32")
    ap.add_argument("--cgls-p", type=int, default=4)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_shift needs a CUDA device")
    if a.out:
        open(a.out, "w").close()

    def emit(rec):                                    # line by line, so a cut-short run keeps what it measured
        print(json.dumps(rec), flush=True)
        if a.out:
            with open(a.out, "a") as fh:
                fh.write(json.dumps(rec) + "\n")

    emit(dict(card=card(), torch=torch.__version__))
    N = a.N
    # ---- CG-Lanczos-shift on get_div_grad(N) ----
    rp, ci, va = P.div_grad_csr(N)
    n = len(rp) - 1
    diag = np.nonzero(ci == np.repeat(np.arange(n), np.diff(rp)))[0]     # where each row's diagonal entry is
    b = torch.ones(n, dtype=torch.float64, device="cuda")
    for p in [int(s) for s in a.p.split(",")]:
        shifts = list(np.logspace(-1, 1, p))
        ws = kb.CgLanczosShiftWorkspace(n, n, p, np.float64, device="cuda")
        A = (rp, ci, va)
        ws.set_operator(A)                            # uploaded once: later solves pass the same object
        runs = {True: [], False: []}
        for fused in (True, False):                   # warm-up
            ws.solve(A, b, shifts, fused=fused)
        for _ in range(a.reps):
            for fused in (True, False):
                runs[fused].append((timed(lambda: ws.solve(A, b, shifts, fused=fused, history=True)), ws.stats.niter))
        st = ws.stats
        launches, d2h = {}, {}
        for fused in (True, False):
            launches[fused], d2h[fused] = per_iteration(ws, A, b, shifts, fused)
        ws.free()
        sep = kb.CgWorkspace(n, n, np.float64, device="cuda")
        t_sep, it_sep = 0.0, []
        for s in shifts:
            vs = va.copy()
            vs[diag] += s
            As = (rp, ci, vs)
            sep.set_operator(As)
            sep.solve(As, b)                          # warm-up of this operator
            t_sep += timed(lambda: sep.solve(As, b))
            it_sep.append(sep.stats.niter)
        sep.free()
        model = bytes_of_solve("cg_lanczos_shift", n, n, len(ci), st)
        for fused in (True, False):
            t, it = min(runs[fused])
            emit(dict(solver="cg_lanczos_shift", path="fused" if fused else "primitive", N=N, n=n, nnz=len(ci), p=p,
                      shifts="logspace(-1, 1, p)", niter=it, solved=st.solved, ms_total=round(1e3 * t, 2),
                      ms_per_iter=round(1e3 * t / it, 3), launches_per_iter=launches[fused], d2h_per_iter=d2h[fused],
                      bytes_model=int(model), model_fraction=round(model / t / PEAK, 3),
                      separate="cg on A + σI", separate_ms_total=round(1e3 * t_sep, 2), separate_niter=it_sep,
                      speedup_vs_separate=round(t_sep / t, 2)))
    del rp, ci, va
    # ---- CGLS-Lanczos-shift on grad_csr(N) ----
    rp, ci, va = P.grad_csr(N)
    m, n = len(rp) - 1, N ** 3
    import scipy.sparse as sp
    G = kb.CsrOperator.from_scipy(sp.csr_matrix((va, ci, rp), shape=(m, n)))
    b = torch.cos(torch.arange(m, dtype=torch.float64, device="cuda"))
    p = a.cgls_p
    shifts = list(np.logspace(-1, 1, p))
    ws = kb.CglsLanczosShiftWorkspace(m, n, p, np.float64, device="cuda")
    runs = {True: [], False: []}
    for fused in (True, False):
        ws.solve(G, b, shifts, fused=fused)
    for _ in range(a.reps):
        for fused in (True, False):
            runs[fused].append((timed(lambda: ws.solve(G, b, shifts, fused=fused, history=True)), ws.stats.niter))
    st = ws.stats
    launches, d2h = {}, {}
    for fused in (True, False):
        launches[fused], d2h[fused] = per_iteration(ws, G, b, shifts, fused)
    ws.free()
    sep = kb.CglsWorkspace(m, n, np.float64, device="cuda")
    t_sep, it_sep = 0.0, []
    for s in shifts:
        sep.solve(G, b, lambda_=s)
        t_sep += timed(lambda: sep.solve(G, b, lambda_=s))
        it_sep.append(sep.stats.niter)
    sep.free()
    model = bytes_of_solve("cgls_lanczos_shift", m, n, len(ci), st)
    for fused in (True, False):
        t, it = min(runs[fused])
        emit(dict(solver="cgls_lanczos_shift", path="fused" if fused else "primitive", N=N, m=m, n=n, nnz=len(ci), p=p,
                  shifts="logspace(-1, 1, p)", niter=it, solved=st.solved, ms_total=round(1e3 * t, 2),
                  ms_per_iter=round(1e3 * t / it, 3), launches_per_iter=launches[fused], d2h_per_iter=d2h[fused],
                  bytes_model=int(model), model_fraction=round(model / t / PEAK, 3),
                  separate="cgls with λ = σ", separate_ms_total=round(1e3 * t_sep, 2), separate_niter=it_sep,
                  speedup_vs_separate=round(t_sep / t, 2)))


if __name__ == "__main__":
    main()
