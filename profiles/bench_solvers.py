"""Throughput of the other three solvers on the BASELINE configs 3 and 4 (+ MINRES on the Poisson matrix), fused
phases vs the primitive path, with the algorithmic-byte roofline of SURVEY.md section 8(d).  One JSON line each.

    python profiles/bench_solvers.py [gmres] [bicgstab] [minres] [car_minares] [--small]

car_minares runs only when named.
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "krylov.jl_b200")]
import numpy as np  # noqa: E402
import torch  # noqa: E402

import krylov_b200 as kb  # noqa: E402
from krylov_b200 import problems as P  # noqa: E402

PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0   # H100 SXM data sheet
small = "--small" in sys.argv
which = [a for a in sys.argv[1:] if not a.startswith("--")] or ["gmres", "bicgstab", "minres", "siblings"]
dev = torch.device("cuda", 0)


def timed(ws, b, reps, **kw):
    st = torch.cuda.ExternalStream(kb.lib().krylov_b200_stream(ws._h), device=dev)
    ws.solve(None, b, **kw)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    l0 = ws.launches
    e0.record(st)
    for _ in range(reps):
        ws.solve(None, b, **kw)
    e1.record(st)
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e-3 / reps, ws.stats.niter, (ws.launches - l0) // reps


def report(name, workload, B_iter, results):
    for fused, (sec, niter, launches) in results.items():
        its = niter / sec
        print(json.dumps(dict(solver=name, workload=workload, fused=bool(fused), iterations_per_s=round(its, 1),
                              us_per_iteration=round(1e6 / its, 1), launches_per_iteration=round(launches / niter, 2),
                              bytes_per_iteration=int(B_iter), achieved_GBs=round(B_iter * its / 1e9, 1),
                              frac_of_measured_hbm=round(B_iter * its / 1e9 / PEAK, 4))), flush=True)


if "gmres" in which:      # config 3: gmres!(restart, memory=30) on kron_unsymmetric(215), 2 full cycles
    N = 64 if small else 215
    rp, ci, va = P.kron_unsymmetric_csr(N, xp=torch, device=dev)
    n, nnz = N ** 3, int(va.numel())
    b = P.csr_matvec_ones(rp, ci, va)
    res = {}
    for fused in (1, 0):
        ws = kb.GmresWorkspace(n, n, np.float64, memory=30, device="cuda")
        ws.set_operator((rp, ci, va))
        res[fused] = timed(ws, b, 2, atol=0.0, rtol=0.0, itmax=60, restart=True, fused=bool(fused))
        ws.free()
    B = nnz * 12 + (n + 1) * 4 + 2 * n * 8 + 64 * n * 8         # B_spmv + 64 n v (cycle average, SURVEY 8d)
    report("gmres(30)", f"kron_unsymmetric({N}) f64, 60 inner iterations/solve", B, res)
    del rp, ci, va, b
    torch.cuda.empty_cache()

if "bicgstab" in which:   # config 4: bicgstab! Float32 on the random CSR, 20 nnz/row + diagonal
    n = 200_000 if small else 5_000_000
    t0 = time.time()
    rp, ci, va = P.random_csr(n, 20, seed=1234, dtype=np.float32)
    nnz = len(va)
    bh = np.add.reduceat(va, rp[:-1].astype(np.int64)).astype(np.float32)
    gen_s = time.time() - t0
    b = torch.from_numpy(bh).to(dev)
    res = {}
    for fused in (1, 0):
        ws = kb.BicgstabWorkspace(n, n, np.float32, device="cuda")
        ws.set_operator((torch.from_numpy(rp).to(dev), torch.from_numpy(ci).to(dev), torch.from_numpy(va).to(dev)))
        res[fused] = timed(ws, b, 2, atol=0.0, rtol=0.0, itmax=50, fused=bool(fused))
        ws.free()
    B = 2 * (nnz * 8 + (n + 1) * 4) + 20 * n * 4                 # 2 (matrix) + 20 n v, v = 4
    report("bicgstab", f"random CSR n={n} nnz={nnz} f32 (generated on host in {gen_s:.0f} s), 50 iterations/solve", B, res)
    torch.cuda.empty_cache()

if "minres" in which:     # MINRES on the config-2 matrix
    N = 64 if small else 215
    rp, ci, va = P.div_grad_csr(N, xp=torch, device=dev)
    n, nnz = N ** 3, int(va.numel())
    b = torch.ones(n, dtype=torch.float64, device=dev)
    res = {}
    for fused in (1, 0):
        ws = kb.MinresWorkspace(n, n, np.float64, device="cuda")
        ws.set_operator((rp, ci, va))
        res[fused] = timed(ws, b, 2, atol=0.0, rtol=0.0, etol=0.0, conlim=1e300, itmax=100, fused=bool(fused))
        ws.free()
    B = nnz * 12 + (n + 1) * 4 + 13 * n * 8
    report("minres", f"get_div_grad({N}) f64, 100 iterations/solve", B, res)

if "siblings" in which:   # SURVEY.md 8f-3: the sibling solvers on the same two matrices (it/s only; primitives + shared fused Arnoldi)
    N = 64 if small else 215
    rp, ci, va = P.kron_unsymmetric_csr(N, xp=torch, device=dev)
    n = N ** 3
    b = P.csr_matvec_ones(rp, ci, va)
    for name, mem, kw in (("fom", 30, dict(restart=True, itmax=60)), ("fgmres", 30, dict(restart=True, itmax=60)),
                          ("dqgmres", 20, dict(itmax=60)), ("diom", 20, dict(itmax=60)), ("cgs", 0, dict(itmax=50))):
        ws = kb.krylov_workspace(name, n, n, np.float64, memory=mem, device="cuda")
        ws.set_operator((rp, ci, va))
        sec, niter, launches = timed(ws, b, 2, atol=0.0, rtol=0.0, **kw)
        print(json.dumps(dict(solver=name, workload=f"kron_unsymmetric({N}) f64, {niter} iterations/solve" + (f", memory {mem}" if mem else ""),
                              iterations_per_s=round(niter / sec, 1), us_per_iteration=round(1e6 * sec / niter, 1),
                              launches_per_iteration=round(launches / niter, 2))), flush=True)
        ws.free()
    del rp, ci, va, b
    torch.cuda.empty_cache()
    rp, ci, va = P.div_grad_csr(N, xp=torch, device=dev)
    b = torch.ones(n, dtype=torch.float64, device=dev)
    for name in ("cr", "cg_lanczos"):
        ws = kb.krylov_workspace(name, n, n, np.float64, device="cuda")
        ws.set_operator((rp, ci, va))
        sec, niter, launches = timed(ws, b, 2, atol=0.0, rtol=0.0, itmax=100)
        print(json.dumps(dict(solver=name, workload=f"get_div_grad({N}) f64, {niter} iterations/solve",
                              iterations_per_s=round(niter / sec, 1), us_per_iteration=round(1e6 * sec / niter, 1),
                              launches_per_iteration=round(launches / niter, 2))), flush=True)
        ws.free()

if "car_minares" in which:  # CAR and MINARES on the config-2 matrix (DESIGN.md §3a byte models)
    N = 64 if small else 215
    rp, ci, va = P.div_grad_csr(N, xp=torch, device=dev)
    n, nnz = N ** 3, int(va.numel())
    b = torch.ones(n, dtype=torch.float64, device=dev)
    for name, vecs, kw in (("car", 20, dict(atol=0.0, rtol=0.0, itmax=100)),
                           ("minares", 17, dict(atol=0.0, rtol=0.0, artol=0.0, itmax=100))):
        res = {}
        for fused in (1, 0):
            ws = kb.krylov_workspace(name, n, n, np.float64, device="cuda")
            ws.set_operator((rp, ci, va))
            res[fused] = timed(ws, b, 2, fused=bool(fused), **kw)
            ws.free()
        B = nnz * 12 + (n + 1) * 4 + vecs * n * 8                  # nnz (v + i) + (n + 1) i + vecs n v, v = 8, i = 4
        report(name, f"get_div_grad({N}) f64, 100 iterations/solve", B, res)
