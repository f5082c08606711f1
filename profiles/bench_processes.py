"""Throughput of the Krylov processes (Float64, k = 30): the fused call (every step enqueued back to back, one read-back)
against the same process restated in Python over the flat primitives kb200_spmv_csr, kb200_dot, kb200_nrm2,
kb200_axpy and kb200_divcopy (one read-back per dot), alternated in the same run.  One JSON line per (process, path)
with steps/s, launches per step, device-to-host copies per call (a torch.profiler run of its own, fused path) and the
fraction of the byte model of DESIGN.md section 3i at 3.35 TB/s; then one line with the card it ran on.

    python profiles/bench_processes.py [--N 215] [--k 30] [--reps 3] [--out FILE]

Workloads, as a user would size them: Lanczos and Arnoldi on get_div_grad(N) (N = 215: 9 938 375 rows); Golub-Kahan on
the divergence of the N^3 grid (problems.div_csr: m = N^3, n = 3 N^2 (N - 1)); non-Hermitian Lanczos and SSY on
kron_unsymmetric(N).  Aᵀ is formed once, outside the timed calls.  b = cos(0, 1, ...), c = sin(0, 1, ...).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "krylov.jl_b200")]
import numpy as np  # noqa: E402
import scipy.sparse as sp  # noqa: E402
import torch  # noqa: E402

import krylov_b200 as kb  # noqa: E402
from krylov_b200 import problems as P  # noqa: E402

PEAK = 3350.0e9   # B/s, H100 SXM data sheet (HBM3)
L = kb._lib.lib()


def mat_bytes(rows, nnz, v=8):
    return nnz * (v + 4) + (rows + 1) * 4


def bytes_per_step(name, m, n, nnz, k, v=8):
    """Algorithmic bytes of one fused step (DESIGN.md section 3i): each SpMV streams its matrix once and gathers its
    input once; every vector an epilogue or a streaming pass touches counts once per read and once per write.
    Lanczos: L1 M + 5n, L2 3n.  Arnoldi at step j: M + 5n, then j - 1 passes of 4n and one of 3n (averaged over k).
    Golub-Kahan: G1 M_A + n + 3m, G2 M_Aᵀ + m + 3n.  Non-Hermitian Lanczos: N1 M + 7n, N2 M + 7n.
    SSY: S1 M_A + n + 4m, S3 3m, S2 M_Aᵀ + m + 4n."""
    MA, MT = mat_bytes(m, nnz, v), mat_bytes(n, nnz, v)
    if name == "hermitian_lanczos":
        return MA + 8 * n * v
    if name == "arnoldi":
        return MA + (5 * n + 3 * n) * v + sum(4 * n * v * (j - 1) for j in range(1, k + 1)) / k
    if name == "golub_kahan":
        return MA + MT + (4 * n + 4 * m) * v
    if name == "nonhermitian_lanczos":
        return 2 * MA + 14 * n * v
    return MA + MT + (5 * n + 8 * m) * v


class Prim:
    """The process restated over the flat primitives of one context (src/krylov_processes.jl line by line)."""

    def __init__(self, ctx):
        self.ctx = ctx

    def spmv(self, A, x, y):
        assert L.kb200_spmv_csr(self.ctx, A._csr, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), 0) == 0

    def dot(self, x, y):
        r = C.c_double()
        L.kb200_dot(self.ctx, 1, x.numel(), C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()), C.byref(r))
        return r.value

    def norm(self, x):
        r = C.c_double()
        L.kb200_nrm2(self.ctx, 1, x.numel(), C.c_void_p(x.data_ptr()), C.byref(r))
        return r.value

    def axpy(self, s, x, y):
        L.kb200_axpy(self.ctx, 1, x.numel(), s, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()))

    def divcopy(self, y, x, s):
        L.kb200_divcopy(self.ctx, 1, x.numel(), C.c_void_p(y.data_ptr()), C.c_void_p(x.data_ptr()), s)

    def run(self, name, A, At, b, c, k):
        if name in ("hermitian_lanczos", "arnoldi"):
            n = b.numel()
            V = torch.empty((k + 1, n), dtype=b.dtype, device="cuda")
            beta = self.norm(b)
            self.divcopy(V[0], b, beta)
            H = np.zeros((k + 1, k))
            for j in range(k):
                q = V[j + 1]
                self.spmv(A, V[j], q)
                rng = range(max(0, j - 1), j + 1) if name == "hermitian_lanczos" else range(j + 1)
                for i in rng:
                    h = H[j, j - 1] if (name == "hermitian_lanczos" and i == j - 1) else self.dot(V[i], q)
                    H[i, j] = h
                    self.axpy(-h, V[i], q)
                H[j + 1, j] = self.norm(q)
                self.divcopy(q, q, H[j + 1, j])
            return
        if name == "golub_kahan":
            m, n = b.numel(), At.shape[0]
            U = torch.empty((k + 1, m), dtype=b.dtype, device="cuda")
            V = torch.empty((k + 1, n), dtype=b.dtype, device="cuda")
            beta = self.norm(b)
            self.divcopy(U[0], b, beta)
            self.spmv(At, U[0], V[0])
            alpha = self.norm(V[0])
            self.divcopy(V[0], V[0], alpha)
            for i in range(k):
                self.spmv(A, V[i], U[i + 1])
                self.axpy(-alpha, U[i], U[i + 1])
                beta = self.norm(U[i + 1])
                self.divcopy(U[i + 1], U[i + 1], beta)
                self.spmv(At, U[i + 1], V[i + 1])
                self.axpy(-beta, V[i], V[i + 1])
                alpha = self.norm(V[i + 1])
                self.divcopy(V[i + 1], V[i + 1], alpha)
            return
        m, n = b.numel(), c.numel()
        V = torch.empty((k + 1, m), dtype=b.dtype, device="cuda")
        U = torch.empty((k + 1, n), dtype=b.dtype, device="cuda")
        if name == "nonhermitian_lanczos":
            cb = self.dot(c, b)
            beta = gamma = abs(cb) ** 0.5
            gamma = cb / beta
        else:
            beta, gamma = self.norm(b), self.norm(c)
        self.divcopy(V[0], b, beta)
        self.divcopy(U[0], c, gamma)
        bprev = gprev = None
        for i in range(k):
            q, p = V[i + 1], U[i + 1]
            if name == "nonhermitian_lanczos":
                self.spmv(A, V[i], q)
                self.spmv(At, U[i], p)
            else:
                self.spmv(A, U[i], q)
                self.spmv(At, V[i], p)
            if i > 0:
                self.axpy(-gprev, V[i - 1], q)
                self.axpy(-bprev, U[i - 1], p)
            alpha = self.dot(U[i], q) if name == "nonhermitian_lanczos" else self.dot(V[i], q)
            self.axpy(-alpha, V[i], q)
            self.axpy(-alpha, U[i], p)
            if name == "nonhermitian_lanczos":
                pq = self.dot(p, q)
                bprev = abs(pq) ** 0.5
                gprev = pq / bprev
            else:
                bprev, gprev = self.norm(q), self.norm(p)
            self.divcopy(q, q, bprev)
            self.divcopy(p, p, gprev)


def workload(name, N):
    if name in ("hermitian_lanczos", "arnoldi"):
        rp, ci, va = P.div_grad_csr(N)
        A = sp.csr_matrix((va, ci, rp))
    elif name == "golub_kahan":
        rp, ci, va = P.div_csr(N)
        A = sp.csr_matrix((va, ci, rp), shape=(len(rp) - 1, 3 * N * N * (N - 1)))
    else:
        rp, ci, va = P.kron_unsymmetric_csr(N)
        A = sp.csr_matrix((va, ci, rp))
    return A


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=215)
    ap.add_argument("--k", type=int, default=30)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--names", default="hermitian_lanczos,arnoldi,golub_kahan,nonhermitian_lanczos,saunders_simon_yip")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_processes needs a CUDA device")
    if a.out:
        open(a.out, "w").close()

    def emit(rec):                                    # line by line, so a cut-short run keeps what it measured
        print(json.dumps(rec), flush=True)
        if a.out:
            with open(a.out, "a") as fh:
                fh.write(json.dumps(rec) + "\n")

    emit(dict(card=card(), torch=torch.__version__))
    for name in a.names.split(","):
        A = workload(name, a.N)
        m, n = A.shape
        Aop, Atop = kb.CsrOperator.from_scipy(A), kb.CsrOperator.from_scipy(sp.csr_matrix(A.T))
        del A
        b = torch.cos(torch.arange(m, dtype=torch.float64, device="cuda"))
        c = torch.sin(torch.arange(n, dtype=torch.float64, device="cuda")) if name in ("nonhermitian_lanczos", "saunders_simon_yip") else None
        kw = {"At": Atop} if name in ("golub_kahan", "nonhermitian_lanczos", "saunders_simon_yip") else {}
        fused = (lambda: getattr(kb, name)(Aop, b, c, a.k, **kw)) if c is not None else (lambda: getattr(kb, name)(Aop, b, a.k, **kw))
        prim = Prim(Aop._ctx)
        primitive = lambda: prim.run(name, Aop, Atop, b, c, a.k)   # noqa: E731
        times = {"fused": [], "primitive": []}
        launches = {}
        for path, f in (("fused", fused), ("primitive", primitive)):           # warm-up, launches per call
            f()
            torch.cuda.synchronize()
            l0 = L.kb200_ctx_launch_count(Aop._ctx)
            f()
            torch.cuda.synchronize()
            launches[path] = (L.kb200_ctx_launch_count(Aop._ctx) - l0) / a.k
        for _ in range(a.reps):
            for path, f in (("fused", fused), ("primitive", primitive)):
                torch.cuda.synchronize()
                t = time.perf_counter()
                f()
                torch.cuda.synchronize()
                times[path].append(time.perf_counter() - t)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fused()
            torch.cuda.synchronize()
        d2h = sum(1 for e in prof.events() if "memcpy" in e.name.lower() and "dtoh" in e.name.lower().replace(" ", ""))
        model = bytes_per_step(name, m, n, Aop.nnz, a.k)
        for path in ("fused", "primitive"):
            t = min(times[path])
            rec = dict(process=name, path=path, N=a.N, k=a.k, m=m, n=n, nnz=Aop.nnz, steps_per_s=round(a.k / t, 1),
                       ms_per_call=round(1e3 * t, 3), launches_per_step=round(launches[path], 2),
                       bytes_per_step_model=int(model), model_fraction=round(model * a.k / t / PEAK, 3))
            if path == "fused":
                rec["d2h_copies_per_call"] = d2h
            emit(rec)
        Aop.free()
        Atop.free()
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
