"""Bit-exact A/B of the solver outputs of library builds: every configuration below runs once per library, and the
outputs must agree exactly -- x byte for byte, niter, status, solved, inconsistent, indefinite, npcCount, Anorm, the
residuals / Aresiduals / Acond histories and the launch count.  Only the timers are ignored.  The configurations run
in chunks of at most CHUNK, each chunk in one child process per library (KB200_LIB selects the .so; "current" is the
tree's build), the libraries alternating chunk by chunk.

    python profiles/ab_outputs.py krylov.jl_b200/lib_ab/libkrylov_b200_<sha>.so

Prints the differences and exits 1 when any configuration differs.  The configurations cover the 13 single
right-hand-side solvers with the fused paths on and off: diagonal M and N, ldiv, warm starts, restart and growth past
`memory`, reorthogonalization, b = 0, itmax = 3, a callback exit, timemax = 0, the solver-specific exits and Float32,
and CG on a constant-coefficient operator (the path of the CsrDict encoding, M = I and a diagonal M, both types), CG's
two-launch kernels (fused = 2), a block-Jacobi M and the in-kernel phase timing (time_kernels).  LSQR and LSMR get the
same treatment; LSLQ, CGLS, CRLS, CRAIG, CRAIGMR, LNLQ, CGNE, CRMR, BiLQ, QMR, BiLQR, TriLQR, CAR and MINARES run
compactly (defaults, Float32, itmax = 3 and a callback exit, fused and not), and each rectangular one once more per
preconditioner it takes (M on the m-space, N on the n-space, CGNE / CRMR's N on the m-space) and per option field it
forwards (λ; the trust-region radius of CGLS / CRLS).  CG, CR, MINRES and CG-Lanczos also run with an N they ignore.
For the two-solution solvers y and the dual history are compared too.
"""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SQUARE = {"cg": "lap", "cr": "lap", "minres": "lap", "cg_lanczos": "lap", "bicgstab": "kron", "cgs": "kron",
          "gmres": "kron", "fom": "kron", "fgmres": "kron", "dqgmres": "kron", "diom": "kron"}
TAKES_N = {"bicgstab", "cgs", "gmres", "fom", "fgmres", "dqgmres", "diom"}
ARNOLDI = {"gmres", "fom", "fgmres"}
COMPACT = {"lslq": "grad", "cgls": "grad", "crls": "grad", "craig": "div", "craigmr": "div", "bilq": "kron",
           "qmr": "kron", "bilqr": "kron", "trilqr": "grad", "car": "lap", "minares": "lap", "lnlq": "div", "cgne": "div",
          "crmr": "div"}
ADJOINT = {"bilqr", "trilqr"}
# the rectangular solvers beyond LSQR / LSMR: the preconditioners they take and whether they forward the radius
RECT = {"lslq": ("M", "N"), "cgls": ("M",), "crls": ("M",), "craig": ("M", "N"), "craigmr": ("M", "N"),
        "lnlq": ("M", "N"), "cgne": ("N",), "crmr": ("N",)}
N_ON_M = {"cgne", "crmr"}
CHUNK = 12


def problems():
    import scipy.sparse as sp
    from krylov_b200.problems import div_grad_csr, kron_unsymmetric_csr, grad_csr

    def csr(t, n, m=None):
        rp, ci, va = t
        return sp.csr_matrix((va, ci, rp), shape=(n, m or n))
    lap = csr(div_grad_csr(6), 216) + sp.diags(np.linspace(0.0, 4.0, 216))        # non-constant diagonal
    dg = csr(div_grad_csr(30, 20, 10), 6000)                                       # constant coefficients: 7 pairs (CsrDict)
    kron = csr(kron_unsymmetric_csr(6), 216) + sp.diags(np.linspace(0.0, 3.0, 216))
    N = 5
    grad = csr(grad_csr(N), 3 * N * N * (N - 1), N ** 3)
    indef = sp.diags([np.ones(9), np.ones(10), np.ones(9)], [-1, 0, 1]) - 10 * sp.identity(10)
    indef12 = sp.diags([np.ones(11), np.ones(12), np.ones(11)], [-1, 0, 1])
    negcurv = sp.lil_matrix(sp.diags([np.ones(9), 4 * np.ones(10), np.ones(9)], [-1, 0, 1]))
    negcurv[8, 8] = -4.0
    d = np.ones(10)
    d[0] = 0.0
    rng = np.random.default_rng(7)
    P = {
        "lap": (lap, np.ones(216)),
        "dg": (dg, rng.standard_normal(6000)),
        "kron": (kron, kron @ np.ones(216)),
        "grad": (grad, rng.standard_normal(grad.shape[0])),
        "div": (grad.T, rng.standard_normal(grad.shape[1])),              # underdetermined: the least-norm solvers
        "indef": (indef, indef @ np.arange(1.0, 11.0)),
        "indef12": (indef12, indef12 @ np.arange(1.0, 13.0)),
        "negcurv": (negcurv, negcurv @ np.arange(1.0, 11.0)),
        "semidef2": (np.array([[1.0, 0.0], [0.0, 0.0]]), np.ones(2)),      # CR linesearch, npcCount = 2
        "zerocurv": (np.array([[0.0, 1.0], [1.0, 0.0]]), np.array([1.0, 0.0])),   # CR: b is a zero-curvature direction
        "bc0": (np.array([[1.0, 2.0], [3.0, 4.0]]), np.array([0.0, 1.0])),  # with c = e1: bᴴc = 0
        "inconsistent": (np.diag(d), np.ones(10)),                        # GMRES / FGMRES inconsistent, FOM breakdown
        "ident": (np.eye(4), np.arange(1.0, 5.0)),                        # MINRES: least-squares exit at iter 1
        "Atb0": (np.array([[1.0], [0.0]]), np.array([0.0, 1.0])),         # LSQR / LSMR: Aᴴb = 0
    }
    return {k: (sp.csr_matrix(A), b) for k, (A, b) in P.items()}


def configs():
    out = []

    def add(solver, prob, fused_both=True, **kw):
        for fused in ((True, False) if fused_both else (True,)):
            out.append(dict(solver=solver, prob=prob, kw=dict(kw, fused=fused)))
    for s, p in SQUARE.items():
        add(s, p)
        add(s, p, M="d")
        add(s, p, M="d", ldiv=True)
        if s in TAKES_N:
            add(s, p, N="d")
            add(s, p, M="d", N="sd")
        add(s, p, x0=True)
        add(s, p, zero_b=True)
        add(s, p, itmax=3)
        add(s, p, callback=3, atol=0.0, rtol=0.0)
        add(s, p, timemax=0.0)
        add(s, p, dtype="float32")
        if s not in TAKES_N:
            add(s, p, N="d")                                          # an N the solver ignores
        if s in ARNOLDI:
            add(s, p, restart=True, memory=5)
            add(s, p, restart=True, memory=5, x0=True)
            add(s, p, restart=True, memory=5, M="d", N="sd")
            add(s, p, restart=False, memory=5)                       # non-restarted growth past memory
            if s != "fom":     # FOM's extra step past `memory` read an unallocated V[k] before the zero column was added
                add(s, p, restart=False, memory=5, callback=7, atol=0.0, rtol=0.0)
            add(s, p, reorthogonalization=True)
            add(s, p, reorthogonalization=True, restart=True, memory=5)
            add(s, "inconsistent")
            add(s, p, dtype="float32", restart=True, memory=5)
        if s in ("dqgmres", "diom"):
            add(s, p, reorthogonalization=True)
            add(s, p, memory=3)
        if s in ("bicgstab", "cgs"):
            add(s, "bc0", c="e1")
    for dtype in ("float64", "float32"):            # the persistent kernel on the constant-coefficient encoding
        add("cg", "dg", dtype=dtype)
        add("cg", "dg", dtype=dtype, M="pos")
        add("cg", "dg", dtype=dtype, itmax=40, atol=0.0, rtol=0.0)
        for prob in ("lap", "dg"):                  # the two-launch kernels
            out.append(dict(solver="cg", prob=prob, kw=dict(dtype=dtype, fused=2)))
    add("cg", "lap", M="bj4")                       # block-Jacobi M, (54, 4, 4) blocks
    add("cg", "dg", time_kernels=True)
    add("cg", "indef", linesearch=True)
    add("cg", "lap", radius=0.5)
    add("cg", "indef12", radius=5.0)
    add("minres", "indef", linesearch=True)
    add("minres", "ident")
    add("minres", "lap", lambda_=0.5)
    add("cr", "indef", linesearch=True)
    add("cr", "semidef2", linesearch=True)
    add("cr", "lap", radius=10.0)
    add("cr", "lap", radius=0.5)
    add("cr", "indef12", radius=5.0)
    add("cr", "indef12")                                                # "Indefinite system and no trust region"
    add("cr", "zerocurv")
    add("cr", "zerocurv", radius=1.0)
    add("cg_lanczos", "negcurv", check_curvature=True)
    for s in ("lsqr", "lsmr"):
        p = "grad"
        add(s, p)
        add(s, p, M="pos")
        add(s, p, N="pos")
        add(s, p, M="pos", N="pos", ldiv=True)
        add(s, p, zero_b=True)
        add(s, "Atb0")
        add(s, p, itmax=3)
        add(s, p, callback=3)
        add(s, p, timemax=0.0)
        add(s, p, lambda_=0.1)
        add(s, p, radius=0.5)
        add(s, p, dtype="float32")
    for s, p in COMPACT.items():
        c = {"c": "ramp"} if s in ADJOINT else {}
        add(s, p, **c)
        add(s, p, dtype="float32", **c)
        add(s, p, itmax=3, **c)
        add(s, p, callback=3, **c)
    for s, slots in RECT.items():
        for which in slots:
            add(s, COMPACT[s], **{which: "pos"})
        add(s, COMPACT[s], lambda_=0.1)
        if s in ("cgls", "crls"):
            add(s, COMPACT[s], radius=0.5)
    return out


def hexf(v):
    return float(v).hex()


def run_chunk(lo, hi, path):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "krylov.jl_b200")]
    import krylov_b200 as kb
    P = problems()
    results = {}
    for cfg in configs()[lo:hi]:
        key = json.dumps(cfg, sort_keys=True)
        kw = dict(cfg["kw"])
        dtype = np.dtype(kw.pop("dtype", "float64"))
        A, b = P[cfg["prob"]]
        m, n = A.shape
        if kw.pop("zero_b", False):
            b = np.zeros_like(b)
        diag = A.diagonal()
        vec = {"d": lambda: 1.0 / diag, "sd": lambda: 1.0 / np.sqrt(diag),
               "pos": lambda ln: np.linspace(0.5, 2.0, ln),
               "bj4": lambda: np.linalg.inv(np.stack([A[k:k + 4, k:k + 4].toarray() for k in range(0, n, 4)]))}
        for which, ln in (("M", m), ("N", m if cfg["solver"] in N_ON_M else n)):
            if which in kw:
                kw[which] = vec["pos"](ln) if kw[which] == "pos" else vec[kw[which]]()
        c = kw.pop("c", None)
        if c == "e1":
            kw["c"] = np.eye(n)[0]
        elif c == "ramp":                           # the adjoint system's right-hand side: n entries
            kw["c"] = np.linspace(-1.0, 2.0, n)
        x0 = 0.5 * np.ones(n) if kw.pop("x0", False) else None
        memory = kw.pop("memory", 0)
        stop_at = kw.pop("callback", None)
        if stop_at:
            cnt = []
            kw["callback"] = lambda w: (cnt.append(1), len(cnt) >= stop_at)[1]
        kw["history"] = True
        if cfg["solver"] in ("lsqr", "lsmr"):
            ws = kb.krylov_workspace(cfg["solver"], m, n, dtype)
        else:
            ws = kb.krylov_workspace(cfg["solver"], m, n, dtype, memory=memory)
        try:
            if x0 is not None:
                ws.warm_start(x0)
            ws.solve(A, b.astype(dtype), **kw)
            st = ws.stats
            res = dict(x=np.ascontiguousarray(ws.x).tobytes().hex(), niter=st.niter, status=st.status, solved=st.solved,
                       launches=ws.launches)
            if cfg["solver"] in ADJOINT:             # AdjointStats
                res.update(solved_primal=st.solved_primal, solved_dual=st.solved_dual,
                           residuals=[hexf(v) for v in st.residuals_primal],
                           residuals_dual=[hexf(v) for v in st.residuals_dual])
            else:
                res.update(inconsistent=st.inconsistent, indefinite=st.indefinite, npcCount=st.npcCount,
                           Anorm=hexf(st.Anorm), residuals=[hexf(v) for v in st.residuals],
                           Aresiduals=[hexf(v) for v in st.Aresiduals], Acond=[hexf(v) for v in st.Acond])
            if hasattr(ws, "y"):                     # the two-solution workspaces
                res["y"] = np.ascontiguousarray(ws.y).tobytes().hex()
        except kb.B200Error as e:
            res = dict(error=str(e))
        finally:
            ws.free()
        results[key] = res
    with open(path, "w") as f:
        json.dump(results, f)


def main():
    libs = [None] + [os.path.abspath(p) for p in sys.argv[1:]]
    cfgs = configs()
    chunks, lo = [], 0
    for i in range(1, len(cfgs) + 1):        # chunks never span two solvers
        if i == len(cfgs) or i - lo == CHUNK or cfgs[i]["solver"] != cfgs[lo]["solver"]:
            chunks.append((lo, i))
            lo = i
    outs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for lo, hi in chunks:
            solver = cfgs[lo]["solver"]
            for lib in libs:
                name = os.path.basename(lib) if lib else "current"
                env = dict(os.environ)
                env.pop("KB200_LIB", None)
                if lib:
                    env["KB200_LIB"] = lib
                path = os.path.join(tmp, f"{name}.{lo}.json")
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", str(lo), str(hi), path], env=env,
                                   capture_output=True, text=True)
                if r.returncode != 0:
                    print("FAILED", name, solver, r.stderr[-2000:])
                    sys.exit(1)
                with open(path) as f:
                    outs.setdefault(name, {}).update(json.load(f))
            print(f"{solver} configurations {lo}..{hi - 1}: done", flush=True)
    ref_name = "current"
    ref = outs[ref_name]
    bad = 0
    for name, other in outs.items():
        if name == ref_name:
            continue
        for key in ref:
            a, b = ref[key], other.get(key)
            if a != b:
                bad += 1
                fields = sorted(k for k in set(a) | set(b or {}) if (b or {}).get(k) != a.get(k))
                print(f"DIFF {name} {key}: {fields}", flush=True)
                for k in fields[:3]:
                    if k != "x":
                        print(f"    {k}: {ref_name}={a.get(k)!r:.200} {name}={(b or {}).get(k)!r:.200}")
    nerr = sum("error" in v for v in ref.values())
    if bad:
        print(f"{bad} of {len(ref)} configurations differ")
        sys.exit(1)
    print(f"all {len(ref)} configurations identical across {len(outs)} libraries ({nerr} of them end in the same error)")


if __name__ == "__main__":
    if len(sys.argv) == 5 and sys.argv[1] == "--child":
        run_chunk(int(sys.argv[2]), int(sys.argv[3]), sys.argv[4])
    else:
        main()
