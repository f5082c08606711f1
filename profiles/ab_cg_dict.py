"""A/B of the constant-coefficient encoding (CsrDict) on the flagship workload: bench.py alternately on a library
build WITHOUT it (the argument, selected with KB200_LIB) and on the tree's build, `--runs` times each, in one process
tree on one GPU.  The first pair runs the full record (CPU leg, parity block) with --dump-outputs, and the dumps of
the two builds must be byte-identical; the other pairs skip the CPU leg.  Appends one JSON line to --out:

    python profiles/ab_cg_dict.py krylov.jl_b200/lib_ab/libkrylov_b200_<sha>.so --out profiles/h100_cg_dict_ab.jsonl

Reported per build: the median `value` (it/s), cfg5.value, the extra records (cfg3 GMRES, cfg4 BiCGSTAB), e2e, and the
in-kernel phase times (roofline.kernels); for the encoded build also the achieved bandwidth against the encoded byte
model B_cg,dict = n + 9nv (+ the dictionary, 96 B) -- bench.py's roofline keeps the CSR model B_cg, so its `frac`
reads above 1 there.
"""
import argparse
import filecmp
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def bench(lib, extra):
    env = dict(os.environ)
    env.pop("KB200_LIB", None)
    if lib:
        env["KB200_LIB"] = lib
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "5", "--warmup", "3"] + extra,
                       env=env, capture_output=True, text=True, cwd=ROOT)
    lines = [l for l in r.stdout.splitlines() if l.startswith("{")]
    if r.returncode != 0 or not lines:
        raise SystemExit(f"bench.py failed ({lib or 'current'}): {r.stderr[-3000:]}")
    return json.loads(lines[-1])


def summary(recs):
    med = lambda f: statistics.median(f(r) for r in recs)
    out = dict(values=[r["value"] for r in recs], value=med(lambda r: r["value"]),
               cfg5_values=[r.get("cfg5", {}).get("value") for r in recs],
               cfg5_value=med(lambda r: r.get("cfg5", {}).get("value") or 0.0),
               e2e=med(lambda r: r["e2e"]["value"]),
               extra={e["config"]: statistics.median(x["value"] for r in recs for x in r.get("extra", []) if x.get("config") == e["config"])
                      for e in recs[0].get("extra", []) if "config" in e},
               kernels=recs[0]["roofline"]["kernels"], frac_csr_model=med(lambda r: r["roofline"]["frac"]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("parent_lib")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    libs = {"parent": os.path.abspath(args.parent_lib), "encoded": None}
    recs = {k: [] for k in libs}
    with tempfile.TemporaryDirectory() as tmp:
        for i in range(args.runs):
            for name, lib in libs.items():
                extra = ["--dump-outputs", os.path.join(tmp, name)] if i == 0 else ["--no-cpu"]
                recs[name].append(bench(lib, extra))
                print(name, i, recs[name][-1]["value"], flush=True)
        same = {f: filecmp.cmp(os.path.join(tmp, "parent", f), os.path.join(tmp, "encoded", f), shallow=False)
                for f in sorted(os.listdir(os.path.join(tmp, "parent")))}
    line = dict(gpu=gpu_info(), runs=args.runs, dumps_identical=same,
                parity_max_rel_dev={k: v[0].get("parity", {}).get("max_rel_dev") for k, v in recs.items()},
                **{k: summary(v) for k, v in recs.items()})
    cfg = recs["encoded"][0]["config"]
    n, iters = cfg["n"], cfg["iters_per_step"]
    b_dict = n + 9 * n * 8 + 96
    enc = line["encoded"]
    enc["bytes_per_iteration_dict"] = b_dict
    enc["GBs_dict"] = b_dict * enc["value"] / 1e9
    k = enc["kernels"]
    for ph, b in (("phase_a", n + 6 * n * 8), ("phase_b", 3 * n * 8)):
        ms = k[ph]["ms"]
        k[ph]["bytes_dict"] = b
        k[ph]["GBs_dict"] = b / (ms * 1e-3) / 1e9 if ms else None
    line["speedup"] = enc["value"] / line["parent"]["value"]
    line["cfg5_speedup"] = enc["cfg5_value"] / line["parent"]["cfg5_value"] if line["parent"]["cfg5_value"] else None
    txt = json.dumps(line)
    print(txt)
    if args.out:
        with open(args.out, "a") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
