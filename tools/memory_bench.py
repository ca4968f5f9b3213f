#!/usr/bin/env python3
"""Device time and memory of the two trace-extension layouts on the 2^20-step collatz proof (bench.py's workload).

  python tools/memory_bench.py [--parent TREE] [--rounds 3]

Cases, each in a fresh process (so the arena and tables of one case do not carry over), run round by round, alternating between the
builds:
  b32_full    extension factor 32, no memory limit (the full layout), this tree and, with --parent, a checkout of the parent commit;
  b32_cosets  extension factor 32, the limit one byte below the full layout's plan (the evaluation-coset layout);
  b128        extension factor 128, no limit: the full layout does not fit on an 80 GB card, the evaluation-coset layout is planned.
Per case: per-stage device ms (median over the proofs after the first), kernel launches, the library's peak bytes (dg_memory_usage;
"n/a" for a build without it) and, for b128, the verdicts of the GPU verifier and the oracle's restated reference verifier.  The card
name and power limit are printed with the numbers."""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def worker(root, case, proofs):
    sys.path.insert(0, root)
    sys.path.insert(1, ROOT)          # bench.build_trace and the oracle of this tree
    import distaff_b200 as dg
    import bench
    tr, _ = bench.build_trace(20)
    ext = 128 if case == "b128" else 32
    opts = dg.ProofOptions(ext, 50, 20)
    limited = hasattr(dg, "set_memory_limit")
    plan = dg.plan_prove(tr.width, tr.length, 1, opts) if limited else None
    if case == "b32_cosets":
        dg.prove(tr, opts)             # tables and transform scratch of this shape, as a long-running user would hold them
        plan = dg.plan_prove(tr.width, tr.length, 1, opts)
        dg.set_memory_limit(plan["fixed_bytes"] + plan["bytes_per_proof"] - 1)
        plan = dg.plan_prove(tr.width, tr.length, 1, opts)
    stages, totals, launches, first = [], [], None, None
    for i in range(proofs):
        p = dg.prove(tr, opts)
        if i == 0:
            first = p.bytes
            continue
        assert p.bytes == first
        stages.append(p.stats["stage_ms"])
        totals.append(p.stats["total_ms"])
        launches = p.stats["kernel_launches"]
    out = {"case": case, "root": root, "plan": plan, "launches": launches, "total_ms": statistics.median(totals),
           "stage_ms": [round(statistics.median(s[j] for s in stages), 3) for j in range(9)],
           "peak_bytes": dg.memory_usage()["peak"] if limited else "n/a", "proof_len": len(first)}
    if case == "b128":
        from oracle import pyoracle as po
        out["dg_verify"] = dg.verify(tr.program_hash, tr.public_inputs, tr.outputs, first)
        out["po_verify"] = po.verify(tr.program_hash, tr.public_inputs, tr.outputs, first)
    print("RESULT " + json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None, help="checkout of the parent commit (built) to run b32_full against")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--proofs", type=int, default=4)
    ap.add_argument("--worker", nargs=2, metavar=("ROOT", "CASE"))
    a = ap.parse_args()
    if a.worker:
        worker(a.worker[0], a.worker[1], a.proofs)
        return
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", card)
    runs = []
    for r in range(a.rounds):
        order = [(ROOT, "b32_full")] + ([(os.path.abspath(a.parent), "b32_full")] if a.parent else []) + [(ROOT, "b32_cosets"), (ROOT, "b128")]
        if r % 2:
            order = order[::-1]
        for root, case in order:
            env = dict(os.environ, DG_LIB_PATH=os.path.join(root, "distaff_b200", "libdistaff_gpu.so"))
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", root, case, "--proofs", str(a.proofs)], capture_output=True,
                               text=True, env=env, cwd=root, timeout=1800)
            line = [ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")]
            if p.returncode or not line:
                print("FAILED", root, case, p.stderr[-2000:])
                continue
            res = json.loads(line[-1][7:])
            res["build"] = "parent" if a.parent and root == os.path.abspath(a.parent) else "this"
            runs.append(res)
            print(json.dumps({k: res[k] for k in ("build", "case", "total_ms", "stage_ms", "launches", "peak_bytes")}), flush=True)
    summary = {}
    for res in runs:
        key = res["build"] + ":" + res["case"]
        s = summary.setdefault(key, {"total_ms": [], "launches": res["launches"], "peak_bytes": res["peak_bytes"], "plan": res["plan"],
                                     "stage_ms": []})
        s["total_ms"].append(res["total_ms"])
        s["stage_ms"].append(res["stage_ms"])
        for v in ("dg_verify", "po_verify"):
            if v in res:
                s[v] = res[v]
    for key, s in summary.items():
        s["stage_ms"] = [round(statistics.median(x[j] for x in s["stage_ms"]), 3) for j in range(9)]
        s["total_ms"] = {"median": round(statistics.median(s["total_ms"]), 3), "min": round(min(s["total_ms"]), 3), "max": round(max(s["total_ms"]), 3)}
        print("SUMMARY", key, json.dumps(s))


if __name__ == "__main__":
    main()
