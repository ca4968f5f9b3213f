#!/usr/bin/env python3
"""One long execution on the GPU: trace_one / execute_one (the sponge from a per-program table, one sequential pass that records
checkpoints, one thread per segment writing the rows) against hostvm.execute (+ prove, which is dg.execute) and trace_batch /
execute_batch with K = 1 (the whole execution on one GPU thread, sponge rounds included).  Wall seconds of one call after a warm-up
call of a small program, and the per-phase device times of the one-execution calls (table, sequential pass, segments; execute_one's
proof).  Every arm's output is compared: trace_one's registers with the host VM's, execute_one's proof with dg.execute's and the K = 1
arms' results.  One JSON line per workload, then a markdown table; every line records the card's name and power limit.

Workloads: collatz at 2^16, 2^18 and 2^20 steps (bench.py's start values; the K = 1 arms are skipped at 2^20, about two minutes each),
fibonacci_program at 2^12 and 2^16 (straight-line: its table is as long as its trace), merkle at 2^14 (four depth-64 paths; RESCR-bound,
and RESCR stays in the sequential pass).

    python tools/trace_one_bench.py [--workloads collatz16,collatz18,collatz20,fib12,fib16,merkle14] [--no-batch]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench                                     # noqa: E402
import distaff_b200 as dg                        # noqa: E402
from distaff_b200 import backend, hostvm          # noqa: E402
from tests import execution_cases as cases        # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception:
        return backend.device_info()["name"], "unknown"


def workload(name):
    """(source, ProgramInputs, num_outputs, K = 1 arms run)"""
    if name.startswith("collatz"):
        log_n = int(name[len("collatz"):])
        return hostvm.COLLATZ_SOURCE, dg.ProgramInputs(secret_a=[bench.collatz_start_for(log_n)]), 1, log_n < 20
    if name in ("fib12", "fib16"):
        return hostvm.fibonacci_program(250 if name == "fib12" else 4000), dg.ProgramInputs([1, 0]), 1, True
    src, a, b = cases.merkle_case(64, 4)
    return src, dg.ProgramInputs(secret_a=a, secret_b=b), 4, True


def timed(f):
    t = time.perf_counter()
    r = f()
    return r, time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="collatz16,collatz18,collatz20,fib12,fib16,merkle14")
    ap.add_argument("--no-batch", action="store_true", help="skip the K = 1 trace_batch / execute_batch arms")
    args = ap.parse_args()
    name, power = card()
    warm = dg.ProgramInputs(secret_a=[7])
    dg.trace_one(hostvm.COLLATZ_SOURCE, warm)
    dg.execute_one(hostvm.COLLATZ_SOURCE, warm)
    dg.execute(hostvm.COLLATZ_SOURCE, secret_a=[7])
    rows = []
    for w in args.workloads.split(","):
        src, x, no, batch = workload(w)
        batch = batch and not args.no_batch
        line = {"workload": w, "gpu": name, "power_limit": power}
        host, line["hostvm_s"] = timed(lambda: hostvm.execute(src, x.public, x.secret_a, x.secret_b, no))
        line["steps"] = int(host.length)
        proof, line["prove_s"] = timed(lambda: dg.prove(host))
        line["dg_execute_s"] = line["hostvm_s"] + line["prove_s"]
        st = {}
        tr, line["trace_one_s"] = timed(lambda: dg.trace_one(src, x, num_outputs=no, stats=st))
        line["trace_one"] = st
        line["trace_one_matches"] = bool(np.array_equal(tr.registers, host.registers))
        st2 = {}
        one, line["execute_one_s"] = timed(lambda: dg.execute_one(src, x, no, stats=st2))
        line["execute_one"] = st2
        line["execute_one_prove_ms"] = one[1].stats["total_ms"]
        line["execute_one_matches"] = one[0] == host.outputs and one[1].bytes == proof.bytes
        if batch:
            tb, line["trace_batch_s"] = timed(lambda: dg.trace_batch(src, [x], num_outputs=no)[0])
            eb, line["execute_batch_s"] = timed(lambda: dg.execute_batch(src, [x], no)[0])
            line["batch_matches"] = bool(np.array_equal(tb.registers, host.registers)) and eb[1].bytes == proof.bytes
        print(json.dumps(line), flush=True)
        rows.append(line)
    print(f"\non {name} at a {power} power limit; wall seconds of one call\n")
    print("| workload | steps | trace_one s (table / sequential / segments ms) | execute_one s | hostvm s | dg.execute s | trace_batch K=1 s | "
          "execute_batch K=1 s | execute_one vs dg.execute |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        s = r["trace_one"]
        print(f"| {r['workload']} | {r['steps']} | {r['trace_one_s']:.3f} ({s['table_ms']:.1f} / {s['sequential_ms']:.1f} / {s['segment_ms']:.1f}) | "
              f"{r['execute_one_s']:.3f} | {r['hostvm_s']:.3f} | {r['dg_execute_s']:.3f} | "
              f"{r.get('trace_batch_s', float('nan')):.3f} | {r.get('execute_batch_s', float('nan')):.3f} | "
              f"{r['dg_execute_s'] / r['execute_one_s']:.1f}x |")


if __name__ == "__main__":
    main()
