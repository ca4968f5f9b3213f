#!/usr/bin/env python3
"""Many executions in one call: trace_many / execute_many (the programs' sponge tables, one sequential launch for every execution, the
rows written by one thread per checkpoint in waves) against trace_programs / execute_programs (every execution on one GPU thread with
the sponge rounds) on the same jobs, and the host VM (hostvm.execute, plus dg.prove for the proofs: dg.execute) where it takes seconds.
After a warm-up call of every arm, the GPU arms run alternating, `--reps` times each, and every result is compared byte for byte with
the other arm's.  Wall seconds of one call (best and median), the tabled call's device phases, one JSON line per workload, then a
markdown table; every line records the card's name and power limit.

Workloads:
  collatz16 / collatz256 / collatz1024   collatz on K seeded starts below 1000 (traces up to 2^16 rows): the loop-heavy case
  collatz20x8                            8 collatz executions of 2^20 steps (bench.py's start), against 8 execute_one / trace_one calls
  suite                                  the 17 jobs of tests/execution_cases.py (16 programs)
  fib12x256                              fibonacci_program at 2^12 steps on 256 inputs: straight-line, where no gain is expected

    python tools/many_bench.py [--workloads collatz16,collatz256,collatz1024,collatz20x8,suite,fib12x256] [--reps 2] [--sweep 256,4096]
"""
import argparse
import json
import os
import random
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench                                     # noqa: E402
import distaff_b200 as dg                        # noqa: E402
from distaff_b200 import hostvm                   # noqa: E402
from tests import execution_cases as cases        # noqa: E402
from tools.trace_one_bench import card            # noqa: E402

X = dg.ProgramInputs


def workload(name):
    """(jobs, the other GPU arm: "programs" or "one", host VM arm run)"""
    if name.startswith("collatz") and "x" not in name:
        k = int(name[len("collatz"):])
        rnd = random.Random(k)
        return [(hostvm.COLLATZ_SOURCE, X(secret_a=[rnd.randrange(1, 1000)])) for _ in range(k)], "programs", k <= 16
    if name == "collatz20x8":
        return [(hostvm.COLLATZ_SOURCE, X(secret_a=[bench.collatz_start_for(20)]))] * 8, "one", False
    if name == "suite":
        return [(src, X(pub, a, b), no) for _, src, pub, a, b, no in cases.SMALL], "programs", True
    fib = hostvm.fibonacci_program(250)
    return [(fib, X([i + 1, i])) for i in range(256)], "programs", False


def timed(f):
    t = time.perf_counter()
    r = f()
    return r, time.perf_counter() - t


def same_traces(a, b):
    return all(type(x) is type(y) and (str(x) == str(y) if isinstance(x, Exception) else np.array_equal(x.registers, y.registers))
               for x, y in zip(a, b)) and len(a) == len(b)


def same_proofs(a, b):
    return all(type(x) is type(y) and (str(x) == str(y) if isinstance(x, Exception) else (x[0] == y[0] and x[1].bytes == y[1].bytes))
               for x, y in zip(a, b)) and len(a) == len(b)


def other_arm(kind, jobs, prove):
    if kind == "programs":
        return (lambda: dg.execute_programs(jobs)) if prove else (lambda: dg.trace_programs(jobs))
    if prove:
        return lambda: [dg.execute_one(j[0], j[1], j[2] if len(j) == 3 else 1) for j in jobs]
    return lambda: [dg.trace_one(j[0], j[1], num_outputs=j[2] if len(j) == 3 else 1) for j in jobs]


def summary(times):
    return {"best": min(times), "median": statistics.median(times)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="collatz16,collatz256,collatz1024,collatz20x8,suite,fib12x256")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--sweep", default="", help="segment_steps values to time trace_many at besides the default, e.g. 256,4096")
    args = ap.parse_args()
    name, power = card()
    warm = [(hostvm.COLLATZ_SOURCE, X(secret_a=[7])), (hostvm.fibonacci_program(13), X([1, 0]))]
    dg.trace_many(warm), dg.execute_many(warm), dg.trace_programs(warm), dg.execute_programs(warm)
    rows = []
    for w in args.workloads.split(","):
        jobs, kind, host = workload(w)
        line = {"workload": w, "executions": len(jobs), "other": kind, "gpu": name, "power_limit": power}
        for prove in (False, True):
            tag = "execute" if prove else "trace"
            many_st = {}
            many = (lambda: dg.execute_many(jobs, stats=many_st)) if prove else (lambda: dg.trace_many(jobs, stats=many_st))
            other = other_arm(kind, jobs, prove)
            a, b = many(), other()                                      # warm-up of both arms, and the comparison
            line[f"{tag}_matches"] = same_proofs(a, b) if prove else same_traces(a, b)
            if not prove:
                line["max_length"] = max(int(t.length) for t in a if not isinstance(t, Exception))
            ta, tb = [], []
            for _ in range(args.reps):
                ta.append(timed(many)[1])
                tb.append(timed(other)[1])
            line[f"{tag}_many_s"], line[f"{tag}_other_s"] = summary(ta), summary(tb)
            line[f"{tag}_many_stats"] = many_st
        for s in [int(v) for v in args.sweep.split(",") if v]:
            st = {}
            _, t = timed(lambda: dg.trace_many(jobs, segment_steps=s, stats=st))
            line.setdefault("sweep", []).append({"segment_steps": s, "trace_s": t, "segments": st["segments"],
                                                 "sequential_ms": st["sequential_ms"], "segment_ms": st["segment_ms"]})
        if host:
            def run_host():
                return [hostvm.execute(j[0], j[1].public, j[1].secret_a, j[1].secret_b, j[2] if len(j) == 3 else 1) for j in jobs]
            traces, line["hostvm_s"] = timed(run_host)
            _, line["dg_execute_s"] = timed(lambda: [dg.prove(t) for t in traces])
            line["dg_execute_s"] += line["hostvm_s"]
        print(json.dumps(line), flush=True)
        rows.append(line)
    print(f"\non {name} at a {power} power limit; wall seconds of one call (best of {args.reps})\n")
    print("| workload | K | longest trace | traces: many / other | with proofs: many / other | host VM (+ prove) | bytes equal |")
    print("|---|---|---|---|---|---|---|")
    for r in rows:
        h = f"{r['hostvm_s']:.2f} ({r['dg_execute_s']:.2f})" if "hostvm_s" in r else "not run"
        other = "trace_programs" if r["other"] == "programs" else f"{r['executions']} x one"
        print(f"| {r['workload']} | {r['executions']} | 2^{int(r['max_length']).bit_length() - 1} | {r['trace_many_s']['best']:.3f} / "
              f"{r['trace_other_s']['best']:.3f} ({other}) | {r['execute_many_s']['best']:.3f} / {r['execute_other_s']['best']:.3f} | {h} | "
              f"{r['trace_matches'] and r['execute_matches']} |")


if __name__ == "__main__":
    main()
