#!/usr/bin/env python3
"""Throughput of per-trace proof options: one prove_traces call with a list of ProofOptions (dg_prove_traces_with_options) against one
prove_traces call per option set (the way a caller proves a mix of security levels without per-trace options).

Workloads: fibonacci traces of 2^8 and 2^12 steps (--sizes), --per-set traces per option set, the option sets (extension factor,
num_queries, grinding factor) of --sets (default 32/50/20, 32/96/24 and 16/50/20), interleaved.  Only option sets that share a (length,
extension factor) partition can share a group: here the first two.

For every size the script prints one JSON line: proofs/s (wall clock) and device ms of both arms, their kernel launches and calls, the
speed-up of the mixed call, and whether both arms gave the same bytes (a workload whose proofs differ is reported as an error, not as a
result).  Each arm is warmed up once; then the two arms alternate, call by call, for --rounds rounds.  The first line names the card and
its power limit (read-only nvidia-smi query).

    python tools/mixed_options_bench.py [--sizes 8,12] [--per-set 16] [--rounds 5] [--sets 32/50/20,32/96/24,16/50/20]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import distaff_b200 as dg                        # noqa: E402
from distaff_b200 import hostvm                   # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, power = [x.strip() for x in out[0].split(",")]
        return {"card": name, "power_limit": power}
    except Exception as e:          # the proofs below still need the device; this only labels the numbers
        return {"card": "unknown", "power_limit": "unknown", "nvidia_smi_error": str(e)}


def fib_traces(log_n, count):
    """count fibonacci traces of 2^log_n steps on different inputs"""
    terms = (1 << log_n) // 16 - 3
    out = [hostvm.execute(hostvm.fibonacci_program(terms), public_inputs=[1 + k, k], num_outputs=1) for k in range(count)]
    assert all(t.length == 1 << log_n for t in out), (log_n, {t.length for t in out})
    return out


def run_mixed(traces, opts):
    t0 = time.perf_counter()
    proofs = dg.prove_traces(traces, opts)
    wall = time.perf_counter() - t0
    st = proofs[0].stats
    return proofs, wall, st["total_ms"], st["kernel_launches"], 1


def run_split(traces, opts):
    """one prove_traces call per option set, in order of first appearance"""
    sets = {}
    for i, o in enumerate(opts):
        sets.setdefault(o, []).append(i)
    proofs = [None] * len(traces)
    wall = dev = 0.0
    launches = 0
    for o, idx in sets.items():
        t0 = time.perf_counter()
        out = dg.prove_traces([traces[i] for i in idx], o)
        wall += time.perf_counter() - t0
        dev += out[0].stats["total_ms"]
        launches += out[0].stats["kernel_launches"]
        for i, p in zip(idx, out):
            proofs[i] = p
    return proofs, wall, dev, launches, len(sets)


def bench(log_n, traces, opts, rounds):
    arms = {"mixed": run_mixed, "per_set": run_split}
    first = {a: f(traces, opts) for a, f in arms.items()}                     # warm-up, and the bytes of both arms
    same = [p.bytes for p in first["mixed"][0]] == [p.bytes for p in first["per_set"][0]]
    line = {"log_n": log_n, "traces": len(traces), "sets": sorted({(o.extension_factor, o.num_queries, o.grinding_factor) for o in opts}),
            "partitions": len({o.extension_factor for o in opts}), "identical": same}
    if not same:
        line["error"] = "the mixed call and the per-set calls gave different proofs"
        return line
    walls = {a: [] for a in arms}
    devs = {a: [] for a in arms}
    for _ in range(rounds):
        for a, f in arms.items():                                          # the arms alternate, call by call
            _, wall, dev, launches, calls = f(traces, opts)
            walls[a].append(wall)
            devs[a].append(dev)
            line[a + "_launches"] = launches
            line[a + "_calls"] = calls
    for a in arms:
        w = statistics.median(walls[a])
        line[a + "_proofs_per_s"] = round(len(traces) / w, 1)
        line[a + "_wall_ms"] = round(1e3 * w, 2)
        line[a + "_wall_ms_spread"] = [round(1e3 * min(walls[a]), 2), round(1e3 * max(walls[a]), 2)]
        line[a + "_device_ms"] = round(statistics.median(devs[a]), 2)
    line["speedup"] = round(line["mixed_proofs_per_s"] / line["per_set_proofs_per_s"], 3)
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--sizes", default="8,12")
    ap.add_argument("--per-set", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--sets", default="32/50/20,32/96/24,16/50/20")
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    sets = [dg.ProofOptions(*[int(x) for x in s.split("/")]) for s in args.sets.split(",")]
    for log_n in [int(x) for x in args.sizes.split(",")]:
        traces = fib_traces(log_n, args.per_set * len(sets))
        opts = [sets[i % len(sets)] for i in range(len(traces))]
        print(json.dumps(bench(log_n, traces, opts, args.rounds)), flush=True)


if __name__ == "__main__":
    main()
