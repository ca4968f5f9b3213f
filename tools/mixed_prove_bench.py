#!/usr/bin/env python3
"""Throughput of batched proving across register shapes: one prove_traces call (dg_prove_traces) against prove_batch, which makes one
dg_prove_batch call per register shape.

Workloads:
  suite   the traces of the 16 distinct programs of tests/execution_cases.py SMALL (2^5 to 2^11 steps, 14 shapes)
  mix8    4 register shapes x --per-shape traces of 2^8 steps (fibonacci programs behind 0 / 4 / 8 / 12 pushes and 0 / 0 / 1 / 2 blocks)
  mix12   the same at 2^12 steps

For every workload the script prints one JSON line: proofs/s (wall clock) and device ms of both arms, their kernel launches and calls,
the speed-up of prove_traces, and whether both arms gave the same bytes (a workload whose proofs differ is reported as an error, not as a
result).  Each arm is warmed up once; then the two arms alternate, call by call, for --rounds rounds.  The first line names the card and
its power limit (read-only nvidia-smi query).

    python tools/mixed_prove_bench.py [--workloads suite,mix8,mix12] [--per-shape 16] [--rounds 5]
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


def suite():
    from tests import execution_cases as cases
    seen, traces = set(), []
    for _, src, pub, a, b, no in cases.SMALL:
        if src in seen:
            continue
        seen.add(src)
        traces.append(hostvm.execute(src, public_inputs=pub, secret_a=a, secret_b=b, num_outputs=no))
    return traces


def fib_variant(extra, blocks, log_n, k):
    """a fibonacci program behind `extra` pushes and inside `blocks` nested blocks, with the most terms whose trace has 2^log_n steps"""
    def source(terms):
        body = hostvm.fibonacci_program(terms)[len("begin "):-len(" end")]
        for _ in range(blocks):
            body = "block " + body + " end"
        return "begin " + "".join("push.%d " % (i + 1) for i in range(extra)) + body + " end"
    terms = (1 << log_n) // 16
    while terms > 2:
        tr = hostvm.execute(source(terms), public_inputs=[1 + k, k], num_outputs=1)
        if tr.length == 1 << log_n:
            return tr
        terms -= 1 if tr.length < (4 << log_n) else max(1, terms // 8)
    raise RuntimeError("no fibonacci variant of 2^%d steps with %d pushes and %d blocks" % (log_n, extra, blocks))


def mix(log_n, per_shape):
    variants = [(0, 0), (4, 0), (8, 1), (12, 2)]
    traces = [fib_variant(e, b, log_n, k) for k in range(per_shape) for (e, b) in variants]
    assert len({(t.width, t.ctx_depth, t.loop_depth) for t in traces}) == len(variants)
    return traces


def run_traces(traces, opts):
    t0 = time.perf_counter()
    proofs = dg.prove_traces(traces, opts)
    wall = time.perf_counter() - t0
    st = proofs[0].stats
    return proofs, wall, st["total_ms"], st["kernel_launches"], 1


def run_batch(traces, opts):
    """prove_batch, one dg_prove_batch call per shape: its calls made here one by one, so that their stats add up"""
    groups = {}
    for i, t in enumerate(traces):
        groups.setdefault((t.width, t.length, t.ctx_depth, t.loop_depth), []).append(i)
    proofs = [None] * len(traces)
    wall = dev = 0.0
    launches = 0
    for idx in groups.values():
        t0 = time.perf_counter()
        out = dg.prove_batch([traces[i] for i in idx], opts)
        wall += time.perf_counter() - t0
        dev += out[0].stats["total_ms"]
        launches += out[0].stats["kernel_launches"]
        for i, p in zip(idx, out):
            proofs[i] = p
    return proofs, wall, dev, launches, len(groups)


def bench(name, traces, rounds, opts):
    arms = {"prove_traces": run_traces, "prove_batch": run_batch}
    first = {a: f(traces, opts) for a, f in arms.items()}                     # warm-up, and the bytes of both arms
    same = [p.bytes for p in first["prove_traces"][0]] == [p.bytes for p in first["prove_batch"][0]]
    line = {"workload": name, "traces": len(traces), "shapes": len({(t.width, t.ctx_depth, t.loop_depth) for t in traces}),
            "lengths": sorted({t.length for t in traces}), "identical": same}
    if not same:
        line["error"] = "prove_traces and prove_batch gave different proofs"
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
        line[a + "_device_ms"] = round(statistics.median(devs[a]), 2)
    line["speedup"] = round(line["prove_traces_proofs_per_s"] / line["prove_batch_proofs_per_s"], 3)
    return line


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workloads", default="suite,mix8,mix12")
    ap.add_argument("--per-shape", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    print(json.dumps(card()), flush=True)
    opts = dg.ProofOptions()
    make = {"suite": suite, "mix8": lambda: mix(8, args.per_shape), "mix12": lambda: mix(12, args.per_shape)}
    for name in args.workloads.split(","):
        print(json.dumps(bench(name, make[name](), args.rounds, opts)), flush=True)


if __name__ == "__main__":
    main()
