#!/usr/bin/env python3
"""Many programs in one call against one call per program: P programs x K inputs through one trace_programs / execute_programs call
(arm "one_call") and through P trace_batch / execute_batch calls (arm "per_program"), the two arms alternating for --rounds rounds.
One JSON line per (workload, mode, arm, round): wall seconds, the one call's shape_ms / write_ms / waves / lanes / launches, whether the
two arms gave the same bytes (traces, or proofs and outputs), and the card's name and power limit; then a markdown table of medians.

Workloads:
  suite  every distinct program of tests/execution_cases.py SMALL on its own inputs, K times each (traces of 2^5 to 2^11 rows)
  fib    P = --fib-programs fibonacci programs, hostvm.fibonacci_program(n) for n = 200, 201, ... (2^11 to 2^12 steps), K inputs each

    python tools/programs_bench.py [--workloads suite,fib] [--fib-programs 64] [--k 4] [--rounds 3] [--modes trace,execute]
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
from distaff_b200 import backend, hostvm          # noqa: E402
from tests import execution_cases as cases        # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, power


def workload(name, k, fib_programs):
    """[(program, [ProgramInputs] of k executions, num_outputs)], one entry per program"""
    if name == "suite":
        seen, progs = set(), []
        for _, src, pub, a, b, no in cases.SMALL:
            if src not in seen:
                seen.add(src)
                progs.append((hostvm.compile_program(src), [dg.ProgramInputs(pub, a, b)] * k, no))
        return progs
    return [(hostvm.compile_program(hostvm.fibonacci_program(200 + p)), [dg.ProgramInputs([i + 1, 3 * i + p]) for i in range(k)], 1)
            for p in range(fib_programs)]


def jobs_of(progs):
    """the jobs of all programs, interleaved: input i of every program before input i + 1 of any"""
    k = max(len(inputs) for _, inputs, _ in progs)
    return [(prog, inputs[i], no) for i in range(k) for prog, inputs, no in progs if i < len(inputs)]


def digest(results):
    out = []
    for r in results:
        assert not isinstance(r, backend.DgError), r
        out.append(r.registers.tobytes() if hasattr(r, "registers") else (tuple(r[0]), r[1].bytes))
    return out


def run(mode, arm, progs, jobs):
    """(wall seconds, results in job order, stats of the one call or None)"""
    stats = {}
    t = time.perf_counter()
    if arm == "one_call":
        res = (dg.trace_programs if mode == "trace" else dg.execute_programs)(jobs, stats=stats)
    else:
        by_prog = {}
        for prog, inputs, no in progs:
            if mode == "trace":
                by_prog[id(prog)] = dg.trace_batch(prog, inputs, num_outputs=no)
            else:
                by_prog[id(prog)] = dg.execute_batch(prog, inputs, num_outputs=no)
        pos = {id(p): 0 for p, _, _ in progs}
        res = []
        for prog, _, _ in jobs:
            res.append(by_prog[id(prog)][pos[id(prog)]])
            pos[id(prog)] += 1
        stats = None
    return time.perf_counter() - t, res, stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="suite,fib")
    ap.add_argument("--fib-programs", type=int, default=64)
    ap.add_argument("--k", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--modes", default="trace,execute")
    args = ap.parse_args()
    name, power = card()
    rows = []
    for wl in args.workloads.split(","):
        progs = workload(wl, args.k, args.fib_programs)
        jobs = jobs_of(progs)
        for mode in args.modes.split(","):
            for arm in ("one_call", "per_program"):             # warm-up: every shape and program once
                run(mode, arm, progs, jobs)
            times = {"one_call": [], "per_program": []}
            for r in range(args.rounds):
                got = {}
                for arm in (("one_call", "per_program") if r % 2 == 0 else ("per_program", "one_call")):
                    s, res, stats = run(mode, arm, progs, jobs)
                    got[arm] = digest(res)
                    times[arm].append(s)
                    line = {"workload": wl, "mode": mode, "arm": arm, "round": r, "programs": len(progs), "K": args.k, "executions": len(jobs),
                            "wall_s": round(s, 4), "card": name, "power_limit": power}
                    if stats:
                        line.update(shape_ms=round(stats["shape_ms"], 2), write_ms=round(stats["write_ms"], 2), waves=stats["waves"],
                                    lanes=stats["lanes"], shape_launches=stats["shape_launches"], write_launches=stats["write_launches"],
                                    prove_groups=stats["prove_groups"])
                    print(json.dumps(line), flush=True)
                same = got["one_call"] == got["per_program"]
                print(json.dumps({"workload": wl, "mode": mode, "round": r, "arms_byte_equal": same}), flush=True)
                assert same, "the two arms differ"
            rows.append((wl, mode, len(progs), args.k, statistics.median(times["one_call"]), statistics.median(times["per_program"])))
    print("\n| workload | mode | programs | K | one call s | one call per program s | speed-up |")
    print("|---|---|---|---|---|---|---|")
    for wl, mode, p, k, one, per in rows:
        print("| %s | %s | %d | %d | %.3f | %.3f | %.1fx |" % (wl, mode, p, k, one, per, per / one))
    print("\ncard: %s, power limit %s (medians of %d alternating rounds)" % (name, power, args.rounds))


if __name__ == "__main__":
    main()
