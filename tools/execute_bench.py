#!/usr/bin/env python3
"""Batched execution against the host VM: traces/s and steps/s of trace_batch (the VM on the GPU, one thread per execution) and of
hostvm on one process and on all cores, and of execute_batch (VM and proofs on the GPU) against hostvm on all cores followed by
prove_batch.  One JSON line per (workload, K), then a markdown table.

Workloads: fibonacci at 2^12 and 2^16 steps (different public inputs), merkle depth 32 (different paths under one leaf index), collatz
over many starts (mixed lengths).  K = 1, 16, 256, 1024 by default.  Host-VM times are measured on a sample of the executions (--host-
sample per process, one round of the pool) and scaled to K; the lines say so.  Every line records the card's name and power limit.

    python tools/execute_bench.py [--ks 1,16,256,1024] [--workloads fib12,fib16,merkle32,collatz] [--no-prove]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

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


def workload(name, k):
    """(source, [ProgramInputs] of k executions, num_outputs)"""
    if name in ("fib12", "fib16"):
        n = 250 if name == "fib12" else 4000
        return hostvm.fibonacci_program(n), [dg.ProgramInputs([i + 1, 3 * i]) for i in range(k)], 1
    if name == "merkle32":
        inputs, src = [], None
        for seed in range(k):
            src, a, b = cases.merkle_case(32, 1, seed=seed, index_of=lambda c: 123456)
            inputs.append(dg.ProgramInputs(secret_a=a, secret_b=b))
        return src, inputs, 4
    return hostvm.COLLATZ_SOURCE, [dg.ProgramInputs(secret_a=[3 + 2 * i]) for i in range(k)], 1


def host_one(args):
    src, pub, a, b, no = args
    return hostvm.execute(src, pub, a, b, no)


def host_args(src, inputs, no):
    return [(src, x.public, x.secret_a, x.secret_b, no) for x in inputs]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1,16,256,1024")
    ap.add_argument("--workloads", default="fib12,fib16,merkle32,collatz")
    ap.add_argument("--host-sample", type=int, default=2, help="executions timed on one host process (then scaled to K)")
    ap.add_argument("--no-prove", action="store_true")
    ap.add_argument("--max-trace-gb", type=float, default=8.0, help="skip trace_batch (host copies of every trace) above this many GB")
    args = ap.parse_args()
    name, power = card()
    cores = os.cpu_count() or 1
    pool = ProcessPoolExecutor(cores)
    rows = []
    for wl in args.workloads.split(","):
        for k in [int(x) for x in args.ks.split(",")]:
            src, inputs, no = workload(wl, k)
            prog = hostvm.compile_program(src)
            shapes = dg.trace_shapes(prog, inputs)
            assert not any(isinstance(x, backend.DgError) for x in shapes)
            steps = sum(s["length"] for s in shapes)                          # padded rows, as the prover sees them
            gpu_s = None
            if sum(16 * s["width"] * s["length"] for s in shapes) <= args.max_trace_gb * 2**30:
                dg.trace_batch(prog, inputs[:1], num_outputs=no)              # warm-up; the timed call runs two shape passes
                t = time.perf_counter()
                traces = dg.trace_batch(prog, inputs, num_outputs=no)
                gpu_s = time.perf_counter() - t
                assert not any(isinstance(x, backend.DgError) for x in traces)
            # host VM, one process: a sample, scaled to K
            sample = host_args(src, inputs[:min(k, args.host_sample)], no)
            t = time.perf_counter()
            for a in sample:
                host_one(a)
            host1_s = (time.perf_counter() - t) * k / len(sample)
            # host VM on all cores: one round of the pool, scaled to K
            rnd = host_args(src, inputs[:min(k, cores)], no)
            t = time.perf_counter()
            host_traces = list(pool.map(host_one, rnd))
            hostn_s = (time.perf_counter() - t) * max(1.0, k / len(rnd))
            line = {"workload": wl, "K": k, "length": max(s["length"] for s in shapes), "card": name, "power_limit": power, "host_cores": cores,
                    "trace_batch_s": round(gpu_s, 4) if gpu_s else None, "trace_batch_traces_per_s": round(k / gpu_s, 2) if gpu_s else None,
                    "trace_batch_steps_per_s": round(steps / gpu_s) if gpu_s else None,
                    "hostvm_1proc_s": round(host1_s, 4), "hostvm_allcores_s": round(hostn_s, 4),
                    "host_note": "host VM timed on %d (one process) and %d (pool) executions, scaled to K" % (len(sample), len(rnd))}
            if not args.no_prove:
                dg.execute_batch(prog, inputs[:1], num_outputs=no)
                t = time.perf_counter()
                res = dg.execute_batch(prog, inputs, num_outputs=no)
                exe_s = time.perf_counter() - t
                assert not any(isinstance(x, backend.DgError) for x in res)
                t = time.perf_counter()
                proofs = dg.prove_batch(host_traces)
                prove_s = (time.perf_counter() - t) * max(1.0, k / len(rnd))
                assert [p.bytes for p in proofs] == [r[1].bytes for r in res[:len(proofs)]]
                line.update(execute_batch_s=round(exe_s, 4), execute_batch_traces_per_s=round(k / exe_s, 2),
                            hostvm_allcores_plus_prove_batch_s=round(hostn_s + prove_s, 4))
            print(json.dumps(line), flush=True)
            rows.append(line)
    print("\n| workload | K | n | trace_batch s | hostvm 1 proc s | hostvm %d cores s | execute_batch s | hostvm %d cores + prove_batch s |" % (cores, cores))
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print("| %s | %d | 2^%d | %s | %.3f | %.3f | %s | %s |" % (r["workload"], r["K"], r["length"].bit_length() - 1,
                                                          r["trace_batch_s"] if r["trace_batch_s"] else "not measured", r["hostvm_1proc_s"],
                                                          r["hostvm_allcores_s"], r.get("execute_batch_s", "not measured"),
                                                          r.get("hostvm_allcores_plus_prove_batch_s", "not measured")))
    print("\ncard: %s, power limit %s" % (name, power))


if __name__ == "__main__":
    main()
