#!/usr/bin/env python3
"""Time of the trace check (dg_check_traces / dg_check_traces_device) against dg_prove of the same input, on one GPU.

Cases (one JSON line each):
  collatz20_device   the 2^20-step x 26-register collatz trace in device memory: check_traces_device vs prove_device
  collatz20_pinned   the same trace in pinned host memory: check_trace vs prove (both upload it)
  fib16_host         fibonacci, 2^16 steps, pageable host memory: check_trace vs prove
  fib8_batch64       64 fibonacci traces of 2^8 steps: one check_traces call vs one prove_batch call
Every arm is warmed up, then the check and prove arms alternate, call by call, --reps times each, with the device synchronised around
every call; the line gives the median and the minimum host wall time of each arm (the call as a user makes it, results on the host), the
prover's stage-3 device time for scale, and check_ok (the honest traces pass).  The first line names the card and its power limit.

  python tools/check_bench.py [--reps 7] [--warmup 2] [--cases collatz20_device,collatz20_pinned,fib16_host,fib8_batch64]
"""
import argparse
import importlib.util
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        name, power = [x.strip() for x in out[0].split(",")]
        return {"card": name, "power_limit": power}
    except Exception as e:          # the calls below still need the device; this only labels the numbers
        return {"card": "unknown", "power_limit": "unknown", "nvidia_smi_error": str(e)}


def collatz_2_20():
    spec = importlib.util.spec_from_file_location("bench", os.path.join(ROOT, "bench.py"))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    tr, _ = bench.build_trace(20)
    assert tr.length == 1 << 20
    return tr


def timed(fn, sync):
    sync()
    t0 = time.perf_counter()
    out = fn()
    sync()
    return (time.perf_counter() - t0) * 1e3, out


def compare(name, check, prove, reps, warmup, sync, extra):
    for _ in range(warmup):
        check()
        prove()
    check_ms, prove_ms, stage3 = [], [], []
    ok = True
    for _ in range(reps):
        ms, reports = timed(check, sync)
        check_ms.append(ms)
        ok = ok and all(r.ok for r in reports)
        ms, proofs = timed(prove, sync)
        prove_ms.append(ms)
        stage3.append(sum(p.stats["stage_ms"][2] for p in proofs) / len(proofs))
    line = {"case": name, "check_ms_median": round(statistics.median(check_ms), 3), "check_ms_min": round(min(check_ms), 3),
            "prove_ms_median": round(statistics.median(prove_ms), 3), "prove_ms_min": round(min(prove_ms), 3),
            "prove_stage3_ms_median": round(statistics.median(stage3), 3),
            "check_over_prove": round(statistics.median(check_ms) / statistics.median(prove_ms), 4), "check_ok": ok, "reps": reps}
    line.update(extra)
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cases", default="collatz20_device,collatz20_pinned,fib16_host,fib8_batch64")
    args = ap.parse_args()
    import torch
    import distaff_b200 as dg
    from distaff_b200 import backend, hostvm
    print(json.dumps(dict(card(), device=backend.device_info()["name"])), flush=True)
    sync = torch.cuda.synchronize
    cases = args.cases.split(",")

    if any(c.startswith("collatz20") for c in cases):
        tr = collatz_2_20()
        regs = np.ascontiguousarray(tr.registers)
        n, w = tr.length, tr.width
        shape = {"n": n, "w": w}
        if "collatz20_device" in cases:
            dbuf = backend.DeviceBuffer(regs.nbytes).upload(regs)
            compare("collatz20_device",
                    lambda: dg.check_traces_device(dbuf, 1, w, n, tr.ctx_depth, tr.loop_depth, [tr.public_inputs], [tr.outputs], [tr.program_hash]),
                    lambda: [dg.prove_device(dbuf, w, n, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs)],
                    args.reps, args.warmup, sync, shape)
            dbuf.free()
        if "collatz20_pinned" in cases:
            pinned = torch.empty(regs.nbytes, dtype=torch.uint8, pin_memory=True)
            pinned.numpy()[:] = regs.reshape(-1).view(np.uint8)
            tp = hostvm.ExecutionTrace(pinned.numpy().view(np.uint64).reshape(regs.shape), tr.ctx_depth, tr.loop_depth, tr.stack_depth,
                                       tr.program_hash, tr.public_inputs, tr.outputs)
            compare("collatz20_pinned", lambda: [dg.check_trace(tp, tp.program_hash)], lambda: [dg.prove(tp)], args.reps, args.warmup, sync,
                    dict(shape, upload_mb=round(regs.nbytes / 1e6, 1)))
    if "fib16_host" in cases:
        tr = hostvm.fibonacci((1 << 16) // 16 - 6)
        assert tr.length == 1 << 16
        compare("fib16_host", lambda: [dg.check_trace(tr, tr.program_hash)], lambda: [dg.prove(tr)], args.reps, args.warmup, sync,
                {"n": tr.length, "w": tr.width})
    if "fib8_batch64" in cases:
        traces = [hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[1 + i, i]) for i in range(64)]
        assert traces[0].length == 1 << 8
        hashes = [t.program_hash for t in traces]
        compare("fib8_batch64", lambda: dg.check_traces(traces, hashes), lambda: dg.prove_batch(traces), args.reps, args.warmup, sync,
                {"n": traces[0].length, "w": traces[0].width, "count": 64})


if __name__ == "__main__":
    main()
