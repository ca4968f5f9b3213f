#!/usr/bin/env python3
"""Kernel time of the constraint evaluation (constraint_eval_smem_kernel) through dg_eval_transitions, for A/B comparisons of builds.

The extended trace is random (every op flag non-binary, so every term of every constraint contributes) with the register shape of the
collatz workload (w = 26).  dg_eval_transitions accepts LDE domains of at most 2^20 rows, so the default is n = 2^16 steps at blowup 16:
2^19 evaluation points, 4096 blocks of 128 threads.  The kernel's device time is read from torch.profiler (CUDA activities) around
--reps calls after --warmup calls, and the median is reported.
    python tools/air_ab.py [--log-n 16] [--log-blowup 4] [--reps 12] [--warmup 2]
    python tools/air_ab.py --alternate LIB_A LIB_B [--rounds 4]     # one process per run (DG_LIB_PATH), the builds alternating
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

KERNEL = "constraint_eval_smem_kernel"


def random_ext(w, rows, seed):
    """canonical field elements: a high limb below 2^64 - 1 keeps every value below M"""
    rng = np.random.default_rng(seed)
    a = np.empty((1, w, rows, 2), dtype=np.uint64)
    a[..., 0] = rng.integers(0, 2**64, size=(1, w, rows), dtype=np.uint64)
    a[..., 1] = rng.integers(0, 2**64 - 1, size=(1, w, rows), dtype=np.uint64)
    return a


def run_once(args):
    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    import distaff_b200 as dg
    from distaff_b200 import backend, hostvm
    tr = hostvm.collatz(7)
    shape = (tr.ctx_depth, tr.loop_depth, tr.stack_depth)
    n, b = 1 << args.log_n, 1 << args.log_blowup
    ext = random_ext(tr.width, n * b, 1234)
    seeds = [bytes(range(32))]
    for _ in range(args.warmup):
        dg.eval_transitions(ext, *shape, b, seeds=seeds)
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.reps):
            dg.eval_transitions(ext, *shape, b, seeds=seeds)
    times = [e.device_time_total / 1000.0 for e in prof.events() if e.device_type == DeviceType.CUDA and KERNEL in e.name]
    if len(times) != args.reps:
        raise SystemExit("expected %d %s launches in the profile, found %d" % (args.reps, KERNEL, len(times)))
    gpu = torch.cuda.get_device_properties(0).name
    print(json.dumps({"lib": backend.LIB_PATH, "device": gpu, "shape": shape, "w": tr.width, "log_n": args.log_n, "blowup": b,
                      "points": 8 * n, "reps": args.reps, "kernel_ms_median": statistics.median(times),
                      "kernel_ms_min": min(times), "kernel_ms_max": max(times)}))


def alternate(args):
    results = {lib: [] for lib in args.alternate}
    cmd = [sys.executable, os.path.abspath(__file__), "--log-n", str(args.log_n), "--log-blowup", str(args.log_blowup),
           "--reps", str(args.reps), "--warmup", str(args.warmup)]
    for _ in range(args.rounds):
        for lib in args.alternate:
            out = subprocess.run(cmd, env=dict(os.environ, DG_LIB_PATH=os.path.abspath(lib)), check=True, capture_output=True, text=True)
            line = json.loads(out.stdout.strip().splitlines()[-1])
            print(json.dumps(line), flush=True)
            results[lib].append(line["kernel_ms_median"])
    for lib, ms in results.items():
        print(json.dumps({"lib": lib, "runs": ms, "mean_ms": statistics.mean(ms), "spread_ms": max(ms) - min(ms)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", type=int, default=16)
    ap.add_argument("--log-blowup", type=int, default=4)
    ap.add_argument("--reps", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--alternate", nargs="+", metavar="LIB", help="builds of libdistaff_gpu.so to compare, one process per run")
    ap.add_argument("--rounds", type=int, default=4)
    args = ap.parse_args()
    if args.reps < 10:
        ap.error("--reps must be at least 10")
    alternate(args) if args.alternate else run_once(args)


if __name__ == "__main__":
    main()
