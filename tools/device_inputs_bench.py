#!/usr/bin/env python3
"""Program inputs built on the host against inputs in device memory, one JSON line per case; every line records the card's name and
power limit, read in the same run.  The two arms of a case alternate after a warm-up of each; lines give the median and the spread (min,
max) of --reps runs per arm.

  membership  prove_membership of K random leaves (smpath) of a 2^20-leaf hasher MerkleTree.  host: the paths from one dg_tree_paths call,
              unpacked and laid out as ProgramInputs in Python, then execute_batch (what prove_membership did before device inputs).
              device: MerkleTree.membership_inputs (one gather launch into device memory), then execute_programs_device.  Wall seconds
              of building the inputs and of the execute call, each ending in a device synchronise; proofs compared by SHA-256.
  collatz     execute_programs of collatz on --collatz inputs (starts 1 .. n) against execute_programs_device of the same inputs in one
              CUDA tensor: wall seconds of the call.  Proofs compared.

    python tools/device_inputs_bench.py [--ks 256,4096,65536] [--reps 3] [--collatz 1024] [--big-reps 1]
"""
import argparse
import hashlib
import json
import os
import random
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import distaff_b200 as dg                        # noqa: E402
from distaff_b200 import api, felt, hostvm        # noqa: E402
from tools.trace_one_bench import card            # noqa: E402


def host_membership_inputs(tree, indexes):
    """the smpath ProgramInputs of the leaves, from one paths() call, as prove_membership laid them out before device inputs"""
    inputs = []
    for i, entries in zip(indexes, tree.paths(indexes)):
        path = api._int_pairs(b"".join(entries))
        a, b, bits = [path[0][0]], [path[0][1]], i
        for node in path[1:]:
            a += [0, node[0]]
            b += [bits & 1, node[1]]
            bits >>= 1
        inputs.append(dg.ProgramInputs([], a, b))
    return inputs


def digest(results):
    h = hashlib.sha256()
    for r in results:
        h.update(r[1].bytes if isinstance(r, tuple) else repr(r).encode())
    return h.hexdigest()


def summary(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4)}


def membership(base, tree, prog, K, reps):
    idx = random.Random(K).sample(range(len(tree)), K)

    def host():
        t0 = time.perf_counter()
        inputs = host_membership_inputs(tree, idx)
        t1 = time.perf_counter()
        res = dg.execute_batch(prog, inputs, num_outputs=2)
        t2 = time.perf_counter()
        return t1 - t0, t2 - t1, digest(res)

    def device():
        t0 = time.perf_counter()
        x = tree.membership_inputs(idx, "smpath")
        t1 = time.perf_counter()
        res = dg.execute_programs_device([prog], [0] * K, x, num_outputs=2)
        t2 = time.perf_counter()
        return t1 - t0, t2 - t1, digest(res)
    arms = {"host": host, "device": device}
    times = {a: ([], []) for a in arms}
    digests = {a: set() for a in arms}
    for a, fn in arms.items():                 # warm-up
        digests[a].add(fn()[2])
    for _ in range(reps):
        for a, fn in arms.items():
            build, call, d = fn()
            times[a][0].append(build)
            times[a][1].append(call)
            digests[a].add(d)
    for a in arms:
        print(json.dumps(dict(base, case="membership", arm=a, leaves=len(tree), k=K, program="smpath", reps=reps,
                              build_inputs_s=summary(times[a][0]), execute_s=summary(times[a][1]),
                              total_s=summary([x + y for x, y in zip(*times[a])]))), flush=True)
    print(json.dumps(dict(base, case="membership_proofs_equal", k=K, equal=len(digests["host"] | digests["device"]) == 1)), flush=True)


def collatz(base, n, reps):
    import torch
    jobs = [(hostvm.COLLATZ_SOURCE, dg.ProgramInputs([], [s])) for s in range(1, n + 1)]
    programs, program_of, inputs, num_outputs = api.pack_jobs(jobs)
    t = torch.from_numpy(felt.from_ints(list(range(1, n + 1))).view(np.int64)).view(torch.uint64).to("cuda")
    x = dg.DeviceInputs(t, [(0, 0)] * n, [(s, 1) for s in range(n)], [(0, 0)] * n)
    arms = {"host": lambda: dg.execute_programs(jobs), "device": lambda: dg.execute_programs_device(programs, program_of, x, num_outputs)}
    times, digests = {a: [] for a in arms}, {a: set() for a in arms}
    for a, fn in arms.items():
        digests[a].add(digest(fn()))
    for _ in range(reps):
        for a, fn in arms.items():
            t0 = time.perf_counter()
            res = fn()
            times[a].append(time.perf_counter() - t0)
            digests[a].add(digest(res))
    for a in arms:
        print(json.dumps(dict(base, case="collatz", arm=a, executions=n, reps=reps, call_s=summary(times[a]))), flush=True)
    print(json.dumps(dict(base, case="collatz_proofs_equal", equal=len(digests["host"] | digests["device"]) == 1)), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="256,4096,65536")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--big-reps", type=int, default=1, help="runs per arm for K >= 65536, whose host arm takes minutes")
    ap.add_argument("--collatz", type=int, default=1024)
    args = ap.parse_args()
    name, power = card()
    base = {"gpu": name, "power_limit": power}
    if args.collatz:
        collatz(base, args.collatz, args.reps)
    ks = [int(k) for k in args.ks.split(",") if k]
    if ks:
        L = 1 << 20
        leaves = np.random.default_rng(2).integers(0, 2**63, size=(L, 2, 2), dtype=np.uint64).tobytes()
        prog = hostvm.compile_program(dg.smpath_program(21))
        with dg.MerkleTree(leaves, "hasher") as tree:
            for K in ks:
                membership(base, tree, prog, K, args.big_reps if K >= 65536 else args.reps)


if __name__ == "__main__":
    main()
