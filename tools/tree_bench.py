#!/usr/bin/env python3
"""Merkle trees kept in device memory (MerkleTree, dg_tree_*) against building the tree again, one JSON line per case; every line records
the card's name and power limit, read in the same run.

  update      dg_tree_update of K random leaves (repeats allowed, so K may exceed L) of a tree of L leaves: wall ms of the call, which
              plans on the host, uploads once, runs one level pass per level (or, when the plan hashes at least half the nodes, builds
              the tree again) and ends in a device synchronise when it reads the root (best of --reps after a warm-up), the digests its
              plan holds, the path it took and its launches; beside it dg_dev_merkle_build_with of the same
              leaves, device ms (CUDA events) and wall ms of the call.
  paths       dg_tree_paths of 256 random leaves: wall ms of the call (one launch, the paths copied back).
  membership  --members leaves of a 2^20-leaf hasher tree, end to end, MerkleTree next to HasherTree: wall seconds to build the tree,
              to get the paths and lay out the smpath inputs, and to run prove_membership (one execute_batch call with proofs).

    python tools/tree_bench.py [--logs 14,20] [--ks 1,16,256,4096,65536] [--reps 3] [--members 256]
"""
import argparse
import ctypes
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import distaff_b200 as dg                        # noqa: E402
from distaff_b200 import backend                 # noqa: E402
from tools.trace_one_bench import card            # noqa: E402

HASH_NAMES = {0: "blake3", 3: "hasher"}


def random_leaves(L, seed):
    """L x 32 bytes of canonical field elements (each below 2^127 < M)"""
    return np.random.default_rng(seed).integers(0, 2**63, size=(L, 2, 2), dtype=np.uint64).tobytes()


def best_wall(fn, reps):
    fn()
    best = None
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        dt = (time.perf_counter() - t) * 1e3
        best = dt if best is None else min(best, dt)
    return best


def plan_digests(indexes, L):
    nodes, total = {L + i for i in indexes}, 0
    while nodes != {1}:
        nodes = {q >> 1 for q in nodes}
        total += len(nodes)
    return total


def rebuild_ms(hash_id, leaves, L, reps):
    d_leaves = backend.DeviceBuffer(L * 32).upload(np.frombuffer(leaves, dtype=np.uint8))
    d_nodes = backend.DeviceBuffer(L * 32)
    ms = ctypes.c_float(0)
    dev = []

    def once():
        backend.check(backend.lib().dg_dev_merkle_build_with(hash_id, d_leaves.ptr, L, d_nodes.ptr, ctypes.byref(ms)))
        dev.append(ms.value)
    wall = best_wall(once, reps)
    d_leaves.free()
    d_nodes.free()
    return min(dev[1:]), wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logs", default="14,20")
    ap.add_argument("--ks", default="1,16,256,4096,65536")
    ap.add_argument("--hashes", default="0,3")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--members", type=int, default=256)
    args = ap.parse_args()
    name, power = card()
    base = {"gpu": name, "power_limit": power}

    for hash_id in (int(h) for h in args.hashes.split(",")):
        hash = HASH_NAMES[hash_id]
        for lg in (int(x) for x in args.logs.split(",")):
            L = 1 << lg
            leaves = random_leaves(L, lg)
            rb_dev, rb_wall = rebuild_ms(hash_id, leaves, L, args.reps)
            with dg.MerkleTree(leaves, hash) as tree:
                rng = random.Random(lg)
                for K in (int(k) for k in args.ks.split(",")):
                    idx = [rng.randrange(L) for _ in range(K)]
                    new = random_leaves(K, K)
                    wall = best_wall(lambda: tree.update(idx, new), args.reps)
                    digests = plan_digests(idx, L)
                    rebuilds = 2 * digests >= L - 1                      # tree_update_rebuilds: the call builds the tree again
                    line = dict(base, case="update", hash=hash, leaves=L, k=K, unique=len(set(idx)), digests=digests, rebuild_digests=L - 1,
                                path="rebuild" if rebuilds else "levels", launches=lg + 1 if rebuilds else 2 * lg + 1, update_call_ms=round(wall, 3), rebuild_device_ms=round(rb_dev, 3),
                                rebuild_call_ms=round(rb_wall, 3), update_over_rebuild=round(wall / rb_wall, 3))
                    print(json.dumps(line), flush=True)
                idx = [rng.randrange(L) for _ in range(256)]
                wall = best_wall(lambda: tree.paths(idx), args.reps)
                print(json.dumps(dict(base, case="paths", hash=hash, leaves=L, k=256, entries=tree.depth, paths_call_ms=round(wall, 3))), flush=True)

    if args.members:
        L = 1 << 20
        raw = np.frombuffer(random_leaves(L, 2), dtype=np.uint64).reshape(-1, 2)
        ints = [int(lo) | int(hi) << 64 for lo, hi in raw.tolist()]
        pairs = list(zip(ints[0::2], ints[1::2]))
        with dg.MerkleTree([(1, 2), (3, 4)] * 2, "hasher") as warm:      # warm-up: module load, constants, prover tables of the smpath trace
            dg.prove_membership(warm, [0])
        idx = random.Random(3).sample(range(L), args.members)
        out = {}
        for arm in ("MerkleTree", "HasherTree"):
            t0 = time.perf_counter()
            tree = dg.MerkleTree(pairs, "hasher") if arm == "MerkleTree" else dg.HasherTree(pairs)
            t1 = time.perf_counter()
            if arm == "MerkleTree":
                tree._membership_inputs(idx, "smpath")
            else:
                [tree.smpath_inputs(i) for i in idx]
            t2 = time.perf_counter()
            res = dg.prove_membership(tree, idx, "smpath")
            t3 = time.perf_counter()
            out[arm] = [r[3].bytes if isinstance(r, tuple) else None for r in res]
            print(json.dumps(dict(base, case="membership", tree=arm, leaves=L, members=args.members, program="smpath", build_s=round(t1 - t0, 3),
                                  paths_and_inputs_s=round(t2 - t1, 3), prove_membership_s=round(t3 - t2, 3),
                                  all_output_root=all(b is not None for b in out[arm]))), flush=True)
            if arm == "MerkleTree":
                tree.close()
        print(json.dumps(dict(base, case="membership_bytes_equal", equal=out["MerkleTree"] == out["HasherTree"])), flush=True)


if __name__ == "__main__":
    main()
