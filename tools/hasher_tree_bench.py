#!/usr/bin/env python3
"""Merkle trees of the VM's hasher (utils::hasher::digest) on the GPU against the host, one JSON line per case; every line records the
card's name and power limit.

  tree        dg_dev_merkle_build_with(3) device time (CUDA events, best of --reps after a warm-up) at L leaves, split into the levels of
              fewer than 2^16 digests (narrow layout, 8 lanes per digest) and the wider ones (wide layout, a thread per digest).  The
              narrow levels of a tree are all the levels of a tree of min(L, 2^16) leaves, so their time is measured as that tree's.
  host        the oracle's or_hasher_digest on one CPU core (digests per second, measured), and the tree time extrapolated from it.
  membership  --members leaves of a 2^20-leaf tree: wall seconds to build the HasherTree (GPU, plus the copy into Python ints), to run
              prove_membership (one execute_batch call: the smpath program and its proofs) and to check every proof in one verify_batch.

    python tools/hasher_tree_bench.py [--logs 10,14,18,20,22] [--reps 3] [--members 256]
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
from oracle import pyoracle as po                # noqa: E402
from tools.trace_one_bench import card            # noqa: E402

WIDE_MIN = 1 << 16                                # HASHER_WIDE_MIN


def leaves_below_m(L, seed):
    """L leaves of 2 elements below 2^127 < M, as (L, 2, 2) uint64 limbs"""
    a = np.random.default_rng(seed).integers(0, 2**63, size=(L, 2, 2), dtype=np.uint64)
    a[:, :, 1] >>= 1
    return a


def tree_ms(d_leaves, d_nodes, L, reps):
    ms = ctypes.c_float(0)
    best = None
    for r in range(reps + 1):
        backend.check(backend.lib().dg_dev_merkle_build_with(3, d_leaves.ptr, L, d_nodes.ptr, ctypes.byref(ms)))
        if r and (best is None or ms.value < best):
            best = ms.value
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logs", default="10,14,18,20,22")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--members", type=int, default=256)
    args = ap.parse_args()
    name, power = card()
    base = {"gpu": name, "power_limit": power}

    # host arm: one core, the oracle's digest of 4 elements
    msg = b"".join(int(v).to_bytes(16, "little") for v in (1, 2, 3, 4))
    out = ctypes.create_string_buffer(32)
    n_host = 300
    t = time.perf_counter()
    for _ in range(n_host):
        po.lib().or_hasher_digest(msg, 4, out)
    host_rate = n_host / (time.perf_counter() - t)

    logs = [int(x) for x in args.logs.split(",")]
    L_max = 1 << max(logs)
    d_leaves = backend.DeviceBuffer(L_max * 32).upload(leaves_below_m(L_max, 1))
    d_nodes = backend.DeviceBuffer(L_max * 32)
    for lg in logs:
        L = 1 << lg
        total = tree_ms(d_leaves, d_nodes, L, args.reps)
        narrow = tree_ms(d_leaves, d_nodes, min(L, WIDE_MIN), args.reps) if L > WIDE_MIN else total
        line = dict(base, case="tree", leaves=L, digests=L - 1, device_ms=round(total, 3), narrow_levels_ms=round(narrow, 3),
                    wide_levels_ms=round(total - narrow, 3), narrow_levels=min(lg, 16), wide_levels=max(lg - 16, 0),
                    gpu_digests_per_s=round((L - 1) / (total / 1e3)),
                    host_digests_per_s_one_core=round(host_rate), host_tree_s_extrapolated=round((L - 1) / host_rate, 1))
        print(json.dumps(line), flush=True)
    del d_leaves, d_nodes

    if args.members:
        L = 1 << 20
        raw = leaves_below_m(L, 2)
        v = raw.reshape(-1, 2)
        ints = [int(lo) | int(hi) << 64 for lo, hi in v.tolist()]
        leaves = list(zip(ints[0::2], ints[1::2]))
        dg.HasherTree(leaves[:WIDE_MIN * 2])                      # warm-up: module load, constants, prover tables of the smpath trace
        warm = dg.HasherTree([(1, 2), (3, 4)] * 2)
        dg.prove_membership(warm, [0])
        t0 = time.perf_counter()
        tree = dg.HasherTree(leaves)
        t1 = time.perf_counter()
        idx = random.Random(3).sample(range(L), args.members)
        res = dg.prove_membership(tree, idx, "smpath")
        t2 = time.perf_counter()
        bad = [r for r in res if not isinstance(r, tuple)]
        verdicts = dg.verify_batch(res) if not bad else []
        t3 = time.perf_counter()
        line = dict(base, case="membership", leaves=L, depth=tree.depth, members=args.members, program="smpath",
                    build_tree_s=round(t1 - t0, 3), execute_batch_with_proofs_s=round(t2 - t1, 3), verify_batch_s=round(t3 - t2, 3),
                    all_output_root=not bad, all_verified=bool(verdicts) and all(x is None for x in verdicts))
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
