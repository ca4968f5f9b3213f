#!/usr/bin/env python3
"""Batch Merkle proofs and path verification on the GPU, one JSON line per case; every line records the card's name and power limit, read
in the same run.  Times are wall ms of one call (host checks, the upload, every launch, the copy back and the synchronise), best of --reps
after a warm-up.

  verify_paths  merkle_verify_paths of K random paths of a 2^20-leaf tree (21 entries each), for the hasher and blake3: ms and digests per
                second (K x 20 digests per call).
  verify_batch  merkle_verify_batch of 64 blake3 batch proofs of 50 random indexes each of a 2^20-leaf tree: ms.
  prove_batch   MerkleTree.prove_batch of 1000 random leaves of a 2^20-leaf tree (the sizing call and the real call): ms.

    python tools/merkle_verify_bench.py [--ks 1024,16384,262144] [--reps 3]
"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import distaff_b200 as dg                        # noqa: E402
from tools.trace_one_bench import card            # noqa: E402


def random_leaves(L, seed):
    """L x 32 bytes of canonical field elements (each below 2^127 < M)"""
    return np.random.default_rng(seed).integers(0, 2**63, size=(L, 2, 2), dtype=np.uint64).tobytes()


def best_wall(fn, reps):
    out = fn()
    best = None
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        dt = (time.perf_counter() - t) * 1e3
        best = dt if best is None else min(best, dt)
    return best, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ks", default="1024,16384,262144")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    name, power = card()
    L, entries = 1 << 20, 21
    rng = np.random.default_rng(1)
    emit = lambda **kw: print(json.dumps(dict(card=name, power_limit=power, **kw)), flush=True)
    for hash in ("hasher", "blake3"):
        with dg.MerkleTree(random_leaves(L, 2), hash) as tree:
            root = tree.root
            for K in [int(k) for k in a.ks.split(",")]:
                idx = rng.integers(0, L, size=K, dtype=np.uint64)
                paths = np.empty((K, entries, 32), dtype=np.uint8)
                for k0 in range(0, K, 1 << 16):
                    part = tree.paths(idx[k0:k0 + (1 << 16)])
                    paths[k0:k0 + len(part)] = np.frombuffer(b"".join(b"".join(p) for p in part), dtype=np.uint8).reshape(-1, entries, 32)
                ms, got = best_wall(lambda: dg.merkle_verify_paths(root, idx, paths, hash), a.reps)
                assert got == [True] * K
                digests = K * (entries - 1)
                emit(case="verify_paths", hash=hash, leaves=L, paths=K, digests=digests, wall_ms=round(ms, 3),
                     digests_per_s=round(digests / ms * 1e3))
            if hash == "blake3":
                pr = random.Random(3)
                items = []
                for _ in range(64):
                    ix = pr.sample(range(L), 50)
                    items.append((root, ix, tree.prove_batch(ix)))
                ms, got = best_wall(lambda: dg.merkle_verify_batch(items, hash), a.reps)
                assert got == [True] * 64
                emit(case="verify_batch", hash=hash, leaves=L, proofs=64, indexes_each=50,
                     proof_digests=sum(len(p.values) + sum(map(len, p.nodes)) for _, _, p in items), wall_ms=round(ms, 3))
                ix = pr.sample(range(L), 1000)
                ms, p = best_wall(lambda: tree.prove_batch(ix), a.reps)
                emit(case="prove_batch", hash=hash, leaves=L, indexes=1000, nodes=sum(map(len, p.nodes)), bytes=len(p.to_bytes()),
                     wall_ms=round(ms, 3))


if __name__ == "__main__":
    main()
