#!/usr/bin/env python3
"""Batched verification (one dg_verify_batch call) against the same proofs verified one by one (K dg_verify calls).

For every shape and batch size K the script prints one JSON line:
  batch_device_ms / batch_wall_ms   one dg_verify_batch call of K proofs (stats.total_ms: upload to download of the groups / host clock)
  batch_host_share                  share of the batch call's wall time outside its device phases (parse, Fiat-Shamir draws, Merkle
                                    plans, packing, the reference's checks, and the Python marshalling of the call)
  seq_wall_ms                       the same K proofs through K dg_verify calls (summed host clock)
  batch_proofs_per_s / seq_proofs_per_s / speedup (wall clock)
  kernel_launches                   of the batch call, and of the K single calls (K times the launches of a batch of one: dg_verify runs
                                    the same pipeline with K = 1)
  identical                         every batched verdict equals the sequential one (all proofs are honest and accepted)
Each arm is warmed up once per shape and K; then the two arms alternate, call by call, until each has at least --min-window-s of work.
The proofs are --distinct different proofs of the shape, repeated up to K.  The first line names the card and its power limit
(read-only nvidia-smi query).

  python tools/verify_bench.py [--shapes fib8,fib12,merkle14] [--ks 1,4,16,64,256,1024] [--min-window-s 0.5] [--distinct 64]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from batch_bench import SHAPES, card  # noqa: E402


def run_shape(key, ks, min_window_s, distinct):
    import distaff_b200 as dg
    from distaff_b200 import backend
    label, make = SHAPES[key]
    traces = [make(k) for k in range(distinct)]
    proofs = dg.prove_batch(traces)
    bad = [p for p in proofs if not isinstance(p, dg.StarkProof)]
    if bad:
        raise bad[0]
    items = [(t.program_hash, t.public_inputs, t.outputs, p.bytes) for t, p in zip(traces, proofs)]
    one = {}
    dg.verify_batch(items[:1])
    dg.verify_batch(items[:1], stats=one)
    L = backend.lib()

    def seq(count):
        return [dg.verify(*items[i % distinct]) for i in range(count)], 0.0, 0

    def batch(count):
        st = {}
        out = dg.verify_batch([items[i % distinct] for i in range(count)], stats=st)
        return out, st["total_ms"], st["kernel_launches"]

    for K in ks:
        arms = {"batch": batch, "seq": seq}
        res = {a: {"dev": 0.0, "wall": 0.0, "reps": 0, "launches": 0, "out": None} for a in arms}
        for fn in arms.values():
            fn(K)                                  # warm-up
        while min(r["wall"] for r in res.values()) < min_window_s * 1000:
            for a, fn in arms.items():
                backend.check(L.dg_dev_sync())
                t = time.perf_counter()
                out, dev, launches = fn(K)
                r = res[a]
                r["wall"] += (time.perf_counter() - t) * 1000
                r["dev"] += dev
                r["reps"] += 1
                r["launches"], r["out"] = launches, out
        b, s = res["batch"], res["seq"]
        b_wall, s_wall, b_dev = b["wall"] / b["reps"], s["wall"] / s["reps"], b["dev"] / b["reps"]
        line = {"shape": label, "K": K, "width": traces[0].width, "log_n": traces[0].length.bit_length() - 1,
                "batch_device_ms": round(b_dev, 3), "batch_wall_ms": round(b_wall, 3), "batch_host_share": round(1 - b_dev / b_wall, 3),
                "seq_wall_ms": round(s_wall, 3), "batch_proofs_per_s": round(K / b_wall * 1000, 1), "seq_proofs_per_s": round(K / s_wall * 1000, 1),
                "speedup": round(s_wall / b_wall, 2), "kernel_launches": {"batch": b["launches"], "seq": K * one["kernel_launches"]},
                "reps": {"batch": b["reps"], "seq": s["reps"]},
                "identical": b["out"] == s["out"] and all(v is None for v in b["out"])}
        print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="fib8,fib12,merkle14")
    ap.add_argument("--ks", default="1,4,16,64,256,1024")
    ap.add_argument("--min-window-s", type=float, default=0.5)
    ap.add_argument("--distinct", type=int, default=64)
    args = ap.parse_args()
    from distaff_b200 import backend
    shapes = args.shapes.split(",")
    for s in shapes:
        if s not in SHAPES:
            ap.error("unknown shape %s (known: %s)" % (s, ",".join(SHAPES)))
    ks = sorted(int(k) for k in args.ks.split(","))
    info = backend.device_info()                  # raises DgError -3 without a device: there is no CPU path to measure
    print(json.dumps(dict(card(), device=info["name"])), flush=True)
    for s in shapes:
        run_shape(s, ks, args.min_window_s, args.distinct)


if __name__ == "__main__":
    main()
