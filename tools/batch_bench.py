#!/usr/bin/env python3
"""Throughput of batched proving (dg_prove_batch_device) against the same traces proven one by one (dg_prove_device).

For every shape and batch size K the script prints one JSON line:
  batch_device_ms / batch_wall_ms   one dg_prove_batch_device call of K proofs (stats.total_ms / host clock around the call)
  seq_device_ms / seq_wall_ms       the same K traces through K dg_prove_device calls (summed)
  batch_proofs_per_s / seq_proofs_per_s / speedup (wall clock), kernel_launches of both arms
  identical                         every batched proof's bytes equal the sequential proof's; a line whose proofs differ is reported
                                    as an error, not as a result
Each arm is warmed up once per shape and K; then the two arms alternate, call by call, until each has at least --min-window-s of work.  The
first line names the card and its power limit (read-only nvidia-smi query).

  python tools/batch_bench.py [--shapes fib8,fib12,merkle14,fib16] [--ks 1,4,16,64,256] [--min-window-s 1.0]
"""
import argparse
import ctypes
import json
import os
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
    except Exception as e:          # the proofs below still need the device; this only labels the numbers
        return {"card": "unknown", "power_limit": "unknown", "nvidia_smi_error": str(e)}


def merkle_trace(k):
    """four depth-64 authentication paths of examples/merkle.rs (2^14 steps); trace k draws its paths with seed k"""
    from distaff_b200 import hostvm
    return hostvm.merkle_paths(64, 4, seed=k)


def fib_trace(log_n, k):
    from distaff_b200 import hostvm
    terms = {8: 13}.get(log_n, (1 << log_n) // 16 - 6)
    tr = hostvm.execute(hostvm.fibonacci_program(terms), public_inputs=[1 + k, k])
    assert tr.length == 1 << log_n, (log_n, tr.length)
    return tr


SHAPES = {
    "fib8": ("fibonacci 2^8", lambda k: fib_trace(8, k)),
    "fib12": ("fibonacci 2^12", lambda k: fib_trace(12, k)),
    "merkle14": ("merkle 2^14 (4 depth-64 paths)", lambda k: merkle_trace(k)),
    "fib16": ("fibonacci 2^16", lambda k: fib_trace(16, k)),
}


def run_shape(key, ks, min_window_s, options):
    import distaff_b200 as dg
    from distaff_b200 import backend, felt
    label, make = SHAPES[key]
    kmax = max(ks)                             # the library splits a batch that does not fit in device memory into groups
    traces = [make(k) for k in range(kmax)]
    t0 = traces[0]
    w, n = t0.width, t0.length
    regs = np.ascontiguousarray(np.stack([t.registers for t in traces]))
    buf = backend.DeviceBuffer(regs.nbytes).upload(regs)
    col_bytes = w * n * 16
    L = backend.lib()
    opt = options._c()

    def seq(count):
        """K dg_prove_device calls; returns (device ms, launches, proof bytes)"""
        dev, launches, out = 0.0, 0, []
        for i in range(count):
            t = traces[i]
            fi, fo = felt.from_ints(t.public_inputs), felt.from_ints(t.outputs)
            h = backend.vp()
            st = backend.DgStats()
            backend.check(L.dg_prove_device(buf.ptr + i * col_bytes, w, n, t.ctx_depth, t.loop_depth, fi.ctypes.data, len(fi), fo.ctypes.data,
                                            len(fo), ctypes.byref(opt), ctypes.byref(h), ctypes.byref(st)))
            p = dg.api._collect(h.value, st)
            dev += p.stats["total_ms"]
            launches += p.stats["kernel_launches"]
            out.append(p.bytes)
        return dev, launches, out

    def batch(count):
        res = dg.prove_batch_device(buf, count, w, n, t0.ctx_depth, t0.loop_depth, [t.public_inputs for t in traces[:count]],
                                    [t.outputs for t in traces[:count]], options)
        bad = [r for r in res if not isinstance(r, dg.StarkProof)]
        if bad:
            raise bad[0]
        return res[0].stats["total_ms"], res[0].stats["kernel_launches"], [r.bytes for r in res]

    def timed(count):
        """both arms, alternating rep by rep (so that clock and power drift hit both alike) until each has min_window_s of work"""
        arms = {"batch": batch, "seq": seq}
        res = {a: {"dev": 0.0, "wall": 0.0, "reps": 0, "launches": 0, "out": None} for a in arms}
        for fn in arms.values():
            fn(count)                              # warm-up (tables, arena sizing for this batch size)
        while min(r["wall"] for r in res.values()) < min_window_s * 1000:
            for a, fn in arms.items():
                backend.check(L.dg_dev_sync())
                t = time.perf_counter()
                dev, launches, out = fn(count)
                backend.check(L.dg_dev_sync())
                r = res[a]
                r["wall"] += (time.perf_counter() - t) * 1000
                r["dev"] += dev
                r["reps"] += 1
                r["launches"], r["out"] = launches, out
        return [(r["dev"] / r["reps"], r["wall"] / r["reps"], r["launches"], r["out"], r["reps"]) for r in (res["batch"], res["seq"])]

    for K in ks:
        (b_dev, b_wall, b_launch, b_out, b_reps), (s_dev, s_wall, s_launch, s_out, s_reps) = timed(K)
        line = {"shape": label, "K": K, "log_n": int(n).bit_length() - 1, "width": w,
                "batch_device_ms": round(b_dev, 3), "batch_wall_ms": round(b_wall, 3),
                "seq_device_ms": round(s_dev, 3), "seq_wall_ms": round(s_wall, 3),
                "batch_proofs_per_s": round(K / b_wall * 1000, 1), "seq_proofs_per_s": round(K / s_wall * 1000, 1),
                "speedup": round(s_wall / b_wall, 2), "kernel_launches": {"batch": b_launch, "seq": s_launch},
                "reps": {"batch": b_reps, "seq": s_reps}, "identical": b_out == s_out}
        if not line["identical"]:
            print(json.dumps({"shape": label, "K": K, "error": "batched proofs differ from the sequential proofs"}), flush=True)
            continue
        print(json.dumps(line), flush=True)
    buf.free()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="fib8,fib12,merkle14,fib16")
    ap.add_argument("--ks", default="1,4,16,64,256")
    ap.add_argument("--min-window-s", type=float, default=1.0)
    args = ap.parse_args()
    import distaff_b200 as dg
    from distaff_b200 import backend
    shapes = args.shapes.split(",")
    for s in shapes:
        if s not in SHAPES:
            ap.error("unknown shape %s (known: %s)" % (s, ",".join(SHAPES)))
    ks = sorted(int(k) for k in args.ks.split(","))
    info = backend.device_info()                  # raises DgError -3 without a device: there is no CPU path to measure
    print(json.dumps(dict(card(), device=info["name"])), flush=True)
    for s in shapes:
        run_shape(s, ks, args.min_window_s, dg.ProofOptions())


if __name__ == "__main__":
    main()
