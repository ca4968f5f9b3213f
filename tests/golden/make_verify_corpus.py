#!/usr/bin/env python3
"""Regenerates tests/golden/verify_corpus.json: the GPU verifier's verdict (return code and message) on a fixed corpus of honest,
tampered, bit-flipped, truncated and extended proofs.

The table was produced by dg_verify of the single-proof verifier, before the verifier became one pipeline shared with
dg_verify_batch, so that both entry points can be checked against behaviour that neither of them defined.  Proofs are deterministic,
so only their SHA-256 and the verdicts are stored: cases() rebuilds every case from the proofs and a fixed seed.  Needs a GPU.   Run:  python tests/golden/make_verify_corpus.py [output path]
"""
import ctypes
import hashlib
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "verify_corpus.json")

# (name, program, proof options): the default options on programs of several register shapes, plus two other option sets.  fib_span
# is proven too, for the reference's tampering cases.
CONFIGS = (("fib13", "fib13", None), ("collatz3", "collatz3", None), ("hash", "hash", None), ("deep_stack", "deep_stack", None),
           ("wide", "wide", None), ("collatz3_e16", "collatz3", (16, 30, 8)), ("fib13_e256", "fib13", (256, 5, 4)))


def proofs(dg):
    """name -> (trace, proof bytes) for every configuration"""
    from tests import programs
    small = programs.small_programs()
    out = {}
    for name, prog, opts in CONFIGS + (("fib_span", "fib_span", None),):
        tr = programs.wide_program() if prog == "wide" else small[prog]
        out[name] = (tr, dg.prove(tr, dg.ProofOptions(*opts) if opts else None).bytes)
    return out


def cases(proof_map):
    """[(case id, program_hash, public_inputs, outputs, proof bytes)] in a fixed order"""
    rng = random.Random(20261015)
    out = []
    for name, _, _ in CONFIGS:
        tr, proof = proof_map[name]
        L = len(proof)
        args = (tr.program_hash, tr.public_inputs, tr.outputs)
        out.append((f"{name}/honest",) + args + (proof,))
        # header (trace root, domain / ctx / loop / stack depth, op count), the body, and the tail (remainder, nonce, options)
        offsets = [0, 31, 32, 33, 34, 35, 36, 40] + sorted(rng.randrange(44, L - 16) for _ in range(40)) + \
                  [L - 20, L - 12, L - 8, L - 5, L - 4, L - 3, L - 2, L - 1]
        for off in offsets:
            bit = rng.randrange(8)
            bad = bytearray(proof)
            bad[off] ^= 1 << bit
            out.append((f"{name}/flip/{off}/{bit}",) + args + (bytes(bad),))
        for cut in (0, 10, 100, L // 2, L - 1):
            out.append((f"{name}/truncate/{cut}",) + args + (proof[:cut],))
        for extra in (b"\0", b"\x01" * 16):
            out.append((f"{name}/append/{len(extra)}",) + args + (proof + extra,))
    # src/tests/mod.rs:32-63: wrong inputs, wrong outputs, wrong program hash
    tr, proof = proof_map["fib_span"]
    bad_hash = bytes([1]) + tr.program_hash[1:]
    out.append(("fib_span/honest", tr.program_hash, tr.public_inputs, tr.outputs, proof))
    out.append(("fib_span/tamper/inputs", tr.program_hash, [1, 1], tr.outputs, proof))
    out.append(("fib_span/tamper/outputs", tr.program_hash, tr.public_inputs, [5], proof))
    out.append(("fib_span/tamper/program_hash", bad_hash, tr.public_inputs, tr.outputs, proof))
    return out


def verify_one(program_hash, public_inputs, outputs, proof):
    """dg_verify -> (return code, message): the rejection string for DG_ERR_REJECTED, dg_last_error() for other failures"""
    from distaff_b200 import backend, felt
    fi, fo = felt.from_ints(public_inputs), felt.from_ints(outputs)
    msg = ctypes.create_string_buffer(512)
    L = backend.lib()
    rc = L.dg_verify(bytes(program_hash), fi.ctypes.data, len(fi), fo.ctypes.data, len(fo), proof, len(proof), msg, len(msg))
    if rc == 0:
        return 0, ""
    if rc == -6:
        return rc, msg.value.decode()
    return rc, L.dg_last_error().decode()


def main():
    import distaff_b200 as dg
    path = sys.argv[1] if len(sys.argv) > 1 else PATH
    pm = proofs(dg)
    table = {cid: list(verify_one(*rest)) for cid, *rest in cases(pm)}
    doc = {"proof_sha256": {k: hashlib.sha256(v[1]).hexdigest() for k, v in sorted(pm.items())}, "cases": table}
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    json.dump(doc, open(path, "w"), indent=1)
    codes = {}
    for rc, _ in table.values():
        codes[rc] = codes.get(rc, 0) + 1
    print("wrote", path, len(table), "cases, return codes", codes)


if __name__ == "__main__":
    main()
