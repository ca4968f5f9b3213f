"""-m gpu tests of batched proving (dg_prove_batch / prove_batch): every proof of a batch must be byte-identical to the single-trace
proof of the same trace (which test_gpu_prove.py pins to the CPU oracle), whatever else the batch holds."""
import hashlib
import json
import os
import subprocess
import sys

import pytest

from tests import programs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "oracle_proofs.json")


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    backend.device_info()
    return distaff_b200


@pytest.fixture(scope="module")
def small():
    return programs.small_programs()


def fib_traces(k):
    """k fibonacci 2^8-step traces (fibonacci_program(13)) with different public-input pairs"""
    from distaff_b200 import hostvm
    return [hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[1 + i, i]) for i in range(k)]


def merkle_trace(depth, seed, po):
    """examples/merkle.rs with its path seeds changed in byte 3: traces of one shape, different paths and leaf indexes"""
    from distaff_b200 import hostvm
    s1 = bytes([1, 2, 3, seed] + [0] * 28)
    s2 = bytes([4, 5, 6, seed] + [0] * 28)
    p0, p1 = po.prng_vector(s1, depth), po.prng_vector(s2, depth)
    leaf_index = p0[0] % (2 ** (depth - 1))
    a, b = [p0[0]], [p1[0]]
    index = leaf_index + 2 ** (depth - 1)
    for i in range(1, depth):
        a += [0, p0[i]]
        b += [index & 1, p1[i]]
        index >>= 1
    for i in range(1, depth):
        a.append(p0[i])
        b.append(p1[i])
    return hostvm.execute(hostvm.merkle_program(depth, leaf_index), secret_a=a, secret_b=b, num_outputs=4)


def test_fibonacci_batch_is_byte_identical(dg, po):
    traces = fib_traces(16)
    batch = dg.prove_batch(traces)
    assert len(batch) == 16
    for i, (tr, proof) in enumerate(zip(traces, batch)):
        assert isinstance(proof, dg.StarkProof), proof
        assert proof.bytes == dg.prove(tr).bytes, i
    for i in (0, 7, 15):                          # a few against the CPU oracle directly
        tr = traces[i]
        ref = po.prove(tr.registers, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs)
        assert ref.error is None
        assert batch[i].bytes == ref.proof, i
        assert po.verify(tr.program_hash, tr.public_inputs, tr.outputs, batch[i].bytes) is None


def test_mixed_shapes_are_grouped(dg, po, small):
    golden = json.load(open(GOLDEN))
    names = list(small)
    batch = dg.prove_batch([small[n] for n in names])
    assert len(batch) == len(names)
    for name, proof in zip(names, batch):
        assert proof.bytes == dg.prove(small[name]).bytes, name
        assert hashlib.sha256(proof.bytes).hexdigest() == golden[name]["proof_sha256"], name
    for name in ("fib13", "collatz3", "hash"):
        tr = small[name]
        ref = po.prove(tr.registers, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs)
        assert batch[names.index(name)].bytes == ref.proof, name


def test_merkle_paths_of_one_depth(dg, po):
    traces = [merkle_trace(16, s, po) for s in range(4)]
    assert len({(t.registers.shape, t.ctx_depth, t.loop_depth) for t in traces}) == 1
    batch = dg.prove_batch(traces)
    for i, (tr, proof) in enumerate(zip(traces, batch)):
        assert proof.bytes == dg.prove(tr).bytes, i
    ref = po.prove(traces[1].registers, traces[1].ctx_depth, traces[1].loop_depth, traces[1].public_inputs, traces[1].outputs)
    assert batch[1].bytes == ref.proof


def distinct_traces(prog):
    """three different traces of one shape for each program of the option sweep"""
    from distaff_b200 import hostvm
    if prog == "fib13":
        return fib_traces(3)
    if prog == "collatz3":
        return [hostvm.collatz(s) for s in (3, 5, 6)]                  # all 2^11 steps x 26 registers
    return [hostvm.execute("begin pad.2 hash.2 end", public_inputs=[a, a + 1], num_outputs=2) for a in (5, 7, 9)]


@pytest.mark.parametrize("prog,ext,queries,grinding", [("collatz3", 16, 30, 8), ("collatz3", 64, 20, 12), ("collatz3", 128, 10, 0),
                                                        ("fib13", 256, 5, 4), ("collatz3", 256, 5, 4), ("hash", 128, 128, 1)])
def test_other_proof_options_in_batch_form(dg, prog, ext, queries, grinding):
    opts = dg.ProofOptions(ext, queries, grinding)
    traces = distinct_traces(prog)
    assert len({(t.registers.shape, t.ctx_depth, t.loop_depth) for t in traces}) == 1
    batch = dg.prove_batch(traces, opts)
    assert len({p.bytes for p in batch}) == 3
    for i, (tr, proof) in enumerate(zip(traces, batch)):
        assert proof.bytes == dg.prove(tr, opts).bytes, i


def test_failed_trace_does_not_change_the_others(dg, small):
    from distaff_b200 import backend, hostvm
    traces = fib_traces(5)
    tr = traces[2]
    regs = tr.registers.copy()
    regs[tr.width - 1, 100, 0] += 1              # as in test_invalid_trace_is_reported_not_proven
    traces[2] = hostvm.ExecutionTrace(regs, tr.ctx_depth, tr.loop_depth, tr.stack_depth, tr.program_hash, tr.public_inputs, tr.outputs)
    batch = dg.prove_batch(traces)
    assert isinstance(batch[2], backend.DgError) and batch[2].code == -5
    with pytest.raises(backend.DgError) as single:
        dg.prove(traces[2])
    assert str(batch[2]) == str(single.value)          # the message dg_prove gives, with the failing step
    for i in (0, 1, 3, 4):
        assert batch[i].bytes == dg.prove(traces[i]).bytes, i


def test_host_rng_callbacks_give_the_same_batch(dg, po):
    from distaff_b200 import backend, felt
    calls = {"field": 0, "positions": 0}

    def draw_field(seed, count):
        calls["field"] += 1
        return felt.from_ints(po.prng_vector(seed, count)).tobytes()

    def draw_positions(seed, domain, ext, nq):
        calls["positions"] += 1
        return po.query_positions(seed, domain, ext, nq)

    traces = fib_traces(4)
    want = [p.bytes for p in dg.prove_batch(traces)]
    try:
        backend.set_rng_callbacks(draw_field, draw_positions)
        got = [p.bytes for p in dg.prove_batch(traces)]
    finally:
        backend.set_rng_callbacks()
    assert got == want
    assert calls["positions"] == 4 and calls["field"] >= 3 * 4


def test_group_splitting_gives_the_same_bytes(dg):
    """DG_BATCH_GROUP=3 splits a batch of 7 into groups of 3, 3 and 1 (in a fresh process, as a user would set it)"""
    traces = fib_traces(7)
    one_group = dg.prove_batch(traces)
    want = [hashlib.sha256(p.bytes).hexdigest() for p in one_group]
    code = ("import hashlib, sys; sys.path.insert(0, %r)\n"
            "import distaff_b200 as dg\n"
            "from distaff_b200 import hostvm\n"
            "traces = [hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[1 + i, i]) for i in range(7)]\n"
            "batch = dg.prove_batch(traces)\n"
            "print(' '.join(hashlib.sha256(p.bytes).hexdigest() for p in batch))\n"
            "print(batch[0].stats['kernel_launches'])\n" % ROOT)
    env = dict(os.environ, DG_BATCH_GROUP="3")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.strip().splitlines()
    assert lines[-2].split() == want
    assert int(lines[-1]) > one_group[0].stats["kernel_launches"]          # three groups: three pipelines


def test_large_batch_is_split_to_fit_one_launch(dg):
    """3300 traces of 20 registers are more than one launch holds (the DEEP evaluation puts every column of every proof on the grid's
    y dimension, at most 65535): the batch is split into groups by itself, and every proof still equals its single proof"""
    assert "DG_BATCH_GROUP" not in os.environ
    distinct = fib_traces(100)
    single = [dg.prove(t).bytes for t in distinct]
    batch = dg.prove_batch([distinct[i % 100] for i in range(3300)])
    assert all(isinstance(p, dg.StarkProof) for p in batch)
    for i, p in enumerate(batch):
        assert p.bytes == single[i % 100], i
    assert batch[0].stats["kernel_launches"] <= 2 * 2 * dg.prove(distinct[0]).stats["kernel_launches"]     # two groups


def test_device_entry_point(dg):
    import numpy as np
    from distaff_b200 import backend
    traces = fib_traces(5)
    tr = traces[0]
    regs = np.ascontiguousarray(np.stack([t.registers for t in traces]))
    buf = backend.DeviceBuffer(regs.nbytes).upload(regs)
    dev = dg.prove_batch_device(buf, 5, tr.width, tr.length, tr.ctx_depth, tr.loop_depth, [t.public_inputs for t in traces],
                                [t.outputs for t in traces])
    host = dg.prove_batch(traces)
    assert [p.bytes for p in dev] == [p.bytes for p in host]
    one = dg.prove_batch_device(buf, 1, tr.width, tr.length, tr.ctx_depth, tr.loop_depth, [tr.public_inputs], [tr.outputs])
    assert one[0].bytes == dg.prove(tr).bytes


def test_batch_shares_launches(dg):
    """every stage is launched once for the whole batch: 16 proofs cost at most twice the launches of one"""
    traces = fib_traces(16)
    dg.prove_batch(traces)
    single = dg.prove(traces[0]).stats["kernel_launches"]
    batch = dg.prove_batch(traces)[0].stats["kernel_launches"]
    print("kernel launches: one proof %d, batch of 16 %d" % (single, batch))
    assert batch <= 2 * single


def test_whole_call_errors_raise(dg, small):
    from distaff_b200 import backend
    with pytest.raises(backend.DgError) as e:
        dg.prove_batch([small["fib13"]], _BadOptions())
    assert e.value.code == -1


class _BadOptions:
    """extension factor 8: rejected by the library for the whole call (ProofOptions itself refuses to build it)"""

    def _c(self):
        from distaff_b200 import backend
        return backend.DgOptions(8, 50, 20, 0)
