"""-m gpu tests of proving under a device-memory limit (dg_set_memory_limit).  With the limit just below what the full layout needs,
plan_prove must report the evaluation-coset layout, and every proof must be byte-identical to the proof without a limit and to the CPU
oracle's: the trace extension is hashed chunk by chunk, only the 8 evaluation cosets are kept, and opened rows outside them are computed
from the trace polynomials.  The query positions of the proofs show that both kinds of opened row occur."""
import contextlib
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from tests import programs

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
KINDS = {"retained": 0, "computed": 0}       # opened rows of every proof checked here, by kind


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    backend.device_info()
    yield distaff_b200
    distaff_b200.set_memory_limit(0)


@contextlib.contextmanager
def below_full(dg, width, length, count=1, options=None):
    """sets the limit one byte below what the full layout needs for one proof of this shape; yields the plan under the limit"""
    plan = dg.plan_prove(width, length, 1, options)
    assert plan["layout"] == "full" and plan["coset_chunk"] == plan["retained_cosets"], plan
    limit = plan["fixed_bytes"] + plan["bytes_per_proof"] - 1
    dg.set_memory_limit(limit)
    try:
        lim = dg.plan_prove(width, length, count, options)
        assert lim["layout"] == "eval_cosets" and lim["retained_cosets"] == 8 and lim["coset_chunk"] < (options or dg.ProofOptions()).extension_factor, lim
        assert lim["bytes_per_proof"] + lim["fixed_bytes"] <= limit, (lim, limit)
        yield lim
    finally:
        dg.set_memory_limit(0)


def count_rows(po, tr, proof, options):
    """tallies the proof's opened rows: in a retained coset (c = 0 mod b / 8) or computed from the polynomials"""
    b = options.extension_factor
    for pos in po.query_positions(proof.pow_seed, tr.length * b, b, options.num_queries):
        KINDS["retained" if (pos % b) % (b // 8) == 0 else "computed"] += 1


def check_limited(dg, po, tr, options=None):
    options = options or dg.ProofOptions()
    want = dg.prove(tr, options)
    with below_full(dg, tr.width, tr.length, 1, options):
        got = dg.prove(tr, options)
    assert got.bytes == want.bytes
    ref = po.prove(tr.registers, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs, ext=options.extension_factor,
                   num_queries=options.num_queries, grinding=options.grinding_factor)
    assert ref.error is None, ref.error
    assert got.bytes == ref.proof
    count_rows(po, tr, got, options)
    return got


@pytest.mark.parametrize("steps", [13, 250], ids=["fib_2_8", "fib_2_12"])
def test_fibonacci(dg, po, steps):
    from distaff_b200 import hostvm
    tr = hostvm.fibonacci(steps)
    assert tr.length in (256, 4096)
    check_limited(dg, po, tr)


def test_merkle_depth_128(dg, po):
    """the longest authentication path the host VM's merkle program takes: 2^13 steps"""
    tr = programs.merkle_example(128, po)
    assert tr.width == 26 and tr.length == 1 << 13
    check_limited(dg, po, tr)


def test_32_step_trace(dg, po):
    from tests.test_gpu_short_traces import LOGIC, run
    tr = run(LOGIC, [1, 1, 0, 1])
    assert tr.length == 32
    check_limited(dg, po, tr)


def test_widest_vm_shape(dg, po):
    from tests.test_gpu_air import vm_traces
    tr = vm_traces()["widest"]
    assert tr.width == 70
    check_limited(dg, po, tr)


@pytest.mark.parametrize("ext,queries,grinding", [(16, 30, 8), (64, 20, 12), (256, 16, 4)])
def test_extension_factors(dg, po, ext, queries, grinding):
    from distaff_b200 import hostvm
    check_limited(dg, po, hostvm.fibonacci(13), dg.ProofOptions(ext, queries, grinding))


def test_both_kinds_of_opened_row_occurred():
    """runs after the proofs above (file order): both the retained-slab fetch and the computed rows were exercised"""
    assert KINDS["retained"] > 0 and KINDS["computed"] > 0, KINDS


def fib_traces(k):
    from distaff_b200 import hostvm
    return [hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[1 + i, i]) for i in range(k)]


def test_batch_gives_the_single_proofs(dg):
    from distaff_b200 import backend, hostvm
    traces = fib_traces(5)
    tr = traces[2]
    regs = tr.registers.copy()
    regs[tr.width - 1, 100, 0] += 1
    traces[2] = hostvm.ExecutionTrace(regs, tr.ctx_depth, tr.loop_depth, tr.stack_depth, tr.program_hash, tr.public_inputs, tr.outputs)
    want = dg.prove_batch(traces)
    with pytest.raises(backend.DgError) as single:
        dg.prove(traces[2])
    with below_full(dg, tr.width, tr.length, 5):
        got = dg.prove_batch(traces)
    assert isinstance(got[2], backend.DgError) and got[2].code == -5
    assert str(got[2]) == str(want[2]) == str(single.value)
    for i in (0, 1, 3, 4):
        assert got[i].bytes == want[i].bytes == dg.prove(traces[i]).bytes, i


def test_batch_group_split_under_the_limit(dg):
    """DG_BATCH_GROUP=3 (a fresh process, as a user would set it) with the limit below the full layout: the single proofs"""
    traces = fib_traces(7)
    want = [hashlib.sha256(dg.prove(t).bytes).hexdigest() for t in traces]
    code = ("import hashlib, sys; sys.path.insert(0, %r)\n"
            "import distaff_b200 as dg\n"
            "from distaff_b200 import hostvm\n"
            "traces = [hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[1 + i, i]) for i in range(7)]\n"
            "dg.prove(traces[0])\n"
            "p = dg.plan_prove(traces[0].width, traces[0].length, 1)\n"
            "dg.set_memory_limit(p['fixed_bytes'] + p['bytes_per_proof'] - 1)\n"
            "p = dg.plan_prove(traces[0].width, traces[0].length, 7)\n"
            "batch = dg.prove_batch(traces)\n"
            "print(p['layout'], p['group'])\n"
            "print(' '.join(hashlib.sha256(b.bytes).hexdigest() for b in batch))\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, DG_BATCH_GROUP="3"), cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.strip().splitlines()
    assert lines[-1].split() == want
    layout, group = lines[-2].split()
    assert layout == "eval_cosets" and int(group) <= 3, lines[-2]


def test_rng_callbacks_see_the_same_sequence(dg, po):
    from distaff_b200 import backend, felt, hostvm
    seen = []

    def draw_field(seed, count):
        seen.append(("field", seed, count))
        return felt.from_ints(po.prng_vector(seed, count)).tobytes()

    def draw_positions(seed, domain, ext, nq):
        seen.append(("positions", seed, domain, ext, nq))
        return po.query_positions(seed, domain, ext, nq)

    tr = hostvm.fibonacci(200)
    try:
        backend.set_rng_callbacks(draw_field, draw_positions)
        want = dg.prove(tr).bytes
        free = list(seen)
        seen.clear()
        with below_full(dg, tr.width, tr.length):
            got = dg.prove(tr).bytes
    finally:
        backend.set_rng_callbacks()
    assert got == want
    assert seen == free and len(seen) >= 4


def test_collatz_2_20_under_16_gb(dg, po):
    import bench
    gold = json.load(open(os.path.join(HERE, "golden", "collatz_2_20.json")))
    tr, name = bench.build_trace(20)
    assert name == gold["name"]
    assert hashlib.sha256(np.ascontiguousarray(tr.registers).tobytes()).hexdigest() == gold["trace_sha256"]
    limit = 16 << 30
    dg.set_memory_limit(limit)
    try:
        plan = dg.plan_prove(tr.width, tr.length)
        assert plan["layout"] == "eval_cosets", plan
        proof = dg.prove(tr)
        assert hashlib.sha256(proof.bytes).hexdigest() == gold["proof_sha256"]
        assert dg.memory_usage()["peak"] <= limit, (dg.memory_usage(), plan)
        assert dg.prove(tr).bytes == proof.bytes                     # a second proof, on the arena sized within the limit
        assert dg.memory_usage()["peak"] <= limit
    finally:
        dg.set_memory_limit(0)


def test_collatz_2_20_at_extension_factor_128(dg, po):
    """the full layout does not fit on an 80 GB card at b = 128; the evaluation-coset layout does"""
    import torch
    import bench
    tr, _ = bench.build_trace(20)
    opts = dg.ProofOptions(128, 50, 20)
    plan = dg.plan_prove(tr.width, tr.length, 1, opts)
    free = torch.cuda.mem_get_info()[0]
    if free < plan["bytes_per_proof"] + plan["fixed_bytes"]:
        pytest.skip("free device memory %d is below the plan %s" % (free, plan))
    assert plan["layout"] == "eval_cosets", plan
    proof = dg.prove(tr, opts)
    assert dg.prove(tr, opts).bytes == proof.bytes
    assert dg.verify(tr.program_hash, tr.public_inputs, tr.outputs, proof.bytes) is None
    assert po.verify(tr.program_hash, tr.public_inputs, tr.outputs, proof.bytes) is None


def test_limit_errors(dg):
    from distaff_b200 import backend
    dg.set_memory_limit(1 << 20)
    try:
        with pytest.raises(backend.DgError) as e:
            dg.plan_prove(26, 1 << 20)
        assert e.value.code == -1 and "bytes" in str(e.value)
        from distaff_b200 import hostvm
        with pytest.raises(backend.DgError) as e:
            dg.prove(hostvm.fibonacci(200))
        assert e.value.code == -1
    finally:
        dg.set_memory_limit(0)
    u = dg.memory_usage()
    assert u["held"] >= 0 and u["peak"] >= u["held"]
