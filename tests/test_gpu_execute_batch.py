"""Batched execution on the GPU (dg_trace_batch / dg_execute_batch): traces byte-identical to the host VM's, proofs byte-identical to
dg.execute's and to the golden oracle proofs, failures with the host VM's messages beside unaffected executions."""
import hashlib
import json
import os

import numpy as np
import pytest

import distaff_b200 as dg
from distaff_b200 import backend, hostvm
from tests import execution_cases as cases

pytestmark = pytest.mark.gpu
GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_proofs.json")))
Inputs = dg.ProgramInputs


def _same(a, b):
    assert a.registers.shape == b.registers.shape
    assert np.array_equal(a.registers, b.registers)
    assert (a.ctx_depth, a.loop_depth, a.stack_depth) == (b.ctx_depth, b.loop_depth, b.stack_depth)
    assert a.program_hash == b.program_hash and a.outputs == b.outputs


@pytest.mark.parametrize("case", cases.SMALL, ids=[c[0] for c in cases.SMALL])
def test_golden_programs(case):
    name, src, pub, a, b, no = case
    g = GOLDEN[name]
    tr = dg.trace_batch(src, [Inputs(pub, a, b)], num_outputs=no)[0]
    assert not isinstance(tr, backend.DgError), tr
    assert hashlib.sha256(tr.registers.tobytes()).hexdigest() == g["trace_sha256"]
    assert (tr.length, tr.width, tr.ctx_depth, tr.loop_depth, tr.stack_depth) == (g["n"], g["w"], g["ctx"], g["loop"], g["stack"])
    assert tr.program_hash.hex() == g["program_hash"]
    outputs, proof = dg.execute_batch(hostvm.compile_program(src), [Inputs(pub, a, b)], num_outputs=no)[0]
    assert hashlib.sha256(proof.bytes).hexdigest() == g["proof_sha256"]
    assert outputs == [int(x) for x in g["outputs"]]


def _check_traces(src, inputs, no=1):
    got = dg.trace_batch(src, inputs, num_outputs=no)
    for x, tr in zip(inputs, got):
        assert not isinstance(tr, backend.DgError), tr
        _same(tr, hostvm.execute(src, x.public, x.secret_a, x.secret_b, no))
    shapes = dg.trace_shapes(src, inputs)               # the shapes-only call reports what the full call reports
    for tr, s in zip(got, shapes):
        assert (s["width"], s["length"], s["ctx_depth"], s["loop_depth"], s["stack_depth"]) == (
            tr.width, tr.length, tr.ctx_depth, tr.loop_depth, tr.stack_depth)
    return got


def test_collatz_starts_1_to_64_mix_lengths():
    got = _check_traces(hostvm.COLLATZ_SOURCE, [Inputs(secret_a=[s]) for s in range(1, 65)])
    assert len({tr.length for tr in got}) > 1


def test_fibonacci_on_64_public_input_pairs():
    rng = np.random.default_rng(1)
    pairs = [[int(rng.integers(0, 2**62)), int(rng.integers(0, 2**62))] for _ in range(64)]
    _check_traces(hostvm.fibonacci_program(64), [Inputs(p) for p in pairs])


def test_merkle_on_32_paths_under_one_leaf_index():
    inputs, src0 = [], None
    for seed in range(32):
        src, a, b = cases.merkle_case(32, 1, seed=seed, index_of=lambda c: 123456)
        src0 = src0 or src
        assert src == src0
        inputs.append(Inputs(secret_a=a, secret_b=b))
    _check_traces(src0, inputs, no=4)


def test_compare_and_range_hints_on_varied_inputs():
    rng = np.random.default_rng(2)
    inputs = []
    for i in range(48):
        x = int(rng.integers(0, 2**31))
        y = x if i % 5 == 0 else int(rng.integers(0, 2**31))
        inputs.append(Inputs([x, y]))
    _check_traces(cases.COMPARE_SOURCE, inputs, no=4)


def test_proofs_equal_execute_and_verify():
    src = hostvm.COLLATZ_SOURCE
    inputs = [Inputs(secret_a=[s]) for s in (3, 7, 27, 3, 12)]
    got = dg.execute_batch(src, inputs)
    for x, (outputs, proof) in zip(inputs, got):
        ref_out, ref = dg.execute(src, x.public, x.secret_a, x.secret_b)
        assert outputs == ref_out and proof.bytes == ref.bytes
        assert dg.verify(hostvm.compile_program(src).hash, x.public, outputs, proof) is None


FAIL_SOURCE = "begin read if.true read assert else read while.true push.1 end end swap end"
FAIL_CASES = [
    ("good", Inputs([5, 6], [1, 1])),
    ("assert", Inputs([5, 6], [1, 0])),
    ("underflow", Inputs([], [1, 1])),
    ("empty tape", Inputs([5, 6], [1])),
    ("non-binary branch", Inputs([5, 6], [2, 1])),
    ("good2", Inputs([7, 8], [0, 0])),
    ("tape B longer", Inputs([5, 6], [1, 1], [1, 2, 3])),
    ("9 public inputs", Inputs(list(range(9)), [1, 1])),
    ("never stops", Inputs([5, 6], [0, 1])),
]


def test_failures_beside_good_executions():
    inputs = [x for _, x in FAIL_CASES]
    traces = dg.trace_batch(FAIL_SOURCE, inputs, max_steps=2**10)
    proofs = dg.execute_batch(FAIL_SOURCE, inputs, max_steps=2**10)
    for (name, x), tr, pr in zip(FAIL_CASES, traces, proofs):
        if name.startswith("good"):
            _same(tr, hostvm.execute(FAIL_SOURCE, x.public, x.secret_a, x.secret_b))
            ref_out, ref = dg.execute(FAIL_SOURCE, x.public, x.secret_a, x.secret_b)
            assert pr[0] == ref_out and pr[1].bytes == ref.bytes
            continue
        if name == "never stops":
            expected = "execution exceeds 1024 steps"
        else:
            with pytest.raises(RuntimeError) as e:
                hostvm.execute(FAIL_SOURCE, x.public, x.secret_a, x.secret_b)
            expected = str(e.value)[len("vm: "):]
        for got in (tr, pr):
            assert isinstance(got, backend.DgError) and got.code == -7, (name, got)
            assert str(got) == "distaff_gpu error -7: " + expected, name


def _fib_inputs(k):
    return [Inputs([i + 1, 2 * i]) for i in range(k)]


def test_batch_group_gives_the_same_bytes(monkeypatch):
    src = hostvm.fibonacci_program(100)
    ref = dg.execute_batch(src, _fib_inputs(5))
    ref_tr = dg.trace_batch(src, _fib_inputs(5))
    monkeypatch.setenv("DG_BATCH_GROUP", "2")
    got = dg.execute_batch(src, _fib_inputs(5))
    assert [p.bytes for _, p in got] == [p.bytes for _, p in ref]
    for a, b in zip(dg.trace_batch(src, _fib_inputs(5)), ref_tr):
        _same(a, b)


def test_memory_limit_forces_groups_and_holds():
    src = hostvm.fibonacci_program(600)
    k = 6
    ref = dg.execute_batch(src, _fib_inputs(k))
    tr = dg.trace_batch(src, _fib_inputs(1))[0]
    plan = dg.plan_prove(tr.width, tr.length, k)
    limit = plan["fixed_bytes"] + 2 * plan["bytes_per_proof"] + (256 << 20)
    try:
        dg.set_memory_limit(limit)
        assert dg.plan_prove(tr.width, tr.length, k)["group"] < k
        got = dg.execute_batch(src, _fib_inputs(k))
        assert [p.bytes for _, p in got] == [p.bytes for _, p in ref]
        assert dg.memory_usage()["peak"] <= limit
    finally:
        dg.set_memory_limit(0)


def test_tape_scratch_is_enlarged():
    prog = cases.tape_growing_program()
    tr = dg.trace_batch(prog, [Inputs(), Inputs()], num_outputs=2)
    for t in tr:
        assert not isinstance(t, backend.DgError), t
        _same(t, hostvm.execute_program(prog, num_outputs=2))


_FIRST_CALL = """
import sys
sys.path.insert(0, {root!r})
import numpy as np
import distaff_b200 as dg
from distaff_b200 import backend, hostvm
from tests import execution_cases as cases
what = sys.argv[1]
if what == "hash_shapes":            # the first call of the process is a shape pass over RESCR
    src = "begin pad.2 hash.2 push.0 dup.2 drop eq if.true push.1 else push.2 push.3 end end"
    ref = hostvm.execute(src, [5, 6], num_outputs=2)
    s = dg.trace_shapes(src, [dg.ProgramInputs([5, 6])])[0]
    assert (s["width"], s["length"], s["stack_depth"]) == (ref.width, ref.length, ref.stack_depth), (s, ref.width, ref.length)
    tr = dg.trace_batch(src, [dg.ProgramInputs([5, 6])], num_outputs=2)[0]
    assert np.array_equal(tr.registers, ref.registers) and tr.outputs == ref.outputs
else:                                # the first call of the process is execute_batch of merkle paths
    src, a, b = cases.merkle_case(16, 2)
    got = dg.execute_batch(src, [dg.ProgramInputs(secret_a=a, secret_b=b)], num_outputs=4)[0]
    assert not isinstance(got, backend.DgError), got
    out, proof = dg.execute(src, [], a, b, num_outputs=4)
    assert got[0] == out and got[1].bytes == proof.bytes
print("ok")
"""


@pytest.mark.parametrize("what", ["hash_shapes", "merkle_execute"])
def test_rescr_on_the_first_call_of_a_process(what):
    """the constants of the hasher round are on the device before the first shape pass, not only after a write pass"""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _FIRST_CALL.format(root=root), what], capture_output=True, text=True, cwd=root, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
