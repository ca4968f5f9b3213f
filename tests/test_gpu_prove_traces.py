"""-m gpu tests of batched proving across register shapes (dg_prove_traces / prove_traces): traces of any widths, depths and lengths in one
call.  Every proof must be byte-identical to the single-trace proof of the same trace (which test_gpu_prove.py pins to the CPU oracle),
whatever else the call holds, and the call must launch each stage once per group, plus one constraint launch per extra register shape."""
import hashlib
import json
import os
import random

import pytest

from tests import programs

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "oracle_proofs.json")


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    backend.device_info()
    yield distaff_b200
    distaff_b200.set_memory_limit(0)


@pytest.fixture(scope="module")
def small():
    return programs.small_programs()


@pytest.fixture(scope="module")
def pool(small, po):
    """name -> trace: the small programs, fibonacci variants (20 registers), merkle paths (26 / 27 registers) and the 65-register trace"""
    from distaff_b200 import hostvm
    P = dict(small)
    for i in range(3):
        P["fib_%d" % i] = hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[3 + i, i])
    P["collatz5"] = hostvm.collatz(5)
    P["collatz6"] = hostvm.collatz(6)
    P["merkle16"] = programs.merkle_example(16, po)
    P["merkle_paths"] = programs.merkle_paths(8, 2, po)
    P["wide"] = programs.wide_program()
    return P


@pytest.fixture(scope="module")
def singles(dg, pool):
    return {name: dg.prove(tr).bytes for name, tr in pool.items()}


def shape(tr):
    return (tr.width, tr.ctx_depth, tr.loop_depth)


def check(dg, names, pool, singles, result):
    assert len(result) == len(names)
    for name, proof in zip(names, result):
        assert isinstance(proof, dg.StarkProof), (name, proof)
        assert proof.bytes == singles[name], name


def test_pool_covers_the_shapes(pool):
    widths = {tr.width for tr in pool.values()}
    assert {20, 26, 65} <= widths and (27 in widths or 26 in widths), widths
    assert pool["wide"].width == 65


def test_one_length_many_shapes(dg, pool, singles, small):
    """the largest set of shapes that share a length, shuffled with repeats: every proof equals its single proof and the golden hash"""
    golden = json.load(open(GOLDEN))
    by_len = {}
    for name, tr in pool.items():
        by_len.setdefault(tr.length, []).append(name)
    length = max(by_len, key=lambda n: len({shape(pool[m]) for m in by_len[n]}))
    names = by_len[length] * 2
    random.Random(1).shuffle(names)
    assert len({shape(pool[m]) for m in names}) >= 3, (length, names)
    result = dg.prove_traces([pool[m] for m in names])
    check(dg, names, pool, singles, result)
    for name, proof in zip(names, result):
        if name in small:
            assert hashlib.sha256(proof.bytes).hexdigest() == golden[name]["proof_sha256"], name


def test_every_shape_and_length_shuffled(dg, po, pool, singles):
    names = list(pool)
    random.Random(7).shuffle(names)
    assert len({pool[m].length for m in names}) >= 3
    result = dg.prove_traces([pool[m] for m in names])
    check(dg, names, pool, singles, result)
    # every proof is accepted by the GPU verifier (batched) and by the oracle's
    items = [(pool[m].program_hash, pool[m].public_inputs, pool[m].outputs, p) for m, p in zip(names, result)]
    assert dg.verify_batch(items) == [None] * len(names)
    for m, p in zip(names, result):
        tr = pool[m]
        assert po.verify(tr.program_hash, tr.public_inputs, tr.outputs, p.bytes) is None, m


def test_wide_and_fibonacci_against_the_oracle(dg, po, pool):
    names = ["fib_0", "wide", "fib13", "merkle16", "wide"]
    result = dg.prove_traces([pool[m] for m in names])
    for m in ("wide", "merkle16"):
        tr = pool[m]
        ref = po.prove(tr.registers, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs)
        assert ref.error is None
        assert result[names.index(m)].bytes == ref.proof, m
    assert result[1].bytes == result[4].bytes


def test_short_traces_of_several_shapes(dg, pool, singles):
    """16..64-step traces take the constraint kernel's SHORT layout, once per shape of the group"""
    names = [m for m, tr in pool.items() if tr.length <= 64]
    assert len({shape(pool[m]) for m in names}) >= 2, names
    assert len({pool[m].length for m in names}) >= 1
    names = names + names[::-1]
    result = dg.prove_traces([pool[m] for m in names])
    check(dg, names, pool, singles, result)


def test_corrupted_trace_in_the_middle(dg, pool, singles):
    from distaff_b200 import backend, hostvm
    names = ["collatz3", "fib_0", "wide", "fib_1", "merkle16", "hash"]
    traces = [pool[m] for m in names]
    tr = traces[3]
    regs = tr.registers.copy()
    regs[tr.width - 1, 100, 0] += 1              # as in test_invalid_trace_is_reported_not_proven
    traces[3] = hostvm.ExecutionTrace(regs, tr.ctx_depth, tr.loop_depth, tr.stack_depth, tr.program_hash, tr.public_inputs, tr.outputs)
    result = dg.prove_traces(traces)
    assert isinstance(result[3], backend.DgError) and result[3].code == -5
    with pytest.raises(backend.DgError) as single:
        dg.prove(traces[3])
    assert str(result[3]) == str(single.value)
    for i, m in enumerate(names):
        if i != 3:
            assert result[i].bytes == singles[m], m


def _recorder(po, log):
    from distaff_b200 import felt

    def draw_field(seed, count):
        log.append(("field", seed, count))
        return felt.from_ints(po.prng_vector(seed, count)).tobytes()

    def draw_positions(seed, domain, ext, nq):
        log.append(("positions", seed, domain))
        return po.query_positions(seed, domain, ext, nq)
    return draw_field, draw_positions


def test_rng_callbacks_see_the_documented_order(dg, po, pool, singles, monkeypatch):
    """length groups in order of first appearance, input order inside a length: with groups of one trace the calls are the
    concatenation of the single proofs' calls in that order; in one group each trace's calls are its own, and the first draws of the
    traces of a length come in input order"""
    from distaff_b200 import backend
    names = ["fib_0", "collatz3", "wide", "fib_1", "merkle16", "fib13", "collatz5"]
    traces = [pool[m] for m in names]
    own = {}
    try:
        for m in names:
            log = []
            backend.set_rng_callbacks(*_recorder(po, log))
            assert dg.prove(pool[m]).bytes == singles[m]
            own[m] = log
        lengths = []
        for tr in traces:
            if tr.length not in lengths:
                lengths.append(tr.length)
        expect_order = [m for n in lengths for m, tr in zip(names, traces) if tr.length == n]
        log = []
        backend.set_rng_callbacks(*_recorder(po, log))
        result = dg.prove_traces(traces)
        check(dg, names, pool, singles, result)
        for m in names:                                    # every trace's calls are its own, in its own order
            mine = [e for e in log if any(e[1] == o[1] for o in own[m])]
            assert mine == own[m], m
        firsts = [next(m for m in names if own[m][0][1] == e[1]) for e in log if any(own[m][0][1] == e[1] for m in names)]
        assert firsts == expect_order, (firsts, expect_order)
        monkeypatch.setenv("DG_BATCH_GROUP", "1")
        log = []
        backend.set_rng_callbacks(*_recorder(po, log))
        result = dg.prove_traces(traces)
        check(dg, names, pool, singles, result)
        assert log == [e for m in expect_order for e in own[m]]
    finally:
        backend.set_rng_callbacks()


def test_group_limit_and_memory_limit_give_the_same_bytes(dg, pool, singles, monkeypatch):
    names = ["fib_0", "collatz3", "wide", "fib_1", "merkle16", "fib13", "hash", "fib_2"]
    traces = [pool[m] for m in names]
    monkeypatch.setenv("DG_BATCH_GROUP", "2")
    check(dg, names, pool, singles, dg.prove_traces(traces))
    monkeypatch.delenv("DG_BATCH_GROUP")
    # a limit below what the full layout needs for one proof of the widest shape of the largest length: the evaluation-coset layout
    tr = max(traces, key=lambda t: (t.length, t.width))
    plan = dg.plan_prove(tr.width, tr.length, 1)
    assert plan["layout"] == "full"
    dg.set_memory_limit(plan["fixed_bytes"] + plan["bytes_per_proof"] - 1)
    try:
        assert dg.plan_prove(tr.width, tr.length, 1)["layout"] == "eval_cosets"
        check(dg, names, pool, singles, dg.prove_traces(traces))
    finally:
        dg.set_memory_limit(0)


def test_device_entry_point(dg, pool, singles):
    import numpy as np
    from distaff_b200 import backend
    names = ["wide", "fib_0", "collatz3", "fib_1", "merkle16"]
    traces = [pool[m] for m in names]
    bufs = [backend.DeviceBuffer(np.ascontiguousarray(t.registers).nbytes).upload(np.ascontiguousarray(t.registers)) for t in traces]
    result = dg.prove_traces_device(bufs, [t.width for t in traces], [t.length for t in traces], [t.ctx_depth for t in traces],
                                    [t.loop_depth for t in traces], [t.public_inputs for t in traces], [t.outputs for t in traces])
    check(dg, names, pool, singles, result)


def test_launches_of_mixed_shapes(dg, pool):
    """S register shapes of one length cost at most the launches of a one-shape batch of as many traces (of the widest shape, so that
    the upload chunks are no fewer) plus one constraint launch for each shape after the first.  Without grinding, so that the proof-of-work
    search, whose rounds depend on the nonces found, is one round in both calls."""
    opts = dg.ProofOptions(32, 50, 0)
    by_len = {}
    for name, tr in pool.items():
        by_len.setdefault(tr.length, []).append(name)
    for length, names in by_len.items():
        shapes = {shape(pool[m]) for m in names}
        if len(shapes) < 2:
            continue
        widest = max(names, key=lambda m: pool[m].width)
        mixed = dg.prove_traces([pool[m] for m in names], opts)[0].stats["kernel_launches"]
        one = dg.prove_batch([pool[widest]] * len(names), opts)[0].stats["kernel_launches"]
        print("length %d: %d shapes, %d traces: %d launches (one shape: %d)" % (length, len(shapes), len(names), mixed, one))
        assert mixed <= one + len(shapes) - 1, (length, mixed, one, len(shapes))


def test_one_shape_call_matches_prove_batch(dg, pool):
    from tests.test_gpu_prove_batch import fib_traces
    traces = fib_traces(6)
    batch = dg.prove_batch(traces)
    mixed = dg.prove_traces(traces)
    assert [p.bytes for p in mixed] == [p.bytes for p in batch]
    assert mixed[0].stats["kernel_launches"] == batch[0].stats["kernel_launches"]
