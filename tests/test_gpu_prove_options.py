"""-m gpu tests of per-trace proof options (prove_traces / prove_traces_device / execute_programs / execute_many with a list of
ProofOptions): every proof equals the single proof of its trace with its own options, whatever else the call holds; num_queries and
grinding_factor may differ inside one group at no extra launches, and each extension factor is a partition of its own."""
import random

import pytest

from tests import programs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    backend.device_info()
    yield distaff_b200
    distaff_b200.set_memory_limit(0)


@pytest.fixture(scope="module")
def fibs():
    """six traces of one shape and length (fibonacci, 2^8 steps, 20 registers) on different inputs"""
    from distaff_b200 import hostvm
    return [hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[3 + i, i]) for i in range(6)]


@pytest.fixture(scope="module")
def pool(po):
    """name -> trace of several shapes and lengths: 16 to 2^10 steps, 20 to 65 registers"""
    from distaff_b200 import hostvm
    small = programs.small_programs()
    P = {m: small[m] for m in ("fib13", "collatz3", "hash", "deep_ctx", "nested_loops", "stack_ops")}
    P["collatz5"] = hostvm.collatz(5)
    P["merkle16"] = programs.merkle_example(16, po)
    P["wide"] = programs.wide_program()
    return P


@pytest.fixture(scope="module")
def single(dg):
    """prove(trace, options).bytes, cached by (id(trace), options)"""
    cache = {}

    def get(trace, options):
        key = (id(trace), options)
        if key not in cache:
            cache[key] = dg.prove(trace, options).bytes
        return cache[key]
    return get


def O(ext=32, queries=50, grinding=20):
    import distaff_b200
    return distaff_b200.ProofOptions(ext, queries, grinding)


# the mix of test 1: num_queries 1, 50 and 128, grinding 0, 8 and 20, in every pairing
MIX = [O(32, 1, 0), O(32, 50, 8), O(32, 128, 20), O(32, 50, 0), O(32, 128, 8), O(32, 1, 20)]


def check(dg, traces, opts, result, single):
    assert len(result) == len(traces)
    for i, (tr, o, proof) in enumerate(zip(traces, opts, result)):
        assert isinstance(proof, dg.StarkProof), (i, proof)
        assert proof.bytes == single(tr, o), (i, o)
        assert proof.options == o, (i, proof.options, o)


def _verify_all(dg, traces, proofs):
    verdicts = dg.verify_batch([(t.program_hash, t.public_inputs, t.outputs, p) for t, p in zip(traces, proofs)])
    assert verdicts == [None] * len(traces), verdicts


def test_one_shape_under_mixed_queries_and_grinding(dg, po, fibs, single):
    result = dg.prove_traces(fibs, MIX)
    check(dg, fibs, MIX, result, single)
    _verify_all(dg, fibs, result)
    # two small cases against the oracle
    for i in (0, 4):
        tr, o = fibs[i], MIX[i]
        ref = po.prove(tr.registers, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs, ext=o.extension_factor,
                       num_queries=o.num_queries, grinding=o.grinding_factor)
        assert ref.error is None, ref.error
        assert result[i].bytes == ref.proof, i


def _launches(dg, traces, opts):
    dg.prove_traces(traces, opts)                    # warm-up: tables of a new extension factor are built by the first call
    return dg.prove_traces(traces, opts)[0].stats["kernel_launches"]


def test_mixed_queries_cost_no_launches(dg, fibs):
    """without grinding, so that every proof-of-work search is one round: a group of mixed num_queries launches what a uniform one does"""
    mixed = [O(32, q, 0) for q in (1, 50, 128, 50, 1, 128)]
    n_mixed = _launches(dg, fibs, mixed)
    for q in (1, 50, 128):
        assert n_mixed == _launches(dg, fibs, O(32, q, 0)), q


def test_launches_add_up_across_extension_factors(dg, fibs):
    """extension factors 16 / 32 / 64 are three partitions: the launches of one mixed call are those of three uniform calls"""
    exts = [16, 32, 64, 16, 32, 64]
    mixed = _launches(dg, fibs, [O(b, 50, 0) for b in exts])
    parts = sum(_launches(dg, [t for t, e in zip(fibs, exts) if e == b], O(b, 50, 0)) for b in (16, 32, 64))
    assert mixed == parts, (mixed, parts)


def _mixed_call(pool):
    """every trace of the pool twice, under extension factors 16 / 32 / 64 and mixed queries and grinding, shuffled"""
    rng = random.Random(3)
    names = list(pool) * 2
    rng.shuffle(names)
    choices = [O(16, 50, 8), O(32, 1, 0), O(32, 128, 20), O(64, 7, 4), O(16, 128, 0), O(32, 50, 20)]
    opts = [choices[rng.randrange(len(choices))] for _ in names]
    return names, opts


def test_mixed_shapes_lengths_and_extension_factors(dg, pool, single):
    names, opts = _mixed_call(pool)
    traces = [pool[m] for m in names]
    assert len({(t.length, o.extension_factor) for t, o in zip(traces, opts)}) >= 6
    result = dg.prove_traces(traces, opts)
    check(dg, traces, opts, result, single)
    _verify_all(dg, traces, result)


def test_device_entry_point(dg, pool, single):
    """every trace in an allocation of its own; allocations of one size often lie back to back, and such traces must not be read as
    one slab"""
    import numpy as np
    from distaff_b200 import backend
    names, opts = _mixed_call(pool)
    traces = [pool[m] for m in names]
    bufs = [backend.DeviceBuffer(np.ascontiguousarray(t.registers).nbytes).upload(np.ascontiguousarray(t.registers)) for t in traces]
    result = dg.prove_traces_device(bufs, [t.width for t in traces], [t.length for t in traces], [t.ctx_depth for t in traces],
                                    [t.loop_depth for t in traces], [t.public_inputs for t in traces], [t.outputs for t in traces], opts)
    check(dg, traces, opts, result, single)


def test_corrupted_trace_in_the_middle(dg, fibs, single):
    from distaff_b200 import backend, hostvm
    traces = list(fibs)
    tr = traces[3]
    regs = tr.registers.copy()
    regs[tr.width - 1, 100, 0] += 1
    traces[3] = hostvm.ExecutionTrace(regs, tr.ctx_depth, tr.loop_depth, tr.stack_depth, tr.program_hash, tr.public_inputs, tr.outputs)
    opts = [O(32, 1, 0), O(16, 50, 8), O(32, 128, 20), O(32, 50, 8), O(16, 1, 20), O(32, 50, 0)]
    result = dg.prove_traces(traces, opts)
    assert isinstance(result[3], backend.DgError) and result[3].code == -5
    with pytest.raises(backend.DgError) as alone:
        dg.prove(traces[3], opts[3])
    assert str(result[3]) == str(alone.value)
    for i in (0, 1, 2, 4, 5):
        assert result[i].bytes == single(traces[i], opts[i]), i


def _recorder(po, log):
    from distaff_b200 import felt

    def draw_field(seed, count):
        log.append(("field", seed, count))
        return felt.from_ints(po.prng_vector(seed, count)).tobytes()

    def draw_positions(seed, domain, ext, nq):
        log.append(("positions", seed, domain, nq))
        return po.query_positions(seed, domain, ext, nq)
    return draw_field, draw_positions


def test_rng_callbacks_see_partitions_in_order_of_first_appearance(dg, po, pool, fibs, single, monkeypatch):
    """partitions (length, extension factor) in order of first appearance, input order inside: with groups of one trace the calls are
    the single proofs' calls in that order; in one call each trace's calls are its own and the first draws come in that order"""
    from distaff_b200 import backend
    traces = [fibs[0], pool["collatz3"], fibs[1], pool["wide"], fibs[2], pool["collatz5"], fibs[3], pool["hash"]]
    opts = [O(32, 50, 8), O(32, 1, 0), O(16, 128, 0), O(32, 7, 4), O(32, 128, 20), O(16, 50, 8), O(16, 1, 20), O(64, 50, 0)]
    keys = [(t.length, o.extension_factor) for t, o in zip(traces, opts)]
    seen = []
    for k in keys:
        if k not in seen:
            seen.append(k)
    expect = [i for k in seen for i in range(len(traces)) if keys[i] == k]
    assert expect != list(range(len(traces)))
    for tr, o in zip(traces, opts):                  # the single proofs before any callback is registered
        single(tr, o)
    own = []
    try:
        for tr, o in zip(traces, opts):
            log = []
            backend.set_rng_callbacks(*_recorder(po, log))
            assert dg.prove(tr, o).bytes == single(tr, o)
            own.append(log)
        log = []
        backend.set_rng_callbacks(*_recorder(po, log))
        check(dg, traces, opts, dg.prove_traces(traces, opts), single)
        for i in range(len(traces)):
            mine = [e for e in log if any(e[1] == x[1] for x in own[i])]
            assert mine == own[i], i
        firsts = [next(i for i in range(len(traces)) if own[i][0][1] == e[1]) for e in log if any(own[i][0][1] == e[1] for i in range(len(traces)))]
        assert firsts == expect, (firsts, expect)
        monkeypatch.setenv("DG_BATCH_GROUP", "1")
        log = []
        backend.set_rng_callbacks(*_recorder(po, log))
        check(dg, traces, opts, dg.prove_traces(traces, opts), single)
        assert log == [e for i in expect for e in own[i]]
    finally:
        backend.set_rng_callbacks()


def test_equal_options_list_is_the_single_options_call(dg, pool, fibs):
    traces = list(fibs[:3]) + [pool["collatz3"], pool["wide"], pool["hash"]]
    for o in (O(), O(16, 1, 0)):
        dg.prove_traces(traces, o)                   # warm-up: tables of a new shape are built by the first call
        one = dg.prove_traces(traces, o)
        listed = dg.prove_traces(traces, [o] * len(traces))
        assert [p.bytes for p in listed] == [p.bytes for p in one]
        assert listed[0].stats["kernel_launches"] == one[0].stats["kernel_launches"]


def test_invalid_options_of_one_trace_fail_the_call(dg, fibs):
    from distaff_b200 import backend
    bad = O()
    bad.num_queries = 129
    with pytest.raises(backend.DgError) as e:
        dg.prove_traces(fibs[:3], [O(), O(16, 1, 0), bad])
    assert e.value.code == -1 and "trace 2: num_queries must be in 1..128" in str(e.value)
    bad = O()
    bad.extension_factor = 512
    with pytest.raises(backend.DgError) as e:
        dg.prove_traces(fibs[:3], [O(), bad, O()])
    assert e.value.code == -1 and "trace 1: extension_factor must be a power of 2" in str(e.value)


def _jobs():
    from distaff_b200 import hostvm
    X = __import__("distaff_b200").ProgramInputs
    fib = hostvm.fibonacci_program(13)
    jobs = [(fib, X([i + 1, i])) for i in range(4)]
    jobs += [(hostvm.COLLATZ_SOURCE, X([], [s])) for s in (3, 5, 6)]
    jobs += [("begin pad.2 hash.2 end", X([5 + i, 6]), 2) for i in range(2)]
    opts = [O(32, 1, 0), O(16, 50, 8), O(32, 128, 20), O(16, 50, 8), O(32, 50, 0), O(16, 7, 4), O(32, 1, 0), O(64, 50, 8), O(32, 128, 20)]
    return jobs, opts


@pytest.mark.parametrize("call", ["execute_programs", "execute_many"])
def test_execute_calls_with_per_job_options(dg, call):
    from distaff_b200 import hostvm
    run = getattr(dg, call)
    jobs, opts = _jobs()
    got = run(jobs, opts)
    for o in set(opts):                          # each job's result is that of the same call with its options alone
        alone = run(jobs, o)
        for i, (job_o, res) in enumerate(zip(opts, got)):
            if job_o == o:
                assert not isinstance(res, Exception), (i, res)
                assert res[0] == alone[i][0] and res[1].bytes == alone[i][1].bytes, (i, o)
                assert res[1].options == o
    items = []
    for job, (outputs, proof) in zip(jobs, got):
        prog = job[0] if not isinstance(job[0], str) else hostvm.compile_program(job[0])
        items.append((prog.hash, job[1].public, outputs, proof))
    assert dg.verify_batch(items) == [None] * len(items)
