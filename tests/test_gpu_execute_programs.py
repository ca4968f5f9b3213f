"""Executing many programs in one call on the GPU (dg_trace_programs / dg_execute_programs): traces byte-identical to the host VM's,
proofs byte-identical to execute_batch of each program alone, to dg.execute's and to the golden oracle proofs; same-shape traces of
different programs proven together; one write launch for every shape of a wave; each program's executions in warps of their own."""
import hashlib
import json
import os

import numpy as np
import pytest

import distaff_b200 as dg
from distaff_b200 import backend, hostvm
from tests import execution_cases as cases
from tests.test_gpu_execute_batch import FAIL_CASES, FAIL_SOURCE

pytestmark = pytest.mark.gpu
GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "oracle_proofs.json")))
X = dg.ProgramInputs


def _same(a, b):
    assert a.registers.shape == b.registers.shape
    assert np.array_equal(a.registers, b.registers)
    assert (a.ctx_depth, a.loop_depth, a.stack_depth) == (b.ctx_depth, b.loop_depth, b.stack_depth)
    assert a.program_hash == b.program_hash and a.outputs == b.outputs and a.public_inputs == b.public_inputs


def _host(job):
    src, x = job[0], job[1]
    return hostvm.execute(src, x.public, x.secret_a, x.secret_b, job[2] if len(job) == 3 else 1)


def _mixed_suite():
    """(jobs, golden names): every program of the suite twice, collatz, fibonacci, merkle and compare on several inputs each, interleaved"""
    runs = [[((src, X(pub, a, b), no), name)] * 2 for name, src, pub, a, b, no in cases.SMALL]
    runs.append([((hostvm.COLLATZ_SOURCE, X([], [s])), None) for s in (5, 6, 27)])
    runs.append([((hostvm.fibonacci_program(50), X([i + 1, 3 * i])), None) for i in range(3)])
    merkle = [cases.merkle_case(16, 1, seed=s, index_of=lambda c: 777) for s in range(3)]
    runs.append([((src, X([], a, b), 4), None) for src, a, b in merkle])
    runs.append([((cases.COMPARE_SOURCE, X([x, y]), 4), None) for x, y in ((5, 9), (9, 5), (7, 7))])
    jobs, names = [], []
    for r in range(max(len(run) for run in runs)):
        for run in runs:
            if r < len(run):
                jobs.append(run[r][0])
                names.append(run[r][1])
    return jobs, names


def test_mixed_suite_traces_and_proofs():
    jobs, names = _mixed_suite()
    assert len({j[0] for j in jobs}) >= 18
    stats = {}
    traces = dg.trace_programs(jobs, stats=stats)
    for job, tr in zip(jobs, traces):
        assert not isinstance(tr, backend.DgError), tr
        _same(tr, _host(job))
    assert stats["waves"] == 1 and stats["write_launches"] == 1, stats
    got = dg.execute_programs(jobs)
    hashes = {j[0]: hostvm.compile_program(j[0]).hash for j in jobs}
    distinct = list(hashes.values())
    for job, name, res in zip(jobs, names, got):
        assert not isinstance(res, backend.DgError), res
        src, x = job[0], job[1]
        no = job[2] if len(job) == 3 else 1
        outputs, proof = res
        alone = dg.execute_batch(src, [x], num_outputs=no)[0]
        assert outputs == alone[0] and proof.bytes == alone[1].bytes
        ref_out, ref = dg.execute(src, x.public, x.secret_a, x.secret_b, num_outputs=no)
        assert outputs == ref_out and proof.bytes == ref.bytes
        if name is not None:
            assert hashlib.sha256(proof.bytes).hexdigest() == GOLDEN[name]["proof_sha256"], name
        h = hashes[src]
        assert dg.verify(h, x.public, outputs, proof) is None
        other = next(d for d in distinct if d != h)
        assert dg.verify(other, x.public, outputs, proof) is not None


def test_same_shape_programs_are_proven_together():
    a, b = "begin push.1 push.2 add end", "begin push.1 push.3 add end"
    ha, hb = hostvm.compile_program(a).hash, hostvm.compile_program(b).hash
    assert ha != hb
    jobs = [(a, X([i])) if i % 2 == 0 else (b, X([i])) for i in range(6)]
    shapes = {(t.width, t.length) for t in dg.trace_programs(jobs)}
    assert len(shapes) == 1
    stats = {}
    got = dg.execute_programs(jobs, stats=stats)
    assert stats["prove_groups"] == 1, stats
    for (src, x), (outputs, proof) in zip(jobs, got):
        alone = dg.execute_batch(src, [x])[0]
        assert outputs == alone[0] and proof.bytes == alone[1].bytes
        assert dg.verify(ha if src == a else hb, x.public, outputs, proof) is None


def _three_shapes():
    jobs = [(hostvm.fibonacci_program(13), X([i + 1, i])) for i in range(3)]
    jobs += [(hostvm.COLLATZ_SOURCE, X([], [s])) for s in (3, 27, 97)]
    jobs += [(cases.COMPARE_SOURCE, X([i, 2 * i]), 4) for i in range(1, 4)]
    return jobs[0::3] + jobs[1::3] + jobs[2::3]


def test_one_write_launch_for_every_shape_and_waves_under_batch_group(monkeypatch):
    jobs = _three_shapes()
    stats, pstats = {}, {}
    traces = dg.trace_programs(jobs, stats=stats)
    assert len({(t.width, t.length) for t in traces}) >= 3
    assert stats["waves"] == 1 and stats["write_launches"] == 1, stats
    proofs = dg.execute_programs(jobs, stats=pstats)
    assert pstats["waves"] == 1 and pstats["write_launches"] == 1, pstats
    monkeypatch.setenv("DG_BATCH_GROUP", "2")
    stats2, pstats2 = {}, {}
    for a, b in zip(dg.trace_programs(jobs, stats=stats2), traces):
        _same(a, b)
    assert stats2["waves"] == stats2["write_launches"] == (len(jobs) + 1) // 2, stats2
    got = dg.execute_programs(jobs, stats=pstats2)
    assert pstats2["waves"] > 1
    assert [g[1].bytes for g in got] == [p[1].bytes for p in proofs] and [g[0] for g in got] == [p[0] for p in proofs]


def test_each_program_starts_a_warp():
    a, b = hostvm.fibonacci_program(13), hostvm.fibonacci_program(20)
    jobs = [(a, X([i, 1])) for i in range(5)] + [(b, X([i, 2])) for i in range(40)]
    stats = {}
    traces = dg.trace_programs(jobs[::-1], stats=stats)
    assert stats["lanes"] == 96 and stats["waves"] == 1, stats
    for job, tr in zip(jobs[::-1], traces):
        _same(tr, _host(job))


def test_failures_beside_other_programs_and_the_step_cap():
    jobs, expected = [], []
    for i, (name, x) in enumerate(FAIL_CASES):
        jobs.append((FAIL_SOURCE, x))
        jobs.append((hostvm.fibonacci_program(13), X([i, 1])))
    jobs.insert(3, (hostvm.COLLATZ_SOURCE, X([], [27])))       # more than 2^10 steps
    for job in jobs:
        if (job[1].public == [5, 6] and job[1].secret_a == [0, 1]) or job[0] == hostvm.COLLATZ_SOURCE:
            expected.append("execution exceeds 1024 steps")
            continue
        try:
            _host(job)
            expected.append(None)
        except RuntimeError as e:
            expected.append(str(e)[len("vm: "):])
    cap = 2**10
    traces = dg.trace_programs(jobs, max_steps=cap)
    proofs = dg.execute_programs(jobs, max_steps=cap)
    assert sum(e is None for e in expected) >= 10
    for job, want, tr, pr in zip(jobs, expected, traces, proofs):
        if want is None:
            _same(tr, _host(job))
            alone = dg.execute_batch(job[0], [job[1]], max_steps=cap)[0]
            assert pr[0] == alone[0] and pr[1].bytes == alone[1].bytes
            continue
        for got in (tr, pr):
            assert isinstance(got, backend.DgError) and got.code == -7, (job, got)
            assert str(got) == "distaff_gpu error -7: " + want


def test_outputs_per_execution():
    src = cases.COMPARE_SOURCE
    jobs = [(src, X([5, 9]), 0), (src, X([5, 9]), 2), (src, X([9, 5]), 4), (hostvm.fibonacci_program(13), X([1, 0]), 1)]
    got = dg.execute_programs(jobs)
    for (s, x, no), (outputs, proof) in zip(jobs, got):
        assert len(outputs) == no
        alone = dg.execute_batch(s, [x], num_outputs=no)[0]
        assert outputs == alone[0] and proof.bytes == alone[1].bytes


def test_memory_limit_holds_and_bytes_are_unchanged():
    fib = hostvm.fibonacci_program(600)
    jobs = [(fib, X([i + 1, 2 * i])) for i in range(6)] + [(hostvm.COLLATZ_SOURCE, X([], [s])) for s in (7, 9)]
    ref = dg.execute_programs(jobs)
    ref_traces = dg.trace_programs(jobs)
    tr = ref_traces[0]
    plan = dg.plan_prove(tr.width, tr.length, 6)
    limit = plan["fixed_bytes"] + 2 * plan["bytes_per_proof"] + (256 << 20)
    try:
        dg.set_memory_limit(limit)
        assert dg.plan_prove(tr.width, tr.length, 6)["group"] < 6
        got = dg.execute_programs(jobs)
        assert [g[1].bytes for g in got] == [r[1].bytes for r in ref] and [g[0] for g in got] == [r[0] for r in ref]
        for a, b in zip(dg.trace_programs(jobs), ref_traces):
            _same(a, b)
        assert dg.memory_usage()["peak"] <= limit
    finally:
        dg.set_memory_limit(0)
