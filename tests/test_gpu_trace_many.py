"""Many executions from sponge tables in one call (dg_trace_many / dg_execute_many) against the batch path (dg_trace_programs /
dg_execute_programs): every case of tests/vm_cases.py in one call, inconsistent encodings mixed with consistent ones, proofs against
execute_programs, the golden oracle proofs and the oracle's verifier, bench.py's 2^20-step collatz beside short executions, the
one-execution case against trace_one, waves and sequential re-runs under a memory limit, the step cap, failures beside successes and the
RNG callback order."""
import hashlib
import json
import os
import random
import re

import numpy as np
import pytest

import distaff_b200 as dg
from distaff_b200 import backend, felt, hostvm
from tests import execution_cases as ec
from tests import vm_cases as vc
from tests.test_gpu_trace_one import _switch_with_unread_hash

pytestmark = pytest.mark.gpu
X = dg.ProgramInputs
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = json.load(open(os.path.join(ROOT, "tests", "golden", "oracle_proofs.json")))
INCONSISTENT = {"hash of the last iteration doesn't match loop image", "wrong switch hash"}


def _same(got, want):
    if isinstance(want, backend.DgError):
        assert isinstance(got, backend.DgError) and (got.code, str(got)) == (want.code, str(want)), (got, want)
        return
    assert not isinstance(got, backend.DgError), got
    assert got.registers.shape == want.registers.shape and np.array_equal(got.registers, want.registers)
    assert (got.ctx_depth, got.loop_depth, got.stack_depth) == (want.ctx_depth, want.loop_depth, want.stack_depth)
    assert got.program_hash == want.program_hash and got.outputs == want.outputs and got.public_inputs == want.public_inputs


def _same_proofs(got, want):
    assert len(got) == len(want)
    for g, w in zip(got, want):
        if isinstance(w, backend.DgError):
            assert isinstance(g, backend.DgError) and (g.code, str(g)) == (w.code, str(w)), (g, w)
        else:
            assert not isinstance(g, backend.DgError), g
            assert g[0] == w[0] and g[1].bytes == w[1].bytes


def _jobs(cases):
    return [(c.program, c.inputs, c.num_outputs) for c in cases]


@pytest.mark.parametrize("segment_steps", [16, 0])
def test_every_case_in_one_call_matches_trace_programs(segment_steps):
    cases = vc.edge_cases() + vc.catalogue_cases() + vc.generated_cases() + vc.boundary_cases()
    assert len(cases) >= 4000
    jobs = _jobs(cases)
    st = {}
    got = dg.trace_many(jobs, segment_steps=segment_steps, stats=st)
    want = dg.trace_programs(jobs)
    for c, g, w in zip(cases, got, want):
        _same(g, w)
    ok = sum(not isinstance(w, backend.DgError) for w in want)
    assert st["segment_steps"] == (segment_steps or 1024)
    assert st["fallback_programs"] == sum(c.name in INCONSISTENT for c in cases) and st["fallback_programs"] >= 2, st
    assert st["table_levels"] >= 2 and st["sequential_launches"] >= 1 and st["waves"] >= 1, st
    print(f"segment_steps {segment_steps}: {st['segments']} segments for {ok} successful executions")
    if segment_steps == 16:
        assert st["segments"] > 2 * ok, st


def _consistency_mix():
    cat = {c.name: c for c in vc.catalogue_cases()}
    bad = [cat[n] for n in sorted(INCONSISTENT)]
    good = [c for c in vc.edge_cases()[:12]]
    jobs = []
    for i, c in enumerate(good):
        jobs.append((c.program, c.inputs, c.num_outputs))
        if i % 4 == 1:
            b = bad[(i // 4) % len(bad)]
            jobs.append((b.program, b.inputs, b.num_outputs))
    return jobs


@pytest.mark.parametrize("segment_steps", [16, 0])
def test_inconsistent_programs_run_on_the_batch_path_in_the_same_call(segment_steps):
    jobs = _consistency_mix()
    n_programs = len(dg.api.pack_jobs(jobs)[0])
    st = {}
    got = dg.trace_many(jobs, segment_steps=segment_steps, stats=st)
    for g, w in zip(got, dg.trace_programs(jobs)):
        _same(g, w)
    assert st["fallback_programs"] == len(INCONSISTENT) and st["tabled_programs"] == n_programs - len(INCONSISTENT), st
    assert st["fallback"]["shape_launches"] >= 1 and st["fallback"]["write_launches"] >= 1, st
    _same_proofs(dg.execute_many(jobs, segment_steps=segment_steps), dg.execute_programs(jobs))


def _proving_jobs():
    """(jobs, golden names): every program of tests/execution_cases.py, collatz, fibonacci and merkle, interleaved and shuffled"""
    runs = [((src, X(pub, a, b), no), name) for name, src, pub, a, b, no in ec.SMALL]
    runs += [((hostvm.COLLATZ_SOURCE, X([], [s])), None) for s in (5, 27, 97)]
    runs += [((hostvm.fibonacci_program(50), X([i + 1, 3 * i])), None) for i in range(2)]
    runs += [((src, X([], a, b), 4), None) for src, a, b in [ec.merkle_case(16, 1, seed=s, index_of=lambda c: 777) for s in range(2)]]
    random.Random(7).shuffle(runs)
    return [r[0] for r in runs], [r[1] for r in runs]


def test_proofs_equal_execute_programs_golden_and_the_verifier(po):
    jobs, names = _proving_jobs()
    st = {}
    got = dg.execute_many(jobs, stats=st)
    want = dg.execute_programs(jobs)
    _same_proofs(got, want)
    assert st["fallback_programs"] == 0 and st["prove_groups"] >= 1, st
    golden = 0
    for name, (outputs, proof) in zip(names, got):
        if name is not None and name in GOLDEN:
            assert hashlib.sha256(proof.bytes).hexdigest() == GOLDEN[name]["proof_sha256"], name
            golden += 1
    assert golden >= 10
    hashes = {j[0]: hostvm.compile_program(j[0]).hash for j in jobs}
    for job, (outputs, proof) in list(zip(jobs, got))[:4]:
        h = hashes[job[0]]
        assert po.verify(h, job[1].public, outputs, proof.bytes) is None
        other = next(v for v in hashes.values() if v != h)
        assert po.verify(other, job[1].public, outputs, proof.bytes) is not None


def test_bench_collatz_2_20_beside_short_executions():
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "collatz_2_20.json")))
    start = int(re.search(r"start=(\d+)", gold["name"]).group(1))
    jobs = [(hostvm.COLLATZ_SOURCE, X([], [27])), (hostvm.COLLATZ_SOURCE, X([], [start])), (hostvm.fibonacci_program(50), X([1, 0])),
            (hostvm.COLLATZ_SOURCE, X([], [5]))]
    st = {}
    traces = dg.trace_many(jobs, stats=st)
    tr = traces[1]
    assert tr.length == 2**20 and st["fallback_programs"] == 0 and st["segments"] > 500, st
    assert hashlib.sha256(np.ascontiguousarray(tr.registers).tobytes()).hexdigest() == gold["trace_sha256"]
    for i in (0, 2, 3):
        _same(traces[i], dg.trace_programs([jobs[i]])[0])
    got = dg.execute_many(jobs)
    assert got[1][0] == tr.outputs and hashlib.sha256(got[1][1].bytes).hexdigest() == gold["proof_sha256"]
    for i in (0, 2, 3):
        w = dg.execute_programs([jobs[i]])[0]
        assert got[i][0] == w[0] and got[i][1].bytes == w[1].bytes


@pytest.mark.parametrize("segment_steps", [16, 0])
def test_one_execution_equals_trace_one(segment_steps):
    for job in [(hostvm.COLLATZ_SOURCE, X([], [97])), (ec.IF_ELSE, X([], [1])), (hostvm.fibonacci_program(40), X([1, 1]))]:
        many, one = {}, {}
        got = dg.trace_many([job], segment_steps=segment_steps, stats=many)[0]
        want = dg.trace_one(job[0], job[1], segment_steps=segment_steps, stats=one)
        _same(got, want)
        assert many["segments"] == one["segments"] and many["checkpoints"] == one["checkpoints"] and many["logged"] == one["logged"]


def test_waves_and_sequential_reruns_under_a_memory_limit(monkeypatch):
    starts = [27, 5, 871, 97, 7, 6171, 27, 3, 871, 97, 6171, 27] * 2
    jobs = [(hostvm.COLLATZ_SOURCE, X([], [s])) for s in starts] + [(hostvm.fibonacci_program(60), X([1, 2]))]
    want = dg.trace_programs(jobs)
    free = {}
    for g, w in zip(dg.trace_many(jobs, segment_steps=16, stats=free), want):
        _same(g, w)
    assert free["sequential_launches"] == 1 and free["waves"] == 1, free
    monkeypatch.setenv("DG_BATCH_GROUP", "2")
    st = {}
    try:
        dg.set_memory_limit(1)                     # frees the proof arena; what stays held are the library's persistent tables
        dg.set_memory_limit(dg.memory_usage()["held"] + (192 << 20))
        got = dg.trace_many(jobs, segment_steps=16, stats=st)
    finally:
        dg.set_memory_limit(0)
    for g, w in zip(got, want):
        _same(g, w)
    assert st["waves"] > 1 and st["sequential_launches"] > 1, st
    assert st["segments"] == free["segments"] and st["logged"] == free["logged"]


def test_step_cap_for_several_executions_at_once():
    cases = vc.boundary_cases()
    jobs = _jobs(cases)
    for c in cases[:6]:
        last = int(c.name.split()[-1])
        for cap in (last, last + 1):
            want = dg.trace_programs(jobs, max_steps=cap)
            for seg in (16, 0):
                got = dg.trace_many(jobs, max_steps=cap, segment_steps=seg)
                for g, w in zip(got, want):
                    _same(g, w)
            at = cases.index(c)
            if cap == last:
                assert isinstance(got[at], backend.DgError) and str(got[at]).endswith(f"execution exceeds {cap} steps")
            else:
                assert not isinstance(got[at], backend.DgError)


def test_a_failing_execution_changes_nothing_else():
    src = hostvm.COLLATZ_SOURCE
    jobs = [(src, X([], [27])), (src, X([], [])), (src, X([], [31])), (src, X([], [2**128 - 1])), (src, X([], [27])),
            ("begin push.1 push.2 add assert end", X()), (src, X([], [41]))]
    got = dg.trace_many(jobs, segment_steps=16)
    want = dg.trace_programs(jobs)
    for g, w in zip(got, want):
        _same(g, w)
    assert sum(isinstance(g, backend.DgError) for g in got) == 3
    _same(got[0], dg.trace_many([jobs[0]])[0])
    _same(got[4], got[0])
    _same_proofs(dg.execute_many(jobs, segment_steps=16), dg.execute_programs(jobs))


def test_rng_callbacks_follow_the_documented_order(po):
    seen = []

    def draw_field(seed, count):
        seen.append(("field", bytes(seed), count))
        return felt.from_ints(po.prng_vector(seed, count)).tobytes()

    def draw_positions(seed, domain, ext, nq):
        seen.append(("positions", bytes(seed), domain, ext, nq))
        return po.query_positions(seed, domain, ext, nq)

    unread = _switch_with_unread_hash()             # inconsistent, and its execution succeeds: proven on the batch path
    fallback = [(unread.program, unread.inputs, unread.num_outputs)]
    tabled = [(hostvm.COLLATZ_SOURCE, X([], [s])) for s in (9, 27)] + [(hostvm.fibonacci_program(13), X([1, i])) for i in range(2)]
    tabled += [(ec.COMPARE_SOURCE, X([3, 4]), 4)]
    jobs = [tabled[0], tabled[2]] + fallback + tabled[1:2] + tabled[3:]
    try:
        backend.set_rng_callbacks(draw_field, draw_positions)
        dg.execute_programs(fallback)
        want = list(seen)
        seen.clear()
        dg.execute_programs([j for j in jobs if j not in fallback])
        want += seen
        seen.clear()
        dg.execute_many(jobs)
    finally:
        backend.set_rng_callbacks()
    assert len(want) >= 8 and seen == want
