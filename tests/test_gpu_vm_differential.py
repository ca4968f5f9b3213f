"""The GPU VM (vm.cu, execute.cu) against the host VM on the case sets of tests/vm_cases.py: edge operands of every op, the failure
catalogue and a few hundred generated programs.  Every trace byte for byte, every failure with the host VM's message and step, the
shapes-only call against the full one, failures only the write pass can see between successes of one shape slab, the trace-length and
step-cap boundaries, and -- since the host VM is itself a restatement -- the traces against the AIR and a sample of proofs against the
oracle's verifier."""
import ctypes
import functools

import numpy as np
import pytest

import distaff_b200 as dg
from distaff_b200 import api, backend, felt
from tests import vm_cases as vc

pytestmark = pytest.mark.gpu
X = dg.ProgramInputs
EXECUTION = -7
HASH_MESSAGE = "program hash does not match trace hash"
LOOP_IMAGE_MESSAGE = "hash of the last iteration doesn't match loop image"


@functools.lru_cache(maxsize=None)
def _cases():
    cases = vc.edge_cases() + vc.catalogue_cases() + vc.generated_cases() + vc.boundary_cases()
    return cases, [vc.host(c) for c in cases]


def _jobs(cases):
    return [(c.program, c.inputs, c.num_outputs) for c in cases]


def _same(got, want):
    assert not isinstance(got, backend.DgError), got
    assert got.registers.shape == want.registers.shape
    assert np.array_equal(got.registers, want.registers)
    assert (got.ctx_depth, got.loop_depth, got.stack_depth) == (want.ctx_depth, want.loop_depth, want.stack_depth)
    assert got.program_hash == want.program_hash and got.outputs == want.outputs and got.public_inputs == want.public_inputs


def _failed(got, message):
    assert isinstance(got, backend.DgError) and got.code == EXECUTION, got
    assert str(got) == f"distaff_gpu error {EXECUTION}: {message}"


def _shapes_only(jobs, max_steps=api.MAX_STEPS):
    """dg_trace_programs with registers_out = NULL: per job, the info dict or the DgError"""
    programs, cprogs, program_of, arr, _, keep = api._programs_args(jobs)
    k = len(jobs)
    info = (backend.DgExecutionInfo * k)()
    status = (ctypes.c_int * k)()
    backend.check(backend.lib().dg_trace_programs(cprogs, len(programs), k, program_of, arr, int(max_steps), info, None, status, None))
    errors = api._messages(list(status))
    del keep
    return [e if e is not None else {f: int(getattr(info[i], f)) for f, _ in backend.DgExecutionInfo._fields_} for i, e in enumerate(errors)]


def _execute_raw(jobs):
    """dg_execute_programs, returning (results as execute_programs returns them, the whole outputs16 array (k, 8) of ints)"""
    programs, cprogs, program_of, arr, num_outputs, keep = api._programs_args(jobs)
    k = len(jobs)
    opt = dg.ProofOptions()._c()
    handles = (backend.vp * k)()
    outputs = np.zeros((k, 8, 2), dtype=np.uint64)
    outputs[:] = 0xAB                                       # whatever the caller's buffer held
    status = (ctypes.c_int * k)()
    pst, st = backend.DgStats(), backend.DgExecutionStats()
    backend.check(backend.lib().dg_execute_programs(cprogs, len(programs), k, program_of, arr, (backend.u32 * k)(*num_outputs),
                                                   api.MAX_STEPS, ctypes.byref(opt), handles, outputs.ctypes.data, status, ctypes.byref(pst),
                                                   ctypes.byref(st)))
    errors = api._messages(list(status))
    del keep
    res = [e if e is not None else (felt.to_ints(outputs[i, :num_outputs[i]]), api._collect(handles[i], pst)) for i, e in enumerate(errors)]
    return res, [felt.to_ints(outputs[i]) for i in range(k)]


def test_every_case_matches_the_host_vm_and_the_air():
    cases, want = _cases()
    jobs = _jobs(cases)
    assert len(jobs) >= 4000
    got = dg.trace_programs(jobs)
    good = []
    for c, w, g in zip(cases, want, got):
        if isinstance(w, str):
            _failed(g, w)
        else:
            _same(g, w)
            good.append(w)
    assert 0.5 < len(good) / len(cases) < 0.9
    # the shapes-only call reports what the full call reports, but for the failures that need the sponge
    for c, w, s in zip(cases, want, _shapes_only(jobs)):
        if isinstance(w, str) and not w.startswith((HASH_MESSAGE, LOOP_IMAGE_MESSAGE)):
            _failed(s, w)
            continue
        assert not isinstance(s, backend.DgError), (c.name, s)
        if not isinstance(w, str):
            assert (s["width"], s["length"], s["ctx_depth"], s["loop_depth"], s["stack_depth"]) == (
                w.width, w.length, w.ctx_depth, w.loop_depth, w.stack_depth), c.name
    # the host VM restates the reference, so the traces both VMs agree on are checked against the AIR as well
    reports = dg.check_traces(good, [t.program_hash for t in good])
    bad = [str(r) for r in reports if not r.ok]
    assert not bad, bad[:3]


def test_the_catalogue_on_the_gpu():
    cat = vc.failure_catalogue()
    reached = [e for e in cat.values() if isinstance(e, vc.Reached) and e.max_steps is None]
    got = dg.trace_programs(_jobs([e.case for e in reached]))
    for e, g in zip(reached, got):
        _failed(g, e.message if e.step is None else f"{e.message} at step {e.step}")
    cap = cat["VM_CAP"]
    _failed(dg.trace_programs(_jobs([cap.case]), max_steps=cap.max_steps)[0], cap.message)
    for name, e in cat.items():
        if isinstance(e, vc.Unreachable) and e.program is not None:       # ruled out by validation: the call is rejected
            with pytest.raises(backend.DgError) as err:
                dg.trace_programs([(e.program, X(), 1)])
            assert err.value.code == -1 and "invalid program encoding" in str(err.value), name
    for case, message in vc.input_failures():
        _failed(dg.trace_programs([(case.program, case.inputs, 1), ("begin add end", X([1, 2]), 1)])[0], message)


def _slab_jobs():
    """a loop program and copies of it with a wrong program hash or loop image, alternating in one shape slab"""
    src = vc.LOOP_SOURCE
    bad = [vc.encoding(src, hash32=bytes(32)), vc.failure_catalogue()["VM_LOOP_IMAGE"].case.program]
    jobs, want = [], []
    for i in range(9):
        x = X([i, 2**64 + i])
        if i % 3 == 0:
            jobs.append((src, x, 2))
        else:
            jobs.append((bad[i % 3 - 1], x, 2))
        want.append(vc.host(vc.Case("", *jobs[-1])))
    return jobs, want


@pytest.mark.parametrize("group", [None, "2"])
def test_failures_only_the_write_pass_sees_between_successes(group, monkeypatch):
    if group:
        monkeypatch.setenv("DG_BATCH_GROUP", group)
    jobs, want = _slab_jobs()
    assert {w.split(" at step")[0] for w in want if isinstance(w, str)} == {HASH_MESSAGE, LOOP_IMAGE_MESSAGE}
    shapes = _shapes_only(jobs)
    assert len({(s["width"], s["length"]) for s in shapes}) == 1          # one slab; the shape pass sees no failure
    stats = {}
    res, outputs = _execute_raw(jobs)
    got = dg.execute_programs(jobs, stats=stats)
    if group:
        assert stats["waves"] == 5, stats
    good = [w for w in want if not isinstance(w, str)]
    ref = dg.prove_batch(good)
    it = iter(ref)
    for j, w, r, g, out in zip(jobs, want, res, got, outputs):
        if isinstance(w, str):
            _failed(r, w)
            _failed(g, w)
            assert out == [0] * 8
            continue
        p = next(it)
        assert r[0] == g[0] == w.outputs and r[1].bytes == g[1].bytes == p.bytes
        assert out[:2] == w.outputs and out[2:] == [0] * 6


def test_a_sample_of_proofs_against_the_host_and_the_verifier(po):
    cases, want = _cases()
    good = [(c, w) for c, w in zip(cases, want) if not isinstance(w, str)]
    picked = good[::max(1, len(good) // 20)][:20]
    got = dg.execute_programs(_jobs([c for c, _ in picked]))
    ref = dg.prove_batch([w for _, w in picked])
    for (c, w), g, p in zip(picked, got, ref):
        assert not isinstance(g, backend.DgError), (c.name, g)
        assert g[0] == w.outputs and g[1].bytes == p.bytes, c.name
        assert po.verify(w.program_hash, w.public_inputs, w.outputs, g[1].bytes) is None, c.name


def test_trace_length_and_step_cap_boundaries():
    for c in vc.boundary_cases():
        want = vc.host(c)
        last = int(c.name.split()[-1])
        _same(dg.trace_programs(_jobs([c]), max_steps=last + 1)[0], want)
        assert want.length == 2 ** last.bit_length()           # 2^k - 1 fills 2^k rows, 2^k + 15 needs 2^(k + 1)
        for cap in (last, 16):
            _failed(dg.trace_programs(_jobs([c]), max_steps=cap)[0], f"execution exceeds {cap} steps")
            _failed(_shapes_only(_jobs([c]), max_steps=cap)[0], f"execution exceeds {cap} steps")
