"""One execution split across GPU threads (dg_trace_one / dg_execute_one) against the host VM: every case of tests/vm_cases.py at the
library's segment length and at 16 steps (so that segments start inside loops, after BREAK, around switches and at depth 15), the
fallback for inconsistent block hashes, the step cap, proofs against dg.execute and the oracle's verifier, and bench.py's 2^20-step
collatz trace against its golden digests."""
import ctypes
import hashlib
import json
import os
import re

import numpy as np
import pytest

import distaff_b200 as dg
from distaff_b200 import backend, hostvm
from tests import execution_cases as ec
from tests import vm_cases as vc

pytestmark = pytest.mark.gpu
X = dg.ProgramInputs
EXECUTION = -7
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _same(got, want):
    assert got.registers.shape == want.registers.shape
    assert np.array_equal(got.registers, want.registers)
    assert (got.ctx_depth, got.loop_depth, got.stack_depth) == (want.ctx_depth, want.loop_depth, want.stack_depth)
    assert got.program_hash == want.program_hash and got.outputs == want.outputs and got.public_inputs == want.public_inputs


def _run(case, segment_steps, max_steps=dg.api.MAX_STEPS):
    """(trace or DgError, stats)"""
    st = {}
    try:
        return dg.trace_one(case.program, case.inputs, max_steps=max_steps, num_outputs=case.num_outputs, segment_steps=segment_steps,
                            stats=st), st
    except backend.DgError as e:
        return e, st


def _run_sized(case, want, segment_steps):
    """dg_trace_one once, with the buffer sized from the host VM's trace (trace_one sizes it with a call without registers first)"""
    if isinstance(want, str):
        return _run(case, segment_steps)
    prog, cprog, arr, keep = dg.api._execution_args(case.program, [case.inputs])
    regs = np.zeros_like(want.registers)
    info, st = backend.DgExecutionInfo(), backend.DgTraceOneStats()
    rc = backend.lib().dg_trace_one(ctypes.byref(cprog), arr, dg.api.MAX_STEPS, segment_steps, ctypes.byref(info), regs.ctypes.data,
                                    ctypes.byref(st))
    del keep
    stats = {f: getattr(st, f) for f, _ in backend.DgTraceOneStats._fields_}
    if rc != 0:
        return backend.DgError(rc, backend.lib().dg_last_error().decode()), stats
    assert (info.width, info.length, info.ctx_depth, info.loop_depth, info.stack_depth) == (
        want.width, want.length, want.ctx_depth, want.loop_depth, want.stack_depth), case.name
    return hostvm.ExecutionTrace(regs, info.ctx_depth, info.loop_depth, info.stack_depth, prog.hash, list(case.inputs.public),
                                 want.outputs), stats


def _check(case, want, got):
    if isinstance(want, str):
        assert isinstance(got, backend.DgError) and got.code == EXECUTION, (case.name, got)
        assert str(got) == f"distaff_gpu error {EXECUTION}: {want}", case.name
    else:
        assert not isinstance(got, backend.DgError), (case.name, got)
        _same(got, want)


# the hand-made encodings whose block hashes do not match their blocks on some path
INCONSISTENT = {"hash of the last iteration doesn't match loop image", "wrong switch hash"}


@pytest.mark.parametrize("segment_steps", [16, 0])
def test_every_case_matches_the_host_vm(segment_steps):
    cases = vc.edge_cases() + vc.catalogue_cases() + vc.generated_cases() + vc.boundary_cases()
    assert len(cases) >= 4000
    segments = checkpointed = 0
    for c in cases:
        want = vc.host(c)
        got, st = _run_sized(c, want, segment_steps)
        _check(c, want, got)
        if st:
            assert st["fallback"] == (1 if c.name in INCONSISTENT else 0), c.name
            segments += st["segments"]
            checkpointed += st["segments"] > 1
            assert st["segment_steps"] == (segment_steps or 1024)
    print(f"segment_steps {segment_steps}: {segments} segments, {checkpointed} of {len(cases)} executions in more than one")
    if segment_steps == 16:
        assert segments > 2 * len(cases) and checkpointed > 500


def _switch_with_unread_hash():
    """IF_SOURCE taking the true branch, with a wrong true-branch hash: only the false branch's end_block reads it, so Program::hash is
    the compiled one and the execution succeeds, but the encoding is inconsistent"""
    p = hostvm.compile_program(vc.IF_SOURCE)
    b = vc.block_index(p, 2)
    hs = [int.from_bytes(bytes(getattr(p.blocks[b], f)), "little") for f in ("hash0", "hash1", "hash2")]
    return vc.Case("unread switch hash", vc.encoding(vc.IF_SOURCE, block_hashes={b: ((hs[0] + 1) % vc.M, hs[1], hs[2])}), X([], [1]), 1)


def _skipped_loop_with_wrong_image():
    src = "begin noop while.true push.1 push.0 end end"
    p = hostvm.compile_program(src)
    b = vc.block_index(p, 3)
    hs = [int.from_bytes(bytes(getattr(p.blocks[b], f)), "little") for f in ("hash0", "hash1", "hash2")]
    return vc.Case("skipped loop, wrong image", vc.encoding(src, block_hashes={b: ((hs[0] + 1) % vc.M, hs[1], hs[2])}), X([0]), 1)


@pytest.mark.parametrize("segment_steps", [16, 0])
def test_inconsistent_encodings_fall_back_to_the_batch_path(segment_steps):
    cat = vc.failure_catalogue()
    image = cat["VM_LOOP_IMAGE"]
    got, st = _run(image.case, segment_steps)
    _check(image.case, f"{image.message} at step {image.step}", got)
    assert st["fallback"] == 1
    wrong_switch = [c for c in vc.catalogue_cases() if c.name == "wrong switch hash"][0]
    got, st = _run(wrong_switch, segment_steps)
    _check(wrong_switch, vc.host(wrong_switch), got)
    assert st["fallback"] == 1
    # a wrong Program::hash alone is consistent: the tabled path reports it at the end
    h = cat["VM_HASH"]
    got, st = _run(h.case, segment_steps)
    _check(h.case, h.message, got)
    assert st["fallback"] == 0
    for c in (_switch_with_unread_hash(), _skipped_loop_with_wrong_image()):
        want = vc.host(c)
        assert not isinstance(want, str), (c.name, want)
        got, st = _run(c, segment_steps)
        _check(c, want, got)
        assert st["fallback"] == 1, c.name
        out, proof = dg.execute_one(c.program, c.inputs, c.num_outputs, segment_steps=segment_steps, stats=st)
        assert st["fallback"] == 1 and out == want.outputs and proof.bytes == dg.prove(want).bytes, c.name


@pytest.mark.parametrize("segment_steps", [16, 0])
def test_step_cap(segment_steps):
    for c in vc.boundary_cases():
        want = vc.host(c)
        last = int(c.name.split()[-1])
        _same(_run(c, segment_steps, max_steps=last + 1)[0], want)
        for cap in (last, 16):
            _check(c, f"execution exceeds {cap} steps", _run(c, segment_steps, max_steps=cap)[0])
    cap = vc.failure_catalogue()["VM_CAP"]
    _check(cap.case, cap.message, _run(cap.case, segment_steps, max_steps=cap.max_steps)[0])


@pytest.mark.parametrize("segment_steps", [16, 0])
def test_proofs_equal_execute_and_the_verifier_accepts(po, segment_steps):
    for name, src, pub, a, b, no in ec.SMALL:
        outputs, proof = dg.execute(src, pub, a, b, no)
        st = {}
        got = dg.execute_one(src, X(pub, a, b), no, segment_steps=segment_steps, stats=st)
        assert st["fallback"] == 0, name
        assert got[0] == outputs and got[1].bytes == proof.bytes, name
        assert po.verify(hostvm.compile_program(src).hash, pub, outputs, got[1].bytes) is None, name
    with pytest.raises(backend.DgError) as e:
        dg.execute_one("begin assert end", X([2]))
    assert e.value.code == EXECUTION and str(e.value).endswith("ASSERT failed at step 2")


def test_bench_collatz_2_20_against_the_golden_digests():
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "collatz_2_20.json")))
    start = int(re.search(r"start=(\d+)", gold["name"]).group(1))
    st = {}
    tr = dg.trace_one(hostvm.COLLATZ_SOURCE, X([], [start]), stats=st)
    assert tr.length == 2**20 and st["fallback"] == 0 and st["segments"] > 500, st
    assert hashlib.sha256(np.ascontiguousarray(tr.registers).tobytes()).hexdigest() == gold["trace_sha256"]
    out, proof = dg.execute_one(hostvm.COLLATZ_SOURCE, X([], [start]), stats=st)
    assert out == tr.outputs and st["fallback"] == 0
    assert hashlib.sha256(proof.bytes).hexdigest() == gold["proof_sha256"]
