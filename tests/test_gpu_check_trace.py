"""-m gpu tests of the trace check (dg_check_traces / dg_check_traces_device, check_trace / check_traces / check_traces_device): honest VM
traces pass with zero masks; random rows at every register shape and in both kernel layouts give the oracle's per-step masks bit for bit
(or_eval_transition_raw at every step); corrupted traces name exactly the constraints and steps the oracle finds, and the lowest one is the
step dg.prove and the oracle prover report; wrong boundary rows, op counts and program hashes are reported; batches, device traces and
split groups give each trace the report it gets alone."""
import os
import subprocess
import sys

import numpy as np
import pytest

from tests.test_gpu_air import SHAPES, SHAPE_IDS, VIOLATIONS, constraint_names, corrupt, first_steps, oracle_step, shape_of, vm_traces, width

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    backend.device_info()
    return distaff_b200


def make_trace(regs, shape, program_hash=bytes(32), inputs=(), outputs=()):
    from distaff_b200 import hostvm
    return hostvm.ExecutionTrace(regs, shape[0], shape[1], shape[2], program_hash, list(inputs), list(outputs))


def with_registers(tr, regs):
    return first_steps(tr, tr.length, regs)


def oracle_masks(po, regs, shape, n, steps=None):
    """the oracle's per-step masks: bit j of word j // 32 at step k is set when transition constraint j of rows k and k + 1 (evaluation
    step 8k) is nonzero; the exempt step n - 1 stays 0"""
    T = len(constraint_names(shape))
    out = np.zeros((n, 3), dtype=np.uint32)
    raw = np.zeros((128, 2), dtype=np.uint64)
    L = po.lib()
    for k in (range(n - 1) if steps is None else steps):
        cur, nxt = np.ascontiguousarray(regs[:, k]), np.ascontiguousarray(regs[:, k + 1])
        assert L.or_eval_transition_raw(cur.ctypes.data, nxt.ctypes.data, *shape, n, 8 * k, raw.ctypes.data) == T
        for j in np.nonzero(raw[:T].any(axis=1))[0]:
            out[k, j >> 5] |= np.uint32(1 << (int(j) & 31))
    return out


def mask_bits(masks, T):
    """(n, 3) uint32 -> (n, T) bool, column j = constraint j"""
    return np.unpackbits(np.ascontiguousarray(masks).view(np.uint8).reshape(-1, 12), axis=1, bitorder="little")[:, :T].astype(bool)


def assert_masks_equal(got, want, shape):
    if np.array_equal(got, want):
        return
    names = constraint_names(shape)
    k = int(np.nonzero((got != want).any(axis=1))[0][0])
    g, w = mask_bits(got[k:k + 1], len(names))[0], mask_bits(want[k:k + 1], len(names))[0]
    pytest.fail("shape %s, step %d: kernel only %s; oracle only %s" % (
        shape, k, [names[j] for j in np.nonzero(g & ~w)[0]], [names[j] for j in np.nonzero(w & ~g)[0]]))


def assert_consistent(rep, masks, shape):
    """the report's counts and lowest steps are those of its masks"""
    names = constraint_names(shape)
    bits = mask_bits(masks, len(names))
    per = bits.sum(axis=0)
    assert rep.n_constraints == len(names)
    assert rep.transitions == {names[j]: (int(per[j]), int(np.argmax(bits[:, j]))) for j in range(len(names)) if per[j]}
    rows = bits.any(axis=1)
    assert rep.violating_steps == int(rows.sum())
    assert rep.first_step == (int(np.argmax(rows)) if rows.any() else None)


def fields(rep):
    return (rep.ok, rep.first_step, rep.violating_steps, rep.transitions, rep.boundary, rep.first_row_registers, rep.last_row_registers,
            rep.op_count, rep.op_count_ok, rep.program_hash_matches)


def last_op_counter(tr):
    from distaff_b200 import felt
    return felt.to_ints(tr.registers[0, tr.length - 1])[0]


# ---- 1. honest traces -------------------------------------------------------------------------------------------------------------------
def honest_traces(po):
    from distaff_b200 import hostvm
    from tests import programs
    t = vm_traces()
    return {"fib13": t["fib13"], "collatz3": t["collatz3"], "wide65": t["wide65"], "widest": t["widest"],
            "merkle": programs.merkle_example(20, po), "fib4096": hostvm.fibonacci(250)}


@pytest.mark.parametrize("name", ["fib13", "collatz3", "wide65", "widest", "merkle", "fib4096"])
def test_honest_trace_is_ok(dg, po, name):
    """every mask is zero (the exempt step n - 1 as well), the op count is the last row's, and the program hash matches"""
    tr = honest_traces(po)[name]
    rep = dg.check_trace(tr, tr.program_hash, masks=True)
    assert rep.ok, str(rep)
    assert rep.masks.shape == (tr.length, 3) and not rep.masks.any()
    assert rep.first_step is None and rep.violating_steps == 0 and rep.transitions == {} and rep.boundary == []
    assert rep.op_count == last_op_counter(tr) >= 16 and rep.op_count_ok
    assert rep.program_hash_matches == 1
    assert str(rep).startswith("trace ok")
    assert dg.check_trace(tr).program_hash_matches == -1


# ---- 2. random rows: every shape, both layouts ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [16, 64, 128, 256, 1024])
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_random_rows_match_the_oracle(dg, po, shape, n):
    """uniformly random rows break nearly every constraint at nearly every step: two traces in one launch, masks equal the oracle's bit
    for bit, and the counts and lowest steps follow from the masks"""
    from distaff_b200 import felt
    w = width(shape)
    traces = [make_trace(felt.random_elements(w * n, 31 * n + q + 7 * sum(shape)).reshape(w, n, 2), shape) for q in range(2)]
    reps = dg.check_traces(traces, masks=True)
    for tr, rep in zip(traces, reps):
        assert_masks_equal(rep.masks, oracle_masks(po, tr.registers, shape, n), shape)
        assert_consistent(rep, rep.masks, shape)
        assert not rep.ok and rep.first_step == 0
        assert not rep.masks[n - 1].any()


# ---- 3. corrupted VM traces -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("where", VIOLATIONS)
def test_corrupted_stack_register(dg, po, where):
    """a stack register changed at two steps: exactly the oracle's constraints and steps, and first_step is the step dg.prove and the
    oracle prover name"""
    from distaff_b200 import backend
    tr = corrupt(vm_traces()["fib13"], VIOLATIONS[where])
    rep = dg.check_trace(tr, tr.program_hash, masks=True)
    assert_masks_equal(rep.masks, oracle_masks(po, tr.registers, shape_of(tr), tr.length), shape_of(tr))
    assert_consistent(rep, rep.masks, shape_of(tr))
    # transitions t - 1 and t of each changed step t (adjacent changes cancel in the transition between them)
    broken = set(int(k) for k in np.nonzero(rep.masks.any(axis=1))[0])
    assert min(VIOLATIONS[where]) - 1 in broken and broken <= {t + d for t in VIOLATIONS[where] for d in (-1, 0)}
    ref = po.prove(tr.registers, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs)
    assert rep.first_step == oracle_step(ref.error) == min(VIOLATIONS[where]) - 1
    with pytest.raises(backend.DgError) as e:
        dg.prove(tr)
    assert e.value.code == -5 and oracle_step(str(e.value)) == rep.first_step
    assert not rep.ok and rep.boundary == [] and rep.program_hash_matches == 1


def break_decoder(tr, kind, t):
    regs = tr.registers.copy()
    if kind == "op bit":
        regs[5, t] = (2, 0)                                   # cf op bit 0 is neither 0 nor 1
        name = "op bit 0 binary"
    elif kind == "op counter":
        regs[0, t:, 0] += 1                                   # the counter skips one value between steps t - 1 and t
        name = "op counter"
    else:
        regs[1, t, 0] += 1                                    # sponge register 0
        name = None
    return with_registers(tr, regs), name


@pytest.mark.parametrize("kind", ["op bit", "op counter", "sponge"])
def test_broken_decoder_register(dg, po, kind):
    """a non-binary op bit, a skipped op counter, a wrong sponge value: the report names that decoder constraint, as the oracle does"""
    t = 77
    tr, name = break_decoder(vm_traces()["fib13"], kind, t)
    rep = dg.check_trace(tr, masks=True)
    shape = shape_of(tr)
    assert_masks_equal(rep.masks, oracle_masks(po, tr.registers, shape, tr.length), shape)
    assert_consistent(rep, rep.masks, shape)
    if name:
        assert name in rep.transitions, str(rep)
        assert rep.transitions[name][1] == (t - 1 if kind == "op counter" else t)
    else:
        assert any(n.startswith("sponge") for n in rep.transitions), str(rep)
    assert rep.first_step in (t - 1, t)


# ---- 4. boundary errors ---------------------------------------------------------------------------------------------------------------
def test_wrong_public_inputs(dg, po):
    """the first-row user-stack registers that disagree with the claimed inputs are named; dg.prove still proves the trace, and both
    verifiers reject the proof"""
    tr = vm_traces()["fib13"]
    assert tr.public_inputs == [1, 0]
    bad = make_trace(tr.registers, shape_of(tr), tr.program_hash, [2, 5], tr.outputs)
    rep = dg.check_trace(bad, tr.program_hash)
    stk = 15 + tr.ctx_depth + tr.loop_depth
    assert rep.first_row_registers == [stk, stk + 1] and rep.last_row_registers == []
    assert rep.boundary == ["first row: user stack 0 (register %d) is 1, expected input 2" % stk,
                            "first row: user stack 1 (register %d) is 0, expected input 5" % (stk + 1)]
    assert rep.first_step is None and not rep.ok and "boundary" in str(rep)
    proof = dg.prove(bad)
    assert dg.verify(tr.program_hash, bad.public_inputs, bad.outputs, proof) is not None
    assert po.verify(tr.program_hash, bad.public_inputs, bad.outputs, proof.bytes) is not None


def test_wrong_outputs(dg, po):
    tr = vm_traces()["collatz3"]
    stk = 15 + tr.ctx_depth + tr.loop_depth
    bad = make_trace(tr.registers, shape_of(tr), tr.program_hash, tr.public_inputs, [tr.outputs[0] + 1])
    rep = dg.check_trace(bad, tr.program_hash)
    assert rep.first_row_registers == [] and rep.last_row_registers == [stk]
    assert rep.boundary == ["last row: user stack 0 (register %d) is %d, expected output %d" % (stk, tr.outputs[0], tr.outputs[0] + 1)]
    assert not rep.ok
    proof = dg.prove(bad)
    assert dg.verify(tr.program_hash, bad.public_inputs, bad.outputs, proof) is not None
    assert po.verify(tr.program_hash, bad.public_inputs, bad.outputs, proof.bytes) is not None


def test_nonzero_first_op_counter(dg, po):
    """the whole op counter shifted by 5: the counter still counts, so the only transition that breaks is the op combination at the
    BEGIN step 0 (op counter times the negated ld / hd bit products), and the first row's op counter breaks its boundary assertion"""
    tr = vm_traces()["fib13"]
    regs = tr.registers.copy()
    regs[0, :, 0] += 5
    bad = with_registers(tr, regs)
    rep = dg.check_trace(bad, tr.program_hash, masks=True)
    assert_masks_equal(rep.masks, oracle_masks(po, bad.registers, shape_of(bad), bad.length), shape_of(bad))
    assert rep.transitions == {"op combination (ld, hd)": (1, 0)} and rep.first_step == 0
    assert rep.first_row_registers == [0] and rep.boundary == ["first row: op counter (register 0) is 5, expected 0"]
    assert rep.op_count == last_op_counter(tr) + 5 and not rep.ok


def test_wrong_program_hash(dg):
    tr = vm_traces()["fib13"]
    rep = dg.check_trace(tr, bytes(32))
    assert rep.program_hash_matches == 0 and not rep.ok
    assert rep.first_step is None and rep.boundary == [] and "program hash" in str(rep)


def test_short_prefix_has_too_few_operations(dg):
    tr = first_steps(vm_traces()["widest"], 16)
    rep = dg.check_trace(tr, tr.program_hash)
    assert rep.op_count == last_op_counter(tr) < 16 and not rep.op_count_ok and not rep.ok
    assert "at least 16" in str(rep)


# ---- 5. batches -----------------------------------------------------------------------------------------------------------------------
def mixed_traces():
    from distaff_b200 import hostvm
    t = vm_traces()
    fib = t["fib13"]
    wrong_in = make_trace(fib.registers, shape_of(fib), fib.program_hash, [3, 3], fib.outputs)
    return [fib, t["collatz3"], corrupt(fib, [41, 201]), hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[2, 1]), t["wide65"], wrong_in]


def test_mixed_batch_equals_single_checks(dg):
    traces = mixed_traces()
    hashes = [t.program_hash for t in traces]
    reps = dg.check_traces(traces, hashes)
    assert [r.ok for r in reps] == [True, True, False, True, True, False]
    for tr, h, rep in zip(traces, hashes, reps):
        assert fields(rep) == fields(dg.check_trace(tr, h))


def same_shape_traces():
    from distaff_b200 import hostvm
    traces = [hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[1 + i, i]) for i in range(5)]
    traces[2] = corrupt(traces[2], [35, 60])
    t = traces[4]
    traces[4] = make_trace(t.registers, shape_of(t), t.program_hash, t.public_inputs, [t.outputs[0] + 2])
    return traces


def test_device_traces_equal_host_traces(dg):
    """proof-major device registers used in place: the reports and the device masks equal the host call's"""
    from distaff_b200 import backend
    traces = same_shape_traces()
    k, w, n = len(traces), traces[0].width, traces[0].length
    hashes = [t.program_hash for t in traces]
    host = dg.check_traces(traces, hashes, masks=True)
    regs = np.stack([t.registers for t in traces])
    buf = backend.DeviceBuffer(regs.nbytes).upload(regs)
    d_masks = backend.DeviceBuffer(k * n * 12)
    dev = dg.check_traces_device(buf, k, w, n, traces[0].ctx_depth, traces[0].loop_depth, [t.public_inputs for t in traces],
                                 [t.outputs for t in traces], hashes, d_masks=d_masks)
    assert [fields(r) for r in dev] == [fields(r) for r in host]
    assert np.array_equal(d_masks.download((k, n, 3), np.uint32), np.stack([r.masks for r in host]))
    assert not host[2].ok and host[4].last_row_registers == [15 + traces[4].ctx_depth + traces[4].loop_depth]


def test_group_splitting_gives_the_same_reports(dg):
    """DG_BATCH_GROUP=2 splits a batch of 5 into groups of 2, 2 and 1 (in a fresh process, as a user would set it)"""
    want = [str(fields(r)) for r in dg.check_traces(same_shape_traces(), [t.program_hash for t in same_shape_traces()])]
    code = ("import sys; sys.path.insert(0, %r)\n"
            "import distaff_b200 as dg\n"
            "from tests.test_gpu_check_trace import fields, same_shape_traces\n"
            "traces = same_shape_traces()\n"
            "for r in dg.check_traces(traces, [t.program_hash for t in traces]): print(str(fields(r)))\n" % ROOT)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, DG_BATCH_GROUP="2"), cwd=ROOT,
                       timeout=600)
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip().splitlines()[-5:] == want


# ---- 6. a long trace: the many-block reduction ----------------------------------------------------------------------------------------
def test_long_trace_corrupted_near_the_end(dg, po):
    from distaff_b200 import hostvm
    tr = hostvm.fibonacci(4000)
    n = tr.length
    assert n == 1 << 16
    assert dg.check_trace(tr, tr.program_hash).ok
    t = n - 100
    bad = corrupt(tr, [t])
    rep = dg.check_trace(bad, tr.program_hash, masks=True)
    assert rep.first_step == t - 1
    assert set(np.nonzero(rep.masks.any(axis=1))[0]) == {t - 1, t}
    assert_masks_equal(rep.masks[t - 1:t + 1], oracle_masks(po, bad.registers, shape_of(bad), n, steps=[t - 1, t])[t - 1:t + 1], shape_of(bad))
    assert_consistent(rep, rep.masks, shape_of(bad))
