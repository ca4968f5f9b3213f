"""Pins oracle/air.h against the reference's TraceState tests (/root/reference/src/stark/trace/trace_state.rs:500-579)
and checks that every transition constraint vanishes on genuine VM traces (the property the reference asserts at
/root/reference/src/stark/constraints/evaluator.rs:152-157)."""
import numpy as np

M = 2**128 - 45 * 2**40 + 1


def _flags(po, row, cd=1, ld=0, sd=2):
    a = po.fvec(row)
    out = np.zeros((46, 2), dtype=np.uint64)
    po.lib().or_op_flags(a.ctypes.data, cd, ld, sd, out.ctypes.data)
    v = po.ints(out)
    return v[:8], v[8:40], v[40:44], v[44], v[45]


def test_op_flags_reference_vectors(po):
    cf, ld, hd, begin, noop = _flags(po, [101, 1, 2, 3, 4, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 15, 16, 17])
    assert cf == [1, 0, 0, 0, 0, 0, 0, 0] and ld == [0] * 32 and hd == [0, 0, 0, 0] and (begin, noop) == (1, 0)
    cf, ld, hd, begin, noop = _flags(po, [101, 1, 2, 3, 4, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 15, 16, 17])
    assert cf == [0] * 7 + [1] and ld == [0] * 31 + [1] and hd == [0, 0, 0, 1] and (begin, noop) == (0, 1)
    cf, ld, hd, begin, noop = _flags(po, [101, 1, 2, 3, 4, 1, 0, 0, 1, 0, 0, 0, 0, 1, 0, 15, 16, 17])
    assert cf == [0, 1, 0, 0, 0, 0, 0, 0] and ld == [0, 1] + [0] * 30 and hd == [0, 1, 0, 0] and (begin, noop) == (0, 0)
    cf, ld, hd, _, _ = _flags(po, [101, 1, 2, 3, 4, 1, 1, 0, 1, 1, 0, 0, 0, 0, 1, 15, 16, 17])
    assert cf == [0, 0, 0, 1, 0, 0, 0, 0] and ld == [0, 0, 0, 1] + [0] * 28 and hd == [0, 0, 1, 0]


def test_ld_flag_quirk_uses_cf_bit(po):
    # trace_state.rs:301: ld_op_flags[2] = (1 - ld0) * cf_bits[1]
    row = [0, 0, 0, 0, 0, 0, 1, 0, 0, 1, 0, 0, 0, 1, 1, 0, 0, 0]   # cf=[0,1,0], ld=[0,1,0,0,0], hd=[1,1]
    _, ld, _, _, _ = _flags(po, row)
    assert ld[2] == 1
    row[6] = 0                                                     # cf=[0,0,0]: the flag for ld index 2 disappears
    _, ld, _, _, _ = _flags(po, row)
    assert ld[2] == 0


def _rows(trace, step):
    return trace.registers[:, step, :].copy()


def test_transition_constraints_vanish_on_vm_traces(po):
    from distaff_b200 import hostvm
    programs = [
        hostvm.fibonacci(6),
        hostvm.execute("begin push.3 push.5 add push.7 mul dup inv mul not not end", num_outputs=1),
        hostvm.collatz(3),
        hostvm.execute("begin pad.2 hash.2 end", public_inputs=[5, 6], num_outputs=2),
        hostvm.execute("begin push.5 push.11 gt.8 push.7 push.3 lt.8 and end", num_outputs=1),
        hostvm.execute("begin read.ab read.ab swap.2 drop choose push.9 eq end", secret_a=[3, 1], secret_b=[4, 7], num_outputs=1),
    ]
    for tr in programs:
        n = tr.length
        out = np.zeros((64, 2), dtype=np.uint64)
        for step in range(n - 1):
            cur, nxt = _rows(tr, step), _rows(tr, step + 1)
            k = po.lib().or_eval_transition_raw(cur.ctypes.data, nxt.ctypes.data, tr.ctx_depth, tr.loop_depth, tr.stack_depth,
                                                n, step * 8, out.ctypes.data)
            vals = po.ints(out[:k])
            assert all(v == 0 for v in vals), (step, [i for i, v in enumerate(vals) if v])
        # a corrupted next row must violate something
        cur, nxt = _rows(tr, 3), _rows(tr, 4)
        nxt[tr.width - 1, 0] ^= np.uint64(1)
        k = po.lib().or_eval_transition_raw(cur.ctypes.data, nxt.ctypes.data, tr.ctx_depth, tr.loop_depth, tr.stack_depth,
                                            n, 3 * 8, out.ctypes.data)
        assert any(v != 0 for v in po.ints(out[:k]))


def test_decoder_flow_ops_reference_vectors(po):
    """the literal expected vectors of the reference's own unit tests for enforce_{begin,tend,fend,loop,wrap,break,void}
    (/root/reference/src/stark/constraints/decoder/flow_ops.rs mod tests; fixture: tests/golden/ref_decoder_flow_cases.json, made by
    tests/golden/make_ref_decoder_cases.py).  The reference calls one enforce_* with op_flag = 1; here the first state carries the op
    bits of that operation, so the oracle's full decoder evaluation has exactly that flag set."""
    import json
    import os
    from distaff_b200 import felt
    flow_code = {"hacc": 0, "begin": 1, "tend": 2, "fend": 3, "loop": 4, "wrap": 5, "break": 6, "void": 7}
    cases = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_decoder_flow_cases.json")))["cases"]
    assert len(cases) == 30

    def row(st, code):
        v = [st["step"]] + st["sponge"] + [(code >> i) & 1 for i in range(3)] + [1] * 7 + st["ctx"] + st["loop"] + [101]
        return felt.from_ints(v)

    out = np.zeros((64, 2), dtype=np.uint64)
    for c in cases:
        cd, ld = len(c["state1"]["ctx"]), len(c["state1"]["loop"])
        assert c["op_flag"] == 1 and len(c["state2"]["ctx"]) == cd and len(c["state2"]["loop"]) == ld
        cur = row(c["state1"], flow_code[c["op"]])
        nxt = row(c["state2"], flow_code[c["state2"]["flow_op"].lower()])
        k = po.lib().or_eval_transition_raw(cur.ctypes.data, nxt.ctypes.data, cd, ld, 1, 16, 8 * c["state1"]["step"], out.ctypes.data)
        want = [int(x) for x in c["expected"]]
        got = po.ints(out[:k])[15:15 + len(want)]
        assert got == want, (c["op"], c["state1"], c["state2"], got)


def _sponge_round(po, state, op_code, op_value, step):
    from distaff_b200 import felt
    st = felt.from_ints(state)
    c, v = felt.from_ints([op_code]), felt.from_ints([op_value])
    po.lib().or_sponge_round(st.ctypes.data, c.ctypes.data, v.ctypes.data, step)
    return felt.to_ints(st)


def _decoder_eval(po, cur, nxt, cd, ld, step):
    from distaff_b200 import felt
    out = np.zeros((64, 2), dtype=np.uint64)
    a, b = felt.from_ints(cur), felt.from_ints(nxt)
    k = po.lib().or_eval_transition_raw(a.ctypes.data, b.ctypes.data, cd, ld, 1, 16, step, out.ctypes.data)
    return po.ints(out[:k])[:20 + max(cd, 1) + max(ld, 1)]          # decoder constraints only


def test_decoder_hacc_reference_vectors(po):
    """decoder/sponge.rs mod tests (op_hacc): literal expectations 0 / M - 1 / M - 9 for the four sponge constraints"""
    M = 2**128 - 45 * 2**40 + 1
    push = [0, 1, 2, 3, 4, 0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0, 0]            # HACC + PUSH  (op code = 0b00_11111 = 31)
    other = [0, 1, 2, 3, 4, 0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 0, 0]           # HACC + an op with hd = 11, ld = 00000 (op code 96)

    def build_state(sponge, push_value):
        return [0] + list(sponge) + [1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, push_value]

    def op_code(state):
        return sum(state[8 + i] << i for i in range(5)) + (state[13] << 5) + (state[14] << 6)

    cases = [(push, 7, 7, [0, 0, 0, 0]), (other, 0, 9, [0, 0, 0, 0]), (push, 7, 6, [0, M - 1, 0, 0]), (other, 9, 9, [0, M - 9, 0, 0])]
    for state1, absorbed, next_top, want in cases:
        sponge = _sponge_round(po, [1, 2, 3, 4], op_code(state1), absorbed, 0)
        got = _decoder_eval(po, state1, build_state(sponge, next_top), 1, 0, 0)[15:19]
        assert got == want, (state1, got)


def test_decoder_begin_and_hacc_transitions(po):
    """decoder/tests.rs: enforce_begin / enforce_hacc through the whole Decoder::evaluate (trace length 16, extension 8)"""
    ok = lambda ev: all(v == 0 for v in ev)
    step = 15 * 8
    s1 = [0, 3, 5, 7, 9, 1, 0, 0, 1, 1, 1, 1, 1, 1, 1, 0, 11]
    assert ok(_decoder_eval(po, s1, [0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 3, 11], 1, 0, step))
    assert not ok(_decoder_eval(po, [0, 3, 5, 7, 9, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1, 0, 11], [0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 3, 11], 1, 0, step))
    assert not ok(_decoder_eval(po, s1, [0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 11], 1, 0, step))
    assert not ok(_decoder_eval(po, s1, [0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 5, 11], 1, 0, step))
    assert not ok(_decoder_eval(po, s1, [0, 3, 5, 7, 9, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 3, 11], 1, 0, step))

    PUSH, ADD = 0b0011111, 0b1101000                     # processor/opcodes.rs:46-92 (hd bits | ld bits)
    def hacc(state1, state2, code, value, sponge_step, eval_step):
        st2 = list(state2)
        st2[1:5] = _sponge_round(po, st2[1:5], code, value, sponge_step)
        return _decoder_eval(po, state1, st2, 1, 0, eval_step)
    p1 = [1, 3, 5, 7, 9, 0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0, 11]
    assert ok(hacc(p1, [2, 3, 5, 7, 9, 1, 0, 0, 1, 1, 1, 1, 1, 1, 1, 0, 9], PUSH, 9, 0, 0))
    assert ok(hacc(p1, [2, 3, 5, 7, 9, 1, 0, 0, 1, 1, 1, 1, 1, 1, 1, 0, 9], PUSH, 9, 8, 8 * 8))
    a1 = [1, 3, 5, 7, 9, 0, 0, 0, 0, 0, 0, 1, 0, 1, 1, 0, 0]
    assert ok(hacc(a1, [2, 3, 5, 7, 9, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 0, 0], ADD, 0, 0, 0))
    assert not ok(hacc(p1, [2, 3, 5, 7, 9, 1, 0, 0, 1, 1, 1, 1, 1, 1, 1, 0, 11], PUSH, 9, 0, 0))
    assert not ok(hacc([1, 3, 5, 7, 9, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 0, 11], [2, 3, 5, 7, 9, 1, 0, 0, 1, 1, 1, 1, 1, 1, 1, 0, 9], PUSH, 9, 0, 0))
    assert not ok(hacc([1, 3, 5, 7, 9, 0, 0, 0, 0, 0, 0, 1, 0, 1, 1, 0, 9], [2, 3, 5, 7, 9, 0, 0, 0, 1, 1, 1, 1, 1, 1, 1, 0, 0], ADD, 9, 0, 0))


def test_decoder_op_bits_reference_tests(po):
    """decoder/op_bits.rs mod tests: op_bits_are_binary (literal 3*3 - 3 at the offending position), invalid_op_combinations,
    invalid_op_alignment and invalid_op_sequence, with the masks passed explicitly as the reference tests do"""
    from distaff_b200 import felt
    NOOP, PUSH, ADD = 0b1111111, 0b0011111, 0b1101000
    HACC, BEGIN, TEND, FEND, LOOP, WRAP, BREAK, VOID = range(8)

    def state(flow, user, counter=0, cf_bits=None, u_bits=None):
        cf = cf_bits if cf_bits is not None else [(flow >> i) & 1 for i in range(3)]
        ub = u_bits if u_bits is not None else [(user >> i) & 1 for i in range(7)]
        return [counter, 0, 0, 0, 0] + cf + ub + [0, 0]                 # ctx depth 1, loop depth 0, stack depth 1

    def op_bits(cur, nxt, masks):
        out = np.zeros((64, 2), dtype=np.uint64)
        a, b = felt.from_ints(cur), felt.from_ints(nxt)
        ark, mk = felt.from_ints([0] * 8), felt.from_ints(masks)
        po.lib().or_decoder_run_raw(a.ctypes.data, b.ctypes.data, 1, 0, 1, ark.ctypes.data, mk.ctypes.data, out.ctypes.data)
        return po.ints(out[:15])

    def evaluate_state(st, masks, inc_counter):
        return op_bits(st, state(VOID, NOOP, st[0] + (1 if inc_counter else 0)), masks)

    ok = [0] * 15
    # op_bits_are_binary
    assert evaluate_state(state(VOID, NOOP, 1), [0, 0, 0], False) == ok
    for i in range(3):
        cf = [1, 1, 1]; cf[i] = 3
        want = [0] * 10; want[i] = 3 * 3 - 3
        assert evaluate_state(state(0, 0, 0, cf_bits=cf, u_bits=[1] * 7), [0, 0, 0], False)[:10] == want
    for i in range(7):
        ub = [1] * 7; ub[i] = 3
        want = [0] * 10; want[i + 3] = 3 * 3 - 3
        assert evaluate_state(state(0, 0, 0, cf_bits=[0, 0, 0], u_bits=ub), [0, 0, 0], False)[:10] == want
    # invalid_op_combinations
    for cf_op in range(8):
        assert evaluate_state(state(cf_op, 0, 1), [0, 0, 0], False) != ok
    for cf_op in range(1, 8):
        for user_op in range(127):
            assert evaluate_state(state(cf_op, user_op, 1), [0, 0, 0], False) != ok
        assert evaluate_state(state(cf_op, NOOP, 1), [0, 0, 0], False) == ok
    # invalid_op_alignment
    for flow, bad in ((TEND, [1, 0, 0]), (FEND, [1, 0, 0]), (BEGIN, [0, 1, 0]), (LOOP, [0, 1, 0]), (WRAP, [0, 1, 0]), (BREAK, [0, 1, 0])):
        st = state(flow, NOOP, 1)
        assert evaluate_state(st, [0, 0, 0], False) == ok
        assert evaluate_state(st, bad, False) != ok
    st = state(HACC, PUSH, 1)
    assert evaluate_state(st, [0, 0, 0], True) == ok
    assert evaluate_state(st, [0, 0, 1], True) != ok
    # invalid_op_sequence
    assert op_bits(state(HACC, ADD, 1), state(VOID, NOOP, 2), [0, 0, 0]) == ok
    assert op_bits(state(VOID, NOOP, 1), state(VOID, NOOP, 1), [0, 0, 0]) == ok
    assert op_bits(state(VOID, NOOP, 1), state(HACC, ADD, 1), [0, 0, 0]) != ok


def test_enforce_left_shift_reference_vectors(po):
    """constraints/utils.rs mod tests: the four literal vectors of enforce_left_shift"""
    from distaff_b200 import felt
    v = felt.from_ints([1, 2, 3, 4, 5, 6, 7, 8])
    one = felt.from_ints([1])
    for frm, num, want in ((1, 1, [1, 1, 1, 1, 1, 1, 1, 8]), (2, 2, [2, 2, 2, 2, 2, 2, 7, 8]), (2, 1, [0, 1, 1, 1, 1, 1, 1, 8]), (6, 4, [0, 0, 4, 4, 5, 6, 7, 8])):
        out = np.zeros((8, 2), dtype=np.uint64)
        po.lib().or_enforce_left_shift(v.ctypes.data, v.ctypes.data, 8, frm, num, one.ctypes.data, out.ctypes.data)
        assert po.ints(out) == want, (frm, num)


def test_trace_state_layout_reference_vectors(po):
    """trace_state.rs mod tests from_vec / op_code: register order (op_counter, sponge, cf, ld, hd, ctx, loop, user stack), zero padding
    of the three stacks to at least 1 / 1 / 8 entries, and op_code = sum of the seven user-op bits weighted by powers of two"""
    from distaff_b200 import felt

    def fields(cd, ld, sd, row):
        out = np.zeros((80, 2), dtype=np.uint64)
        a = felt.from_ints(row)
        k = po.lib().or_trace_state_fields(a.ctypes.data, cd, ld, sd, out.ctypes.data)
        return po.ints(out[:k])

    head = [101, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14]
    assert fields(0, 0, 2, head + [15, 16])[:-1] == head + [0] + [0] + [15, 16, 0, 0, 0, 0, 0, 0]
    assert fields(1, 0, 2, head + [15, 16, 17])[:-1] == head + [15] + [0] + [16, 17, 0, 0, 0, 0, 0, 0]
    assert fields(2, 1, 9, head + list(range(15, 27)))[:-1] == head + [15, 16] + [17] + list(range(18, 27))
    base = [101, 1, 2, 3, 4, 1, 1, 1]
    for bits, code in (([0] * 7, 0), ([1] * 7, 127), ([1, 1, 1, 1, 1, 1, 0], 63), ([1, 0, 0, 0, 0, 1, 1], 97)):
        assert fields(1, 0, 2, base + bits + [15, 16, 17])[-1] == code


def test_eval_transitions_is_the_provers_transition_loop(po):
    """or_eval_transitions over the extended trace: with the trace root as seed it gives the prover's t_evals; on a trace corrupted at
    two separated steps it fails with the prover's message, which names the lowest violating step; without the check it gives a value
    at every step"""
    import re
    from distaff_b200 import hostvm
    tr = hostvm.fibonacci(13)
    n, b = tr.length, 16
    ref = po.prove(tr.registers, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs, ext=b, num_queries=8, grinding=0, keep_large=True)
    assert ref.error is None
    ext = po.extend(tr.registers, b)
    assert all(np.array_equal(ext[j], ref.vector("extended", j)) for j in range(tr.width))
    vals, err = po.eval_transitions(ext, tr.ctx_depth, tr.loop_depth, tr.stack_depth, b, ref.digest("trace_root"), check=True)
    assert err is None and np.array_equal(vals, ref.vector("t_evals"))
    assert not vals[0:8 * (n - 1):8].any() and vals[8 * (n - 1)].any()

    regs = tr.registers.copy()
    regs[tr.width - 1, 201, 0] += 1                 # transitions 200 and 201 break
    regs[tr.width - 1, 41, 0] += 1                  # transitions 40 and 41 break
    bad = po.prove(regs, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs, ext=b, num_queries=8, grinding=0)
    assert bad.error is not None and re.search(r"\bstep 40\b", bad.error), bad.error
    vals, err = po.eval_transitions(po.extend(regs, b), tr.ctx_depth, tr.loop_depth, tr.stack_depth, b, bytes(32), check=True)
    assert vals is None and err == bad.error
    vals, err = po.eval_transitions(po.extend(regs, b), tr.ctx_depth, tr.loop_depth, tr.stack_depth, b, bytes(32), check=False)
    assert err is None and vals[8 * 40].any() and vals[8 * 201].any()
