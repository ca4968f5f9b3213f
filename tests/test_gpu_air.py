"""-m gpu tests of the constraint-evaluation kernel (air.cu), called directly through dg_eval_transitions and compared with the CPU
oracle's transition loop (or_eval_transitions) value for value: register shapes across the whole range the prover accepts (ctx 0..16,
loop 0..8, stack 1..32, up to 71 registers), the SHORT layout (n < 128) and the one-block-per-coset layout, extension factors 16 / 32 /
256, random, constant and op-bit-pattern rows, batches of entries, and the prover's trace-domain check, which must name the lowest
violating step.  On a mismatch the failure names the shape, the step and the raw constraints that differ (or_eval_transition_raw against
the kernel run with one-hot coefficients).  Also: the kernels' unreduced accumulator at every group length up to its documented bound,
and the widest register shape the host VM emits, proven end to end."""
import functools
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

M = 2**128 - 45 * 2**40 + 1

# (ctx, loop, stack)
SHAPES = [(0, 0, 1), (0, 0, 7), (1, 0, 8), (0, 1, 8), (1, 1, 9), (2, 1, 10), (3, 2, 11), (4, 3, 12),
          (0, 8, 31), (16, 0, 8), (15, 8, 32), (16, 8, 32)]
SHAPE_IDS = ["c%dl%ds%d" % s for s in SHAPES]


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    backend.device_info()
    return distaff_b200


def width(shape):
    return 15 + sum(shape)


def seeds(count, salt):
    return [bytes([q, salt & 255, salt >> 8, 0x5A]) + bytes(28) for q in range(count)]


def random_ext(shape, n, b, seed):
    from distaff_b200 import felt
    return felt.random_elements(width(shape) * n * b, seed).reshape(width(shape), n * b, 2)


def const_ext(shape, n, b, value):
    a = np.empty((width(shape), n * b, 2), dtype=np.uint64)
    a[..., 0], a[..., 1] = value & (2**64 - 1), value >> 64
    return a


def constraint_names(shape):
    cd, ld, sd = shape
    return ([f"op bit {i} binary" for i in range(10)] + ["op counter", "op combination (ld, hd)", "op combination (cf)", "void sequence",
                                                          "op alignment"]
            + [f"sponge {i}" for i in range(4)] + ["loop image"] + [f"ctx stack {i}" for i in range(max(cd, 1))]
            + [f"loop stack {i}" for i in range(max(ld, 1))] + ["stack aux 0", "stack aux 1"] + [f"stack slot {i}" for i in range(sd)])


def diagnose(dg, po, ext, shape, b, step):
    """which raw constraints the kernel gets wrong at `step`: the kernel with coefficient A one-hot at constraint j (B = 0) returns
    constraint j's value, compared with or_eval_transition_raw on the same two rows"""
    from distaff_b200 import felt
    names = constraint_names(shape)
    T = len(names)
    N = ext.shape[1]
    n = N // b
    i = step * (b // 8)
    cur, nxt = np.ascontiguousarray(ext[:, i]), np.ascontiguousarray(ext[:, (i + b) % N])
    raw = np.zeros((128, 2), dtype=np.uint64)
    k = po.lib().or_eval_transition_raw(cur.ctypes.data, nxt.ctypes.data, *shape, n, step, raw.ctypes.data)
    assert k == T
    want = felt.to_ints(raw[:T])
    coefs = np.zeros((T, 2 * T, 2), dtype=np.uint64)
    for j in range(T):
        coefs[j, j, 0] = 1
    got = []
    for j in range(T):              # one entry per call: the slab of a long trace is large
        vals, _ = dg.eval_transitions(ext[None], *shape, b, coefs=coefs[j:j + 1])
        got.append(felt.to_ints(vals[0, step])[0])
    bad = ["%s (kernel %d, oracle %d)" % (names[j], got[j], want[j]) for j in range(T) if got[j] != want[j]]
    return "shape (ctx, loop, stack) %s, n %d, blowup %d, step %d (trace step %d, coset %d): %s" % (
        shape, n, b, step, step // 8, step % 8, "; ".join(bad) or "raw constraints agree, the combination differs")


def compare(dg, po, ext, shape, b, salt, check=False):
    """kernel on `count` entries in one launch vs the oracle entry by entry; returns (values, first_violation)"""
    sd = seeds(ext.shape[0], salt)
    vals, first = dg.eval_transitions(ext, *shape, b, seeds=sd, check=check)
    for q in range(ext.shape[0]):
        want, err = po.eval_transitions(ext[q], *shape, b, sd[q], check)
        assert err is None, err
        if not np.array_equal(vals[q], want):
            step = int(np.nonzero((vals[q] != want).any(axis=1))[0][0])
            pytest.fail("entry %d of %d: %s" % (q, ext.shape[0], diagnose(dg, po, ext[q], shape, b, step)))
        assert first[q] == 0
    return vals, first


RANDOM_CASES = ([(s, 16, 16, 3) for s in SHAPES] + [(s, 32, 16, 2) for s in SHAPES] + [(s, 64, 32, 1) for s in SHAPES]
                + [(s, 128, 16, 1) for s in SHAPES] + [(s, 256, 32, 1) for s in SHAPES]
                + [((1, 1, 9), 32, 32, 2), ((15, 8, 32), 256, 16, 3),
                   ((2, 1, 10), 16, 256, 1), ((16, 8, 32), 16, 256, 1), ((4, 3, 12), 1024, 16, 1), ((16, 8, 32), 1024, 32, 1)])


@pytest.mark.parametrize("shape,n,b,count", RANDOM_CASES, ids=["%s-n%d-b%d-x%d" % ("c%dl%ds%d" % c[0], *c[1:]) for c in RANDOM_CASES])
def test_random_rows(dg, po, shape, n, b, count):
    """uniformly random rows: every op flag is non-binary, so every term of every constraint contributes"""
    ext = np.stack([random_ext(shape, n, b, 1000 * n + 10 * b + q + sum(shape)) for q in range(count)])
    compare(dg, po, ext, shape, b, salt=n + b)


@pytest.mark.parametrize("n,b", [(16, 16), (128, 32)])
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_constant_rows(dg, po, shape, n, b):
    """rows of all 0, all 1 and all M - 1, three entries of one launch"""
    ext = np.stack([const_ext(shape, n, b, v) for v in (0, 1, M - 1)])
    compare(dg, po, ext, shape, b, salt=7)


@pytest.mark.parametrize("shape", [(0, 0, 1), (1, 0, 8), (3, 2, 11), (0, 8, 31), (16, 8, 32)], ids=lambda s: "c%dl%ds%d" % s)
def test_every_op_bit_pattern(dg, po, shape):
    """the 8n = 1024 steps of entries 0 and 2 take all 1024 binary patterns of the 10 op bits (in two different orders), the other
    registers random; entry 1 is random throughout"""
    n, b = 128, 16
    stride = b // 8
    ext = np.stack([random_ext(shape, n, b, 77 + q) for q in range(3)])
    for q, mult in ((0, 1), (2, 397)):
        for s in range(8 * n):
            pattern = (s * mult) % 1024
            for bit in range(10):
                ext[q, 5 + bit, s * stride] = ((pattern >> bit) & 1, 0)
    compare(dg, po, ext, shape, b, salt=11)


def test_random_rows_fail_at_step_0(dg, po):
    """with the prover's check, random rows violate at almost every trace step of every block: the kernel reports the lowest, step 0,
    as the oracle does"""
    shape, n, b = (1, 1, 9), 256, 16
    ext = np.stack([random_ext(shape, n, b, 5 + q) for q in range(2)])
    sd = seeds(2, 3)
    _, first = dg.eval_transitions(ext, *shape, b, seeds=sd, check=True)
    for q in range(2):
        _, err = po.eval_transitions(ext[q], *shape, b, sd[q], True)
        assert err is not None and re.search(r"\bat step 0\b", err), err
    assert first == [1, 1]


# ---- honest and corrupted VM traces with the prover's check ----------------------------------------------------------------------------
def widest_source():
    """ctx 15, loop 8, stack 32: w = 70, the widest register file the host VM emits (it reports at most 15 contexts)"""
    loops = "push.1 while.true " * 8 + "push.0 end " * 8
    return "begin " + " ".join(f"push.{i + 1}" for i in range(31)) + " " + "block push.1 add " * 15 + "end " * 15 + loops + "end"


def first_steps(tr, n, regs=None):
    from distaff_b200 import hostvm
    regs = tr.registers[:, :n].copy() if regs is None else regs
    return hostvm.ExecutionTrace(regs, tr.ctx_depth, tr.loop_depth, tr.stack_depth, tr.program_hash, tr.public_inputs, tr.outputs)


@functools.lru_cache(maxsize=None)
def vm_traces():
    from distaff_b200 import hostvm
    from tests import programs
    wide = hostvm.execute(widest_source(), num_outputs=2)
    return {"fib13": hostvm.fibonacci(13), "collatz3": hostvm.collatz(3), "wide65": programs.wide_program(),
            "widest16": first_steps(wide, 16), "widest": wide}


def shape_of(tr):
    return (tr.ctx_depth, tr.loop_depth, tr.stack_depth)


def corrupt(tr, steps):
    """adds 1 to the last stack register at each of `steps`: transitions t - 1 and t break for each t"""
    regs = tr.registers.copy()
    for t in steps:
        regs[tr.width - 1, t, 0] += 1
    return first_steps(tr, tr.length, regs)


def oracle_step(message):
    m = re.search(r"at step (\d+) ", message)
    assert m, message
    return int(m.group(1))


@pytest.mark.parametrize("name,b", [("fib13", 16), ("fib13", 32), ("collatz3", 16), ("wide65", 16), ("widest16", 32), ("widest", 16)])
def test_honest_vm_trace(dg, po, name, b):
    """an honest trace passes the check with the oracle's values, although its last transition (step n - 1 -> 0) breaks: that one is
    exempt"""
    tr = vm_traces()[name]
    n = tr.length
    ext = po.extend(tr.registers, b)[None]
    vals, first = compare(dg, po, ext, shape_of(tr), b, salt=n, check=True)
    assert not vals[0, 0:8 * (n - 1):8].any()
    cur, nxt = np.ascontiguousarray(tr.registers[:, n - 1]), np.ascontiguousarray(tr.registers[:, 0])
    raw = np.zeros((128, 2), dtype=np.uint64)
    k = po.lib().or_eval_transition_raw(cur.ctypes.data, nxt.ctypes.data, *shape_of(tr), n, 8 * (n - 1), raw.ctypes.data)
    assert raw[:k].any(), "the wrap-around transition of an honest trace should break"


# fib13 has 256 steps: the trace-domain steps k of one coset fill two 128-thread blocks
VIOLATIONS = {"blocks": [41, 201], "blocks_reversed": [201, 41], "warp": [35, 60], "adjacent": [100, 101], "far": [3, 250]}


@pytest.mark.parametrize("where", VIOLATIONS)
@pytest.mark.parametrize("b", [16, 32])
def test_lowest_violating_step(dg, po, where, b):
    """a trace that violates at several steps reports the lowest one, the step the oracle (and the reference's sequential loop) names"""
    tr = corrupt(vm_traces()["fib13"], VIOLATIONS[where])
    want = min(VIOLATIONS[where]) - 1
    ext = po.extend(tr.registers, b)
    sd = seeds(1, 9)
    _, err = po.eval_transitions(ext, *shape_of(tr), b, sd[0], True)
    assert err is not None and oracle_step(err) == want, err
    _, first = dg.eval_transitions(ext[None], *shape_of(tr), b, seeds=sd, check=True)
    assert first == [want + 1]


def test_violation_in_one_batch_entry(dg, po):
    """three same-shape traces in one launch, the middle one corrupted at two steps: it reports its lowest step, and the other two
    entries give their oracle values and their values alone"""
    from distaff_b200 import hostvm
    b = 16
    traces = [hostvm.execute(hostvm.fibonacci_program(13), public_inputs=p) for p in ([1, 0], [2, 1], [3, 5])]
    traces[1] = corrupt(traces[1], [150, 20])
    ext = np.stack([po.extend(t.registers, b) for t in traces])
    shape = shape_of(traces[0])
    sd = seeds(3, 21)
    vals, first = dg.eval_transitions(ext, *shape, b, seeds=sd, check=True)
    assert first == [0, 20, 0]
    _, err = po.eval_transitions(ext[1], *shape, b, sd[1], True)
    assert oracle_step(err) == 19
    for q in (0, 2):
        want, err = po.eval_transitions(ext[q], *shape, b, sd[q], True)
        assert err is None and np.array_equal(vals[q], want), q
        alone, f = dg.eval_transitions(ext[q:q + 1], *shape, b, seeds=sd[q:q + 1], check=True)
        assert f == [0] and np.array_equal(alone[0], vals[q]), q


@pytest.mark.parametrize("where", ["blocks", "warp", "far"])
def test_prove_names_the_lowest_violating_step(dg, po, where):
    """dg.prove and dg.prove_batch of a trace corrupted at two separated steps fail with the step po.prove names; the single and batch
    messages are equal"""
    from distaff_b200 import backend, hostvm
    tr = corrupt(vm_traces()["fib13"], VIOLATIONS[where])
    ref = po.prove(tr.registers, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs)
    want = oracle_step(ref.error)
    assert want == min(VIOLATIONS[where]) - 1
    with pytest.raises(backend.DgError) as single:
        dg.prove(tr)
    assert single.value.code == -5 and oracle_step(str(single.value)) == want, str(single.value)
    other = hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[2, 1])
    batch = dg.prove_batch([other, tr, other])
    assert isinstance(batch[1], backend.DgError) and str(batch[1]) == str(single.value)
    assert batch[0].bytes == batch[2].bytes == dg.prove(other).bytes


@pytest.mark.parametrize("steps", [16, None], ids=["16_steps", "full"])
def test_widest_vm_shape_end_to_end(dg, po, steps):
    """ctx 15, loop 8, stack 32 (w = 70): the proof equals the oracle's byte for byte, and both verifiers accept the full trace's proof.
    The 16-step prefix claims fewer than 16 operations, which the reference's verifier rejects (verifier.rs:34-37): both verifiers
    give that verdict"""
    tr = vm_traces()["widest"]
    assert (tr.width, tr.ctx_depth, tr.loop_depth, tr.stack_depth) == (70, 15, 8, 32)
    if steps:
        tr = first_steps(tr, steps)
    proof = dg.prove(tr)
    ref = po.prove(tr.registers, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs)
    assert ref.error is None, ref.error
    assert proof.bytes == ref.proof
    verdict = None if not steps else "Verification of minimum operation count failed"
    assert dg.verify(tr.program_hash, tr.public_inputs, tr.outputs, proof) == verdict
    assert po.verify(tr.program_hash, tr.public_inputs, tr.outputs, proof.bytes) == verdict


# ---- the unreduced accumulator ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("length", [1, 2, 7, 71, 78, 127, 128])
def test_unreduced_accumulator_up_to_128_products(dg, length):
    """wide_set / wide_add / reduce of `length` products (fe_reduce_wide is documented for up to 128; the constraint kernel folds up to
    78, the per-register combinations w <= 71) == Python integers, for all-(M - 1) operands (the largest sum), the crafted operand
    pairs of tools/gen_mul_vectors.py and random operands"""
    import importlib.util
    import os
    from distaff_b200 import felt
    spec = importlib.util.spec_from_file_location(
        "gen_mul_vectors", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools", "gen_mul_vectors.py"))
    gen_mul_vectors = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen_mul_vectors)
    pairs = gen_mul_vectors.pairs()
    xs = [M - 1] * (3 * length) + [p[0] for p in pairs] + felt.to_ints(felt.random_elements(40 * length, length))
    ys = [M - 1] * (3 * length) + [p[1] for p in pairs] + felt.to_ints(felt.random_elements(40 * length, length + 1000))
    xs += xs[:(-len(xs)) % length]
    ys += ys[:(-len(ys)) % length]
    groups = len(xs) // length
    want = [sum(x * y for x, y in zip(xs[g * length:(g + 1) * length], ys[g * length:(g + 1) * length])) % M for g in range(groups)]
    assert felt.to_ints(dg.field_dot(felt.from_ints(xs), felt.from_ints(ys), length)) == want
