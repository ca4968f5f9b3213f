"""-m gpu tests of traces shorter than the constraint kernel's 128-step block: 16-step traces (the shortest the API accepts; the VM never
emits fewer than 32 steps) and same-shape batches of 16- and 32-step traces.  Every proof must equal the CPU oracle's, and every proof of
a batch the single proof of the same trace."""
import pytest

pytestmark = pytest.mark.gpu

LOGIC = "begin not and or end"                  # 32 steps
HASH = "begin pad.2 hash.2 end"                 # 64 steps


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    backend.device_info()
    return distaff_b200


def run(src, inputs):
    from distaff_b200 import hostvm
    return hostvm.execute(src, public_inputs=inputs, num_outputs=2)


def first_steps(tr, n, regs=None):
    """the first n steps of a VM trace (or `regs` in their place), with the trace's claimed outputs: transitions 0..n-2 are those of
    the full trace, and the last step is exempt from the transition constraints"""
    from distaff_b200 import hostvm
    regs = tr.registers[:, :n].copy() if regs is None else regs
    return hostvm.ExecutionTrace(regs, tr.ctx_depth, tr.loop_depth, tr.stack_depth, tr.program_hash, tr.public_inputs, tr.outputs)


def oracle_proof(po, tr):
    ref = po.prove(tr.registers, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs)
    assert ref.error is None, ref.error
    return ref.proof


def logic_traces(n):
    """three different n-step traces of one shape (n = 16 or 32)"""
    traces = [run(LOGIC, p) for p in ([1, 1, 0, 1], [0, 1, 1, 0], [1, 0, 0, 1])]
    return [first_steps(t, n) for t in traces]


@pytest.mark.parametrize("src,inputs,size", [(LOGIC, [1, 1, 0, 1], 32606), (HASH, [5, 6], 35702)], ids=["logic", "hash"])
def test_16_step_trace(dg, po, src, inputs, size):
    tr = first_steps(run(src, inputs), 16)
    assert tr.length == 16
    proof = dg.prove(tr)
    assert len(proof.bytes) == size
    assert proof.bytes == oracle_proof(po, tr)


@pytest.mark.parametrize("n", [16, 32])
def test_short_batch(dg, po, n):
    traces = logic_traces(n)
    assert len({(t.registers.shape, t.ctx_depth, t.loop_depth) for t in traces}) == 1 and traces[0].length == n
    batch = dg.prove_batch(traces)
    assert len({p.bytes for p in batch}) == 3
    for i, (tr, proof) in enumerate(zip(traces, batch)):
        assert proof.bytes == dg.prove(tr).bytes, i
        assert proof.bytes == oracle_proof(po, tr), i


@pytest.mark.parametrize("n", [16, 32])
def test_failed_trace_in_short_batch(dg, n):
    from distaff_b200 import backend
    traces = logic_traces(n)
    want = [dg.prove(t).bytes for t in traces]
    regs = traces[1].registers.copy()
    regs[traces[1].width - 1, n - 1, 0] += 1     # the last stack register at the last step: only transition n-2 -> n-1 breaks
    traces[1] = first_steps(traces[1], n, regs)
    batch = dg.prove_batch(traces)
    assert isinstance(batch[1], backend.DgError) and batch[1].code == -5
    with pytest.raises(backend.DgError) as single:
        dg.prove(traces[1])
    assert str(batch[1]) == str(single.value)          # the message dg_prove gives, with the failing step
    assert "step %d " % (n - 2) in str(single.value)
    assert [batch[0].bytes, batch[2].bytes] == [want[0], want[2]]
