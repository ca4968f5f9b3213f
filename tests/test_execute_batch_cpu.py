"""CPU-side checks of batched execution: the program encoding (hostvm.compile_program) carries everything the VM needs -- the host VM
run on the decoded encoding gives the same trace as on the source -- the library rejects bad encodings before touching a device, and
the new entry points have no CPU path."""
import ctypes
import os

import numpy as np
import pytest

from distaff_b200 import hostvm
from tests import execution_cases as cases


def _same(a, b):
    assert a.registers.shape == b.registers.shape
    assert np.array_equal(a.registers, b.registers)
    assert (a.ctx_depth, a.loop_depth, a.stack_depth) == (b.ctx_depth, b.loop_depth, b.stack_depth)
    assert a.outputs == b.outputs and a.program_hash == b.program_hash and a.public_inputs == b.public_inputs


def _lib_or_skip():
    from distaff_b200 import backend
    if not os.path.exists(backend.LIB_PATH):
        pytest.skip("libdistaff_gpu.so not built (run __graft_entry__.build())")
    return backend


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_restated_cases_are_small_programs():
    from tests import programs
    P = programs.small_programs()
    assert [c[0] for c in cases.SMALL] == list(P)
    for name, src, pub, a, b, no in cases.SMALL:
        _same(hostvm.execute(src, pub, a, b, no), P[name])
    _same(hostvm.execute(cases.WIDE_SOURCE, num_outputs=2), programs.wide_program())


@pytest.mark.parametrize("case", cases.SMALL, ids=[c[0] for c in cases.SMALL])
def test_encoding_runs_like_the_source(case):
    name, src, pub, a, b, no = case
    prog = hostvm.compile_program(src)
    ref = hostvm.execute(src, pub, a, b, no)
    assert prog.hash == ref.program_hash
    _same(hostvm.execute_program(prog, pub, a, b, no), ref)


def test_encoding_of_wide_collatz_and_merkle():
    prog = hostvm.compile_program(cases.WIDE_SOURCE)
    _same(hostvm.execute_program(prog, num_outputs=2), hostvm.execute(cases.WIDE_SOURCE, num_outputs=2))
    prog = hostvm.compile_program(hostvm.COLLATZ_SOURCE)
    for start in (1, 2, 7, 27, 97):
        _same(hostvm.execute_program(prog, secret_a=[start]), hostvm.collatz(start))
    _lib_or_skip()
    src, a, b = cases.merkle_case(8, 2)
    _same(hostvm.execute_program(hostvm.compile_program(src), secret_a=a, secret_b=b, num_outputs=4), hostvm.merkle_paths(8, 2))


def test_encoding_errors_match_the_source():
    prog = hostvm.compile_program(hostvm.COLLATZ_SOURCE)
    for args in (dict(), dict(public_inputs=list(range(9)), secret_a=[3]), dict(secret_a=[3], secret_b=[1, 2])):
        with pytest.raises(RuntimeError) as e1:
            hostvm.execute(hostvm.COLLATZ_SOURCE, **args)
        with pytest.raises(RuntimeError) as e2:
            hostvm.execute_program(prog, **args)
        assert str(e1.value) == str(e2.value)


def test_wrong_hash_in_the_encoding_fails_the_execution():
    prog = hostvm.compile_program(hostvm.fibonacci_program(13))
    prog.hash = bytes(32)
    with pytest.raises(RuntimeError, match="program hash does not match trace hash"):
        hostvm.execute_program(prog, public_inputs=[1, 0])


def _call(backend, prog, k=1, max_steps=1 << 10):
    from distaff_b200 import api
    _, cprog, arr, keep = api._execution_args(prog, [api.ProgramInputs([1, 0])] * k)
    info = (backend.DgExecutionInfo * k)()
    status = (ctypes.c_int * k)()
    rc = backend.lib().dg_trace_batch(ctypes.byref(cprog), k, arr, max_steps, info, None, status)
    return rc, backend.lib().dg_last_error().decode()


def test_bad_encodings_are_rejected_on_the_host():
    backend = _lib_or_skip()
    src = "begin push.1 if.true push.2 else push.3 end add end"
    prog = hostvm.compile_program(src)
    bad = hostvm.compile_program(src)
    bad.children[bad.root_first + 1] = 99                       # out-of-range child index
    rc, msg = _call(backend, bad)
    assert rc == -1 and "out of range" in msg, msg
    bad = hostvm.compile_program(src)
    sp = bad.children[bad.root_first]
    bad.blocks[sp].count -= 1                                  # a span of the wrong length
    rc, msg = _call(backend, bad)
    assert rc == -1 and "span length must be one less than a multiple of 16" in msg, msg
    bad = hostvm.compile_program(src)
    bad.children[bad.root_first] = bad.children[bad.root_first + 1]     # a list that starts with a Switch
    rc, msg = _call(backend, bad)
    assert rc == -1 and "must start with a Span block" in msg, msg
    rc, msg = _call(backend, prog, max_steps=8)
    assert rc == -1 and "max_steps" in msg


def test_no_cpu_path():
    backend = _lib_or_skip()
    if _has_gpu():
        pytest.skip("a GPU is present (covered by tests/test_gpu_execute_batch.py)")
    import distaff_b200 as dg
    rc, msg = _call(backend, hostvm.compile_program(hostvm.fibonacci_program(13)))
    assert rc == -3 and "no CPU path" in msg
    for fn in (dg.trace_batch, dg.execute_batch, dg.trace_shapes):
        with pytest.raises(backend.DgError) as e:
            fn(hostvm.fibonacci_program(13), [dg.ProgramInputs([1, 0])])
        assert e.value.code == -3
    assert dg.execute_batch(hostvm.fibonacci_program(13), []) == []


def test_tape_growing_encoding_runs_on_the_host_vm():
    tr = hostvm.execute_program(cases.tape_growing_program(), num_outputs=2)
    assert tr.length == 256


def test_shared_blocks_are_validated_once():
    """14 levels of 10 references each: a tree walk would visit 10^14 lists; the validator checks each shared list once.  16 levels
    nest deeper than the context stack allows."""
    import time
    backend = _lib_or_skip()
    prog = cases.shared_block_program()
    t = time.perf_counter()
    rc, msg = _call(backend, prog)
    assert time.perf_counter() - t < 5
    assert rc in (0, -3), msg                    # valid: it runs (and stops at max_steps) or there is no device
    deeper = cases.shared_block_program(levels=16)
    rc, msg = _call(backend, deeper)
    assert rc == -1 and "nested more than 15 deep" in msg, msg


def test_output_count_is_checked_before_the_device():
    """dg_execute_batch rejects more than 8 outputs on the host, as every execution entry rejects bad arguments, with or without a GPU"""
    backend = _lib_or_skip()
    from distaff_b200 import api
    _, cprog, arr, keep = api._execution_args(hostvm.fibonacci_program(13), [api.ProgramInputs([1, 0])])
    opt = api.ProofOptions()._c()
    handles = (backend.vp * 1)()
    out = np.zeros((9, 2), dtype=np.uint64)
    status = (ctypes.c_int * 1)()
    rc = backend.lib().dg_execute_batch(ctypes.byref(cprog), 1, arr, 9, 1 << 10, ctypes.byref(opt), handles, out.ctypes.data, status, None)
    del keep
    assert (rc, backend.lib().dg_last_error().decode()) == (-1, "cannot have more than 8 outputs")
    assert handles[0] is None
