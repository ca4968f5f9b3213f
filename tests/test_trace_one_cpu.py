"""CPU-side checks of dg_trace_one / dg_execute_one: bad arguments and encodings are rejected before any device is touched (so these
tests pass without a GPU), and a valid call has no CPU path."""
import ctypes
import os

import numpy as np
import pytest

import distaff_b200 as dg
from distaff_b200 import backend, hostvm
from tests import vm_cases as vc

X = dg.ProgramInputs


def _lib():
    if not os.path.exists(backend.LIB_PATH):
        pytest.skip("libdistaff_gpu.so not built (run __graft_entry__.build())")
    return backend.lib()


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def _trace(program, max_steps=1024, segment_steps=0, inputs=None):
    L = _lib()
    _, cprog, arr, keep = dg.api._execution_args(program, [inputs or X([1, 2])])
    info, st = backend.DgExecutionInfo(), backend.DgTraceOneStats()
    rc = L.dg_trace_one(ctypes.byref(cprog) if cprog is not None else None, arr, max_steps, segment_steps, ctypes.byref(info), None,
                        ctypes.byref(st))
    del keep
    return rc, L.dg_last_error().decode()


def _execute(program, num_outputs=1, max_steps=1024, segment_steps=0, outputs=True, options=True):
    L = _lib()
    _, cprog, arr, keep = dg.api._execution_args(program, [X([1, 2])])
    opt = dg.ProofOptions()._c()
    handle = backend.vp()
    out = np.zeros((8, 2), dtype=np.uint64)
    rc = L.dg_execute_one(ctypes.byref(cprog), arr, num_outputs, max_steps, segment_steps, ctypes.byref(opt) if options else None,
                          ctypes.byref(handle), out.ctypes.data if outputs else None, None, None, None)
    del keep
    assert handle.value is None
    return rc, L.dg_last_error().decode()


@pytest.mark.parametrize("segment_steps", [1, 8, 15, 24, 48, 1000, 2**40 + 1])
def test_segment_steps_must_be_a_power_of_two_of_at_least_16(segment_steps):
    for rc, msg in (_trace("begin add end", segment_steps=segment_steps), _execute("begin add end", segment_steps=segment_steps)):
        assert rc == -1 and msg == "segment_steps must be 0 or a power of two of at least 16"


def test_bad_encodings_and_arguments_are_rejected_before_the_device():
    for name, e in vc.failure_catalogue().items():
        if isinstance(e, vc.Unreachable) and e.program is not None:
            for rc, msg in (_trace(e.program), _execute(e.program)):
                assert rc == -1 and msg.startswith("invalid program encoding"), (name, msg)
    assert _trace("begin add end", max_steps=15) == (-1, "max_steps must be at least 16")
    assert _execute("begin add end", num_outputs=9) == (-1, "cannot have more than 8 outputs")
    assert _execute("begin add end", num_outputs=1, outputs=False) == (-1, "null outputs")
    assert _execute("begin add end", options=False) == (-1, "null argument")
    L = _lib()
    assert L.dg_trace_one(None, None, 1024, 0, None, None, None) == -1 and L.dg_last_error() == b"null argument"


def test_valid_calls_have_no_cpu_path():
    if _has_gpu():
        pytest.skip("a GPU is present")
    for rc, msg in (_trace("begin add end", segment_steps=16), _execute(hostvm.COLLATZ_SOURCE, segment_steps=2**20)):
        assert rc == -3 and "no CPU path" in msg
    with pytest.raises(backend.DgError) as e:
        dg.trace_one("begin add end", X([1, 2]))
    assert e.value.code == -3
