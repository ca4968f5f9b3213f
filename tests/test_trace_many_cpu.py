"""CPU-side checks of dg_trace_many / dg_execute_many: the exports, every argument check before any device is touched (so these tests
pass without a GPU), DG_ERR_NO_DEVICE for a valid call without a device, and the Python argument checks."""
import ctypes
import os

import numpy as np
import pytest

import distaff_b200 as dg
from distaff_b200 import backend, hostvm
from tests import vm_cases as vc

X = dg.ProgramInputs
INVALID, NO_DEVICE = -1, -3


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


def _call(jobs, count=None, program_of=None, max_steps=1024, segment_steps=0, num_outputs=None, null_inputs=False, outputs=True):
    """(rc of dg_trace_many, rc of dg_execute_many), each with dg_last_error()"""
    L = _lib()
    programs, cprogs, of, arr, no, keep = dg.api._programs_args(jobs)
    k = len(jobs) if count is None else count
    if program_of is not None:
        of = (backend.u32 * len(program_of))(*program_of)
    inputs = None if null_inputs else arr
    n = max(k, len(jobs))
    info = (backend.DgExecutionInfo * n)()
    status = (ctypes.c_int * n)()
    st = backend.DgManyStats()
    rc = L.dg_trace_many(cprogs, len(programs), k, of, inputs, max_steps, segment_steps, info, None, status, ctypes.byref(st))
    traced = (rc, L.dg_last_error().decode())
    opt = dg.ProofOptions()._c()
    handles = (backend.vp * n)()
    out = np.zeros((n, 8, 2), dtype=np.uint64)
    n_out = (backend.u32 * n)(*(num_outputs or no))
    rc = L.dg_execute_many(cprogs, len(programs), k, of, inputs, n_out, max_steps, segment_steps, ctypes.byref(opt), handles,
                           out.ctypes.data if outputs else None, status, None, ctypes.byref(st))
    executed = (rc, L.dg_last_error().decode())
    assert all(h is None for h in handles)
    del keep
    return traced, executed


JOBS = [("begin add end", X([1, 2])), (hostvm.COLLATZ_SOURCE, X([], [27])), ("begin add end", X([3, 4]))]


def test_exports():
    L = _lib()
    for name in ("dg_trace_many", "dg_execute_many"):
        assert hasattr(L, name) and name in backend.EXPORTS
    assert dg.trace_many is dg.api.trace_many and dg.execute_many is dg.api.execute_many
    names = [f for f, _ in backend.DgManyStats._fields_]
    assert names[:3] == ["table_ms", "sequential_ms", "segment_ms"] and names[-1] == "fallback"


def test_argument_checks_before_the_device():
    both = lambda rc, msg, **kw: [r == (rc, msg) for r in _call(JOBS, **kw)]    # noqa: E731
    assert both(INVALID, "at least one execution is needed", count=0) == [True, True]
    assert all(both(INVALID, "program_of[1] = 5 is out of range: the call has 2 programs", program_of=[0, 5, 0]))
    assert all(both(INVALID, "null argument", null_inputs=True))
    assert all(both(INVALID, "max_steps must be at least 16", max_steps=15))
    for s in (1, 8, 15, 24, 1000, 2**40 + 1):
        assert all(both(INVALID, "segment_steps must be 0 or a power of two of at least 16", segment_steps=s))
    traced, executed = _call(JOBS, num_outputs=[1, 9, 1])
    assert executed == (INVALID, "cannot have more than 8 outputs") and traced[0] != INVALID
    assert _call(JOBS, outputs=False)[1] == (INVALID, "null outputs")
    L = _lib()
    assert L.dg_trace_many(None, 1, 1, None, None, 1024, 0, None, None, None, None) == INVALID and L.dg_last_error() == b"null argument"


def test_bad_encodings_name_their_program():
    for name, e in vc.failure_catalogue().items():
        if isinstance(e, vc.Unreachable) and e.program is not None:
            for rc, msg in _call([("begin add end", X([1, 2])), (e.program, X([1, 2]))]):
                assert rc == INVALID and msg.startswith("program 1: invalid program encoding"), (name, msg)


def test_valid_calls_have_no_cpu_path():
    if _has_gpu():
        pytest.skip("a GPU is present")
    for rc, msg in _call(JOBS, segment_steps=16):
        assert rc == NO_DEVICE and "no CPU path" in msg
    for f in (dg.trace_many, dg.execute_many):
        with pytest.raises(backend.DgError) as e:
            f(JOBS)
        assert e.value.code == NO_DEVICE


def test_python_argument_checks():
    for f in (dg.trace_many, dg.execute_many):
        assert f([]) == []
        for s in (8, 24, -16):
            with pytest.raises(ValueError, match="segment_steps"):
                f(JOBS, segment_steps=s)
        with pytest.raises(ValueError, match="a job is"):
            f([("begin add end",)])
        with pytest.raises(ValueError, match="more than 8 outputs"):
            f([("begin add end", X([1, 2]), 9)])
