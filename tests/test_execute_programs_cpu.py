"""CPU-side checks of executing many programs in one call (dg_trace_programs / dg_execute_programs): the exports, the argument checks
that run before the device is touched, the job packing of trace_programs / execute_programs, and no CPU path."""
import ctypes
import os

import pytest

from distaff_b200 import api, backend, hostvm
from tests import execution_cases as cases

FIB = hostvm.fibonacci_program(13)
IF_ELSE = cases.IF_ELSE


def _lib_or_skip():
    if not os.path.exists(backend.LIB_PATH):
        pytest.skip("libdistaff_gpu.so not built (run __graft_entry__.build())")
    return backend.lib()


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


def test_exports():
    for name in ("dg_trace_programs", "dg_execute_programs"):
        assert name in backend.EXPORTS
    assert [f for f, _ in backend.DgExecutionStats._fields_] == ["shape_launches", "write_launches", "waves", "prove_groups", "lanes",
                                                                  "shape_ms", "write_ms"]
    assert ctypes.sizeof(backend.DgExecutionStats) == 32
    L = _lib_or_skip()
    assert L.dg_trace_programs and L.dg_execute_programs


def _call(programs, program_of, inputs=None, num_outputs=None, n_programs=None, execute=False):
    """one dg_trace_programs (or dg_execute_programs) call of compiled programs; returns (rc, last error)"""
    L = _lib_or_skip()
    k = len(program_of)
    inputs = inputs or [api.ProgramInputs([1, 0], [1])] * k
    cprogs = (backend.DgProgram * max(len(programs), 1))(*[p.c_struct() for p in programs])
    keep, arr = [], (backend.DgProgramInputs * k)()
    for i, x in enumerate(inputs):
        vals = [api.felt.from_ints(v) for v in (x.public, x.secret_a, x.secret_b)]
        keep += vals
        arr[i] = backend.DgProgramInputs(vals[0].ctypes.data, len(vals[0]), vals[1].ctypes.data, len(vals[1]), vals[2].ctypes.data, len(vals[2]))
    of = (backend.u32 * k)(*program_of)
    status = (ctypes.c_int * k)()
    n = len(programs) if n_programs is None else n_programs
    if execute:
        opt = api.ProofOptions()._c()
        handles = (backend.vp * k)()
        outs = (ctypes.c_uint8 * (128 * k))()
        no = (backend.u32 * k)(*(num_outputs or [1] * k))
        rc = L.dg_execute_programs(cprogs, n, k, of, arr, no, 1 << 10, ctypes.byref(opt), handles, ctypes.cast(outs, backend.vp), status, None, None)
    else:
        info = (backend.DgExecutionInfo * k)()
        rc = L.dg_trace_programs(cprogs, n, k, of, arr, 1 << 10, info, None, status, None)
    return rc, L.dg_last_error().decode()


def test_program_of_out_of_range():
    progs = [hostvm.compile_program(FIB), hostvm.compile_program(IF_ELSE)]
    for execute in (False, True):
        rc, msg = _call(progs, [0, 1, 2, 0], execute=execute)
        assert rc == -1 and "program_of[2] = 2 is out of range" in msg, msg


def test_bad_encoding_is_named_by_its_program():
    good, bad = hostvm.compile_program(FIB), hostvm.compile_program(IF_ELSE)
    bad.children[bad.root_first + 1] = 99
    for execute in (False, True):
        rc, msg = _call([good, bad], [0, 1], execute=execute)
        assert rc == -1 and msg.startswith("program 1: invalid program encoding:") and "out of range" in msg, msg
    rc, msg = _call([bad], [0])                       # one program: the message has no prefix, as dg_trace_batch's
    assert rc == -1 and msg.startswith("invalid program encoding:"), msg
    empty = hostvm.compile_program(FIB)
    empty.n_blocks = 0                                # a table entry without blocks
    rc, msg = _call([good, empty], [0, 1])
    assert rc == -1 and msg == "program 1: invalid program encoding: null or empty arrays", msg


def test_more_than_8_outputs():
    progs = [hostvm.compile_program(FIB), hostvm.compile_program(IF_ELSE)]
    rc, msg = _call(progs, [0, 1, 1], num_outputs=[1, 8, 9], execute=True)
    assert rc == -1 and "cannot have more than 8 outputs" in msg, msg


def test_no_programs():
    progs = [hostvm.compile_program(FIB)]
    for execute in (False, True):
        rc, msg = _call(progs, [0], n_programs=0, execute=execute)
        assert rc == -1 and "at least one program is needed" in msg, msg


def test_pack_jobs_compiles_each_source_once_and_keeps_job_order():
    calls = []

    def compile_counting(src):
        calls.append(src)
        return hostvm.compile_program(src)
    shared = hostvm.compile_program(cases.COMPARE_SOURCE)
    X = api.ProgramInputs
    jobs = [(FIB, X([1, 0])), (IF_ELSE, X([], [1]), 1), (shared, X([3, 4]), 4), (FIB, X([2, 1]), 0), (shared, X([5, 6]), 4),
            (IF_ELSE, X([], [0])), (hostvm.COLLATZ_SOURCE, X([], [7]))]
    programs, program_of, inputs, num_outputs = api.pack_jobs(jobs, compile=compile_counting)
    assert sorted(calls) == sorted([FIB, IF_ELSE, hostvm.COLLATZ_SOURCE])        # each distinct source once; the Program not at all
    assert len(programs) == 4 and programs[2] is shared
    assert program_of == [0, 1, 2, 0, 2, 1, 3]
    assert [p.hash for p in programs] == [hostvm.compile_program(s).hash for s in (FIB, IF_ELSE, cases.COMPARE_SOURCE, hostvm.COLLATZ_SOURCE)]
    assert inputs == [j[1] for j in jobs]
    assert num_outputs == [1, 1, 4, 0, 4, 1, 1]
    with pytest.raises(ValueError):
        api.pack_jobs([(FIB, X(), 9)])
    with pytest.raises(ValueError):
        api.pack_jobs([(FIB,)])


def test_no_cpu_path():
    _lib_or_skip()
    if _has_gpu():
        pytest.skip("a GPU is present (covered by tests/test_gpu_execute_programs.py)")
    import distaff_b200 as dg
    progs = [hostvm.compile_program(FIB), hostvm.compile_program(IF_ELSE)]
    for execute in (False, True):
        rc, msg = _call(progs, [0, 1, 0], execute=execute)
        assert rc == -3 and "no CPU path" in msg, msg
    jobs = [(FIB, dg.ProgramInputs([1, 0])), (IF_ELSE, dg.ProgramInputs([], [1]))]
    for fn in (dg.trace_programs, dg.execute_programs):
        with pytest.raises(backend.DgError) as e:
            fn(jobs)
        assert e.value.code == -3
        assert fn([]) == []
