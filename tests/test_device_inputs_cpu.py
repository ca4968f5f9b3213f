"""CPU-side checks of program inputs in device memory (dg_*_device_inputs, dg_tree_membership_inputs): every whole-call rejection, with
its message, before the device is touched; DeviceInputs argument checking; and no CPU path."""
import ctypes
import os

import numpy as np
import pytest

from distaff_b200 import api, backend, hostvm

FIB = hostvm.fibonacci_program(13)
ENTRIES = ("dg_trace_programs_device_inputs", "dg_execute_programs_device_inputs", "dg_trace_many_device_inputs",
           "dg_execute_many_device_inputs")
FAKE = 0x7f0000000000          # an aligned address that no check reads through


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


class Desc:
    """a dg_device_inputs_t over host arrays, one range per execution and region"""

    def __init__(self, ranges, d_values=FAKE, n_values=64):
        k = len(ranges)
        self.first = [np.array([r[j][0] for r in ranges], dtype=np.uint64) for j in range(3)]
        self.n_pub = np.array([r[0][1] for r in ranges], dtype=np.uint32)
        self.n_ab = [np.array([r[j][1] for r in ranges], dtype=np.uint64) for j in (1, 2)]
        p64, p32 = ctypes.POINTER(backend.u64), ctypes.POINTER(backend.u32)
        self.c = backend.DgDeviceInputs(d_values, n_values, self.first[0].ctypes.data_as(p64), self.n_pub.ctypes.data_as(p32),
                                        self.first[1].ctypes.data_as(p64), self.n_ab[0].ctypes.data_as(p64),
                                        self.first[2].ctypes.data_as(p64), self.n_ab[1].ctypes.data_as(p64))
        assert k == len(self.n_pub)


def _call(entry, desc, count=None, programs=None, program_of=None, num_outputs=None, segment_steps=0, max_steps=1 << 10, options=True):
    """one call of a device-inputs entry; returns (rc, last error)"""
    L = _lib_or_skip()
    programs = programs or [hostvm.compile_program(FIB)]
    k = count if count is not None else len(desc.n_pub) if desc is not None else 1
    cprogs = (backend.DgProgram * len(programs))(*[p.c_struct() for p in programs])
    of = (backend.u32 * max(k, 1))(*(program_of or [0] * k))
    status = (ctypes.c_int * max(k, 1))()
    d = ctypes.byref(desc.c) if desc is not None else None
    fn = getattr(L, entry)
    if "execute" in entry:
        opts = (backend.DgOptions * max(k, 1))(*[api.ProofOptions()._c()] * max(k, 1)) if options else None
        handles = (backend.vp * max(k, 1))()
        outs = (ctypes.c_uint8 * (128 * max(k, 1)))()
        no = (backend.u32 * max(k, 1))(*(num_outputs or [1] * k))
        args = (cprogs, len(programs), k, of, d, no, max_steps) + ((segment_steps,) if "many" in entry else ()) + (
            opts, handles, ctypes.cast(outs, backend.vp), status, None, None)
    else:
        info = (backend.DgExecutionInfo * max(k, 1))()
        args = (cprogs, len(programs), k, of, d, max_steps) + ((segment_steps,) if "many" in entry else ()) + (info, None, status, None)
    rc = fn(*args)
    return rc, L.dg_last_error().decode()


GOOD = [((0, 2), (2, 1), (3, 0)), ((5, 0), (5, 0), (5, 0)), ((0, 2), (0, 3), (2, 3))]      # shared and overlapping ranges


def test_exports():
    for name in ENTRIES + ("dg_tree_membership_inputs",):
        assert name in backend.EXPORTS
    assert [f for f, _ in backend.DgDeviceInputs._fields_] == ["d_values", "n_values", "public_first", "n_public", "secret_a_first",
                                                               "n_secret_a", "secret_b_first", "n_secret_b"]
    assert ctypes.sizeof(backend.DgDeviceInputs) == 64
    L = _lib_or_skip()
    for name in ENTRIES + ("dg_tree_membership_inputs",):
        assert getattr(L, name)


@pytest.mark.parametrize("entry", ENTRIES)
def test_null_descriptor_and_arrays(entry):
    rc, msg = _call(entry, None, count=1)
    assert rc == -1 and msg == "null device inputs", msg
    for field in ("public_first", "n_public", "secret_a_first", "n_secret_a", "secret_b_first", "n_secret_b"):
        d = Desc(GOOD)
        setattr(d.c, field, None)
        rc, msg = _call(entry, d)
        assert rc == -1 and msg == "device inputs: null offset or count array", (field, msg)


@pytest.mark.parametrize("entry", ENTRIES)
def test_null_or_unaligned_values(entry):
    for addr, want in ((None, "device inputs: d_values is null"), (FAKE + 8, "device inputs: d_values is not 16-byte aligned")):
        rc, msg = _call(entry, Desc(GOOD, d_values=addr))
        assert rc == -1 and msg == want, msg
        # only one non-empty range still needs the buffer
        rc, msg = _call(entry, Desc([((0, 0), (9, 1), (0, 0))], d_values=addr))
        assert rc == -1 and msg == want, msg


@pytest.mark.parametrize("entry", ENTRIES)
def test_ranges_past_the_buffer(entry):
    cases = [
        ([((60, 5), (0, 0), (0, 0))], "device inputs of execution 0: public inputs [60, + 5) ends past n_values = 64"),
        ([((0, 0), (0, 1), (0, 0)), ((0, 0), (64, 1), (0, 0))], "device inputs of execution 1: tape A [64, + 1) ends past n_values = 64"),
        ([((0, 0), (0, 0), (2**64 - 1, 2))], "device inputs of execution 0: tape B [18446744073709551615, + 2) overflows"),
        ([((0, 0), (0, 65), (0, 0))], "device inputs of execution 0: tape A [0, + 65) ends past n_values = 64"),
    ]
    for ranges, want in cases:
        rc, msg = _call(entry, Desc(ranges))
        assert rc == -1 and msg == want, msg


@pytest.mark.parametrize("entry", ENTRIES)
def test_checks_of_the_host_forms_come_first(entry):
    """the arguments the host forms check are rejected with the host forms' messages"""
    rc, msg = _call(entry, Desc(GOOD), count=0)
    assert rc == -1 and "at least one execution is needed" in msg, msg
    rc, msg = _call(entry, Desc(GOOD), program_of=[0, 1, 0])
    assert rc == -1 and "program_of[1] = 1 is out of range" in msg, msg
    rc, msg = _call(entry, Desc(GOOD), max_steps=8)
    assert rc == -1 and "max_steps must be at least 16" in msg, msg
    if "execute" in entry:
        rc, msg = _call(entry, Desc(GOOD), num_outputs=[1, 9, 1])
        assert rc == -1 and "cannot have more than 8 outputs" in msg, msg
        rc, msg = _call(entry, Desc(GOOD), options=False)
        assert rc == -1 and "null argument" in msg, msg
    if "many" in entry:
        rc, msg = _call(entry, Desc(GOOD), segment_steps=24)
        assert rc == -1 and "segment_steps must be 0 or a power of two" in msg, msg


def test_empty_ranges_need_no_buffer_and_per_execution_failures_are_not_whole_call():
    """9 public inputs and a short tape A fail their executions only: they pass the whole-call checks and reach the device"""
    _lib_or_skip()
    if _has_gpu():
        pytest.skip("a GPU is present (covered by tests/test_gpu_device_inputs.py)")
    for entry in ENTRIES:
        for ranges, addr in (([((0, 0), (0, 0), (0, 0))], None), ([((0, 9), (0, 1), (0, 2))], FAKE), (GOOD, FAKE)):
            rc, msg = _call(entry, Desc(ranges, d_values=addr))
            assert rc == -3 and "no CPU path" in msg, (entry, msg)


def test_tree_membership_inputs_null_arguments():
    L = _lib_or_skip()
    out = backend.DgDeviceInputs()
    idx = np.zeros(1, dtype=np.uint64)
    assert L.dg_tree_membership_inputs(None, 0, idx.ctypes.data, 1, None, 0, ctypes.byref(out)) == -1
    assert L.dg_last_error().decode() == "null argument"
    assert L.dg_tree_membership_inputs(FAKE, 0, idx.ctypes.data, 1, None, 0, None) == -1
    assert L.dg_last_error().decode() == "null argument"


def test_device_inputs_argument_checking():
    buf = (FAKE, 64)
    x = api.DeviceInputs(buf, [(0, 1), (1, 0)], [(2, 3), (0, 0)], np.array([[5, 1], [6, 0]]))
    assert x.count == 2 and x.n_values == 64 and x._c.d_values == FAKE and x._c.n_public[0] == 1 and x._c.secret_b_first[1] == 6
    empty = api.DeviceInputs((None, 0), [], [], [])
    assert empty.count == 0
    with pytest.raises(TypeError):
        api.DeviceInputs(np.zeros((4, 2), dtype=np.uint64), [], [], [])          # host memory is not device memory
    with pytest.raises(TypeError):
        api.DeviceInputs(FAKE, [], [], [])                                       # a pointer needs its length
    for n in (-1, 2**64, 1.5):
        with pytest.raises(ValueError):
            api.DeviceInputs((FAKE, n), [], [], [])
    with pytest.raises(ValueError, match="one range per execution"):
        api.DeviceInputs(buf, [(0, 1)], [(0, 1), (1, 1)], [(0, 0)])
    for bad in ([(0, 1, 2)], [(-1, 1)], [(0, 2**64)], [("0", 1)], np.array([[0, -1]]), np.array([1, 2, 3])):
        with pytest.raises(ValueError):
            api.DeviceInputs(buf, bad, [(0, 0)] * len(bad), [(0, 0)] * len(bad))
    with pytest.raises(ValueError, match="public-input count"):
        api.DeviceInputs(buf, [(0, 2**32)], [(0, 0)], [(0, 0)])
    x = api.DeviceInputs(buf, [(0, 1)] * 3, [(0, 0)] * 3, [(0, 0)] * 3)
    for fn in (api.trace_programs_device, api.execute_programs_device, api.trace_many_device, api.execute_many_device):
        with pytest.raises(ValueError, match="program_of"):
            fn([FIB], [0, 0], x)
        with pytest.raises(ValueError, match="num_outputs"):
            fn([FIB], [0, 0, 0], x, num_outputs=[1, 1])
        with pytest.raises(ValueError, match="8 outputs"):
            fn([FIB], [0, 0, 0], x, num_outputs=9)
        with pytest.raises(TypeError):
            fn([FIB], [0], [api.ProgramInputs()])
        assert fn([FIB], [], api.DeviceInputs((None, 0), [], [], [])) == []
    with pytest.raises(ValueError, match="one ProofOptions per execution"):
        api.execute_programs_device([FIB], [0, 0, 0], x, options=[api.ProofOptions()])


def test_no_cpu_path():
    _lib_or_skip()
    if _has_gpu():
        pytest.skip("a GPU is present (covered by tests/test_gpu_device_inputs.py)")
    x = api.DeviceInputs((FAKE, 64), [(0, 2)], [(2, 0)], [(2, 0)])
    for fn in (api.trace_programs_device, api.execute_programs_device, api.trace_many_device, api.execute_many_device):
        with pytest.raises(backend.DgError) as e:
            fn([FIB], [0], x)
        assert e.value.code == -3
