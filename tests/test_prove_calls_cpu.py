"""Every prove and trace-check entry point checks its traces, their public input / output counts and its options on the host, before it
touches the device: the table of bad inputs of tests/test_gpu_argument_checks.py through all eight prove entries and both check entries,
the messages that follow the form of a trace (host dg_trace_t or device registers) whatever the entry, and valid traces that still need
a device.  No test here needs a GPU: every call fails before the context is created."""
import ctypes
import os

import pytest

from tests.test_gpu_argument_checks import CASES, CHECK_CASES, INVALID, LENGTH, Traces

NO_DEVICE = -3
# entry: (form of its traces, whether it names the trace in its messages, whether it takes one set of options per trace)
PROVE_ENTRIES = {
    "dg_prove": ("host", False, False),
    "dg_prove_device": ("device", False, False),
    "dg_prove_batch": ("host", False, False),
    "dg_prove_batch_device": ("device", False, False),
    "dg_prove_traces": ("host", True, False),
    "dg_prove_traces_with_options": ("host", True, True),
    "dg_prove_traces_device": ("device", True, False),
    "dg_prove_traces_device_with_options": ("device", True, True),
}
CHECK_ENTRIES = {"dg_check_traces": "host", "dg_check_traces_device": "device"}


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.fixture(scope="module")
def backend():
    from distaff_b200 import backend
    if not os.path.exists(backend.LIB_PATH):
        pytest.skip("libdistaff_gpu.so not built (run __graft_entry__.build())")
    return backend


@pytest.fixture(scope="module")
def dev(backend):
    """device memory for the registers of the device entries (never read: the calls fail first); without a device, an address that is
    never dereferenced"""
    L = backend.lib()
    p = ctypes.c_void_p()
    if not _has_gpu() or L.dg_dev_alloc(ctypes.byref(p), 1 << 20) != 0:
        yield 0x1000
        return
    yield p.value
    L.dg_dev_free(p)


def _prove(backend, entry, tr, k, shape, opt, dev):
    """calls a prove entry with k traces of one shape (w, n, ctx depth, loop depth): tr's host traces and public inputs, or k device
    traces at dev; returns (code, message)"""
    L = backend.lib()
    w, n, cd, ld = shape
    form, _, per_trace = PROVE_ENTRIES[entry]
    options = (backend.DgOptions * k)(*[opt] * k) if per_trace else ctypes.byref(opt)
    handles = (backend.vp * k)()
    status = (ctypes.c_int * k)()
    io = (tr.in_ptrs, tr.n_in, tr.out_ptrs, tr.n_out)
    if entry == "dg_prove":
        rc = L.dg_prove(tr.traces, tr.in_ptrs[0], tr.n_in[0], None, 0, options, handles, None)
    elif entry == "dg_prove_device":
        rc = L.dg_prove_device(dev, w, n, cd, ld, tr.in_ptrs[0], tr.n_in[0], None, 0, options, handles, None)
    elif entry == "dg_prove_batch_device":
        rc = L.dg_prove_batch_device(dev, k, w, n, cd, ld, *io, options, handles, status, None)
    elif form == "host":
        rc = getattr(L, entry)(tr.traces, k, *io, options, handles, status, None)
    else:
        arr = lambda t, x: (t * k)(*[x] * k)
        rc = getattr(L, entry)(arr(backend.vp, dev), arr(backend.u32, w), arr(backend.u64, n), arr(backend.u32, cd), arr(backend.u32, ld), k,
                               *io, options, handles, status, None)
    return rc, L.dg_last_error().decode()


def _check(backend, entry, tr, k, shape, dev):
    L = backend.lib()
    w, n, cd, ld = shape
    reports = (backend.DgTraceReport * k)()
    io = (tr.in_ptrs, tr.n_in, tr.out_ptrs, tr.n_out)
    if entry == "dg_check_traces":
        rc = L.dg_check_traces(tr.traces, k, *io, None, reports, None)
    else:
        rc = L.dg_check_traces_device(dev, k, w, n, cd, ld, *io, None, reports, None)
    return rc, L.dg_last_error().decode()


def _count(entry):
    return 1 if entry in ("dg_prove", "dg_prove_device") else 2


@pytest.mark.parametrize("entry", list(PROVE_ENTRIES))
@pytest.mark.parametrize("case", list(CASES))
def test_prove_entries_reject_bad_traces_on_the_host(backend, dev, entry, case):
    """every case of the table, on every prove entry, fails with the message of the trace's form before the device is touched; a
    per-trace entry names the trace, and its options when they are per trace"""
    (w, n, cd, ld, ext, ni), host_msg, dev_msg = CASES[case]
    form, names_trace, per_trace = PROVE_ENTRIES[entry]
    k = _count(entry)
    msg = host_msg if form == "host" else dev_msg or host_msg
    if names_trace and (per_trace or not case.startswith("extension")):
        msg = "trace 0: " + msg
    tr = Traces(backend, [(w, n, cd, ld)] * k, ni)
    assert _prove(backend, entry, tr, k, (w, n, cd, ld), backend.DgOptions(ext, 50, 20, 0), dev) == (INVALID, msg)


@pytest.mark.parametrize("entry", list(CHECK_ENTRIES))
@pytest.mark.parametrize("case", CHECK_CASES)
def test_check_entries_reject_bad_traces_on_the_host(backend, dev, entry, case):
    (w, n, cd, ld, _, ni), host_msg, dev_msg = CASES[case]
    msg = host_msg if CHECK_ENTRIES[entry] == "host" else dev_msg or host_msg
    tr = Traces(backend, [(w, n, cd, ld)] * 2, ni)
    assert _check(backend, entry, tr, 2, (w, n, cd, ld), dev) == (INVALID, msg)


@pytest.mark.parametrize("entry", ["dg_prove_traces_device", "dg_prove_traces_device_with_options"])
@pytest.mark.parametrize("shape,msg", [
    ((128, 16, 0, 0), "execution trace cannot have more than 128 registers"),
    ((15, 16, 0, 0), "user stack must consist of at least one register"),
], ids=["width_128", "width_15"])
def test_per_trace_device_entries_report_the_register_shape(backend, dev, entry, shape, msg):
    """a device trace's width outside 16..127 is reported as TraceShape::of_trace reports it, as the one-shape device entries do"""
    tr = Traces(backend, [shape] * 2, 0)
    assert _prove(backend, entry, tr, 2, shape, backend.DgOptions(32, 50, 20, 0), dev) == (INVALID, "trace 0: " + msg)
    assert _prove(backend, "dg_prove_device", tr, 1, shape, backend.DgOptions(32, 50, 20, 0), dev) == (INVALID, msg)


class FakeTraces:
    """k host traces of one shape whose columns are never read (the calls fail before any upload), and no public inputs"""

    def __init__(self, backend, shape, k):
        w, n, cd, ld = shape
        self.cols = (backend.vp * w)(*[0x1000] * w)
        self.traces = (backend.DgTrace * k)(*[backend.DgTrace(self.cols, w, n, cd, ld)] * k)
        self.in_ptrs, self.n_in = (backend.vp * k)(), (backend.u32 * k)()
        self.out_ptrs, self.n_out = (backend.vp * k)(), (backend.u32 * k)()


@pytest.mark.parametrize("entry", list(PROVE_ENTRIES) + list(CHECK_ENTRIES))
def test_every_entry_takes_the_prove_length_bound(backend, dev, entry):
    """2^31 steps of 16 registers are 512 GiB: every entry, the trace check included, rejects the length before the device"""
    shape = (16, 1 << 31, 0, 0)
    k = _count(entry)
    tr = FakeTraces(backend, shape, k)
    if entry in CHECK_ENTRIES:
        assert _check(backend, entry, tr, k, shape, dev) == (INVALID, LENGTH)
    else:
        prefix = "trace 0: " if PROVE_ENTRIES[entry][1] else ""
        assert _prove(backend, entry, tr, k, shape, backend.DgOptions(32, 50, 20, 0), dev) == (INVALID, prefix + LENGTH)


@pytest.mark.parametrize("entry", list(PROVE_ENTRIES) + list(CHECK_ENTRIES))
def test_valid_traces_still_need_a_device(backend, entry):
    """valid traces pass the host check on every entry and then fail for want of a device: there is no CPU path"""
    if _has_gpu():
        pytest.skip("a GPU is present (the GPU tests prove and check these traces)")
    from distaff_b200 import hostvm
    fib = hostvm.fibonacci(13)
    shape = (fib.registers.shape[0], fib.length, fib.ctx_depth, fib.loop_depth)
    k = _count(entry)
    tr = Traces(backend, [shape] * k, 2)
    if entry in CHECK_ENTRIES:
        rc, msg = _check(backend, entry, tr, k, shape, 0x1000)
    else:
        rc, msg = _prove(backend, entry, tr, k, shape, backend.DgOptions(32, 50, 20, 0), 0x1000)
    assert rc == NO_DEVICE and "no CPU path" in msg, msg
