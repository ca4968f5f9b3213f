"""Every C entry point that takes a register shape rejects a bad one with a fixed (code, message): a table of bad inputs, each run
against dg_prove, dg_prove_device, dg_prove_batch, dg_prove_batch_device, dg_check_traces(_device), dg_eval_transitions and
dg_host_constraint_name.  Every input fails its argument checks before any kernel runs."""
import ctypes

import numpy as np
import pytest

INVALID = -1
LENGTH = "execution trace length must be a power of 2 and at least 16"
WIDE_HOST = "invalid trace"
WIDE_DEVICE = "execution trace cannot have more than 128 registers"
SHAPE = "register shape out of range"

# name: (width, length, ctx depth, loop depth, extension factor, public inputs), then the message of a host trace and of a device trace
CASES = {
    "ctx_depth": ((40, 16, 17, 0, 32, 0), "context depth cannot be greater than 16", None),
    "loop_depth": ((40, 16, 0, 9, 32, 0), "loop depth cannot be greater than 8", None),
    "width_128": ((128, 16, 0, 0, 32, 0), WIDE_HOST, WIDE_DEVICE),
    "no_user_stack": ((16, 16, 1, 0, 32, 0), "user stack must consist of at least one register", None),
    "stack_depth_33": ((48, 16, 0, 0, 32, 0), "stack depth cannot be greater than 32", None),
    "length_24": ((20, 24, 1, 0, 32, 0), LENGTH, None),
    "extension_8": ((20, 16, 1, 0, 8, 0), "extension_factor must be a power of 2 between 16 and 256", None),
    "extension_512": ((20, 16, 1, 0, 512, 0), "extension_factor must be a power of 2 between 16 and 256", None),
    "inputs_9": ((20, 16, 1, 0, 32, 9), "cannot have more than 8 public inputs / outputs", None),
}
# the trace check takes no proof options
CHECK_CASES = [k for k in CASES if not k.startswith("extension")]


@pytest.fixture(scope="module")
def L():
    from distaff_b200 import backend
    return backend.lib()


@pytest.fixture(scope="module")
def dev(L):
    """device memory for the registers of every case (never read: the calls fail first)"""
    p = ctypes.c_void_p()
    assert L.dg_dev_alloc(ctypes.byref(p), 1 << 20) == 0
    yield p.value
    L.dg_dev_free(p)


class Traces:
    """count host traces of one shape (zero registers), their public inputs and what the calls take"""

    def __init__(self, backend, shapes, n_inputs):
        self.regs = [np.zeros((w, n, 2), dtype=np.uint64) for (w, n, _, _) in shapes]
        self.cols = [(backend.vp * w)(*[r[j].ctypes.data for j in range(w)]) for r, (w, _, _, _) in zip(self.regs, shapes)]
        self.traces = (backend.DgTrace * len(shapes))(*[backend.DgTrace(c, w, n, cd, ld) for c, (w, n, cd, ld) in zip(self.cols, shapes)])
        k = len(shapes)
        self.inputs = np.zeros((max(n_inputs, 1), 2), dtype=np.uint64)
        self.in_ptrs = (backend.vp * k)(*[self.inputs.ctypes.data] * k)
        self.n_in = (backend.u32 * k)(*[n_inputs] * k)
        self.out_ptrs = (backend.vp * k)()
        self.n_out = (backend.u32 * k)()


def message(L, rc):
    return rc, L.dg_last_error().decode()


def prove_host(L, backend, tr, k, opt):
    handles = (backend.vp * k)()
    status = (ctypes.c_int * k)()
    if k == 0:
        return message(L, L.dg_prove(tr.traces, tr.in_ptrs[0], tr.n_in[0], None, 0, ctypes.byref(opt), handles, None))
    return message(L, L.dg_prove_batch(tr.traces, k, tr.in_ptrs, tr.n_in, tr.out_ptrs, tr.n_out, ctypes.byref(opt), handles, status, None))


def check_host(L, backend, tr, k):
    reports = (backend.DgTraceReport * k)()
    return message(L, L.dg_check_traces(tr.traces, k, tr.in_ptrs, tr.n_in, tr.out_ptrs, tr.n_out, None, reports, None))


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_prove(L, dev, case):
    from distaff_b200 import backend
    (w, n, cd, ld, ext, ni), host_msg, dev_msg = CASES[case]
    opt = backend.DgOptions(ext, 50, 20, 0)
    tr = Traces(backend, [(w, n, cd, ld)], ni)
    assert prove_host(L, backend, tr, 0, opt) == (INVALID, host_msg)
    assert prove_host(L, backend, tr, 1, opt) == (INVALID, host_msg)
    handle = backend.vp()
    rc = L.dg_prove_device(dev, w, n, cd, ld, tr.in_ptrs[0], ni, None, 0, ctypes.byref(opt), ctypes.byref(handle), None)
    assert message(L, rc) == (INVALID, dev_msg or host_msg)
    handles = (backend.vp * 2)()
    status = (ctypes.c_int * 2)()
    tr2 = Traces(backend, [(w, n, cd, ld)] * 2, ni)
    rc = L.dg_prove_batch_device(dev, 2, w, n, cd, ld, tr2.in_ptrs, tr2.n_in, tr2.out_ptrs, tr2.n_out, ctypes.byref(opt), handles, status, None)
    assert message(L, rc) == (INVALID, dev_msg or host_msg)
    assert prove_host(L, backend, tr2, 2, opt) == (INVALID, host_msg)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CHECK_CASES)
def test_check_traces(L, dev, case):
    from distaff_b200 import backend
    (w, n, cd, ld, _, ni), host_msg, dev_msg = CASES[case]
    for k in (1, 2):
        tr = Traces(backend, [(w, n, cd, ld)] * k, ni)
        assert check_host(L, backend, tr, k) == (INVALID, host_msg)
        reports = (backend.DgTraceReport * k)()
        rc = L.dg_check_traces_device(dev, k, w, n, cd, ld, tr.in_ptrs, tr.n_in, tr.out_ptrs, tr.n_out, None, reports, None)
        assert message(L, rc) == (INVALID, dev_msg or host_msg)


@pytest.mark.gpu
def test_mixed_shapes_and_null_columns(L):
    from distaff_b200 import backend
    opt = backend.DgOptions(32, 50, 20, 0)
    for other in ((21, 16, 1, 0), (20, 32, 1, 0), (20, 16, 2, 0), (20, 16, 1, 1)):      # width, length, ctx depth, loop depth differ
        tr = Traces(backend, [(20, 16, 1, 0), other], 0)
        assert prove_host(L, backend, tr, 2, opt) == (INVALID, "all traces of a batch must have the same width, length, context depth and loop depth")
        assert check_host(L, backend, tr, 2) == (INVALID, "all traces of a call must have the same width, length, context depth and loop depth")
    for k, at in ((1, 0), (2, 0), (2, 1)):
        tr = Traces(backend, [(20, 16, 1, 0)] * k, 0)
        tr.cols[at][7] = None
        if k == 1:
            assert prove_host(L, backend, tr, 0, opt) == (INVALID, "null register column")
        assert prove_host(L, backend, tr, k, opt) == (INVALID, "null register column")
        assert check_host(L, backend, tr, k) == (INVALID, "null register column")


@pytest.mark.gpu
@pytest.mark.parametrize("shape,sizes,msg", [
    ((17, 0, 4), (4, 5), SHAPE), ((0, 9, 4), (4, 5), SHAPE), ((0, 0, 0), (4, 5), SHAPE), ((0, 0, 33), (4, 5), SHAPE),
    ((2 ** 32 - 1, 0, 4), (4, 5), SHAPE), ((0, 2 ** 32 - 1, 4), (4, 5), SHAPE), ((0, 0, 2 ** 32 - 1), (4, 5), SHAPE),
    ((1, 0, 4), (3, 5), "trace length or extension factor out of range"), ((1, 0, 4), (4, 3), "trace length or extension factor out of range"),
], ids=["ctx_17", "loop_9", "stack_0", "stack_33", "ctx_max", "loop_max", "stack_max", "log_n_3", "log_blowup_3"])
def test_eval_transitions(L, shape, sizes, msg):
    ext = np.zeros(16, dtype=np.uint64)
    seeds = np.zeros(32, dtype=np.uint8)
    out = np.zeros(16, dtype=np.uint64)
    first = (ctypes.c_uint32 * 1)()
    rc = L.dg_eval_transitions(ext.ctypes.data, 1, *shape, *sizes, seeds.ctypes.data, None, 1, out.ctypes.data, first)
    assert message(L, rc) == (INVALID, msg)


@pytest.mark.parametrize("shape,index,msg", [
    ((17, 0, 4), 0, SHAPE), ((0, 9, 4), 0, SHAPE), ((0, 0, 0), 0, SHAPE), ((0, 0, 33), 0, SHAPE), ((2 ** 32 - 1, 0, 4), 0, SHAPE),
    ((0, 2 ** 32 - 1, 4), 0, SHAPE), ((0, 0, 2 ** 32 - 1), 0, SHAPE),
    ((1, 0, 4), 28, "constraint index out of range"), ((16, 8, 32), 78, "constraint index out of range"),
], ids=["ctx_17", "loop_9", "stack_0", "stack_33", "ctx_max", "loop_max", "stack_max", "index_28", "index_78"])
def test_constraint_name(shape, index, msg):
    from distaff_b200 import backend
    import os
    if not os.path.exists(backend.LIB_PATH):
        pytest.skip("libdistaff_gpu.so not built (run __graft_entry__.build())")
    L = backend.lib()
    buf = ctypes.create_string_buffer(64)
    assert message(L, L.dg_host_constraint_name(*shape, index, buf, 64)) == (INVALID, msg)
