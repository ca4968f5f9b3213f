"""CPU-side checks of batched proving across register shapes (dg_prove_traces / prove_traces): every argument is checked on the host
before the device is touched (a bad entry is named), the call fails loudly without a device, and the grouping of the traces by length,
memory and shape (dg_host_group_traces) is what the call runs."""
import ctypes
import os

import numpy as np
import pytest


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


def _c_traces(backend, traces):
    """dg_trace_t entries (and what keeps their columns alive) for hostvm traces"""
    regs = [np.ascontiguousarray(t.registers, dtype=np.uint64) for t in traces]
    cols = [(backend.vp * r.shape[0])(*[r[j].ctypes.data for j in range(r.shape[0])]) for r in regs]
    ts = (backend.DgTrace * len(traces))(*[backend.DgTrace(c, r.shape[0], r.shape[1], t.ctx_depth, t.loop_depth)
                                          for c, r, t in zip(cols, regs, traces)])
    return ts, (regs, cols)


def _call(backend, ts, count, inputs=None):
    opt = backend.DgOptions(32, 50, 20, 0)
    handles = (backend.vp * max(count, 1))()
    status = (ctypes.c_int * max(count, 1))()
    rc = backend.lib().dg_prove_traces(ts, count, inputs[0] if inputs else None, inputs[1] if inputs else None, None, None, ctypes.byref(opt),
                                       handles, status, None)
    return rc, backend.lib().dg_last_error().decode()


def test_count_zero_and_null_arrays_are_invalid():
    backend = _lib_or_skip()
    from distaff_b200 import hostvm
    rc, msg = _call(backend, None, 0)
    assert rc == -1 and "at least one trace" in msg
    rc, msg = _call(backend, None, 2)
    assert rc == -1 and "null argument" in msg
    ts, keep = _c_traces(backend, [hostvm.fibonacci(13)])
    opt = backend.DgOptions(32, 50, 20, 0)
    status = (ctypes.c_int * 1)()
    assert backend.lib().dg_prove_traces(ts, 1, None, None, None, None, ctypes.byref(opt), None, status, None) == -1
    assert backend.lib().dg_prove_traces(ts, 1, None, None, None, None, None, (backend.vp * 1)(), status, None) == -1
    u32, u64 = backend.u32, backend.u64
    rc = backend.lib().dg_prove_traces_device(None, (u32 * 1)(20), (u64 * 1)(256), (u32 * 1)(0), (u32 * 1)(0), 1, None, None, None, None,
                                              ctypes.byref(opt), (backend.vp * 1)(), status, None)
    assert rc == -1 and "null argument" in backend.lib().dg_last_error().decode()
    rc = backend.lib().dg_prove_traces_device((backend.vp * 1)(0x1000), None, (u64 * 1)(256), (u32 * 1)(0), (u32 * 1)(0), 1, None, None, None,
                                              None, ctypes.byref(opt), (backend.vp * 1)(), status, None)
    assert rc == -1
    rc = backend.lib().dg_prove_traces_device(None, None, None, None, None, 0, None, None, None, None, ctypes.byref(opt), (backend.vp * 1)(),
                                              status, None)
    assert rc == -1 and "at least one trace" in backend.lib().dg_last_error().decode()
    del keep


@pytest.mark.parametrize("field,value,expected", [
    ("length", 100, "power of 2"),
    ("length", 8, "power of 2"),
    ("width", 200, "invalid trace"),
    ("ctx_depth", 17, "context depth cannot be greater than 16"),
    ("loop_depth", 9, "loop depth cannot be greater than 8"),
    ("width", 15 + 1 + 1, "user stack must consist of at least one register"),
    ("width", 15 + 1 + 1 + 33, "stack depth cannot be greater than 32"),
])
def test_bad_shape_names_its_entry_before_the_device(field, value, expected):
    """a shape dg_prove rejects fails the whole call with DG_ERR_INVALID, naming the entry -- with or without a GPU: nothing runs"""
    backend = _lib_or_skip()
    from distaff_b200 import hostvm
    traces = [hostvm.fibonacci(13), hostvm.collatz(3), hostvm.fibonacci(13)]
    ts, keep = _c_traces(backend, traces)
    setattr(ts[1], field, value)
    if field == "width" and value < 128:
        ts[1].ctx_depth, ts[1].loop_depth = 1, 1           # collatz's depths; the width leaves a stack of 0 or 33 registers
    rc, msg = _call(backend, ts, 3)
    assert rc == -1, msg
    assert msg.startswith("trace 1: ") and expected in msg, msg
    del keep


def test_bad_inputs_and_null_columns_name_their_entry():
    backend = _lib_or_skip()
    from distaff_b200 import felt, hostvm
    traces = [hostvm.fibonacci(13), hostvm.collatz(3), hostvm.fibonacci(13)]
    ts, keep = _c_traces(backend, traces)
    pub = felt.from_ints(list(range(9)))
    inputs = ((backend.vp * 3)(pub.ctypes.data, pub.ctypes.data, pub.ctypes.data), (backend.u32 * 3)(2, 1, 9))
    rc, msg = _call(backend, ts, 3, inputs)
    assert rc == -1 and msg.startswith("trace 2: ") and "more than 8 public inputs" in msg, msg
    inputs = ((backend.vp * 3)(pub.ctypes.data, None, pub.ctypes.data), (backend.u32 * 3)(2, 1, 2))
    rc, msg = _call(backend, ts, 3, inputs)
    assert rc == -1 and msg.startswith("trace 1: ") and "null public inputs" in msg, msg
    keep[1][2][5] = None
    rc, msg = _call(backend, ts, 3)
    assert rc == -1 and msg.startswith("trace 2: ") and "null register column" in msg, msg


def test_no_cpu_fallback_without_a_device():
    backend = _lib_or_skip()
    if _has_gpu():
        pytest.skip("a GPU is present (covered by tests/test_gpu_prove_traces.py)")
    import distaff_b200 as dg
    from distaff_b200 import hostvm
    traces = [hostvm.fibonacci(13), hostvm.collatz(3), hostvm.execute("begin pad.2 hash.2 end", public_inputs=[5, 6], num_outputs=2)]
    ts, keep = _c_traces(backend, traces)
    rc, msg = _call(backend, ts, 3)
    assert rc == -3 and "no CPU path" in msg
    with pytest.raises(backend.DgError) as e:
        dg.prove_traces(traces)
    assert e.value.code == -3 and "no CPU path" in str(e.value)
    with pytest.raises(backend.DgError) as e:
        dg.prove_traces_device([0x1000, 0x2000], [20, 26], [256, 2048], [0, 1], [0, 1], [[1, 0], []], [[0], [1]])
    assert e.value.code == -3
    del keep


# ---- grouping --------------------------------------------------------------------------------------------------------------------------
def _group(lengths, shapes, foot, budget, cap):
    _lib_or_skip()
    import distaff_b200 as dg
    return dg.group_traces(lengths, [s[0] for s in shapes], [s[1] for s in shapes], [s[2] for s in shapes], foot, budget, cap)


FIB, COLLATZ, MERKLE, WIDE = (20, 0, 0), (26, 1, 1), (27, 1, 1), (65, 15, 3)


def test_lengths_in_order_of_first_appearance():
    lengths = [2048, 256, 2048, 4096, 256, 256]
    groups = _group(lengths, [FIB] * 6, [1] * 6, 100, 100)
    assert groups == [[0, 2], [1, 4, 5], [3]]


def test_shapes_are_adjacent_in_first_appearance_order():
    shapes = [FIB, COLLATZ, FIB, WIDE, COLLATZ, MERKLE, FIB]
    groups = _group([256] * 7, shapes, [1] * 7, 100, 100)
    assert groups == [[0, 2, 6, 1, 4, 3, 5]]


def test_groups_are_cut_by_budget_cap_and_launch_width():
    shapes = [FIB, WIDE, FIB, FIB, WIDE]
    # footprints: bytes of each trace; a group holds at most 10 bytes
    assert _group([256] * 5, shapes, [3, 6, 3, 3, 6], 10, 100) == [[0, 1], [2, 3], [4]]
    # the count cap ($DG_BATCH_GROUP)
    assert _group([256] * 5, shapes, [1] * 5, 100, 2) == [[0, 1], [2, 3], [4]]
    # a trace larger than the budget still runs, alone
    assert _group([256] * 3, [FIB] * 3, [1, 50, 1], 10, 100) == [[0], [1], [2]]
    # sum of widths <= 65535: 1008 wide traces fill one launch, the 1009th starts the next group
    groups = _group([256] * 1009, [WIDE] * 1009, [1] * 1009, 1 << 40, 1 << 20)
    assert [len(g) for g in groups] == [1008, 1]


def test_one_shape_is_cut_as_the_batch_plan():
    """a one-shape call is cut as dg_prove_batch cuts it: groups of plan.group consecutive traces"""
    groups = _group([1024] * 7, [COLLATZ] * 7, [5] * 7, 15, 3)
    assert groups == [[0, 1, 2], [3, 4, 5], [6]]
