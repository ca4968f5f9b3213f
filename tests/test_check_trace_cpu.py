"""CPU-side checks of the trace check (dg_check_traces / check_trace): constraint names come from the library without a device and match
the evaluation order the AIR tests use, and the check itself fails loudly (no CPU path) without a CUDA device."""
import ctypes
import os

import pytest

from tests.test_gpu_air import SHAPES, constraint_names


def _backend_or_skip():
    from distaff_b200 import backend
    if not os.path.exists(backend.LIB_PATH):
        pytest.skip("libdistaff_gpu.so not built (run __graft_entry__.build())")
    return backend


def _skip_if_gpu():
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        pytest.skip("a GPU is present (covered by tests/test_gpu_check_trace.py)")


@pytest.mark.parametrize("shape", SHAPES + [(0, 0, 32), (16, 8, 1)], ids=lambda s: "c%dl%ds%d" % s)
def test_constraint_names_match_the_evaluation_order(shape):
    _backend_or_skip()
    import distaff_b200 as dg
    want = constraint_names(shape)
    assert [dg.constraint_name(*shape, j) for j in range(len(want))] == want


def test_constraint_name_limits():
    backend = _backend_or_skip()
    L = backend.lib()
    buf = ctypes.create_string_buffer(64)
    T = len(constraint_names((16, 8, 32)))
    assert T == 78
    assert L.dg_host_constraint_name(16, 8, 32, T - 1, buf, 64) == 0 and buf.value == b"stack slot 31"
    assert L.dg_host_constraint_name(16, 8, 32, T, buf, 64) == -1                 # one past the last constraint
    assert L.dg_host_constraint_name(0, 0, 1, 25, buf, 64) == -1                  # T = 25 for the smallest shape
    assert L.dg_host_constraint_name(0, 0, 1, 24, buf, 64) == 0 and buf.value == b"stack slot 0"
    for bad in ((17, 0, 8), (0, 9, 8), (0, 0, 0), (0, 0, 33)):                   # shapes dg_prove rejects
        assert L.dg_host_constraint_name(*bad, 0, buf, 64) == -1, bad
    small = ctypes.create_string_buffer(7)
    assert L.dg_host_constraint_name(0, 0, 1, 0, small, 7) == 0 and small.value == b"op bit"      # truncated, NUL-terminated


def test_check_trace_raises_without_a_device():
    _backend_or_skip()
    _skip_if_gpu()
    import distaff_b200 as dg
    from distaff_b200 import backend, hostvm
    tr = hostvm.fibonacci(13)
    with pytest.raises(backend.DgError) as e:
        dg.check_trace(tr, tr.program_hash)
    assert e.value.code == -3 and "no CPU path" in str(e.value)
    with pytest.raises(backend.DgError) as e:
        dg.check_traces_device(0x1000, 2, tr.width, tr.length, tr.ctx_depth, tr.loop_depth, [[1, 0], [1, 0]], [[0], [0]])
    assert e.value.code == -3


def test_check_of_no_trace_is_invalid():
    backend = _backend_or_skip()
    reports = (backend.DgTraceReport * 1)()
    assert backend.lib().dg_check_traces(None, 0, None, None, None, None, None, reports, None) == -1
    assert backend.lib().dg_check_traces_device(None, 0, 20, 256, 0, 0, None, None, None, None, None, reports, None) == -1
