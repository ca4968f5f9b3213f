"""CPU-side checks of batched proving (dg_prove_batch / prove_batch): the entry points are bound, reject an empty batch, and fail
loudly with "no CPU path" when there is no CUDA device."""
import ctypes
import os

import pytest


def _lib_or_skip():
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
        pytest.skip("a GPU is present (covered by tests/test_gpu_prove_batch.py)")


def test_empty_batch_is_invalid():
    backend = _lib_or_skip()
    opt = backend.DgOptions(32, 50, 20, 0)
    handles = (backend.vp * 1)()
    status = (ctypes.c_int * 1)()
    rc = backend.lib().dg_prove_batch(None, 0, None, None, None, None, ctypes.byref(opt), handles, status, None)
    assert rc == -1 and "at least one trace" in backend.lib().dg_last_error().decode()
    rc = backend.lib().dg_prove_batch_device(None, 0, 20, 256, 0, 0, None, None, None, None, ctypes.byref(opt), handles, status, None)
    assert rc == -1


def test_batch_has_no_cpu_fallback():
    backend = _lib_or_skip()
    _skip_if_gpu()
    import numpy as np
    from distaff_b200 import hostvm
    tr = hostvm.fibonacci(13)
    regs = np.ascontiguousarray(tr.registers, dtype=np.uint64)
    w, n = regs.shape[0], regs.shape[1]
    cols = (backend.vp * w)(*[regs[j].ctypes.data for j in range(w)])
    traces = (backend.DgTrace * 2)(backend.DgTrace(cols, w, n, tr.ctx_depth, tr.loop_depth), backend.DgTrace(cols, w, n, tr.ctx_depth, tr.loop_depth))
    opt = backend.DgOptions(32, 50, 20, 0)
    handles = (backend.vp * 2)()
    status = (ctypes.c_int * 2)()
    rc = backend.lib().dg_prove_batch(traces, 2, None, None, None, None, ctypes.byref(opt), handles, status, None)
    assert rc == -3 and "no CPU path" in backend.lib().dg_last_error().decode()


def test_prove_batch_raises_without_a_device():
    _lib_or_skip()
    _skip_if_gpu()
    import distaff_b200 as dg
    from distaff_b200 import backend, hostvm
    traces = [hostvm.fibonacci(13), hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[2, 1]), hostvm.collatz(3)]
    with pytest.raises(backend.DgError) as e:
        dg.prove_batch(traces)
    assert e.value.code == -3 and "no CPU path" in str(e.value)
    with pytest.raises(backend.DgError) as e:
        dg.prove_batch_device(0x1000, 2, 20, 256, 0, 0, [[1, 0], [1, 0]], [[0], [0]])
    assert e.value.code == -3


def test_prove_batch_of_nothing_is_empty():
    _lib_or_skip()
    import distaff_b200 as dg
    assert dg.prove_batch([]) == []
