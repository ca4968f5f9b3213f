"""CPU-side checks of the device-memory interface (dg_set_memory_limit, dg_memory_usage, dg_plan_prove): the exports are bound, every
entry fails with DG_ERR_NO_DEVICE without a CUDA device, and the Python wrappers reject bad arguments before calling the library."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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
        pytest.skip("a GPU is present (covered by tests/test_gpu_memory_limit.py)")


NAMES = ("dg_set_memory_limit", "dg_memory_usage", "dg_plan_prove")


def test_exports_are_declared_and_bound():
    backend = _backend_or_skip()
    header = open(os.path.join(ROOT, "include", "distaff_gpu.h")).read()
    for name in NAMES:
        assert re.search(r"\bint %s\(" % name, header), name
        assert name in backend.EXPORTS
        assert getattr(backend.lib(), name).restype is ctypes.c_int
    assert "DG_LAYOUT_FULL 0" in header and "DG_LAYOUT_EVAL_COSETS 1" in header
    # the plan struct: int32 + 3 x uint32 + 3 x uint64
    assert ctypes.sizeof(backend.DgProvePlan) == 40


def test_without_a_device_every_entry_fails_with_no_device():
    backend = _backend_or_skip()
    _skip_if_gpu()
    L = backend.lib()
    held, peak = ctypes.c_size_t(0), ctypes.c_size_t(0)
    opt = backend.DgOptions(32, 50, 20, 0)
    plan = backend.DgProvePlan()
    assert L.dg_set_memory_limit(1 << 30) == -3
    assert L.dg_set_memory_limit(0) == -3
    assert L.dg_memory_usage(ctypes.byref(held), ctypes.byref(peak)) == -3
    assert L.dg_plan_prove(26, 1 << 20, 1, ctypes.byref(opt), ctypes.byref(plan)) == -3
    import distaff_b200 as dg
    for call in (lambda: dg.set_memory_limit(1 << 30), dg.memory_usage, lambda: dg.plan_prove(26, 1 << 20)):
        with pytest.raises(backend.DgError) as e:
            call()
        assert e.value.code == -3 and "no CPU path" in str(e.value)


def test_python_argument_checks():
    _backend_or_skip()
    import distaff_b200 as dg
    with pytest.raises(ValueError):
        dg.set_memory_limit(-1)
    for args in ((0, 256), (128, 256), (26, 15), (26, 100), (26, 256, 0)):
        with pytest.raises(ValueError):
            dg.plan_prove(*args)
    with pytest.raises(AssertionError):
        dg.plan_prove(26, 256, 1, dg.ProofOptions(extension_factor=512))
