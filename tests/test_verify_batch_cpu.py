"""CPU-side checks of batched verification (dg_verify_batch / verify_batch): an empty batch or a null array is refused for the whole
call, and without a CUDA device the call fails loudly with "no CPU path"."""
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
        pytest.skip("a GPU is present (covered by tests/test_gpu_verify_batch.py)")


def _arrays(backend, k, proof=b"not a proof"):
    """the ten arguments after `count` for k copies of one (program hash, no inputs / outputs, proof)"""
    h = ctypes.create_string_buffer(32)
    p = ctypes.create_string_buffer(proof, len(proof))
    ptr = lambda b: ctypes.cast(b, backend.vp)  # noqa: E731
    keep = (h, p)
    return keep, [(backend.vp * k)(*[ptr(h)] * k), (backend.vp * k)(), (backend.u32 * k)(), (backend.vp * k)(), (backend.u32 * k)(),
                  (backend.vp * k)(*[ptr(p)] * k), (ctypes.c_size_t * k)(*[len(proof)] * k), (ctypes.c_int * k)(*[7] * k), None]


def test_empty_batch_and_null_arrays_are_invalid():
    backend = _lib_or_skip()
    L = backend.lib()
    keep, args = _arrays(backend, 1)
    assert L.dg_verify_batch(0, *args) == -1
    assert "at least one proof" in L.dg_last_error().decode()
    for i in (0, 5, 6, 7):                    # program hashes, proof bytes, proof lengths, status
        bad = list(args)
        bad[i] = None
        assert L.dg_verify_batch(1, *bad) == -1 and "null argument" in L.dg_last_error().decode(), i
    assert list(args[7]) == [7]               # a whole-call error leaves every status unset


def test_batch_has_no_cpu_fallback():
    backend = _lib_or_skip()
    _skip_if_gpu()
    keep, args = _arrays(backend, 3)
    rc = backend.lib().dg_verify_batch(3, *args)
    assert rc == -3 and "no CPU path" in backend.lib().dg_last_error().decode()
    assert list(args[7]) == [7, 7, 7]


def test_verify_batch_raises_without_a_device():
    _lib_or_skip()
    _skip_if_gpu()
    import distaff_b200 as dg
    from distaff_b200 import backend
    with pytest.raises(backend.DgError) as e:
        dg.verify_batch([(bytes(32), [1, 0], [3], b"not a proof")] * 2)
    assert e.value.code == -3 and "no CPU path" in str(e.value)


def test_verify_batch_of_nothing_is_empty():
    _lib_or_skip()
    import distaff_b200 as dg
    assert dg.verify_batch([]) == []
