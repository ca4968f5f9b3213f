"""CPU-side checks of per-trace proof options (dg_prove_traces_with_options and the execute calls' _with_options forms): the partition by
(length, extension factor) and the groups the call runs (dg_host_group_traces_with_options), ProofOptions.security_level against hand
computation, StarkProof.options on the oracle's proof bytes, the Python argument checks and the per-trace option checks of the C-ABI, which
run before the device is touched."""
import ctypes
import os
import random

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("dg_prove_traces_with_options", "dg_prove_traces_device_with_options", "dg_execute_programs_with_options",
               "dg_execute_many_with_options", "dg_host_group_traces_with_options")


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


def test_new_symbols_are_exported():
    backend = _lib_or_skip()
    L = ctypes.CDLL(backend.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert hasattr(L, name), name
        assert name in backend.EXPORTS, name


# ---- partitions and groups -------------------------------------------------------------------------------------------------------
FIB, COLLATZ, WIDE = (20, 0, 0), (26, 1, 1), (65, 15, 3)


def _group(lengths, shapes, foot, budget, cap, factors=None):
    _lib_or_skip()
    import distaff_b200 as dg
    return dg.group_traces(lengths, [s[0] for s in shapes], [s[1] for s in shapes], [s[2] for s in shapes], foot, budget, cap,
                           extension_factors=factors)


def test_partitions_by_length_and_extension_factor_in_order_of_first_appearance():
    lengths = [256, 256, 2048, 256, 2048, 256, 256]
    factors = [32, 16, 32, 32, 32, 64, 16]
    assert _group(lengths, [FIB] * 7, [1] * 7, 100, 100, factors) == [[0, 3], [1, 6], [2, 4], [5]]


def test_groups_inside_a_partition_are_cut_and_ordered_as_before():
    shapes = [FIB, WIDE, COLLATZ, FIB, WIDE, FIB, COLLATZ]
    factors = [16, 32, 16, 16, 32, 16, 16]
    # partition (256, 16): traces 0, 2, 3, 5, 6 cut by a 10-byte budget, then grouped by shape; partition (256, 32): 1, 4
    assert _group([256] * 7, shapes, [3, 6, 3, 3, 6, 3, 3], 10, 100, factors) == [[0, 3, 2], [5, 6], [1], [4]]
    assert _group([256] * 7, shapes, [1] * 7, 100, 2, factors) == [[0, 2], [3, 5], [6], [1, 4]]


def test_equal_extension_factors_give_todays_groups():
    rng = random.Random(7)
    for _ in range(50):
        k = rng.randint(1, 40)
        lengths = [rng.choice([16, 256, 1024, 4096]) for _ in range(k)]
        shapes = [rng.choice([FIB, COLLATZ, WIDE]) for _ in range(k)]
        foot = [rng.randint(1, 6) for _ in range(k)]
        budget, cap = rng.randint(1, 20), rng.randint(1, 8)
        today = _group(lengths, shapes, foot, budget, cap)
        for b in (16, 32, 256):
            assert _group(lengths, shapes, foot, budget, cap, [b] * k) == today


def test_a_different_extension_factor_splits_a_length():
    """the mix of test_gpu_prove_options.test_launches_add_up_across_extension_factors: three partitions of one length"""
    assert _group([256] * 6, [FIB] * 6, [1] * 6, 100, 100, [16, 32, 64, 16, 32, 64]) == [[0, 3], [1, 4], [2, 5]]


def test_group_traces_argument_checks():
    _lib_or_skip()
    import distaff_b200 as dg
    with pytest.raises(ValueError, match="one per trace"):
        dg.group_traces([256, 256], [20, 20], [0, 0], [0, 0], [1, 1], 10, 10, extension_factors=[32])


# ---- security level ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ext,queries,grinding,optimistic,conservative", [
    (32, 50, 20, 120, 50),       # the defaults: log2(32 / 8) = 2 bits per query; 100 >= 80 adds the grinding factor, 50 does not
    (16, 50, 20, 50, 25),        # 1 bit per query: never 80
    (16, 80, 20, 100, 40),       # exactly 80 counts
    (16, 79, 20, 79, 39),
    (256, 128, 32, 672, 352),    # 5 bits per query: 640 + 32, 320 + 32
    (64, 27, 0, 81, 39),         # 3 bits: 81 >= 80, plus grinding 0
    (64, 1, 32, 3, 0),           # conservative: 1 // 2 = 0 queries
])
def test_security_level(ext, queries, grinding, optimistic, conservative):
    import distaff_b200 as dg
    o = dg.ProofOptions(ext, queries, grinding)
    assert o.security_level() == optimistic
    assert o.security_level(optimistic=True) == optimistic
    assert o.security_level(optimistic=False) == conservative


def test_proof_options_compare_by_value():
    import distaff_b200 as dg
    assert dg.ProofOptions() == dg.ProofOptions(32, 50, 20)
    assert dg.ProofOptions(32, 50, 20) != dg.ProofOptions(32, 50, 21)
    assert len({dg.ProofOptions(), dg.ProofOptions(32, 50, 20), dg.ProofOptions(16)}) == 2
    assert repr(dg.ProofOptions(16, 7, 3)) == "ProofOptions(extension_factor=16, num_queries=7, grinding_factor=3)"


# ---- StarkProof.options --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ext,queries,grinding", [(32, 50, 20), (16, 1, 0), (64, 128, 8), (128, 9, 3), (16, 50, 2)])
def test_stark_proof_options_from_oracle_bytes(po, ext, queries, grinding):
    import distaff_b200 as dg
    from distaff_b200 import hostvm
    tr = hostvm.fibonacci(13)
    ref = po.prove(tr.registers, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs, ext=ext, num_queries=queries, grinding=grinding)
    assert ref.error is None, ref.error
    proof = dg.StarkProof(ref.proof, None, None, None, None, None)
    assert proof.options == dg.ProofOptions(ext, queries, grinding)


def test_stark_proof_options_reject_other_hashes_and_short_bytes():
    import distaff_b200 as dg
    with pytest.raises(ValueError, match="hash function 1"):
        dg.StarkProof(b"\x00" * 10 + bytes([5, 50, 20, 1]), None, None, None, None, None).options
    with pytest.raises(ValueError, match="too short"):
        dg.StarkProof(b"\x05\x32", None, None, None, None, None).options


# ---- argument checks ------------------------------------------------------------------------------------------------------------------
def test_python_option_lists_must_match_the_call():
    _lib_or_skip()
    import distaff_b200 as dg
    from distaff_b200 import hostvm
    traces = [hostvm.fibonacci(13), hostvm.collatz(3)]
    with pytest.raises(ValueError, match="one ProofOptions per trace"):
        dg.prove_traces(traces, [dg.ProofOptions()])
    with pytest.raises(ValueError, match="one ProofOptions per trace"):
        dg.prove_traces(traces, [dg.ProofOptions()] * 3)
    with pytest.raises(TypeError, match="ProofOptions"):
        dg.prove_traces(traces, [dg.ProofOptions(), (32, 50, 20)])
    with pytest.raises(ValueError, match="one ProofOptions per trace"):
        dg.prove_traces_device([0x1000], [20], [256], [0], [0], [[1, 0]], [[0]], [])
    jobs = [(hostvm.fibonacci_program(13), dg.ProgramInputs([1, 0]))] * 3
    with pytest.raises(ValueError, match="one ProofOptions per job"):
        dg.execute_programs(jobs, [dg.ProofOptions()] * 2)
    with pytest.raises(ValueError, match="one ProofOptions per job"):
        dg.execute_many(jobs, [dg.ProofOptions()] * 4)
    with pytest.raises(ValueError, match="one ProofOptions per job"):
        dg.execute_programs([], [dg.ProofOptions()])
    assert dg.execute_programs([], []) == []


def _bad(**fields):
    """a ProofOptions that ProofOptions() would refuse: the C-ABI's own checks see it"""
    import distaff_b200 as dg
    o = dg.ProofOptions()
    for k, v in fields.items():
        setattr(o, k, v)
    return o


@pytest.mark.parametrize("fields,message", [
    ({"extension_factor": 8}, "extension_factor must be a power of 2 between 16 and 256"),
    ({"extension_factor": 48}, "extension_factor must be a power of 2 between 16 and 256"),
    ({"num_queries": 0}, "num_queries must be in 1..128"),
    ({"num_queries": 129}, "num_queries must be in 1..128"),
    ({"grinding_factor": 33}, "grinding factor cannot be greater than 32"),
])
def test_bad_options_of_one_trace_fail_the_call_on_the_host(fields, message):
    """checked with the traces, before the device: the same error with or without a GPU"""
    backend = _lib_or_skip()
    import distaff_b200 as dg
    from distaff_b200 import hostvm
    traces = [hostvm.fibonacci(13), hostvm.collatz(3), hostvm.fibonacci(13)]
    with pytest.raises(backend.DgError) as e:
        dg.prove_traces(traces, [dg.ProofOptions(), dg.ProofOptions(16, 1, 0), _bad(**fields)])
    assert e.value.code == -1 and ("trace 2: " + message) in str(e.value), str(e.value)
    with pytest.raises(backend.DgError) as e:
        dg.prove_traces_device([0x1000, 0x2000], [20, 20], [256, 256], [0, 0], [0, 0], [[1, 0], [1, 0]], [[0], [0]],
                               [_bad(**fields), dg.ProofOptions()])
    assert e.value.code == -1 and ("trace 0: " + message) in str(e.value), str(e.value)
    jobs = [(hostvm.fibonacci_program(13), dg.ProgramInputs([1, 0]))] * 2
    for call in (dg.execute_programs, dg.execute_many):
        with pytest.raises(backend.DgError) as e:
            call(jobs, [dg.ProofOptions(), _bad(**fields)])
        assert e.value.code == -1 and ("execution 1: " + message) in str(e.value), str(e.value)


def test_unsupported_hash_of_one_trace_fails_the_call():
    backend = _lib_or_skip()
    from distaff_b200 import hostvm
    L = backend.lib()
    tr = hostvm.fibonacci(13)
    import numpy as np
    regs = np.ascontiguousarray(tr.registers, dtype=np.uint64)
    cols = (backend.vp * tr.width)(*[regs[j].ctypes.data for j in range(tr.width)])
    ts = (backend.DgTrace * 2)(*[backend.DgTrace(cols, tr.width, tr.length, tr.ctx_depth, tr.loop_depth)] * 2)
    opts = (backend.DgOptions * 2)(backend.DgOptions(32, 50, 20, 0), backend.DgOptions(32, 50, 20, 2))
    handles = (backend.vp * 2)()
    status = (ctypes.c_int * 2)()
    rc = L.dg_prove_traces_with_options(ts, 2, None, None, None, None, opts, handles, status, None)
    assert rc == -1 and L.dg_last_error().decode().startswith("trace 1: unsupported hash function")
    assert list(handles) == [None, None]


def test_no_cpu_fallback_without_a_device():
    backend = _lib_or_skip()
    if _has_gpu():
        pytest.skip("a GPU is present (covered by tests/test_gpu_prove_options.py)")
    import distaff_b200 as dg
    from distaff_b200 import hostvm
    traces = [hostvm.fibonacci(13), hostvm.collatz(3)]
    with pytest.raises(backend.DgError) as e:
        dg.prove_traces(traces, [dg.ProofOptions(), dg.ProofOptions(16, 1, 0)])
    assert e.value.code == -3 and "no CPU path" in str(e.value)
    with pytest.raises(backend.DgError) as e:
        dg.execute_programs([(hostvm.fibonacci_program(13), dg.ProgramInputs([1, 0]))], [dg.ProofOptions(16, 1, 0)])
    assert e.value.code == -3
