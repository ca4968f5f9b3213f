"""Program inputs in device memory (dg_*_device_inputs, DeviceInputs) against the same inputs given on the host: traces, proofs,
statuses, messages and the stats' launch, wave and group figures of all four calls on the execution corpus; layouts (ranges in reverse
order, shared tapes, empty tapes, 0 to 8 public inputs, a range at the end of the buffer, programs interleaved, the batch-path fallback of
the tabled calls); per-execution failures of bad values in every region and position; and membership proofs of a device MerkleTree
(dg_tree_membership_inputs) against a HasherTree's."""
import ctypes
import random

import numpy as np
import pytest

import distaff_b200 as dg
from distaff_b200 import api, backend, felt, hostvm
from tests import execution_cases as ec
from tests.test_gpu_execute_batch import FAIL_CASES, FAIL_SOURCE
from tests.test_gpu_execute_programs import _mixed_suite
from tests.test_gpu_trace_one import _switch_with_unread_hash

pytestmark = pytest.mark.gpu
X = dg.ProgramInputs
M = 2**128 - 45 * 2**40 + 1


def _tensor(values):
    import torch
    a = felt.from_ints(values).reshape(-1, 2) if values else np.zeros((0, 2), dtype=np.uint64)
    return torch.from_numpy(a.view(np.int64)).view(torch.uint64).to("cuda")


def _device(inputs, reverse=False, pad=0):
    """DeviceInputs of ProgramInputs: every region's values in one tensor, executions (and the regions of each) in reverse buffer order
    when `reverse`, `pad` unused values before them"""
    vals, ranges = [0] * pad, [[None] * len(inputs) for _ in range(3)]
    order = list(range(len(inputs)))[::-1] if reverse else range(len(inputs))
    for i in order:
        x = inputs[i]
        regions = ((0, x.public), (1, x.secret_a), (2, x.secret_b))
        for r, region in (regions[::-1] if reverse else regions):
            ranges[r][i] = (len(vals), len(region))
            vals += region
    return dg.DeviceInputs(_tensor(vals), *ranges)


def _no_ms(d):
    return {k: _no_ms(v) if isinstance(v, dict) else v for k, v in d.items() if not k.endswith("_ms")}


def _same_trace(got, want):
    if isinstance(want, backend.DgError):
        assert isinstance(got, backend.DgError) and (got.code, str(got)) == (want.code, str(want)), (got, want)
        return
    assert not isinstance(got, backend.DgError), got
    assert got.registers.shape == want.registers.shape and np.array_equal(got.registers, want.registers)
    assert (got.ctx_depth, got.loop_depth, got.stack_depth) == (want.ctx_depth, want.loop_depth, want.stack_depth)
    assert got.program_hash == want.program_hash and got.outputs == want.outputs and got.public_inputs == want.public_inputs


def _same_proof(got, want):
    if isinstance(want, backend.DgError):
        assert isinstance(got, backend.DgError) and (got.code, str(got)) == (want.code, str(want)), (got, want)
        return
    assert not isinstance(got, backend.DgError), got
    assert got[0] == want[0] and got[1].bytes == want[1].bytes


def _both(jobs, device_inputs=None, calls=("trace_programs", "execute_programs", "trace_many", "execute_many"), verify=True):
    """every call of `calls` on the jobs, host form against device form (device_inputs, default _device of the jobs' inputs)"""
    programs, program_of, inputs, num_outputs = api.pack_jobs(jobs)
    d = device_inputs or _device(inputs)
    out = {}
    for name in calls:
        hs, ds = {}, {}
        host = getattr(dg, name)(jobs, stats=hs)
        dev = getattr(dg, name + "_device")(programs, program_of, d, num_outputs, stats=ds)
        assert len(dev) == len(host)
        for g, w in zip(dev, host):
            (_same_trace if name.startswith("trace") else _same_proof)(g, w)
        assert _no_ms(ds) == _no_ms(hs), (name, ds, hs)
        if verify and name.startswith("execute"):
            items = [(programs[program_of[i]].hash, inputs[i].public, r[0], r[1]) for i, r in enumerate(dev) if not isinstance(r, backend.DgError)]
            assert dg.verify_batch(items) == [None] * len(items)
        out[name] = dev
    return out


def test_corpus_host_and_device_forms_agree():
    jobs, _ = _mixed_suite()
    jobs += [(FAIL_SOURCE, x) for _, x in FAIL_CASES]
    for name, src, pub, a, b, no in ec.SMALL:
        jobs.append((src, X(pub, a, b), no))
    out = _both(jobs)
    assert sum(isinstance(r, backend.DgError) for r in out["execute_programs"]) >= 4
    # the same buffer laid out backwards, with unused values before it
    _both(jobs, _device(api.pack_jobs(jobs)[2], reverse=True, pad=5), calls=("trace_programs", "execute_many"), verify=False)


def test_layouts():
    """shared and overlapping ranges, empty tapes, 0 to 8 public inputs, a range ending at the last value, programs interleaved"""
    rng = random.Random(1)
    vals = [rng.randrange(M) for _ in range(40)] + [1, 0, 3, 2, 5, 1]
    t = _tensor(vals)
    n = len(vals)
    fib, collatz, if_else = hostvm.fibonacci_program(13), hostvm.COLLATZ_SOURCE, ec.IF_ELSE
    spec = []                                             # (program, public range, tape A range, tape B range, outputs)
    for k in range(9):
        spec.append((fib, (3 * k, k), (0, 0), (0, 0), 1))                         # 0 to 8 public inputs, no tapes
    spec.append((if_else, (0, 0), (n - 2, 1), (0, 0), 1))                        # tape A: the value 5
    spec.append((collatz, (0, 0), (n - 1, 1), (0, 0), 1))                        # a range ending at n_values - 1
    spec.append((if_else, (0, 0), (n - 2, 2), (n - 1, 1), 1))                    # overlapping tapes
    spec.append((if_else, (0, 0), (n - 2, 2), (n - 1, 1), 1))                    # shared with the one before
    spec.append((fib, (n - 6, 2), (n - 6, 2), (n - 6, 2), 1))                    # one range read three times
    spec.append((ec.COMPARE_SOURCE, (n - 4, 2), (0, 0), (0, 0), 4))
    d = dg.DeviceInputs(t, [s[1] for s in spec], [s[2] for s in spec], [s[3] for s in spec])
    take = lambda r: vals[r[0]:r[0] + r[1]]
    jobs = [(s[0], X(take(s[1]), take(s[2]), take(s[3])), s[4]) for s in spec]
    out = _both(jobs, d)
    assert sum(not isinstance(r, backend.DgError) for r in out["execute_programs"]) >= 10
    # a (device pointer, n) pair, with the public inputs read back range by range
    buf = backend.DeviceBuffer(16 * n).upload(felt.from_ints(vals))
    p = dg.DeviceInputs((buf, n), [s[1] for s in spec], [s[2] for s in spec], [s[3] for s in spec])
    programs, program_of, inputs, num_outputs = api.pack_jobs(jobs)
    for g, w in zip(dg.trace_programs_device(programs, program_of, p, num_outputs), out["trace_programs"]):
        _same_trace(g, w)


def test_tabled_calls_fall_back_to_the_batch_path():
    unread = _switch_with_unread_hash()
    jobs = [(hostvm.COLLATZ_SOURCE, X([], [9])), (unread.program, unread.inputs, unread.num_outputs), (hostvm.fibonacci_program(13), X([1, 2]))]
    jobs += [(unread.program, unread.inputs, unread.num_outputs), (ec.COMPARE_SOURCE, X([3, 4]), 4)]
    programs, program_of, inputs, num_outputs = api.pack_jobs(jobs)
    st = {}
    dg.execute_many_device(programs, program_of, _device(inputs), num_outputs, stats=st)
    assert st["fallback_programs"] == 1 and st["tabled_programs"] == 3, st
    _both(jobs, calls=("trace_many", "execute_many"))


@pytest.mark.parametrize("bad", [M, M + 1, 2**128 - 1])
def test_bad_values_fail_only_their_execution(bad):
    what = ("public input", "tape A value", "tape B value")
    good = [(ec.IF_ELSE, X([], [1])), (hostvm.fibonacci_program(13), X([1, 0]))]
    jobs, want = [], []
    for r in range(3):
        for j in (0, 1, 2):
            regions = [[1, 2, 3], [1, 4, 5], [6, 7, 8]]
            regions[r][j] = bad
            jobs += [good[len(jobs) % 2], (ec.IF_ELSE, X(*regions))]
            want += [None, f"{what[r]} {j} is not a field element"]
    jobs += [(ec.IF_ELSE, X(list(range(9)), [1])), (ec.IF_ELSE, X([], [1], [1, 1]))]
    want += ["expected no more than 8 public inputs", "tape A cannot be shorter than tape B"]
    jobs.append(good[0])
    want.append(None)
    out = _both(jobs)
    for name, results in out.items():
        for r, w in zip(results, want):
            if w is None:
                assert not isinstance(r, backend.DgError), (name, r)
            else:
                assert isinstance(r, backend.DgError) and r.code == -7 and str(r).endswith(w), (name, r, w)


def _pairs(L, seed):
    rng = random.Random(seed)
    return [(rng.randrange(M), rng.randrange(M)) for _ in range(L)]


def _check_membership(tree, ht, indexes, program):
    got = dg.prove_membership(tree, indexes, program)
    want = dg.prove_membership(ht, indexes, program)
    assert len(got) == len(want) == len(indexes)
    for g, w in zip(got, want):
        assert isinstance(g, tuple), g
        assert g[:3] == w[:3] and g[3].bytes == w[3].bytes
    return got


@pytest.mark.parametrize("program", ["smpath", "pmpath"])
def test_membership_of_small_trees(program):
    items = []
    for d in range(1, 13):
        pairs = _pairs(2**d, d)
        with dg.MerkleTree(pairs, "hasher") as tree:
            items += _check_membership(tree, dg.HasherTree(pairs), list(range(2**d)), program)
    assert dg.verify_batch(items) == [None] * len(items)


@pytest.mark.parametrize("program", ["smpath", "pmpath"])
def test_membership_of_a_large_tree_and_after_updates(program):
    L = 2**20
    raw = np.random.default_rng(20).integers(0, 2**63, size=(L, 2, 2), dtype=np.uint64)
    pairs = [(int(a[0]) | int(a[1]) << 64, int(b[0]) | int(b[1]) << 64) for a, b in raw.tolist()]
    indexes = random.Random(4).sample(range(L), 4096)
    with dg.MerkleTree(raw.tobytes(), "hasher") as tree:
        got = _check_membership(tree, dg.HasherTree(pairs), indexes, program)
        assert dg.verify_batch(got) == [None] * len(got)
        changed = indexes[:5] + [0, L - 1]
        new = _pairs(len(changed), 7)
        tree.update(changed, new)
        for i, p in zip(changed, new):
            pairs[i] = p
        after = dg.HasherTree(pairs)
        got = _check_membership(tree, after, changed + indexes[100:110], program)
        assert dg.verify_batch(got) == [None] * len(got)


def test_membership_inputs_layout_and_rejections():
    pairs = _pairs(16, 3)
    ht = dg.HasherTree(pairs)
    with dg.MerkleTree(pairs, "hasher") as tree:
        for program in ("smpath", "pmpath"):
            x = tree.membership_inputs([5, 5, 0, 15], program)
            assert x.count == 4 and x.n_values == 4 * (18 if program == "smpath" else 11)
            for k, i in enumerate([5, 5, 0, 15]):
                want = ht.smpath_inputs(i) if program == "smpath" else ht.pmpath_inputs(i)
                for r, region in enumerate((want.public, want.secret_a, want.secret_b)):
                    f, n = (int(v) for v in x.ranges[r][k])
                    vals = np.zeros((n, 2), dtype=np.uint64)
                    if n:
                        backend.check(backend.lib().dg_dev_download(vals.ctypes.data, x.ptr + 16 * f, 16 * n))
                    assert felt.to_ints(vals) == region, (program, i, r)
            assert tree.membership_inputs([], program).count == 0
            with pytest.raises(backend.DgError, match="index 16 .entry 1. is not a leaf of a tree of 16 leaves"):
                tree.membership_inputs([3, 16], program)
            with pytest.raises(backend.DgError, match="index 16"):
                dg.prove_membership(tree, [3, 16], program)
        L = backend.lib()
        idx = np.array([1, 2], dtype=np.uint64)
        out = backend.DgDeviceInputs()
        assert L.dg_tree_membership_inputs(tree._handle(), 2, idx.ctypes.data, 2, None, 0, ctypes.byref(out)) == -1
        assert "DG_PATH_SMPATH" in L.dg_last_error().decode()
        assert L.dg_tree_membership_inputs(tree._handle(), 0, idx.ctypes.data, 2, None, 0, ctypes.byref(out)) == 0 and out.n_values == 36
        buf = backend.DeviceBuffer(16 * 40)
        assert L.dg_tree_membership_inputs(tree._handle(), 0, idx.ctypes.data, 2, buf.ptr, 35, ctypes.byref(out)) == -1
        assert L.dg_last_error().decode() == "d_values holds 35 values, the inputs need 36"
        assert L.dg_tree_membership_inputs(tree._handle(), 0, idx.ctypes.data, 2, buf.ptr + 8, 36, ctypes.byref(out)) == -1
        assert L.dg_last_error().decode() == "d_values is not 16-byte aligned"
        assert L.dg_tree_membership_inputs(tree._handle(), 0, idx.ctypes.data, 2, buf.ptr, 36, ctypes.byref(out)) == -1
        assert L.dg_last_error().decode() == "null offset or count array in out"
        host = np.zeros(40 * 2, dtype=np.uint64)
        x = tree.membership_inputs([1, 2], "smpath")
        out = backend.DgDeviceInputs.from_buffer_copy(x._c)
        assert L.dg_tree_membership_inputs(tree._handle(), 0, idx.ctypes.data, 2, host.ctypes.data, 40, ctypes.byref(out)) == -1
        assert "is not device memory" in L.dg_last_error().decode()
        buf.free()
    with dg.MerkleTree(bytes(32 * 8), "blake3") as other:
        for program in ("smpath", "pmpath"):
            with pytest.raises(ValueError, match="hasher"):
                dg.prove_membership(other, [0], program)
        L = backend.lib()
        out = backend.DgDeviceInputs()
        assert L.dg_tree_membership_inputs(other._handle(), 0, idx.ctypes.data, 2, None, 0, ctypes.byref(out)) == -1
        assert "hash 3 (hasher)" in L.dg_last_error().decode()


def test_device_values_must_be_device_memory():
    host = np.zeros((4, 2), dtype=np.uint64)
    x = dg.DeviceInputs((host.ctypes.data, 4), [(0, 1)], [(1, 1)], [(2, 1)])
    with pytest.raises(backend.DgError, match="d_values is not device memory"):
        dg.trace_programs_device([hostvm.fibonacci_program(13)], [0], x)
