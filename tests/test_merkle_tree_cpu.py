"""Merkle trees kept in device memory, without a GPU: the exports, the argument checks that run before the device is touched, and the
update plan of dg_tree_update (dg_host_tree_plan) against a Python restatement."""
import ctypes
import os
import random

import numpy as np
import pytest

import distaff_b200 as dg
from distaff_b200 import backend

M = 2**128 - 45 * 2**40 + 1
NAMES = ["dg_tree_new", "dg_tree_new_device", "dg_tree_info", "dg_tree_paths", "dg_tree_update", "dg_tree_read", "dg_tree_free",
         "dg_host_tree_plan"]


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(backend.LIB_PATH):
        pytest.skip("libdistaff_gpu.so not built")
    return backend.lib()


def test_exports(lib):
    for name in NAMES:
        assert hasattr(lib, name), name
    assert "dg_tree_free" in backend.VOID_EXPORTS


def test_argument_checks_before_the_device(lib):
    leaves = bytes(32 * 4)
    handle = backend.vp()
    assert lib.dg_tree_new(0, leaves, 4, None) == -1
    assert lib.dg_tree_new(0, None, 4, ctypes.byref(handle)) == -1
    assert lib.dg_tree_new_device(0, None, 4, ctypes.byref(handle)) == -1
    for hash_id in (-1, 4):
        assert lib.dg_tree_new(hash_id, leaves, 4, ctypes.byref(handle)) == -1
        assert "hash id must be" in lib.dg_last_error().decode()
        assert lib.dg_tree_new_device(hash_id, 1, 4, ctypes.byref(handle)) == -1
    for n in (0, 1, 3, 6):
        assert lib.dg_tree_new(0, bytes(32 * max(n, 1)), n, ctypes.byref(handle)) == -1
        assert "power of 2" in lib.dg_last_error().decode()
        assert lib.dg_tree_new_device(1, 1, n, ctypes.byref(handle)) == -1
    bad = bytearray(32 * 4)
    bad[32 * 2 + 16:32 * 3] = (2**128 - 1).to_bytes(16, "little")
    assert lib.dg_tree_new(3, bytes(bad), 4, ctypes.byref(handle)) == -1
    assert "leaf 2 element 1 is not a field element" in lib.dg_last_error().decode()
    assert handle.value is None
    out = ctypes.create_string_buffer(32)
    assert lib.dg_tree_info(None, None, None, out) == -1
    assert lib.dg_tree_paths(None, (ctypes.c_uint64 * 1)(0), 1, out) == -1
    assert lib.dg_tree_update(None, (ctypes.c_uint64 * 1)(0), out, 1, out) == -1
    assert lib.dg_tree_read(None, out, None) == -1
    lib.dg_tree_free(None)


def test_python_argument_checks():
    with pytest.raises(ValueError, match="hash is one of"):
        dg.MerkleTree(bytes(64), hash="gmimc")
    with pytest.raises(ValueError, match="32 bytes each"):
        dg.MerkleTree(bytes(48))
    with pytest.raises(TypeError):
        dg.MerkleTree([(1, 2), (3, 4)], hash="blake3")              # pairs are hasher leaves only
    with pytest.raises(ValueError):
        dg.MerkleTree([(1, 2), (3, 4, 5)], hash="hasher")
    with pytest.raises(ValueError, match="integer in"):
        dg.MerkleTree([(1, 2), (-1, 4)], hash="hasher")
    with pytest.raises(ValueError, match="integer in"):
        dg.MerkleTree([(1, 2), (2**128, 4)], hash="hasher")
    with pytest.raises(ValueError, match="non-negative"):
        dg.MerkleTree._indexes([0, -1])


def test_shape_errors_come_before_no_device(lib):
    """a bad leaf count is an argument error (DG_ERR_INVALID) with or without a device"""
    with pytest.raises(backend.DgError) as e:
        dg.MerkleTree(bytes(96))
    assert e.value.code == -1 and "power of 2" in str(e.value)


def plan(lib, indexes, L):
    idx = np.array(indexes, dtype=np.uint64)
    cap = 8 + 3 * len(indexes) + 3 * (len(indexes) + 1) * L.bit_length()
    out = np.zeros(cap, dtype=np.uint64)
    written = ctypes.c_size_t(0)
    backend.check(lib.dg_host_tree_plan(idx.ctypes.data, len(idx), L, out.ctypes.data, cap, ctypes.byref(written)))
    v = [int(x) for x in out[:written.value]]
    K, d, T = v[:3]
    leaves, source = v[3:3 + K], v[3 + K:3 + 2 * K]
    at, levels = 3 + 2 * K, []
    for _ in range(d):
        n = v[at]
        levels.append((v[at + 1:at + 1 + n], v[at + 1 + n:at + 1 + 2 * n]))
        at += 1 + 2 * n
    assert at == len(v) and T == sum(len(ids) for ids, _ in levels)
    return leaves, source, levels


def restated(indexes, L):
    """the last occurrence of every index, sorted; per level the sorted unique parents with their first changed child below"""
    last = {i: k for k, i in enumerate(indexes)}
    leaves = sorted(last)
    levels, below = [], [(L + i) for i in leaves]               # heap ids of the leaves: leaf i is node L + i
    while below[0] > 1:
        ids, first = [], []
        for k, c in enumerate(below):
            if not ids or ids[-1] != c >> 1:
                ids.append(c >> 1)
                first.append(k)
        levels.append((ids, first))
        below = ids
    return leaves, [last[i] for i in leaves], levels


@pytest.mark.parametrize("L", [2, 4, 16, 1 << 10, 1 << 20])
def test_plan_matches_the_restatement(lib, L):
    rng = random.Random(L)
    cases = [[0], [L - 1], [0, 1], [L - 2, L - 1], [L - 1, 0], [3 % L, 3 % L, 1 % L, 3 % L], [rng.randrange(L) for _ in range(50)],
             [rng.randrange(min(L, 8)) for _ in range(40)]]
    if L <= 1 << 10:
        cases.append(list(range(L)))
        cases.append(rng.sample(range(L), L))
    for idx in cases:
        got = plan(lib, idx, L)
        want = restated(idx, L)
        assert got == want, idx
        d = L.bit_length() - 1
        assert len(got[2]) == d and got[2][-1] == ([1], [0])
        assert sum(len(ids) for ids, _ in got[2]) <= len(set(idx)) * d


def test_plan_counts(lib):
    L = 1 << 10
    _, _, levels = plan(lib, [5], L)                             # K = 1: one node per level
    assert [len(ids) for ids, _ in levels] == [1] * 10
    _, _, levels = plan(lib, [6, 7], L)                          # siblings share every node
    assert [ids for ids, _ in levels][0] == [(L + 6) >> 1] and sum(len(ids) for ids, _ in levels) == 10
    _, _, levels = plan(lib, list(range(L))[::-1], L)            # every leaf: all L - 1 nodes
    assert sum(len(ids) for ids, _ in levels) == L - 1
    leaves, source, _ = plan(lib, [9, 4, 9, 9, 4, 2], L)         # last occurrence wins
    assert leaves == [2, 4, 9] and source == [5, 4, 3]


def test_plan_rejects_bad_arguments(lib):
    out = np.zeros(64, dtype=np.uint64)
    w = ctypes.c_size_t(0)
    idx = np.array([1, 8, 2], dtype=np.uint64)
    assert lib.dg_host_tree_plan(idx.ctypes.data, 3, 8, out.ctypes.data, 64, ctypes.byref(w)) == -1
    assert "index 8 (entry 1) is not a leaf of a tree of 8 leaves" in lib.dg_last_error().decode()
    assert lib.dg_host_tree_plan(idx.ctypes.data, 1, 6, out.ctypes.data, 64, ctypes.byref(w)) == -1
    assert lib.dg_host_tree_plan(idx.ctypes.data, 3, 16, out.ctypes.data, 4, ctypes.byref(w)) == -1
    assert "buffer too small" in lib.dg_last_error().decode()
