"""Batch Merkle proofs and path verification without a GPU: the exports, every whole-call argument check (DG_ERR_INVALID before any device
is touched), BatchMerkleProof bytes against the oracle's encoding, and the Python restatements of prove_batch / verify / verify_batch
(tests/merkle_batch_refs.py) against the oracle on every case where the crate does not panic, and against the crate's own cases."""
import ctypes
import os
import random

import numpy as np
import pytest

import distaff_b200 as dg
from distaff_b200 import backend
from tests import merkle_batch_refs as R

NAMES = ["dg_tree_prove_batch", "dg_merkle_verify_paths", "dg_merkle_verify_batch"]
ORACLE_HASHES = ["blake3", "rescue", "poseidon"]


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(backend.LIB_PATH):
        pytest.skip("libdistaff_gpu.so not built")
    return backend.lib()


def random_leaves(L, seed):
    """L leaves of canonical field elements (each below 2^127 < M), so that every hash takes them"""
    raw = np.random.default_rng(seed).integers(0, 2**63, size=(L, 2, 2), dtype=np.uint64).tobytes()
    return [raw[32 * i:32 * i + 32] for i in range(L)]


def test_exports(lib):
    for name in NAMES:
        assert hasattr(lib, name), name
    for name in ("BatchMerkleProof", "merkle_verify_paths", "merkle_verify_batch"):
        assert hasattr(dg, name), name
    assert callable(dg.MerkleTree.prove_batch) and callable(dg.MerkleTree.verify) and callable(dg.MerkleTree.verify_batch)


def err(lib):
    return lib.dg_last_error().decode()


def test_verify_paths_argument_checks(lib):
    root, idx, path = b"\0" * 96, (ctypes.c_uint64 * 3)(0, 1, 2), bytes(32 * 3 * 3)
    st = (ctypes.c_int * 3)()
    for hash_id in (-1, 4, 7):
        assert lib.dg_merkle_verify_paths(hash_id, root, 1, idx, path, 3, 3, st) == -1
        assert "hash id must be" in err(lib)
    for entries in (0, 1, 65, 1000):
        assert lib.dg_merkle_verify_paths(0, root, 1, idx, path, entries, 3, st) == -1
        assert "2 to 64 entries" in err(lib)
    for n_roots in (0, 2, 4):
        assert lib.dg_merkle_verify_paths(0, root, n_roots, idx, path, 3, 3, st) == -1
        assert "n_roots" in err(lib)
    for args in ((None, idx, path, st), (root, None, path, st), (root, idx, None, st), (root, idx, path, None)):
        assert lib.dg_merkle_verify_paths(1, args[0], 1, args[1], args[2], 3, 3, args[3]) == -1
        assert "null array" in err(lib)


def test_verify_batch_argument_checks(lib):
    k = 2
    roots = bytes(64)
    idx = (backend.vp * k)()
    n_idx = (backend.u32 * k)()
    proofs = (backend.vp * k)()
    lens = (ctypes.c_size_t * k)()
    st = (ctypes.c_int * k)()
    for hash_id in (-1, 4):
        assert lib.dg_merkle_verify_batch(hash_id, k, roots, idx, n_idx, proofs, lens, st) == -1
        assert "hash id must be" in err(lib)
    full = [roots, idx, n_idx, proofs, lens, st]
    for j in range(len(full)):
        args = list(full)
        args[j] = None
        assert lib.dg_merkle_verify_batch(2, k, *args) == -1
        assert "null array" in err(lib)


def test_prove_batch_argument_checks(lib):
    n = ctypes.c_size_t(0)
    assert lib.dg_tree_prove_batch(None, (ctypes.c_uint64 * 1)(0), 1, None, 0, ctypes.byref(n)) == -1


def test_python_argument_checks():
    with pytest.raises(ValueError, match="hash is one of"):
        dg.merkle_verify_paths(bytes(32), [0], [[bytes(32)] * 3], hash="gmimc")
    with pytest.raises(ValueError, match="hash is one of"):
        dg.merkle_verify_batch([(bytes(32), [0], b"")], hash="sha3")
    with pytest.raises(ValueError, match="one number of entries"):
        dg.merkle_verify_paths(bytes(32), [0, 1], [[bytes(32)] * 3, [bytes(32)] * 4])
    with pytest.raises(ValueError, match="shape"):
        dg.merkle_verify_paths(bytes(32), [0], np.zeros((1, 3, 16), dtype=np.uint8))
    with pytest.raises(ValueError, match="indexes and"):
        dg.merkle_verify_paths(bytes(32), [0, 1], [[bytes(32)] * 3])
    assert dg.merkle_verify_paths(bytes(32), [], []) == [] and dg.merkle_verify_batch([]) == []


def test_whole_call_errors_come_before_no_device(lib):
    """a bad entry count or hash is an argument error (DG_ERR_INVALID) with or without a device"""
    with pytest.raises(backend.DgError) as e:
        dg.merkle_verify_paths(bytes(32), [0], np.zeros((1, 65, 32), dtype=np.uint8))
    assert e.value.code == -1 and "2 to 64 entries" in str(e.value)
    with pytest.raises(backend.DgError) as e:
        dg.MerkleTree.verify(bytes(32), 0, [bytes(32)])
    assert e.value.code == -1


# ---- BatchMerkleProof bytes ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ORACLE_HASHES)
def test_encoding_round_trips_the_oracle_bytes(po, name):
    rng = random.Random(name)
    for L in (2, 8, 64):
        leaves = random_leaves(L, L)
        for idx in ([0], [L - 1], list(range(L)), rng.sample(range(L), max(1, L // 3)), []):
            raw = po.merkle_prove_batch(name, b"".join(leaves), idx)
            p = dg.BatchMerkleProof.from_bytes(raw)
            assert p.to_bytes() == raw and len(p.values) == len(idx) and p.depth == L.bit_length() - 1
            assert dg.BatchMerkleProof.from_bytes(p.to_bytes()) == p
            assert R.encode(p.values, p.nodes, p.depth) == raw


def test_malformed_encodings_are_rejected():
    p = dg.BatchMerkleProof([bytes(range(32))], [[bytes(32), bytes([7] * 32)], []], 5)
    raw = p.to_bytes()
    for bad in (raw[:-1], raw + b"\0", raw[:8], b"", (2**40).to_bytes(8, "little") + raw[8:]):
        with pytest.raises(ValueError, match="not a BatchMerkleProof"):
            dg.BatchMerkleProof.from_bytes(bad)
    assert p != dg.BatchMerkleProof(p.values, p.nodes, 4) and p == dg.BatchMerkleProof.from_bytes(raw)


# ---- the restatements against the oracle --------------------------------------------------------------------------------------------
def index_sets(L, rng):
    sets = [[0], [L - 1], [0, 1], list(range(1, L, 2)), list(range(0, L, 2)), list(range(L)), list(range(L))[::-1], []]
    for _ in range(6):
        s = rng.sample(range(L), rng.randrange(1, L + 1))
        rng.shuffle(s)
        sets.append(s)
    return sets


@pytest.mark.parametrize("name", ORACLE_HASHES)
@pytest.mark.parametrize("L", [2, 4, 8, 32])
def test_prove_batch_restatement_matches_the_oracle(po, name, L):
    h = R.oracle_hash(po, name)
    leaves = random_leaves(L, 7 * L)
    nodes = R.heap(h, leaves)
    assert b"".join(nodes) == po.merkle_nodes(name, b"".join(leaves))
    for idx in index_sets(L, random.Random(L)):
        assert R.encode(*R.prove_batch(leaves, nodes, idx)) == po.merkle_prove_batch(name, b"".join(leaves), idx), idx
    with pytest.raises(R.Panic, match=f"invalid index {L + 1}"):
        R.prove_batch(leaves, nodes, [0, L + 1])
    with pytest.raises(R.Panic, match="repeating indexes detected"):
        R.prove_batch(leaves, nodes, [1, 0, 1])
    with pytest.raises(R.Panic, match="index out of bounds"):
        R.prove_batch(leaves, nodes, [L])


@pytest.mark.parametrize("name", ORACLE_HASHES)
def test_verify_restatement_matches_the_oracle(po, name):
    """every path of a tree is accepted, a path is a batch proof of one index to the oracle, and flips agree"""
    h = R.oracle_hash(po, name)
    L = 16
    leaves = random_leaves(L, 3)
    nodes = R.heap(h, leaves)
    root = nodes[1]
    for i in range(L):
        path = R.prove_batch(leaves, nodes, [i])
        full = [path[0][0]] + path[1][0]
        assert R.verify(root, i, full, h)
        as_batch = lambda p: po.merkle_verify_batch(name, root, [i], R.encode([p[0]], [p[1:]], 4))
        assert as_batch(full) == 1
        for e in range(len(full)):
            bad = list(full)
            bad[e] = bytes([bad[e][0] ^ 1]) + bad[e][1:]
            assert R.verify(root, i, bad, h) == (as_batch(bad) == 1) == False   # noqa: E712
        assert not R.verify(root, i ^ 2, full, h)


def test_verify_reads_only_the_low_index_bits(po):
    """the reference's verify checks an index >= L = 2^(entries - 1) as index mod L"""
    h = R.oracle_hash(po, "blake3")
    L = 8
    leaves = random_leaves(L, 4)
    nodes = R.heap(h, leaves)
    for i in range(L):
        v, n, _ = R.prove_batch(leaves, nodes, [i])
        path = [v[0]] + n[0]
        for big in (i + L, i + 5 * L, i + 2**40, i + 2**63, 2**64 - L + i):
            assert R.verify(nodes[1], big, path, h)
        assert not R.verify(nodes[1], (i ^ 1) + L, path, h)


def mutations(values, nodes, depth, rng):
    """(values, nodes, depth) variants: every value and node flipped, the depth moved, slots shortened and lengthened, values swapped"""
    flip = lambda d: bytes([d[0] ^ 0x80]) + d[1:]
    out = []
    for k in range(len(values)):
        vs = list(values)
        vs[k] = flip(vs[k])
        out.append((vs, nodes, depth))
    for s in range(len(nodes)):
        for j in range(len(nodes[s])):
            ns = [list(x) for x in nodes]
            ns[s][j] = flip(ns[s][j])
            out.append((values, ns, depth))
        if nodes[s]:
            out.append((values, [x if t != s else x[:-1] for t, x in enumerate(nodes)], depth))
        out.append((values, [x if t != s else x + [nodes[s][0] if nodes[s] else values[0]] for t, x in enumerate(nodes)], depth))
    out += [(values, nodes, depth - 1), (values, nodes, depth + 1), (values[:-1], nodes, depth), (values, nodes[:-1], depth),
            (values, nodes + [[]], depth)]
    if len(values) >= 2:
        a, b = rng.sample(range(len(values)), 2)
        vs = list(values)
        vs[a], vs[b] = vs[b], vs[a]
        out.append((vs, nodes, depth))
    return out


@pytest.mark.parametrize("name", ORACLE_HASHES)
@pytest.mark.parametrize("L", [2, 8, 32])
def test_verify_batch_restatement_matches_the_oracle(po, name, L):
    h = R.oracle_hash(po, name)
    rng = random.Random(L + 1)
    leaves = random_leaves(L, 11 * L)
    nodes = R.heap(h, leaves)
    root = nodes[1]
    panics = 0
    for idx in index_sets(L, rng):
        values, pn, depth = R.prove_batch(leaves, nodes, idx)
        cases = [(idx, values, pn, depth)] + [(idx,) + m for m in mutations(values, pn, depth, rng) if m[2] >= 0]
        if idx:
            cases += [(idx[:-1], values, pn, depth), (idx + [L], values, pn, depth), (idx + idx[:1], values, pn, depth),
                      ([(i ^ 1) for i in idx], values, pn, depth)]
        for ix, vs, ns, d in cases:
            want = po.merkle_verify_batch(name, root, ix, R.encode(vs, ns, d))
            try:
                got = R.verify_batch(root, ix, vs, ns, d, h)
            except R.Panic:
                panics += 1
                assert want == 0                  # the oracle returns false where the crate panics
                continue
            assert int(got) == want, (ix, d)
        if idx:
            assert R.verify_batch(root, idx, values, pn, depth, h)
    assert panics > 0


def test_verify_batch_restatement_panics():
    h = lambda m: bytes(32)
    with pytest.raises(R.Panic, match="invalid index 8"):
        R.verify_batch(bytes(32), [1, 8, 3, 3], [], [], 3, h)
    with pytest.raises(R.Panic, match="repeating indexes detected"):
        R.verify_batch(bytes(32), [1, 3, 3], [], [], 3, h)
    with pytest.raises(R.Panic, match="unwrap"):
        R.verify_batch(bytes(32), [], [], [], 3, h)          # no index: no root
    with pytest.raises(R.Panic, match="unwrap"):
        R.verify_batch(bytes(32), [0], [bytes(32)], [[bytes(32)]], 0, h)
    with pytest.raises(R.Panic, match="overflow"):
        R.verify_batch(bytes(32), [0], [bytes(32)], [[bytes(32)]], 64, h)
    assert R.verify_batch(bytes(32), [], [], [[]], 3, h) is False      # nodes.len() != indexes.len() comes before the unwrap


LEAVES8 = [bytes([(37 * i + 11 * j + 5) % 256 for j in range(32)]) for i in range(8)]


def test_the_crates_cases(po):
    """merkle.rs:427-518 (the cases tests/test_oracle_crypto.py pins on the oracle) through the restatements"""
    h = R.oracle_hash(po, "poseidon")
    L = LEAVES8
    hh = lambda a, b: h(a + b)
    nodes = R.heap(h, L)
    assert R.prove_batch(L, nodes, [1]) == ([L[1]], [[L[0], hh(L[2], L[3]), hh(hh(L[4], L[5]), hh(L[6], L[7]))]], 3)
    assert R.prove_batch(L, nodes, [1, 2]) == ([L[1], L[2]], [[L[0], hh(hh(L[4], L[5]), hh(L[6], L[7]))], [L[3]]], 3)
    assert R.prove_batch(L, nodes, [1, 6]) == ([L[1], L[6]], [[L[0], hh(L[2], L[3])], [L[7], hh(L[4], L[5])]], 3)
    assert R.prove_batch(L, nodes, list(range(8))) == (L, [[], [], [], []], 3)
    root = nodes[1]
    p = R.prove_batch(L, nodes, [1])
    assert R.verify_batch(root, [1], *p, h) and not R.verify_batch(root, [2], *p, h)
    p = R.prove_batch(L, nodes, [1, 2])
    assert R.verify_batch(root, [1, 2], *p, h)
    for idx in ([1], [1, 3], [1, 2, 3]):
        assert not R.verify_batch(root, idx, *p, h)
    for idx in ([1, 6], [1, 3, 6], list(range(8))):
        assert R.verify_batch(root, idx, *R.prove_batch(L, nodes, idx), h)
