"""-m gpu: Merkle trees kept in device memory (MerkleTree, dg_tree_*): heaps against merkle_build and the oracle, authentication paths
against MerkleTree::prove (merkle.rs:47-62), leaf updates against a rebuild of the changed leaf list, rejections that leave the tree as it
was, membership proofs against HasherTree's, and the memory a live tree holds."""
import ctypes
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

M = 2**128 - 45 * 2**40 + 1
HASHES = ["blake3", "rescue", "poseidon", "hasher"]
ORACLE_NAMES = {"blake3": "blake3", "rescue": "rescue", "poseidon": "poseidon"}     # the oracle's id 3 is gmimc: the hasher is folded here


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    assert backend.device_info()["sm_count"] > 0
    return distaff_b200


def le(values):
    return b"".join(int(v).to_bytes(16, "little") for v in values)


def ints(raw):
    return [int.from_bytes(raw[16 * k:16 * k + 16], "little") for k in range(len(raw) // 16)]


def random_leaves(L, seed):
    """L x 32 bytes of canonical field elements (each below 2^127 < M), so that every hash takes them"""
    return np.random.default_rng(seed).integers(0, 2**63, size=(L, 2, 2), dtype=np.uint64).tobytes()


def hasher_digest(po, values):
    out = ctypes.create_string_buffer(32)
    po.lib().or_hasher_digest(le(values), len(values), out)
    return out.raw


def oracle_heap(po, hash, leaves):
    if hash in ORACLE_NAMES:
        return po.merkle_nodes(ORACLE_NAMES[hash], leaves)
    L = len(leaves) // 32                    # a fold with the oracle's utils::hasher::digest, as test_gpu_hasher_tree.heap_of does
    nodes = [b"\0" * 32] * L
    level = [leaves[32 * i:32 * i + 32] for i in range(L)]
    m = L // 2
    while m >= 1:
        for i in range(m):
            nodes[m + i] = hasher_digest(po, ints(level[2 * i] + level[2 * i + 1]))
        level = nodes[m:2 * m]
        m //= 2
    return b"".join(nodes)


def prove_path(leaves, nodes, i):
    """MerkleTree::prove (merkle.rs:47-62) restated: leaf i, its sibling, then the sibling of every node from i's parent to the root's child"""
    L = len(leaves) // 32
    leaf = lambda k: leaves[32 * k:32 * k + 32]
    path, index = [leaf(i), leaf(i ^ 1)], (i + L) >> 1
    while index > 1:
        path.append(nodes[32 * (index ^ 1):32 * (index ^ 1) + 32])
        index >>= 1
    return path


@pytest.mark.parametrize("hash", HASHES)
@pytest.mark.parametrize("log_l", [1, 2, 10])
def test_build_and_paths_match_the_oracle(dg, po, hash, log_l):
    L = 1 << log_l
    leaves = random_leaves(L, 10 * log_l + HASHES.index(hash))
    want = oracle_heap(po, hash, leaves)
    with dg.MerkleTree(leaves, hash) as tree:
        assert tree.hash == hash and len(tree) == L and tree.depth == log_l + 1
        assert tree.nodes() == want == dg.merkle_build(leaves, hash)
        assert tree.leaves() == leaves and tree.root == want[32:64]
        paths = tree.paths(range(L))
        assert paths == [prove_path(leaves, want, i) for i in range(L)]
        order = [L - 1, 0, L - 1, L // 2, 0]                     # repeated and unsorted
        assert tree.paths(order) == [paths[i] for i in order]
        assert tree.paths([]) == []


def test_hasher_paths_are_hasher_tree_paths(dg):
    pairs = [(random.Random(i).randrange(M), random.Random(-i).randrange(M)) for i in range(64)]
    ht = dg.HasherTree(pairs)
    with dg.MerkleTree(pairs, "hasher") as tree:
        assert tree.depth == ht.depth and list(ints(tree.root)) == ht.root
        for i, p in zip(range(64), tree.paths(range(64))):
            assert [tuple(ints(e)) for e in p] == ht.path(i)


@pytest.mark.parametrize("log_l", [18, 20])
def test_large_trees(dg, log_l):
    """for the hasher at 2^18 the lower levels run the wide layout and the upper ones the narrow one"""
    L = 1 << log_l
    leaves = random_leaves(L, log_l)
    hashes = ["blake3", "hasher"] if log_l == 18 else ["blake3"]
    for hash in hashes:
        nodes = dg.merkle_build(leaves, hash)
        with dg.MerkleTree(leaves, hash) as tree:
            assert tree.nodes() == nodes
            idx = [0, L - 1, 1, L - 2] + random.Random(log_l).sample(range(L), 60)
            assert tree.paths(idx) == [prove_path(leaves, nodes, i) for i in idx]


def test_device_leaves(dg):
    import torch
    L = 1 << 12
    leaves = random_leaves(L, 3)
    t = torch.frombuffer(bytearray(leaves), dtype=torch.uint8).to("cuda")
    for hash in ("blake3", "hasher"):
        with dg.MerkleTree(t, hash) as a, dg.MerkleTree(leaves, hash) as b:
            assert a.nodes() == b.nodes() and a.leaves() == leaves and a.root == b.root
    with pytest.raises(ValueError):
        dg.MerkleTree(t[:100], "blake3")


def check_update(dg, tree, host, indexes, new):
    """applies the change to the host leaf list first, then to the tree; the tree then equals merkle_build of the host list"""
    for k, i in enumerate(indexes):
        host[32 * i:32 * i + 32] = new[32 * k:32 * k + 32]
    root = tree.update(indexes, new)
    nodes = tree.nodes()
    assert tree.leaves() == bytes(host)
    assert nodes == dg.merkle_build(bytes(host), tree.hash)
    assert root == nodes[32:64] == tree.root


def update_cases(L, seed):
    rng = random.Random(seed)
    return [[rng.randrange(L)], [6, 7], [0, L - 1], [5, 9, 5, 5, 9], rng.sample(range(L), 37), [rng.randrange(L) for _ in range(300)],
            list(range(L))[::-1], rng.sample(range(L), L // 2)]


@pytest.mark.parametrize("hash", HASHES)
def test_updates(dg, hash):
    L = 1 << 10
    host = bytearray(random_leaves(L, 40))
    with dg.MerkleTree(bytes(host), hash) as tree:
        for n, idx in enumerate(update_cases(L, 41)):             # one tree through every case in turn: a sequence of updates
            check_update(dg, tree, host, idx, random_leaves(len(idx), 1000 + n))
        assert tree.update([], b"") == tree.root


def test_repeated_index_last_occurrence_wins(dg):
    L = 16
    with dg.MerkleTree(random_leaves(L, 1), "blake3") as tree:
        a, b, c = (bytes([v]) * 32 for v in (1, 2, 3))
        tree.update([4, 4, 4], a + b + c)
        assert tree.leaves()[32 * 4:32 * 5] == c


def test_updates_at_2_18(dg):
    L = 1 << 18
    rng = random.Random(18)
    for hash in ("hasher", "blake3"):
        host = bytearray(random_leaves(L, 180))
        with dg.MerkleTree(bytes(host), hash) as tree:
            for n, idx in enumerate([[L - 1], [0, 1], rng.sample(range(L), 4096), rng.sample(range(L), 1 << 17)]):
                check_update(dg, tree, host, idx, random_leaves(len(idx), 2000 + n))


def test_rejections_leave_the_tree_unchanged(dg):
    from distaff_b200 import backend
    for hash in ("blake3", "hasher"):
        with dg.MerkleTree(random_leaves(64, 5), hash) as tree:
            leaves, nodes = tree.leaves(), tree.nodes()
            with pytest.raises(backend.DgError, match="index 64 .entry 2. is not a leaf") as e:
                tree.update([1, 2, 64, 3], random_leaves(4, 6))
            assert e.value.code == -1
            with pytest.raises(backend.DgError, match="index 99"):
                tree.paths([0, 99])
            assert tree.leaves() == leaves and tree.nodes() == nodes
            if hash == "hasher":
                bad = bytearray(random_leaves(4, 7))
                bad[32 * 2:32 * 2 + 16] = M.to_bytes(16, "little")
                with pytest.raises(backend.DgError, match="leaf 2 element 0 is not a field element") as e:
                    tree.update([1, 2, 3, 4], bytes(bad))
                assert e.value.code == -1
                assert tree.leaves() == leaves and tree.nodes() == nodes
            with pytest.raises(ValueError):
                tree.update([1, 2], random_leaves(3, 8))


def test_build_rejections(dg):
    from distaff_b200 import backend
    for L in (1, 3):
        with pytest.raises(backend.DgError, match="power of 2") as e:
            dg.MerkleTree(random_leaves(L, 1), "blake3")
        assert e.value.code == -1
    handle = backend.vp()
    assert backend.lib().dg_tree_new(4, random_leaves(4, 1), 4, ctypes.byref(handle)) == -1 and handle.value is None
    bad = bytearray(random_leaves(4, 2))
    bad[32 * 3 + 16:32 * 4] = (M + 5).to_bytes(16, "little")
    with pytest.raises(backend.DgError, match="leaf 3 element 1 is not a field element"):
        dg.MerkleTree(bytes(bad), "hasher")


def test_closed_tree(dg):
    tree = dg.MerkleTree(random_leaves(4, 1))
    tree.close()
    tree.close()
    with pytest.raises(ValueError, match="closed"):
        tree.paths([0])


@pytest.mark.parametrize("program", ["smpath", "pmpath"])
def test_membership_after_updates(dg, po, program):
    from distaff_b200 import backend
    rng = random.Random(64)
    pairs = [(rng.randrange(M), rng.randrange(M)) for _ in range(64)]
    changed = [3, 17, 40, 41]
    new_pairs = [(rng.randrange(M), rng.randrange(M)) for _ in changed]
    after = list(pairs)
    for i, p in zip(changed, new_pairs):
        after[i] = p
    with dg.MerkleTree(pairs, "hasher") as tree:
        old = dg.prove_membership(tree, [17], program)[0]
        old_root = ints(tree.root)[::-1]
        tree.update(changed, new_pairs)
        ht = dg.HasherTree(after)
        assert list(ints(tree.root)) == ht.root
        indexes = changed + [0, 16, 63]
        got = dg.prove_membership(tree, indexes, program)
        want = dg.prove_membership(ht, indexes, program)
        assert all(isinstance(r, tuple) for r in got)
        for g, w in zip(got, want):
            assert g[:3] == w[:3] and g[3].bytes == w[3].bytes
        assert dg.verify_batch(got) == [None] * len(got)
        h, pub, _, proof = old                    # a proof made before the update proves the old root, not the new one
        verdicts = dg.verify_batch([(h, pub, old_root, proof), (h, pub, ht.root[::-1], proof)])
        assert verdicts[0] is None and verdicts[1] is not None
    with dg.MerkleTree(random_leaves(8, 1), "blake3") as other:
        with pytest.raises(ValueError, match="hasher"):
            dg.prove_membership(other, [0], program)
    assert not isinstance(got[0], backend.DgError)


def test_a_live_tree_is_held_memory(dg):
    L = 1 << 20
    with dg.MerkleTree(random_leaves(L, 20), "blake3") as tree:
        assert dg.memory_usage()["held"] >= 64 * L
        tree.update([5], random_leaves(1, 21))
        assert dg.memory_usage()["held"] >= 64 * L
