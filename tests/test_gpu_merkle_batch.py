"""-m gpu: batch Merkle proofs of device trees (MerkleTree.prove_batch, dg_tree_prove_batch) against the oracle's prove_batch and the
restatement of merkle.rs:64-124, and path / batch-proof verification (merkle_verify_paths, merkle_verify_batch) against the restatements
of merkle.rs:127-263 and the oracle: accepted proofs, every single mutation, the crate's panics, malformed bytes, non-canonical elements,
mixed calls, depths the STARK verifier never plans, and calls split into memory groups."""
import random

import numpy as np
import pytest

from tests import merkle_batch_refs as R

pytestmark = pytest.mark.gpu

M = 2**128 - 45 * 2**40 + 1
HASHES = ["blake3", "rescue", "poseidon", "hasher"]


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    assert backend.device_info()["sm_count"] > 0
    return distaff_b200


def random_leaves(L, seed):
    """L x 32 bytes of canonical field elements (each below 2^127 < M), so that every hash takes them"""
    return np.random.default_rng(seed).integers(0, 2**63, size=(L, 2, 2), dtype=np.uint64).tobytes()


def split(raw):
    return [raw[32 * i:32 * i + 32] for i in range(len(raw) // 32)]


def flip(d, k=0):
    return d[:k] + bytes([d[k] ^ 0x40]) + d[k + 1:]


def index_sets(L, rng):
    sets = [[L // 2 + 1 if L > 2 else 1], [L - 2, L - 1], list(range(1, L, 2)), list(range(0, L, 2)), []]
    if L <= 1 << 10:
        sets.append(list(range(L)))
    for size in (1, 3, 50, 1000):
        s = rng.sample(range(L), min(L, size))
        rng.shuffle(s)
        sets.append(s)
    return sets


def err_of(x):
    from distaff_b200 import backend
    assert isinstance(x, backend.DgError), x
    return x


# ---- prove_batch -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hash", HASHES)
@pytest.mark.parametrize("log_l", [1, 2, 3, 10, 14, 20])
def test_prove_batch(dg, po, hash, log_l):
    if log_l == 20 and hash in ("rescue", "poseidon"):
        pytest.skip("2^20 leaves: blake3 and the hasher")
    L = 1 << log_l
    leaves = random_leaves(L, 100 * log_l + HASHES.index(hash))
    rng = random.Random(log_l)
    with dg.MerkleTree(leaves, hash) as tree:
        nodes = tree.nodes()
        oracle = hash == "blake3" or (hash != "hasher" and log_l <= 10)
        if hash in ("rescue", "poseidon") and not oracle:
            assert nodes == po.merkle_nodes(hash, leaves)         # the heap the restatement runs over, checked once
        lv, nv = split(leaves), split(nodes)
        for idx in index_sets(L, rng):
            p = tree.prove_batch(idx)
            assert p.depth == log_l and len(p.values) == len(idx)
            if oracle:
                assert p.to_bytes() == po.merkle_prove_batch(hash, leaves, idx), idx[:8]
            else:
                assert p.to_bytes() == R.encode(*R.prove_batch(lv, nv, idx)), idx[:8]
            assert p.values == [lv[i] for i in idx]                # request order
        # after an update the proof opens the new leaves
        changed = rng.sample(range(L), min(L, 5))
        new = random_leaves(len(changed), 7)
        tree.update(changed, new)
        lv2 = list(lv)
        for k, i in enumerate(changed):
            lv2[i] = new[32 * k:32 * k + 32]
        idx = changed + [i ^ 1 for i in changed if i ^ 1 not in changed]
        idx = list(dict.fromkeys(idx))
        p = tree.prove_batch(idx)
        assert p.to_bytes() == R.encode(*R.prove_batch(lv2, split(tree.nodes()), idx))
        if oracle and log_l <= 10:
            assert p.to_bytes() == po.merkle_prove_batch(hash, b"".join(lv2), idx)


@pytest.mark.parametrize("hash", HASHES)
def test_prove_batch_rejections_leave_the_tree(dg, hash):
    from distaff_b200 import backend
    L = 16
    with dg.MerkleTree(random_leaves(L, 5), hash) as tree:
        root, nodes = tree.root, tree.nodes()
        for idx, msg in (([3, L], f"invalid index {L}"), ([L + 1, 2], f"invalid index {L + 1}"), ([4, 2, 4], "repeating indexes detected"),
                         ([L, 5, 5], "repeating indexes detected"), ([L + 7, 5, 5], f"invalid index {L + 7}")):
            with pytest.raises(backend.DgError) as e:
                tree.prove_batch(idx)
            assert e.value.code == -1 and msg in str(e.value), (idx, str(e.value))
        assert tree.root == root and tree.nodes() == nodes
        empty = tree.prove_batch([])
        assert empty.values == [] and empty.nodes == [] and empty.depth == 4


# ---- verify_paths ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hash", HASHES)
def test_verify_paths(dg, po, hash):
    L, e = 1 << 10, 11
    h = R.oracle_hash(po, hash)
    leaves = random_leaves(L, 40 + HASHES.index(hash))
    with dg.MerkleTree(leaves, hash) as tree:
        root = tree.root
        paths = tree.paths(range(L))
        assert dg.merkle_verify_paths(root, range(L), paths, hash) == [True] * L
        arr = np.frombuffer(b"".join(b"".join(p) for p in paths), dtype=np.uint8).reshape(L, e, 32)
        assert dg.merkle_verify_paths(root, range(L), arr, hash) == [True] * L
        assert dg.merkle_verify_paths(flip(root, 31), range(L), arr, hash) == [False] * L
        # one byte flipped at every entry position of a sample of paths: all rejected
        sample = [0, 1, 2, 3, 512, 777, L - 1]
        flipped, fidx = [], []
        for i in sample:
            for k in range(e):
                q = list(paths[i])
                q[k] = flip(q[k], 3)                            # a low byte: the element stays canonical
                flipped.append(q)
                fidx.append(i)
        assert dg.merkle_verify_paths(root, fidx, flipped, hash) == [False] * len(flipped)
        # indexes >= L: the low d bits are read, as the restatement reads them
        for i in (5, 6, 1000):
            big = [i + L, i + 3 * L, i + 2**40, (i ^ 1) + L, (i ^ 4) + 7 * L]
            got = dg.merkle_verify_paths(root, big, [paths[i]] * len(big), hash)
            assert got == [True, True, True, False, False]
            if hash != "hasher" or i == 5:
                assert got == [R.verify(root, b, paths[i], h) for b in big]
        for i in (0, 777):
            assert dg.MerkleTree.verify(root, i, paths[i], hash) and not dg.MerkleTree.verify(root, i ^ 1, paths[i], hash)


def test_verify_paths_per_path_roots(dg):
    trees = [dg.MerkleTree(random_leaves(1 << 6, s), "poseidon") for s in range(4)]
    roots = [t.root for t in trees]
    idx = [(7 * s + 3) % 64 for s in range(4)]
    paths = [t.paths([i])[0] for t, i in zip(trees, idx)]
    assert dg.merkle_verify_paths(roots, idx, paths, "poseidon") == [True] * 4
    assert dg.merkle_verify_paths(roots[::-1], idx, paths, "poseidon") == [False] * 4
    assert dg.merkle_verify_paths(roots[1], idx, paths, "poseidon") == [False, True, False, False]
    for t in trees:
        t.close()


@pytest.mark.parametrize("hash", ["rescue", "poseidon", "hasher"])
def test_verify_paths_names_noncanonical_elements(dg, hash):
    with dg.MerkleTree(random_leaves(8, 3), hash) as tree:
        paths = tree.paths(range(8))
        bad = list(paths[2])
        bad[3] = bad[3][:16] + M.to_bytes(16, "little")
        got = dg.merkle_verify_paths(tree.root, range(9), paths + [bad], hash)
        assert got[:8] == [True] * 8
        e = err_of(got[8])
        assert e.code == -1 and "entry 3 element 1 is not a field element" in str(e)
        assert dg.merkle_verify_paths(tree.root, [2], [bad], "blake3") == [False]      # blake3 takes any bytes


def test_verify_paths_of_a_large_hasher_tree(dg, po):
    L, K = 1 << 20, 1 << 16
    h = R.oracle_hash(po, "hasher")
    rng = np.random.default_rng(9)
    with dg.MerkleTree(random_leaves(L, 8), "hasher") as tree:
        root = tree.root
        idx = rng.choice(L, size=K, replace=False)
        paths = tree.paths(idx)
        arr = np.frombuffer(b"".join(b"".join(p) for p in paths), dtype=np.uint8).reshape(K, 21, 32).copy()
        assert dg.merkle_verify_paths(root, idx, arr, "hasher") == [True] * K
        sample = rng.choice(K, size=256, replace=False)
        for j, k in enumerate(sample):
            arr[k, j % 21, j % 8] ^= 1                           # a low byte: the element stays canonical
        got = dg.merkle_verify_paths(root, idx, arr, "hasher")
        assert [got[k] for k in sample] == [False] * len(sample) and sum(got) == K - len(sample)
        for k in sample[:4]:                                     # host hasher digests are slow: a few through the restatement
            assert R.verify(root, int(idx[k]), [bytes(x) for x in arr[k]], h) is False


# ---- verify_batch ---------------------------------------------------------------------------------------------------------------------
def mutated(values, nodes, depth, rng):
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
        out.append((values, [x if t != s else x + [values[0] if values else bytes(32)] for t, x in enumerate(nodes)], depth))
    out += [(values, nodes, depth - 1), (values, nodes, depth + 1), (values[:-1], nodes, depth), (values, nodes[:-1], depth)]
    if len(values) >= 2:
        a, b = rng.sample(range(len(values)), 2)
        vs = list(values)
        vs[a], vs[b] = vs[b], vs[a]
        out.append((vs, nodes, depth))
    return out


def expected(root, idx, vs, ns, d, h):
    try:
        return R.verify_batch(root, idx, vs, ns, d, h)
    except R.Panic as p:
        return p


@pytest.mark.parametrize("hash", HASHES)
def test_verify_batch_mutations(dg, po, hash):
    L = 64 if hash == "hasher" else 256
    h = R.oracle_hash(po, hash)
    rng = random.Random(HASHES.index(hash))
    leaves = random_leaves(L, 60 + HASHES.index(hash))
    with dg.MerkleTree(leaves, hash) as tree:
        root = tree.root
        items, want = [], []
        for idx in ([5], [6, 7], [1, 2, 60, 61, 33], rng.sample(range(L), 9)):
            p = tree.prove_batch(idx)
            if hash != "hasher":
                assert p.to_bytes() == po.merkle_prove_batch(hash, leaves, idx)
            items.append((root, idx, p))
            want.append(True)
            for vs, ns, d in mutated(p.values, p.nodes, p.depth, rng):
                items.append((root, idx, R.encode(vs, ns, d)))
                want.append(expected(root, idx, vs, ns, d, h))
            for ix in (idx[:-1], idx + [L], idx + idx[:1], [i ^ 1 for i in idx], []):
                items.append((root, ix, p))
                want.append(expected(root, ix, p.values, p.nodes, p.depth, h))
        got = dg.merkle_verify_batch(items, hash)
        for (r, ix, _), g, w in zip(items, got, want):
            if isinstance(w, R.Panic):
                assert err_of(g).code == -1 and str(w) in str(g), (ix, str(g))
            else:
                assert g is w, ix
        # the oracle agrees wherever the crate does not panic
        if hash != "hasher":
            for (r, ix, p), w in zip(items, want):
                if not isinstance(w, R.Panic):
                    raw = p.to_bytes() if hasattr(p, "to_bytes") else p
                    assert po.merkle_verify_batch(hash, r, ix, raw) == int(w)
        assert dg.MerkleTree.verify_batch(root, [5], items[0][2], hash) is True


def test_verify_batch_panics_and_malformed_bytes(dg):
    L = 32
    with dg.MerkleTree(random_leaves(L, 1), "blake3") as tree:
        root = tree.root
        p = tree.prove_batch([3, 9])
        raw = p.to_bytes()
        cases = [([3, 9, 40], raw, "invalid index 40"), ([3, 9, 3], raw, "repeating indexes detected"),
                 ([], dg.BatchMerkleProof([], [], 5).to_bytes(), "unwrap"), ([0], R.encode([bytes(32)], [[bytes(32)]], 0), "unwrap"),
                 ([3, 9], R.encode(p.values, p.nodes, 64), "overflow"), ([3, 9], raw[:-1], "malformed"), ([3, 9], raw + b"\0", "malformed"),
                 ([3, 9], b"", "malformed"), ([3, 9], (2**50).to_bytes(8, "little") + raw[8:], "malformed")]
        good = (root, [3, 9], p)
        items = [good] + [(root, ix, b) for ix, b, _ in cases] + [good]
        got = dg.merkle_verify_batch(items)
        assert got[0] is True and got[-1] is True
        for (ix, b, msg), g in zip(cases, got[1:-1]):
            assert err_of(g).code == -1 and msg in str(g), (ix, str(g))
        from distaff_b200 import backend
        with pytest.raises(backend.DgError, match="repeating"):
            dg.MerkleTree.verify_batch(root, [3, 3], p)


@pytest.mark.parametrize("hash", ["rescue", "poseidon", "hasher"])
def test_verify_batch_names_noncanonical_elements(dg, hash):
    with dg.MerkleTree(random_leaves(16, 2), hash) as tree:
        p = tree.prove_batch([1, 6])
        bad_v = dg.BatchMerkleProof(list(p.values), p.nodes, p.depth)
        bad_v.values[1] = M.to_bytes(16, "little") + bad_v.values[1][16:]
        bad_n = dg.BatchMerkleProof(p.values, [list(s) for s in p.nodes], p.depth)
        bad_n.nodes[1][1] = bad_n.nodes[1][1][:16] + (2**128 - 1).to_bytes(16, "little")
        got = dg.merkle_verify_batch([(tree.root, [1, 6], p), (tree.root, [1, 6], bad_v), (tree.root, [1, 6], bad_n)], hash)
        assert got[0] is True
        assert "value 1 element 0 is not a field element" in str(err_of(got[1]))
        assert "node 1 of slot 1 element 1 is not a field element" in str(err_of(got[2]))


def test_verify_batch_deep_proofs(dg, po):
    """depths 41-63, which the STARK verifier's plan never takes: a one-index proof folded on the host with blake3"""
    h = R.oracle_hash(po, "blake3")
    rng = random.Random(3)
    items, want = [], []
    for depth in (41, 50, 63):
        index = rng.randrange(2**depth)
        leaf = bytes(rng.randrange(256) for _ in range(32))
        path = [leaf] + [bytes(rng.randrange(256) for _ in range(32)) for _ in range(depth)]
        v = h(path[0] + path[1]) if index & 1 == 0 else h(path[1] + path[0])
        k = (index + 2**depth) >> 1
        for e in path[2:]:
            v = h(v + e) if k & 1 == 0 else h(e + v)
            k >>= 1
        raw = R.encode([leaf], [path[1:]], depth)
        assert R.verify_batch(v, [index], [leaf], [path[1:]], depth, h)
        assert po.merkle_verify_batch("blake3", v, [index], raw) == 1
        items += [(v, [index], raw), (v, [index ^ 1], raw), (flip(v), [index], raw)]
        want += [True, False, False]
        assert dg.merkle_verify_paths(v, [index], [path], "blake3") == [True]
    assert dg.merkle_verify_batch(items) == want


def test_a_mixed_call(dg):
    """one bad entry changes no other verdict: accepted, rejected, panicking and malformed entries of three trees in one call"""
    trees = [dg.MerkleTree(random_leaves(1 << k, k), "poseidon") for k in (3, 7, 12)]
    items, want = [], []
    for t in trees:
        idx = random.Random(len(t)).sample(range(len(t)), 6)
        p = t.prove_batch(idx)
        items += [(t.root, idx, p), (flip(t.root), idx, p), (t.root, idx + idx[:1], p), (t.root, idx, p.to_bytes()[:-2])]
        want += [True, False, "repeating", "malformed"]
    got = dg.merkle_verify_batch(items, "poseidon")
    for g, w in zip(got, want):
        assert g is w if isinstance(w, bool) else w in str(err_of(g))
    for t in trees:
        t.close()


# ---- memory ---------------------------------------------------------------------------------------------------------------------------
def test_memory_groups_and_held_memory(dg):
    L = 1 << 14
    with dg.MerkleTree(random_leaves(L, 77), "rescue") as tree:
        root = tree.root
        rng = random.Random(5)
        idx = list(range(L))
        paths = tree.paths(idx)
        paths[7] = [flip(paths[7][0])] + paths[7][1:]
        items = []
        for k in range(128):
            ix = rng.sample(range(L), 40)
            items.append((root if k % 5 else flip(root), ix, tree.prove_batch(ix)))
        want_p = dg.merkle_verify_paths(root, idx, paths, "rescue")
        want_b = dg.merkle_verify_batch(items, "rescue")
        assert want_p == [k != 7 for k in range(L)] and want_b == [k % 5 != 0 for k in range(128)]
        held = dg.memory_usage()["held"]
        for _ in range(2):                                       # every buffer goes back to the pool before the call returns
            assert dg.merkle_verify_paths(root, idx, paths, "rescue") == want_p
            assert dg.merkle_verify_batch(items, "rescue") == want_b
            assert dg.memory_usage()["held"] == held
        # the paths take ~ 16384 x 650 bytes and the proofs ~ 128 x 56 KB on the device; 3 MiB above what the library holds once its pool
        # is trimmed splits each call into several groups
        dg.set_memory_limit(1)
        try:
            dg.set_memory_limit(dg.memory_usage()["held"] + (3 << 20))
            assert dg.merkle_verify_paths(root, idx, paths, "rescue") == want_p
            assert dg.merkle_verify_batch(items, "rescue") == want_b
        finally:
            dg.set_memory_limit(0)
