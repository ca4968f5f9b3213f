"""-m gpu: utils::hasher::digest on the GPU (hash64 / merkle_build with "hasher"), against the oracle's digest and the GPU VM's RESCR, and
membership proofs of HasherTree leaves through the smpath and pmpath programs."""
import ctypes
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

M = 2**128 - 45 * 2**40 + 1
WIDE_MIN = 1 << 16               # levels of at least this many digests run the wide layout (HASHER_WIDE_MIN)


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


def oracle_digest(po, values):
    out = ctypes.create_string_buffer(32)
    po.lib().or_hasher_digest(le(values), len(values), out)
    return out.raw


def random_elements(n, seed):
    rng = random.Random(seed)
    return [rng.randrange(M) for _ in range(n)]


def test_hash64_matches_the_oracle(dg, po):
    n = 300                                              # not a multiple of any block size
    msgs = [random_elements(4, 1000 + i) for i in range(n)]
    msgs[0] = [0, 0, 0, 0]
    msgs[1] = [M - 1] * 4
    for k in (1, 2, 3):                                  # 1-3 elements: the zero-padded message is the short input
        msgs[1 + k] = msgs[1 + k][:k] + [0] * (4 - k)
    got = dg.hash64(le([v for m in msgs for v in m]), "hasher")
    assert len(got) == 32 * n
    for i, m in enumerate(msgs):
        assert got[32 * i:32 * i + 32] == oracle_digest(po, m), i
    for k in (1, 2, 3):
        assert got[32 * (1 + k):32 * (2 + k)] == oracle_digest(po, msgs[1 + k][:k]), k
    assert dg.hash64(b"", "hasher") == b""


def test_hash64_wide_layout_matches_the_oracle(dg, po):
    n = WIDE_MIN + 3
    raw = np.random.default_rng(5).integers(0, 2**63, size=(n, 4, 2), dtype=np.uint64).tobytes()    # below M
    got = dg.hash64(raw, "hasher")
    for i in list(range(8)) + list(range(n - 8, n)) + random.Random(6).sample(range(n), 48):
        assert got[32 * i:32 * i + 32] == oracle_digest(po, ints(raw[64 * i:64 * i + 64])), i


def test_rescr_of_the_gpu_vm_is_the_hasher(dg):
    """the relation of the reference's hash_operations test (tests/mod.rs:212-269), run by the GPU VM and proven"""
    d = dg.hash64(le([1, 2, 3, 4]), "hasher")
    once = ints(d)[::-1]
    twice = ints(dg.hash64(d + le([0, 0]), "hasher"))[::-1]
    stacked = ints(dg.hash64(le([0, 0] + ints(d)), "hasher"))[::-1]        # hash.4 of [d1, d0, 0, 0] on the stack
    cases = [("begin hash.4 end", [4, 3, 2, 1], once), ("begin hash.4 hash.2 end", [4, 3, 2, 1], twice),
             ("begin hash.4 hash.4 end", [4, 3, 2, 1, 0, 0], stacked)]
    items = []
    for src, pub, want in cases:
        (outputs, proof), = dg.execute_batch(src, [dg.ProgramInputs(pub)], num_outputs=2)
        assert outputs == want, src
        items.append((dg.api.hostvm.compile_program(src).hash, pub, outputs, proof))
    assert dg.verify_batch(items) == [None] * len(items)


def heap_of(po, leaves):
    L = len(leaves)
    nodes = [b"\0" * 32] * L
    level = [le(p) for p in leaves]
    m = L // 2
    while m >= 1:
        for i in range(m):
            nodes[m + i] = oracle_digest(po, ints(level[2 * i] + level[2 * i + 1]))
        level = nodes[m:2 * m]
        m //= 2
    nodes[0] = b"\0" * 32
    return b"".join(nodes)


def random_leaves(L, seed):
    v = random_elements(2 * L, seed)
    return [(v[2 * i], v[2 * i + 1]) for i in range(L)]


@pytest.mark.parametrize("log_l", [1, 2, 3, 6, 10])
def test_merkle_build_matches_the_oracle_heap(dg, po, log_l):
    leaves = random_leaves(1 << log_l, 300 + log_l)
    assert dg.merkle_build(le([v for p in leaves for v in p]), "hasher") == heap_of(po, leaves)


def test_wide_tree_nodes_are_digests_of_their_children(dg, po):
    """a tree whose lower levels run the wide layout and upper levels the narrow one: sampled nodes of every level"""
    L = 4 * WIDE_MIN
    raw = np.random.default_rng(9).integers(0, 2**63, size=(L, 2, 2), dtype=np.uint64).tobytes()
    nodes = dg.merkle_build(raw, "hasher")
    assert nodes[:32] == b"\0" * 32
    full = nodes + raw                                    # node k's children are 2k, 2k + 1 of nodes ++ leaves
    rng = random.Random(10)
    m = L // 2
    while m >= 1:
        for k in ({m, 2 * m - 1} | set(rng.sample(range(m, 2 * m), min(m, 62)))):
            assert nodes[32 * k:32 * k + 32] == oracle_digest(po, ints(full[64 * k:64 * k + 64])), (m, k)
        m //= 2


def test_non_canonical_inputs_and_bad_sizes_are_rejected(dg):
    from distaff_b200 import backend
    msgs = [1, 2, 3, 4] * 3
    msgs[6] = M
    with pytest.raises(backend.DgError, match="message 1 element 2 is not a field element") as e:
        dg.hash64(le(msgs), "hasher")
    assert e.value.code == -1
    leaves = [5] * 8
    leaves[5] = 2**128 - 1
    with pytest.raises(backend.DgError, match="leaf 2 element 1 is not a field element"):
        dg.merkle_build(le(leaves), "hasher")
    for L in (1, 3):
        with pytest.raises(backend.DgError, match="power of 2"):
            dg.merkle_build(le([1, 2] * L), "hasher")
    out = ctypes.create_string_buffer(32)
    assert backend.lib().dg_hash64(4, le([1, 2, 3, 4]), 1, out) == -1
    assert backend.lib().dg_merkle_build_with(4, le([1, 2, 3, 4]), 2, ctypes.create_string_buffer(64)) == -1


@pytest.fixture(scope="module")
def tree64(dg):
    return dg.HasherTree(random_leaves(64, 77))


def test_tree_heap_is_the_oracle_heap(dg, po, tree64):
    assert b"".join(le(p) for p in tree64.nodes) == heap_of(po, tree64.leaves)
    assert tree64.depth == 7 and tree64.root == ints(heap_of(po, tree64.leaves)[32:64])


@pytest.mark.parametrize("program", ["smpath", "pmpath"])
def test_every_leaf_proves_membership(dg, po, tree64, program):
    from distaff_b200 import backend, hostvm
    L = len(tree64.leaves)
    results = dg.prove_membership(tree64, range(L), program)
    assert all(not isinstance(r, backend.DgError) for r in results)
    want = tree64.root[::-1]
    assert all(r[2] == want for r in results)
    assert dg.verify_batch(results) == [None] * L
    for i in (0, 37, L - 1):
        h, pub, outputs, proof = results[i]
        assert po.verify(h, pub, outputs, proof.bytes) is None
        x = tree64.smpath_inputs(i) if program == "smpath" else tree64.pmpath_inputs(i)
        source = dg.smpath_program(tree64.depth) if program == "smpath" else dg.pmpath_program(tree64.depth)
        host_outputs, host_proof = dg.execute(source, x.public, x.secret_a, x.secret_b, num_outputs=2)
        assert host_outputs == outputs and host_proof.bytes == proof.bytes
        assert hostvm.compile_program(source).hash == h

    # a leaf with one changed element does not output the root, and a proof claiming the root for it is rejected
    forged = dg.HasherTree(list(tree64.leaves), nodes=tree64.nodes)
    forged.leaves[5] = (forged.leaves[5][0], (forged.leaves[5][1] + 1) % M)
    bad, = dg.prove_membership(forged, [5], program)
    assert isinstance(bad, backend.DgError) and "not the root" in str(bad)
    x = forged.smpath_inputs(5) if program == "smpath" else forged.pmpath_inputs(5)
    source = dg.smpath_program(7) if program == "smpath" else dg.pmpath_program(7)
    (outputs, proof), = dg.execute_batch(source, [x], num_outputs=2)
    assert outputs != want
    h = hostvm.compile_program(source).hash
    verdict, = dg.verify_batch([(h, x.public, want, proof)])
    assert verdict is not None and verdict == po.verify(h, x.public, want, proof.bytes)


def test_example_program_on_the_tree_tapes(dg, tree64):
    """hostvm.merkle_program(n, i) (examples/merkle.rs:41-57) with the tree's tapes outputs the doubled, reversed root"""
    from distaff_b200 import hostvm
    want = tree64.root[::-1] * 2
    for i in (0, 21, 63):
        a, b = tree64.tapes(i)
        assert hostvm.execute(hostvm.merkle_program(7, i), secret_a=a, secret_b=b, num_outputs=4).outputs == want
        (outputs, _), = dg.execute_batch(hostvm.merkle_program(7, i), [dg.ProgramInputs([], a, b)], num_outputs=4)
        assert outputs == want


def test_leaves_of_a_2_20_leaf_tree(dg):
    L = 1 << 20
    raw = np.random.default_rng(21).integers(0, 2**63, size=(L, 2, 2), dtype=np.uint64)
    leaves = [(int(a[0][0]) | int(a[0][1]) << 64, int(a[1][0]) | int(a[1][1]) << 64) for a in raw]
    tree = dg.HasherTree(leaves)
    assert tree.depth == 21
    indexes = random.Random(22).sample(range(L), 64)
    results = dg.prove_membership(tree, indexes, "smpath", options=dg.ProofOptions())
    assert all(r[2] == tree.root[::-1] for r in results), [r for r in results if not isinstance(r, tuple)][:1]
    assert dg.verify_batch(results[:8]) == [None] * 8
