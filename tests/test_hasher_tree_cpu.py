"""Merkle trees of the VM's hasher without a GPU: paths and tapes of HasherTree on heaps folded with the oracle's hasher::digest, run
through the host VM with the smpath, pmpath and examples/merkle.rs programs, and the argument checks that run before the device is
touched."""
import ctypes
import random

import pytest

import distaff_b200 as dg
from distaff_b200 import hostvm

M = 2**128 - 45 * 2**40 + 1


def oracle_digest(po, values):
    """utils::hasher::digest of 1-4 field elements, by the oracle"""
    out = ctypes.create_string_buffer(32)
    po.lib().or_hasher_digest(b"".join(int(v).to_bytes(16, "little") for v in values), len(values), out)
    return (int.from_bytes(out.raw[:16], "little"), int.from_bytes(out.raw[16:], "little"))


def oracle_heap(po, leaves):
    """nodes[L/2 + i] = digest(leaf[2i] | leaf[2i+1]), nodes[i] = digest(nodes[2i] | nodes[2i+1]), nodes[0] = 0"""
    L = len(leaves)
    nodes = [(0, 0)] * L
    level = leaves
    m = L // 2
    while m >= 1:
        for i in range(m):
            nodes[m + i] = oracle_digest(po, list(level[2 * i]) + list(level[2 * i + 1]))
        level = nodes[m:2 * m]
        m //= 2
    nodes[0] = (0, 0)
    return nodes


def random_leaves(L, seed):
    rng = random.Random(seed)
    return [(rng.randrange(M), rng.randrange(M)) for _ in range(L)]


@pytest.fixture(scope="module", params=[3, 4], ids=["L8", "L16"])
def tree(request, po):
    leaves = random_leaves(1 << request.param, 50 + request.param)
    return dg.HasherTree(leaves, nodes=oracle_heap(po, leaves))


def test_paths_fold_to_the_root(tree, po):
    """compute_merkle_root of examples/merkle.rs:112-146 over every path gives the root"""
    L = len(tree.leaves)
    assert tree.depth == L.bit_length()
    for i in range(L):
        path = tree.path(i)
        assert len(path) == tree.depth and path[0] == tree.leaves[i] and path[1] == tree.leaves[i ^ 1]
        r = i & 1
        v = oracle_digest(po, list(path[r]) + list(path[1 - r]))
        index = (i + L) >> 1
        for node in path[2:]:
            v = oracle_digest(po, list(v) + list(node) if index & 1 == 0 else list(node) + list(v))
            index >>= 1
        assert list(v) == tree.root


def test_tapes_follow_generate_program_inputs(tree):
    """merkle.rs:63-94 restated literally on the path"""
    for i in (0, 1, len(tree.leaves) - 1):
        path = tree.path(i)
        n = len(path)
        a, b, index = [path[0][0]], [path[0][1]], i + 2 ** (n - 1)
        for k in range(1, n):
            a += [0, path[k][0]]
            b += [index & 1, path[k][1]]
            index >>= 1
        a += [p[0] for p in path[1:]]
        b += [p[1] for p in path[1:]]
        assert tree.tapes(i) == (a, b)


def test_sources_are_pinned():
    assert dg.smpath_program(5) == "begin read.ab smpath.5 end"
    assert dg.pmpath_program(21) == "begin read.ab pmpath.21 end"


def test_every_leaf_outputs_the_root_on_the_host_vm(tree):
    n, want = tree.depth, tree.root[::-1]
    sm, pm = dg.smpath_program(n), dg.pmpath_program(n)
    for i in range(len(tree.leaves)):
        x = tree.smpath_inputs(i)
        assert x.public == []
        assert hostvm.execute(sm, x.public, x.secret_a, x.secret_b, num_outputs=2).outputs == want, ("smpath", i)
        x = tree.pmpath_inputs(i)
        assert x.public == [i]
        assert hostvm.execute(pm, x.public, x.secret_a, x.secret_b, num_outputs=2).outputs == want, ("pmpath", i)
        a, b = tree.tapes(i)
        assert hostvm.execute(hostvm.merkle_program(n, i), secret_a=a, secret_b=b, num_outputs=4).outputs == want + want, ("example", i)


def test_a_changed_leaf_does_not_output_the_root(tree):
    n = tree.depth
    x = tree.smpath_inputs(3)
    x.secret_a[0] = (x.secret_a[0] + 1) % M
    assert hostvm.execute(dg.smpath_program(n), x.public, x.secret_a, x.secret_b, num_outputs=2).outputs != tree.root[::-1]
    x = tree.pmpath_inputs(2)                        # a public index that is not the leaf's folds the path in the wrong order
    x.public = [3]
    assert hostvm.execute(dg.pmpath_program(n), x.public, x.secret_a, x.secret_b, num_outputs=2).outputs != tree.root[::-1]


def test_argument_checks_before_the_device():
    leaves = random_leaves(4, 1)
    for bad in ([], leaves[:1], leaves[:3], leaves + leaves[:2]):
        with pytest.raises(ValueError):
            dg.HasherTree(bad, nodes=[(0, 0)] * len(bad))
    with pytest.raises(ValueError):
        dg.HasherTree(leaves, nodes=[(0, 0)] * 2)
    t = dg.HasherTree(leaves, nodes=[(0, 0)] * 4)
    for i in (-1, 4):
        with pytest.raises(IndexError):
            t.path(i)
        with pytest.raises(IndexError):
            t.smpath_inputs(i)
        with pytest.raises(IndexError):
            dg.prove_membership(t, [0, i])
    with pytest.raises(ValueError):
        dg.prove_membership(t, [0], program="mpath")
    for n in (1, 257):
        with pytest.raises(ValueError):
            dg.smpath_program(n)
        with pytest.raises(ValueError):
            dg.pmpath_program(n)
    assert dg.api.HASH_IDS["hasher"] == 3
