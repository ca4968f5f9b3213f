"""Plain Python restatements of MerkleTree::prove_batch, verify and verify_batch (/root/reference/src/crypto/merkle.rs:64-263),
statement by statement, that raise Panic where the crate panics.  The oracle returns false (or fails) in those places instead, so the
panic cases are pinned here; tests/test_merkle_batch_cpu.py checks these restatements against the oracle on every other case.

A hash is a function of 64 bytes to 32 bytes; `oracle_hash(po, name)` gives the oracle's blake3 / rescue / poseidon, and the VM's hasher
(utils::hasher::digest of four little-endian u128 elements: the oracle's hash id 3 is GMiMC, not this one)."""
import ctypes

U64 = 2**64


class Panic(Exception):
    pass


def oracle_hash(po, name):
    if name != "hasher":
        return lambda m: po.hash(name, m)

    def hasher(m):
        out = ctypes.create_string_buffer(32)
        po.lib().or_hasher_digest(bytes(m), 4, out)
        return out.raw
    return hasher


def heap(h, leaves):
    """build_merkle_nodes (merkle.rs:269-294): the heap of a list of 32-byte leaves, nodes[0] zero"""
    L = len(leaves)
    nodes = [b"\0" * 32] * L
    for i in range(L // 2):
        nodes[L // 2 + i] = h(leaves[2 * i] + leaves[2 * i + 1])
    for i in range(L // 2 - 1, 0, -1):
        nodes[i] = h(nodes[2 * i] + nodes[2 * i + 1])
    return nodes


def map_indexes(indexes, max_valid):
    m = {}
    for i, index in enumerate(indexes):
        m[index] = i
        if index > max_valid:
            raise Panic(f"invalid index {index}")
    if len(indexes) != len(m):
        raise Panic("repeating indexes detected")
    return m


def normalize_indexes(indexes):
    return sorted({i - (i & 1) for i in indexes})


def prove_batch(leaves, nodes, indexes):
    """merkle.rs:64-124 over the leaves and heap (lists of 32-byte bytes): (values, nodes, depth)"""
    n = len(leaves)
    index_map = map_indexes(indexes, n)

    def leaf(i):
        if i >= n:
            raise Panic(f"index out of bounds: the len is {n} but the index is {i}")
        return leaves[i]
    values = [None] * len(index_map)
    out = []
    next_indexes = []
    for index in normalize_indexes(indexes):
        v1, v2 = leaf(index), leaf(index + 1)
        i1, i2 = index_map.get(index), index_map.get(index + 1)
        if i1 is not None:
            values[i1] = v1
            if i2 is not None:
                values[i2] = v2
                out.append([])
            else:
                out.append([v2])
        else:
            values[i2] = v2
            out.append([v1])
        next_indexes.append((index + n) >> 1)
    depth = (n & -n).bit_length() - 1                    # trailing_zeros
    for _ in range(1, depth):
        idx, next_indexes = next_indexes, []
        i = 0
        while i < len(idx):
            sibling = idx[i] ^ 1
            if i + 1 < len(idx) and idx[i + 1] == sibling:
                i += 1
            else:
                out[i].append(nodes[sibling])
            next_indexes.append(sibling >> 1)
            i += 1
    return values, out, depth


def verify(root, index, proof, h):
    """merkle.rs:127-151 (usize arithmetic wraps at 2^64)"""
    r = index & 1
    v = h(proof[r] + proof[1 - r])
    index = ((index + 2 ** (len(proof) - 1)) % U64) >> 1
    for i in range(2, len(proof)):
        v = h(v + proof[i]) if index & 1 == 0 else h(proof[i] + v)
        index >>= 1
    return v == root


def verify_batch(root, indexes, values, nodes, depth, h):
    """merkle.rs:154-263"""
    if depth > 63:
        raise Panic("attempt to multiply with overflow")     # usize::pow(2, depth)
    offset = 2 ** depth
    index_map = map_indexes(indexes, offset - 1)
    norm = normalize_indexes(indexes)
    if len(norm) != len(nodes):
        return False
    v = {}
    next_indexes, pointers = [], []
    for i, index in enumerate(norm):
        i1, i2 = index_map.get(index), index_map.get(index + 1)
        if i1 is not None:
            if len(values) <= i1:
                return False
            left = values[i1]
            if i2 is not None:
                if len(values) <= i2:
                    return False
                right = values[i2]
                pointers.append(0)
            else:
                if len(nodes[i]) < 1:
                    return False
                right = nodes[i][0]
                pointers.append(1)
        else:
            if len(nodes[i]) < 1:
                return False
            left = nodes[i][0]
            if i2 is None:
                return False
            if len(values) <= i2:
                return False
            right = values[i2]
            pointers.append(1)
        parent = (offset + index) >> 1
        v[parent] = h(left + right)
        next_indexes.append(parent)
    for _ in range(1, depth):
        idx, next_indexes = next_indexes, []
        i = 0
        while i < len(idx):
            node_index = idx[i]
            sibling_index = node_index ^ 1
            if i + 1 < len(idx) and idx[i + 1] == sibling_index:
                if sibling_index not in v:
                    return False
                sibling = v[sibling_index]
                i += 1
            else:
                pointer = pointers[i]
                if len(nodes[i]) <= pointer:
                    return False
                sibling = nodes[i][pointer]
                pointers[i] += 1
            if node_index not in v:
                return False
            node = v[node_index]
            parent = h(sibling + node) if node_index & 1 else h(node + sibling)
            v[node_index >> 1] = parent
            next_indexes.append(node_index >> 1)
            i += 1
    if 1 not in v:
        raise Panic("called `Option::unwrap()` on a `None` value")
    return root == v[1]


def encode(values, nodes, depth):
    """the bincode of BatchMerkleProof"""
    u64 = lambda n: n.to_bytes(8, "little")
    return u64(len(values)) + b"".join(values) + u64(len(nodes)) + b"".join(u64(len(s)) + b"".join(s) for s in nodes) + bytes([depth])
