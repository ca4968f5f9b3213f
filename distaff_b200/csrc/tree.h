// Merkle trees that stay on the GPU (tree.cu, the dg_tree_* entry points of capi.cu): the leaves and the heap of alg_merkle_build kept in
// device memory, authentication paths of many leaves gathered in one launch, and leaf updates that rehash only the nodes on their paths.
#pragma once
#include "common.cuh"

namespace dg {

struct Tree {
    int hash = 0;                       // DG_HASH_* id of alg_hash64
    unsigned long long L = 0;           // leaves, a power of 2 >= 2
    DevBuf leaves, nodes;               // L x 32 bytes each, from the context's stream-ordered pool; nodes in the heap layout
    uint8_t root[32] = {};              // host copy of nodes[1], refreshed by every build and update
};

// The nodes an update of some leaves rehashes, level by level from the leaves' parents in [L/2, L) up to the root, node 1.
struct TreePlan {
    std::vector<uint64_t> leaves;       // the changed leaves, sorted and unique
    std::vector<uint32_t> source;       // per changed leaf, the position of its last occurrence in the call: the leaf it becomes
    std::vector<uint32_t> level_size;   // per level 1 .. d (L = 2^d), the number of its changed nodes
    std::vector<uint64_t> ids;          // the changed nodes, sorted within each level, level after level
    std::vector<uint32_t> first;        // per changed node, the position in the level below of its first changed child
};
// An update whose plan hashes at least half of the L - 1 nodes scatters the new leaves and builds the whole tree again instead: on an H100
// the level-by-level update of the VM's hash lost to a rebuild at 59 % of the nodes and won at 26 % (DESIGN.md section 7k).
inline bool tree_update_rebuilds(size_t digests, unsigned long long L) { return 2 * digests >= L - 1; }
// indexes are < L (checked by the caller)
TreePlan plan_tree_update(const uint64_t *indexes, uint32_t count, unsigned long long L);

// builds the heap of t.leaves into t.nodes and reads the root
void tree_build(Context &c, Tree &t);
// paths32[k (d + 1) + e], entry e of the authentication path of leaf indexes[k] (MerkleTree::prove order); indexes are < L
void tree_paths(Context &c, const Tree &t, const uint64_t *indexes, uint32_t count, uint8_t *paths32);
// the leaf at the plan's leaves[k] becomes leaves32[source[k]]; rehashes the plan's nodes (or the whole tree, tree_update_rebuilds) and
// reads the root
void tree_update(Context &c, Tree &t, const TreePlan &plan, const uint8_t *leaves32);

}  // namespace dg
