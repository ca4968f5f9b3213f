// Merkle trees that stay on the GPU (tree.cu, the dg_tree_* entry points of capi.cu): the leaves and the heap of alg_merkle_build kept in
// device memory, authentication paths of many leaves gathered in one launch, and leaf updates that rehash only the nodes on their paths.
#pragma once
#include "common.cuh"
#include "host_fs.h"
#include "proof.h"

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
// dg_tree_membership_inputs: the smpath (pmpath false) or pmpath values of leaf indexes[k] at values + k per, per = 4 d + 2 or 2 d + 3 for
// L = 2^d, in one gather launch from the heap; indexes are < L
void tree_membership_inputs(Context &c, const Tree &t, bool pmpath, const uint64_t *indexes, uint32_t count, fe *values);
// the leaf at the plan's leaves[k] becomes leaves32[source[k]]; rehashes the plan's nodes (or the whole tree, tree_update_rebuilds) and
// reads the root
void tree_update(Context &c, Tree &t, const TreePlan &plan, const uint8_t *leaves32);

// ---- batch proofs and path verification (dg_tree_prove_batch, dg_merkle_verify_paths, dg_merkle_verify_batch) ----------------------------
// bytes of the BatchMerkleProof encoding of a prove_batch plan
size_t batch_proof_len(const fs::BatchPlan &plan);
// MerkleTree::prove_batch (merkle.rs:64-124) of the plan's indexes (< L, unique): out receives batch_proof_len(plan) bytes.  One gather
// launch and one copy when the proof holds any digest; the empty proof touches no device.
void tree_prove_batch(Context &c, const Tree &t, const fs::BatchPlan &plan, uint8_t *out);

// MerkleTree::verify (merkle.rs:127-151) of count paths of `entries` entries each: accepted[k] = 1 when path k leads to
// roots32[per_path_root ? k : 0].  One pass per level (a message launch and one alg_hash64 launch), in groups within the memory budget.
void merkle_verify_paths(Context &c, int hash, const uint8_t *roots32, bool per_path_root, const uint64_t *indexes, const uint8_t *paths32,
                         unsigned entries, uint32_t count, uint8_t *accepted);

// MerkleTree::verify_batch (merkle.rs:154-263) as a hashing plan over a pool of 32-byte digests: the caller lays out the proof's values and
// nodes; computed parents get fresh slots from next_slot, in op order.  ok: the ops compute the root into root_slot.  Otherwise `why` says
// where verify_batch returns false, or, with `panic`, gives the reference's panic message.  dg_verify plans depths 1..40 and treats every
// failure as a rejection; the standalone calls plan depths 0..63.
struct MerklePlan {
    std::vector<uint32_t> ops;            // (left, right, out) pool indices
    std::vector<uint32_t> level_start;    // op index where each level starts (+ final end)
    uint32_t root_slot = 0;
    bool ok = false, panic = false;
    std::string why;
};
MerklePlan plan_verify_batch(const std::vector<uint64_t> &indexes_in, int depth, size_t n_values, uint32_t values_base,
                             const std::vector<std::vector<Digest>> &nodes, const std::vector<uint32_t> &nodes_base, uint32_t &next_slot,
                             int min_depth = 1, int max_depth = 40);

// One batch proof of dg_merkle_verify_batch with a plan that is ok, made with values at slots [0, n_values), the nodes of slot i after
// the values and the earlier slots' nodes, computed parents after them.
struct BatchCheck {
    const BatchMerkleProof *proof;
    MerklePlan plan;
};
// accepted[i] = 1 when check i computes its root equal to roots32 + 32 i.  Every group of checks runs level by level with the checks
// aligned at their roots: one gather and one alg_hash64 launch per level, the level's outputs of all checks one run of the pool.
void merkle_verify_batch(Context &c, int hash, const std::vector<BatchCheck> &checks, const uint8_t *const *roots32, uint8_t *accepted);

}  // namespace dg
