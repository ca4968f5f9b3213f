// Merkle trees that stay on the GPU (tree.h): build once with alg_merkle_build, gather the authentication paths of many leaves in one
// launch, and update leaves by rehashing only the nodes on their paths.  An update runs one pass per level: tree_level_kernel writes the
// level below's new values into their slots and gathers this level's 64-byte messages, then alg_hash64 (for hash 3 hasher_digest, with
// its narrow / wide choice) hashes them.  The digest kernels are the measured ones, unchanged.
#include "tree.h"
#include "poly.h"
#include <algorithm>
#include <map>
#include <set>

namespace dg {

TreePlan plan_tree_update(const uint64_t *indexes, uint32_t count, unsigned long long L) {
    TreePlan p;
    std::vector<std::pair<uint64_t, uint32_t>> order(count);            // (index, position): sorted, a run of equal indexes ends with
    for (uint32_t k = 0; k < count; k++) order[k] = {indexes[k], k};   // its last occurrence
    std::sort(order.begin(), order.end());
    p.leaves.reserve(count);
    p.source.reserve(count);
    for (uint32_t k = 0; k < count; k++) {
        if (k + 1 < count && order[k + 1].first == order[k].first) continue;
        p.leaves.push_back(order[k].first);
        p.source.push_back(order[k].second);
    }
    if (p.leaves.empty()) return p;
    // level 1: the parents (L + i) >> 1 of the leaves; level j + 1: the parents q >> 1 of level j, up to the root
    size_t below = 0, n_below = p.leaves.size();
    for (unsigned long long m = L / 2; m >= 1; m >>= 1) {
        const size_t start = p.ids.size();
        for (size_t k = 0; k < n_below; k++) {
            const uint64_t q = m == L / 2 ? (L + p.leaves[k]) >> 1 : p.ids[below + k] >> 1;
            if (p.ids.size() == start || p.ids.back() != q) { p.ids.push_back(q); p.first.push_back((uint32_t)k); }
        }
        p.level_size.push_back((uint32_t)(p.ids.size() - start));
        below = start;
        n_below = p.ids.size() - start;
    }
    return p;
}

// 32-byte items as two uint4.  Thread t < n_below writes the level below's new item src[t] into slot below_ids[t] of `below`.  Thread
// t < n writes message t of this level, the children of node ids[t]: children 2 ids[t] - base and the next of `below`, each taken from
// src when it changed (it is then at position first[t] or first[t] + 1 of below_ids) and from `below` when it did not.  A slot that is
// written is never read from `below`, so the two parts need no ordering.
__global__ void __launch_bounds__(256) tree_level_kernel(const uint4 *src, const unsigned long long *below_ids, unsigned n_below, uint4 *below,
                                                         const unsigned long long *ids, const unsigned *first, unsigned n,
                                                         unsigned long long base, uint4 *msgs) {
    const unsigned long long t = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n_below) {
        const unsigned long long s = below_ids[t];
        below[2 * s] = src[2 * t];
        below[2 * s + 1] = src[2 * t + 1];
    }
    if (t < n) {
        const unsigned long long c = 2 * ids[t] - base, f = first[t];
        const uint4 *a = below_ids[f] == c ? src + 2 * f : below + 2 * c;
        const uint4 *b = below_ids[f] == c + 1 ? src + 2 * f : f + 1 < n_below && below_ids[f + 1] == c + 1 ? src + 2 * (f + 1) : below + 2 * (c + 1);
        msgs[4 * t] = a[0];
        msgs[4 * t + 1] = a[1];
        msgs[4 * t + 2] = b[0];
        msgs[4 * t + 3] = b[1];
    }
}

// thread k of grid row e: entry e of leaf indexes[k]'s path, at k (d + 1) + e of out: leaf i, leaf i ^ 1, then nodes[((L + i) >> 1 >> j) ^ 1]
// for j = e - 2
__global__ void __launch_bounds__(256) tree_paths_kernel(const uint4 *__restrict__ leaves, const uint4 *__restrict__ nodes,
                                                         const unsigned long long *__restrict__ indexes, unsigned count, unsigned long long L,
                                                         uint4 *__restrict__ out) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x, e = blockIdx.y;
    if (k >= count) return;
    const unsigned long long i = indexes[k], t = (unsigned long long)k * gridDim.y + e;
    const uint4 *s = e == 0 ? leaves + 2 * i : e == 1 ? leaves + 2 * (i ^ 1) : nodes + 2 * ((((L + i) >> 1) >> (e - 2)) ^ 1);
    out[2 * t] = s[0];
    out[2 * t + 1] = s[1];
}

void tree_build(Context &c, Tree &t) {
    alg_merkle_build(c, t.hash, t.leaves.p, t.nodes.p, t.L);
    DG_CUDA(cudaMemcpyAsync(t.root, t.nodes.as<uint8_t>() + 32, 32, cudaMemcpyDeviceToHost, c.stream));
    DG_CUDA(cudaStreamSynchronize(c.stream));
}

void tree_paths(Context &c, const Tree &t, const uint64_t *indexes, uint32_t count, uint8_t *paths32) {
    if (count == 0) return;
    const unsigned entries = (unsigned)ceil_log2(t.L) + 1;
    const unsigned long long total = (unsigned long long)count * entries;
    DevBuf d_idx((size_t)count * 8), d_out(total * 32);
    DG_CUDA(cudaMemcpyAsync(d_idx.p, indexes, (size_t)count * 8, cudaMemcpyHostToDevice, c.stream));
    tree_paths_kernel<<<dim3((count + 255) / 256, entries), 256, 0, c.stream>>>(t.leaves.as<uint4>(), t.nodes.as<uint4>(), d_idx.as<unsigned long long>(),
                                                                                 count, t.L, d_out.as<uint4>());
    c.launches++;
    DG_CUDA(cudaGetLastError());
    DG_CUDA(cudaMemcpyAsync(paths32, d_out.p, total * 32, cudaMemcpyDeviceToHost, c.stream));
    DG_CUDA(cudaStreamSynchronize(c.stream));
}

static void launch_level(Context &c, const void *src, const unsigned long long *below_ids, size_t n_below, void *below,
                         const unsigned long long *ids, const unsigned *first, size_t n, unsigned long long base, void *msgs) {
    tree_level_kernel<<<(unsigned)((n_below + 255) / 256), 256, 0, c.stream>>>((const uint4 *)src, below_ids, (unsigned)n_below, (uint4 *)below,
                                                                                ids, first, (unsigned)n, base, (uint4 *)msgs);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

void tree_update(Context &c, Tree &t, const TreePlan &plan, const uint8_t *leaves32) {
    const size_t K = plan.leaves.size(), T = plan.ids.size();
    if (K == 0) return;
    // one upload: the new leaves in plan order, the leaf indexes, and for a level-by-level update the node ids and first-child positions
    const bool rebuild = tree_update_rebuilds(T, t.L);
    const size_t o_idx = K * 32, o_ids = o_idx + K * 8, o_first = o_ids + T * 8, bytes = rebuild ? o_ids : o_first + T * 4;
    std::vector<uint8_t> h(bytes);
    for (size_t k = 0; k < K; k++) memcpy(h.data() + 32 * k, leaves32 + 32 * (size_t)plan.source[k], 32);
    memcpy(h.data() + o_idx, plan.leaves.data(), K * 8);
    if (!rebuild) {
        memcpy(h.data() + o_ids, plan.ids.data(), T * 8);
        memcpy(h.data() + o_first, plan.first.data(), T * 4);
    }
    DevBuf d_plan(bytes);
    DG_CUDA(cudaMemcpyAsync(d_plan.p, h.data(), bytes, cudaMemcpyHostToDevice, c.stream));
    const uint8_t *P = d_plan.as<uint8_t>();
    if (rebuild) {                                               // the new leaves into the leaf buffer, then the whole heap
        launch_level(c, P, (const unsigned long long *)(P + o_idx), K, t.leaves.p, nullptr, nullptr, 0, 0, nullptr);
        tree_build(c, t);
        return;
    }
    DevBuf d_msg((size_t)plan.level_size[0] * 64), d_dig((size_t)plan.level_size[0] * 32);
    const unsigned long long *ids = (const unsigned long long *)(P + o_ids);
    const unsigned *first = (const unsigned *)(P + o_first);
    // level 1: the new leaves into the leaf buffer, and the messages of their parents
    launch_level(c, P, (const unsigned long long *)(P + o_idx), K, t.leaves.p, ids, first, plan.level_size[0], t.L, d_msg.p);
    alg_hash64(c, t.hash, d_msg.p, d_dig.p, plan.level_size[0]);
    size_t at = 0;
    for (size_t j = 1; j < plan.level_size.size(); j++) {       // level j + 1: the digests of level j into the heap, the messages above
        const size_t n_below = plan.level_size[j - 1], n = plan.level_size[j];
        launch_level(c, d_dig.p, ids + at, n_below, t.nodes.p, ids + at + n_below, first + at + n_below, n, 0, d_msg.p);
        alg_hash64(c, t.hash, d_msg.p, d_dig.p, n);
        at += n_below;
    }
    launch_level(c, d_dig.p, ids + at, 1, t.nodes.p, nullptr, nullptr, 0, 0, nullptr);     // the root into nodes[1]
    DG_CUDA(cudaMemcpyAsync(t.root, d_dig.p, 32, cudaMemcpyDeviceToHost, c.stream));
    DG_CUDA(cudaStreamSynchronize(c.stream));
}

// ---- batch Merkle verification as a hashing plan (merkle.rs:154-263) -------------------------------------------------------------
MerklePlan plan_verify_batch(const std::vector<uint64_t> &indexes_in, int depth, size_t n_values, uint32_t values_base,
                             const std::vector<std::vector<Digest>> &nodes, const std::vector<uint32_t> &nodes_base, uint32_t &next_slot,
                             int min_depth, int max_depth) {
    MerklePlan plan;
    auto reject = [&](const std::string &why) { plan.why = why; return plan; };
    auto panic = [&](const std::string &why) { plan.panic = true; plan.why = why; return plan; };
    if (depth < min_depth || depth > max_depth) return reject("depth " + std::to_string(depth) + " is outside " + std::to_string(min_depth) +
                                                              ".." + std::to_string(max_depth));
    const uint64_t offset = 1ULL << depth;
    std::map<uint64_t, uint64_t> index_map;
    for (size_t i = 0; i < indexes_in.size(); i++) {
        if (indexes_in[i] > offset - 1) return panic("invalid index " + std::to_string(indexes_in[i]));     // map_indexes asserts
        index_map[indexes_in[i]] = i;
    }
    if (index_map.size() != indexes_in.size()) return panic("repeating indexes detected");
    std::set<uint64_t> norm;
    for (uint64_t idx : indexes_in) norm.insert(idx - (idx & 1));
    std::vector<uint64_t> indexes(norm.begin(), norm.end());
    if (indexes.size() != nodes.size())
        return reject("the proof has " + std::to_string(nodes.size()) + " node slots for " + std::to_string(indexes.size()) + " index pairs");
    const std::string no_value = "the proof has no value for an index", no_node = "a node slot of the proof is too short";

    std::map<uint64_t, uint32_t> v;                              // node index -> pool slot of its computed hash
    std::vector<uint64_t> next;
    std::vector<size_t> ptrs;
    plan.level_start.push_back(0);
    for (size_t i = 0; i < indexes.size(); i++) {
        const uint64_t index = indexes[i];
        auto i1 = index_map.find(index), i2 = index_map.find(index + 1);
        uint32_t left, right;
        if (i1 != index_map.end()) {
            if (n_values <= i1->second) return reject(no_value);
            left = values_base + (uint32_t)i1->second;
            if (i2 != index_map.end()) {
                if (n_values <= i2->second) return reject(no_value);
                right = values_base + (uint32_t)i2->second;
                ptrs.push_back(0);
            } else {
                if (nodes[i].size() < 1) return reject(no_node);
                right = nodes_base[i];
                ptrs.push_back(1);
            }
        } else {
            if (nodes[i].size() < 1) return reject(no_node);
            left = nodes_base[i];
            if (i2 == index_map.end()) return reject(no_value);
            if (n_values <= i2->second) return reject(no_value);
            right = values_base + (uint32_t)i2->second;
            ptrs.push_back(1);
        }
        const uint32_t out = next_slot++;
        plan.ops.insert(plan.ops.end(), {left, right, out});
        const uint64_t parent = (offset + index) >> 1;
        v[parent] = out;
        next.push_back(parent);
    }
    for (int d = 1; d < depth; d++) {
        plan.level_start.push_back((uint32_t)(plan.ops.size() / 3));
        std::vector<uint64_t> cur = next;
        next.clear();
        std::map<uint64_t, uint32_t> vnext;
        size_t i = 0;
        while (i < cur.size()) {
            const uint64_t node_index = cur[i], sibling_index = node_index ^ 1;
            uint32_t sibling;
            if (i + 1 < cur.size() && cur[i + 1] == sibling_index) {
                auto s = v.find(sibling_index);
                if (s == v.end()) return reject("a sibling was not computed");
                sibling = s->second;
                i += 1;
            } else {
                // the reference indexes proof.nodes and the pointers with the position inside the CURRENT level's list
                if (i >= ptrs.size() || i >= nodes.size()) return reject(no_node);
                const size_t pointer = ptrs[i];
                if (nodes[i].size() <= pointer) return reject(no_node);
                sibling = nodes_base[i] + (uint32_t)pointer;
                ptrs[i] += 1;
            }
            auto nd = v.find(node_index);
            if (nd == v.end()) return reject("a node was not computed");
            const uint32_t out = next_slot++;
            if (node_index & 1) plan.ops.insert(plan.ops.end(), {sibling, nd->second, out});
            else plan.ops.insert(plan.ops.end(), {nd->second, sibling, out});
            const uint64_t parent = node_index >> 1;
            vnext[parent] = out;
            next.push_back(parent);
            i += 1;
        }
        for (auto &kv : vnext) v[kv.first] = kv.second;         // parents join the map (HashMap::insert in the reference)
    }
    plan.level_start.push_back((uint32_t)(plan.ops.size() / 3));
    auto rt = v.find(1);
    if (rt == v.end()) return panic("called `Option::unwrap()` on a `None` value");      // v.get(&1).unwrap()
    plan.root_slot = rt->second;
    plan.ok = true;
    return plan;
}

// ---- batch proofs ------------------------------------------------------------------------------------------------------------------

// digest t of a batch proof in encoding order: refs[t] = index into the leaves, or (1 << 63) | index into the heap
__global__ void __launch_bounds__(256) tree_gather_kernel(const uint4 *__restrict__ leaves, const uint4 *__restrict__ nodes,
                                                          const unsigned long long *__restrict__ refs, unsigned n, uint4 *__restrict__ out) {
    const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const unsigned long long r = refs[t], i = r & ~(1ULL << 63);
    const uint4 *s = (r >> 63 ? nodes : leaves) + 2 * i;
    out[2 * t] = s[0];
    out[2 * t + 1] = s[1];
}

size_t batch_proof_len(const fs::BatchPlan &plan) {
    size_t n = 8 + 32 * plan.value_leaves.size() + 8 + 1;
    for (auto &slot : plan.nodes) n += 8 + 32 * slot.size();
    return n;
}

void tree_prove_batch(Context &c, const Tree &t, const fs::BatchPlan &plan, uint8_t *out) {
    std::vector<unsigned long long> refs(plan.value_leaves.begin(), plan.value_leaves.end());      // values in request order, then the slots
    for (auto &slot : plan.nodes)
        for (const fs::NodeRef &r : slot) refs.push_back(r.leaf ? r.index : (1ULL << 63) | r.index);
    const size_t n = refs.size();
    std::vector<uint8_t> digests(n * 32);
    if (n) {
        DevBuf d((n * 8 + 15) / 16 * 16 + n * 32);
        uint4 *d_out = (uint4 *)(d.as<uint8_t>() + (n * 8 + 15) / 16 * 16);
        DG_CUDA(cudaMemcpyAsync(d.p, refs.data(), n * 8, cudaMemcpyHostToDevice, c.stream));
        tree_gather_kernel<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(t.leaves.as<uint4>(), t.nodes.as<uint4>(), d.as<unsigned long long>(),
                                                                              (unsigned)n, d_out);
        c.launches++;
        DG_CUDA(cudaGetLastError());
        DG_CUDA(cudaMemcpyAsync(digests.data(), d_out, n * 32, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    }
    // the bincode framing around the gathered digests: u64 count + values, u64 count, per slot u64 count + nodes, u8 depth
    auto u64 = [&](uint64_t v) { memcpy(out, &v, 8); out += 8; };
    const uint8_t *d = digests.data();
    auto copy = [&](size_t k) { memcpy(out, d, 32 * k); out += 32 * k; d += 32 * k; };
    u64(plan.value_leaves.size());
    copy(plan.value_leaves.size());
    u64(plan.nodes.size());
    for (auto &slot : plan.nodes) { u64(slot.size()); copy(slot.size()); }
    *out = plan.depth;
}

// ---- path and batch-proof verification -------------------------------------------------------------------------------------------

// message of path k at level e (1 .. entries - 1): at e = 1 entries r = index & 1 and 1 - r of the path; above, the digest so far and
// entry e, in the order bit e - 1 of the index chooses (merkle.rs:131-148: the bits of (index + 2^(entries - 1)) >> 1)
__global__ void __launch_bounds__(256) path_level_kernel(const uint4 *__restrict__ paths, const unsigned long long *__restrict__ indexes,
                                                         const uint4 *__restrict__ v, unsigned count, unsigned entries, unsigned e,
                                                         uint4 *__restrict__ msgs) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    const unsigned long long i = indexes[k];
    const uint4 *p = paths + 2 * (size_t)k * entries, *a, *b;
    if (e == 1) {
        a = p + 2 * (i & 1);
        b = p + 2 * (~i & 1);
    } else if ((i >> (e - 1)) & 1) {
        a = p + 2 * e;
        b = v + 2 * (size_t)k;
    } else {
        a = v + 2 * (size_t)k;
        b = p + 2 * e;
    }
    msgs[4 * (size_t)k] = a[0];
    msgs[4 * (size_t)k + 1] = a[1];
    msgs[4 * (size_t)k + 2] = b[0];
    msgs[4 * (size_t)k + 3] = b[1];
}

// accepted[k] = 1 when digest k equals root k (root_step 1) or the one root (root_step 0)
__global__ void __launch_bounds__(256) path_root_kernel(const uint4 *__restrict__ v, const uint4 *__restrict__ roots, unsigned root_step,
                                                        unsigned count, uint8_t *__restrict__ accepted) {
    const unsigned k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    const uint4 a0 = v[2 * (size_t)k], a1 = v[2 * (size_t)k + 1];
    const uint4 r0 = roots[2 * (size_t)k * root_step], r1 = roots[2 * (size_t)k * root_step + 1];
    accepted[k] = a0.x == r0.x && a0.y == r0.y && a0.z == r0.z && a0.w == r0.w && a1.x == r1.x && a1.y == r1.y && a1.z == r1.z && a1.w == r1.w;
}

// message t of a level of batch proofs: the pool's digests pairs[2 t] | pairs[2 t + 1]
__global__ void __launch_bounds__(256) pool_pairs_kernel(const uint4 *__restrict__ pool, const uint32_t *__restrict__ pairs, unsigned n,
                                                         uint4 *__restrict__ msgs) {
    const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint4 *a = pool + 2 * (size_t)pairs[2 * t], *b = pool + 2 * (size_t)pairs[2 * t + 1];
    msgs[4 * (size_t)t] = a[0];
    msgs[4 * (size_t)t + 1] = a[1];
    msgs[4 * (size_t)t + 2] = b[0];
    msgs[4 * (size_t)t + 3] = b[1];
}

// device bytes a group of verification calls may take (the budget of dg_verify_batch), within dg_set_memory_limit
static const size_t VERIFY_GROUP_BYTES = (size_t)512 << 20;
static size_t align16(size_t n) { return (n + 15) & ~(size_t)15; }

void merkle_verify_paths(Context &c, int hash, const uint8_t *roots32, bool per_path_root, const uint64_t *indexes, const uint8_t *paths32,
                         unsigned entries, uint32_t count, uint8_t *accepted) {
    const size_t budget = memory_budget(c, Budget::FIXED, VERIFY_GROUP_BYTES);
    const size_t per_path = 8 + 32 * (size_t)entries + (per_path_root ? 32 : 0) + 64 + 32 + 1 + 64;     // + alignment slack
    const uint32_t group = (uint32_t)std::max<size_t>(1, std::min<size_t>(count, budget / per_path));
    for (uint32_t k0 = 0; k0 < count; k0 += group) {
        const uint32_t K = std::min(group, count - k0), n_roots = per_path_root ? K : 1;
        const size_t o_paths = align16((size_t)K * 8), o_roots = o_paths + (size_t)K * 32 * entries, o_msgs = o_roots + (size_t)n_roots * 32,
                     o_v = o_msgs + (size_t)K * 64, o_ok = o_v + (size_t)K * 32;
        DevBuf d(o_ok + K);
        uint8_t *D = d.as<uint8_t>();
        DG_CUDA(cudaMemcpyAsync(D, indexes + k0, (size_t)K * 8, cudaMemcpyHostToDevice, c.stream));
        DG_CUDA(cudaMemcpyAsync(D + o_paths, paths32 + (size_t)k0 * 32 * entries, (size_t)K * 32 * entries, cudaMemcpyHostToDevice, c.stream));
        DG_CUDA(cudaMemcpyAsync(D + o_roots, roots32 + (per_path_root ? (size_t)k0 * 32 : 0), (size_t)n_roots * 32, cudaMemcpyHostToDevice, c.stream));
        const unsigned grid = (K + 255) / 256;
        for (unsigned e = 1; e < entries; e++) {
            path_level_kernel<<<grid, 256, 0, c.stream>>>((const uint4 *)(D + o_paths), (const unsigned long long *)D, (const uint4 *)(D + o_v), K,
                                                          entries, e, (uint4 *)(D + o_msgs));
            c.launches++;
            DG_CUDA(cudaGetLastError());
            alg_hash64(c, hash, D + o_msgs, D + o_v, K);
        }
        path_root_kernel<<<grid, 256, 0, c.stream>>>((const uint4 *)(D + o_v), (const uint4 *)(D + o_roots), per_path_root ? 1 : 0, K, D + o_ok);
        c.launches++;
        DG_CUDA(cudaGetLastError());
        DG_CUDA(cudaMemcpyAsync(accepted + k0, D + o_ok, K, cudaMemcpyDeviceToHost, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    }
}

// One group of batch proofs, aligned at their roots: with D the group's largest depth, round r runs level r - (D - depth) of every check
// whose depth reaches it, so the last round holds exactly the root op of every check.  Pool: [the checks' values and nodes | the outputs
// of round 0 | round 1 | ...]; the outputs of global op g are slot n_in + g.
static void verify_batch_group(Context &c, int hash, const std::vector<const BatchCheck *> &g, const std::vector<const uint8_t *> &roots,
                               std::vector<uint8_t *> &accepted) {
    const size_t K = g.size();
    std::vector<uint32_t> in_base(K), n_in(K);
    uint32_t slots = 0, D = 0;
    for (size_t i = 0; i < K; i++) {
        const BatchMerkleProof &p = *g[i]->proof;
        in_base[i] = slots;
        n_in[i] = (uint32_t)p.values.size();
        for (auto &slot : p.nodes) n_in[i] += (uint32_t)slot.size();
        slots += n_in[i];
        D = std::max(D, (uint32_t)g[i]->plan.level_start.size() - 1);
    }
    const uint32_t n_inputs = slots;
    // global op index of every check's ops, round by round
    std::vector<std::vector<uint32_t>> gop(K);
    std::vector<uint32_t> round_start{0};
    uint32_t ops = 0;
    for (uint32_t r = 0; r < D; r++) {
        for (size_t i = 0; i < K; i++) {
            const MerklePlan &pl = g[i]->plan;
            const uint32_t levels = (uint32_t)pl.level_start.size() - 1;
            if (r + levels < D) continue;
            const uint32_t l = r + levels - D;
            for (uint32_t o = pl.level_start[l]; o < pl.level_start[l + 1]; o++) { gop[i].push_back(ops++); }
        }
        round_start.push_back(ops);
    }
    // upload: the input digests, then the (left, right) global slots of every op in global order
    const size_t o_pairs = (size_t)n_inputs * 32, bytes = o_pairs + (size_t)ops * 8;
    std::vector<uint8_t> h(bytes);
    std::vector<uint32_t> pairs((size_t)ops * 2);
    for (size_t i = 0; i < K; i++) {
        const BatchMerkleProof &p = *g[i]->proof;
        uint8_t *at = h.data() + (size_t)in_base[i] * 32;
        for (auto &v : p.values) { memcpy(at, v.data(), 32); at += 32; }
        for (auto &slot : p.nodes) for (auto &v : slot) { memcpy(at, v.data(), 32); at += 32; }
        const MerklePlan &pl = g[i]->plan;
        auto global = [&](uint32_t s) { return s < n_in[i] ? in_base[i] + s : n_inputs + gop[i][s - n_in[i]]; };
        for (size_t o = 0; o < gop[i].size(); o++) {
            DG_REQUIRE(pl.ops[3 * o + 2] == n_in[i] + o, "batch proof plan: outputs out of op order");
            pairs[2 * (size_t)gop[i][o]] = global(pl.ops[3 * o]);
            pairs[2 * (size_t)gop[i][o] + 1] = global(pl.ops[3 * o + 1]);
        }
        DG_REQUIRE(pl.level_start[pl.level_start.size() - 2] + 1 == pl.level_start.back() && pl.root_slot == n_in[i] + gop[i].size() - 1,
                   "batch proof plan: the last level is not the root");
    }
    memcpy(h.data() + o_pairs, pairs.data(), (size_t)ops * 8);
    size_t widest = 1;
    for (uint32_t r = 0; r < D; r++) widest = std::max<size_t>(widest, round_start[r + 1] - round_start[r]);
    const size_t o_pool_ops = o_pairs, o_dev_pairs = align16(o_pool_ops + (size_t)ops * 32), o_msgs = align16(o_dev_pairs + (size_t)ops * 8);
    DevBuf d(o_msgs + widest * 64);
    uint8_t *B = d.as<uint8_t>();
    DG_CUDA(cudaMemcpyAsync(B, h.data(), o_pairs, cudaMemcpyHostToDevice, c.stream));
    DG_CUDA(cudaMemcpyAsync(B + o_dev_pairs, h.data() + o_pairs, (size_t)ops * 8, cudaMemcpyHostToDevice, c.stream));
    for (uint32_t r = 0; r < D; r++) {
        const uint32_t n = round_start[r + 1] - round_start[r];
        pool_pairs_kernel<<<(n + 255) / 256, 256, 0, c.stream>>>((const uint4 *)B, (const uint32_t *)(B + o_dev_pairs) + 2 * (size_t)round_start[r], n,
                                                                (uint4 *)(B + o_msgs));
        c.launches++;
        DG_CUDA(cudaGetLastError());
        alg_hash64(c, hash, B + o_msgs, B + ((size_t)n_inputs + round_start[r]) * 32, n);
    }
    // the last round's outputs are the K roots, in check order
    std::vector<Digest> got(K);
    DG_CUDA(cudaMemcpyAsync(got.data(), B + ((size_t)n_inputs + round_start[D - 1]) * 32, K * 32, cudaMemcpyDeviceToHost, c.stream));
    DG_CUDA(cudaStreamSynchronize(c.stream));
    for (size_t i = 0; i < K; i++) *accepted[i] = memcmp(got[i].data(), roots[i], 32) == 0;
}

void merkle_verify_batch(Context &c, int hash, const std::vector<BatchCheck> &checks, const uint8_t *const *roots32, uint8_t *accepted) {
    const size_t budget = memory_budget(c, Budget::FIXED, VERIFY_GROUP_BYTES);
    std::vector<const BatchCheck *> g;
    std::vector<const uint8_t *> roots;
    std::vector<uint8_t *> out;
    size_t bytes = 0;
    auto flush = [&]() {
        if (g.empty()) return;
        verify_batch_group(c, hash, g, roots, out);
        g.clear(); roots.clear(); out.clear(); bytes = 0;
    };
    for (size_t i = 0; i < checks.size(); i++) {
        const BatchCheck &ck = checks[i];
        size_t in = ck.proof->values.size();
        for (auto &slot : ck.proof->nodes) in += slot.size();
        const size_t ops = ck.plan.ops.size() / 3, b = in * 32 + ops * (32 + 8 + 64) + 64;
        if (!g.empty() && bytes + b > budget) flush();
        g.push_back(&ck); roots.push_back(roots32[i]); out.push_back(accepted + i);
        bytes += b;
    }
    flush();
}

}  // namespace dg
