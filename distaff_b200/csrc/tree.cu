// Merkle trees that stay on the GPU (tree.h): build once with alg_merkle_build, gather the authentication paths of many leaves in one
// launch, and update leaves by rehashing only the nodes on their paths.  An update runs one pass per level: tree_level_kernel writes the
// level below's new values into their slots and gathers this level's 64-byte messages, then alg_hash64 (for hash 3 hasher_digest, with
// its narrow / wide choice) hashes them.  The digest kernels are the measured ones, unchanged.
#include "tree.h"
#include "poly.h"
#include <algorithm>

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

}  // namespace dg
