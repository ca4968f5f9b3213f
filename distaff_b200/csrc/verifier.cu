// GPU verifier for StarkProof bytes: the step after the prove path (SURVEY.md section 8f rank 3).
//
//   stark::verify                      /root/reference/src/stark/verifier.rs:11-75
//   evaluate_constraints / compose_*   /root/reference/src/stark/verifier.rs:79-162
//   fri::verify                        /root/reference/src/stark/fri/verifier.rs:11-131
//   MerkleTree::verify_batch           /root/reference/src/crypto/merkle.rs:154-263
//
// The reference walks the proof sequentially on one core.  Here one pipeline verifies K proofs (dg_verify is K = 1) in three phases:
//   prepare (host, proof by proof in input order): parse, option and PoW checks, query positions, every Fiat-Shamir draw (z, constraint
//      and composition coefficients, FRI folding points), and every batch-Merkle verification as a plan of (left, right, out) hashing
//      steps per tree level -- pure index logic, following verify_batch statement by statement, including its use of the current
//      level's position as the slot of `proof.nodes`.  A proof decided here (malformed bytes, failed PoW, ...) skips the device.
//   device (per group of proofs: one upload, one synchronise), each step one launch for the whole group:
//      1. BLAKE3 of the opened trace rows (one launch per row width) and of the opened FRI rows (the Merkle leaves),
//      2. all Merkle plans of all proofs (one block per tree, one barrier per level),
//      3. the transition constraints at the out-of-domain point z: the prover's constraint kernel (air.cu) in verify mode, one launch
//         per register shape, with the deep values as the two rows of a 128-step stand-in trace, the cycle polynomials evaluated at
//         z^(n/16) and the powers z^inc from the host,
//      4. C(z) from the boundary numerators and the transition value at z (one thread per proof),
//      5. the DEEP composition at every query position (one thread per query, two Fermat inversions each),
//      6. every FRI row folded at its layer's point (closed-form 4-point fold of fri.cu; all layers in parallel, because each layer's
//         opened rows are in the proof and only the equality "fold of layer d == opened value of layer d + 1" chains them).
//   finish (host, per proof): the reference's checks in the reference's order, with its error strings.
#include <algorithm>
#include <array>
#include <map>
#include <set>
#include "air.h"
#include "blake3.cuh"
#include "host_fs.h"
#include "poly.h"
#include "prover.h"
#include "shard.h"

namespace dg {

namespace {

// ---- bincode reader (proof.rs:10-37, fri/mod.rs:17-30, merkle.rs:14-18) -------------------------------------------------------
struct Reader {
    const uint8_t *p, *end;
    bool ok = true;
    Reader(const uint8_t *b, size_t n) : p(b), end(b + n) {}
    bool need(size_t n) { if (!ok || (size_t)(end - p) < n) { ok = false; return false; } return true; }
    uint8_t u8() { if (!need(1)) return 0; return *p++; }
    uint32_t u32() { if (!need(4)) return 0; uint32_t v; memcpy(&v, p, 4); p += 4; return v; }
    uint64_t u64() { if (!need(8)) return 0; uint64_t v; memcpy(&v, p, 8); p += 8; return v; }
    fe felt() { fe v = fe_make(0, 0); if (!need(16)) return v; memcpy(&v, p, 16); p += 16; return v; }
    Digest digest() { Digest d; d.fill(0); if (!need(32)) return d; memcpy(d.data(), p, 32); p += 32; return d; }
    size_t len(size_t elem_bytes) {                              // a Vec length that the remaining bytes can actually hold
        uint64_t n = u64();
        if (!ok || n > (uint64_t)(end - p) / (elem_bytes ? elem_bytes : 1)) { ok = false; return 0; }
        return (size_t)n;
    }
    std::vector<Digest> dvec() { size_t n = len(32); std::vector<Digest> v(n); for (auto &x : v) x = digest(); return v; }
    std::vector<std::vector<Digest>> dvv() { size_t n = len(8); std::vector<std::vector<Digest>> v(n); for (auto &x : v) x = dvec(); return v; }
    std::vector<fe> fvec() { size_t n = len(16); std::vector<fe> v(n); for (auto &x : v) x = felt(); return v; }
};

struct FriLayerProof { Digest root; std::vector<std::array<fe, 4>> values; std::vector<std::vector<Digest>> nodes; uint8_t depth; };
struct ParsedProof {
    Digest trace_root, constraint_root, rem_root;
    uint8_t domain_depth, ctx_depth, loop_depth, stack_depth, c_depth;
    uint32_t op_count;
    std::vector<std::vector<Digest>> trace_nodes, c_nodes;
    std::vector<std::vector<fe>> trace_evaluations;
    std::vector<Digest> c_values;
    std::vector<fe> z1, z2, rem_values;
    std::vector<FriLayerProof> layers;
    uint64_t pow_nonce;
    uint8_t log_ext, num_queries, grinding, hash_id;
};

bool parse_proof(const uint8_t *bytes, size_t n, ParsedProof &P) {
    Reader r(bytes, n);
    P.trace_root = r.digest();
    P.domain_depth = r.u8(); P.ctx_depth = r.u8(); P.loop_depth = r.u8(); P.stack_depth = r.u8();
    P.op_count = r.u32();
    P.trace_nodes = r.dvv();
    { size_t k = r.len(8); P.trace_evaluations.resize(k); for (auto &row : P.trace_evaluations) row = r.fvec(); }
    P.constraint_root = r.digest();
    P.c_values = r.dvec(); P.c_nodes = r.dvv(); P.c_depth = r.u8();
    P.z1 = r.fvec(); P.z2 = r.fvec();
    { size_t k = r.len(41); P.layers.resize(k); }
    for (auto &l : P.layers) {
        l.root = r.digest();
        size_t k = r.len(64);
        l.values.resize(k);
        for (auto &q : l.values) for (int j = 0; j < 4; j++) q[j] = r.felt();
        l.nodes = r.dvv();
        l.depth = r.u8();
    }
    P.rem_root = r.digest();
    P.rem_values = r.fvec();
    P.pow_nonce = r.u64();
    P.log_ext = r.u8(); P.num_queries = r.u8(); P.grinding = r.u8(); P.hash_id = r.u8();
    return r.ok && r.p == r.end;
}

// ---- batch Merkle verification as a hashing plan (merkle.rs:154-263) -------------------------------------------------------------
// pool slots: the caller lays out the proof's values and nodes in a pool of 32-byte digests; computed parents get fresh slots
struct MerklePlan {
    std::vector<uint32_t> ops;            // (left, right, out) pool indices
    std::vector<uint32_t> level_start;    // op index where each level starts (+ final end)
    uint32_t root_slot = 0;
    bool ok = false;
};
MerklePlan plan_verify_batch(const std::vector<uint64_t> &indexes_in, int depth, size_t n_values, uint32_t values_base,
                             const std::vector<std::vector<Digest>> &nodes, const std::vector<uint32_t> &nodes_base, uint32_t &next_slot) {
    MerklePlan plan;
    if (depth < 1 || depth > 40) return plan;
    const uint64_t offset = 1ULL << depth;
    std::map<uint64_t, uint64_t> index_map;
    for (size_t i = 0; i < indexes_in.size(); i++) {
        if (indexes_in[i] > offset - 1) return plan;             // the reference asserts here (map_indexes)
        index_map[indexes_in[i]] = i;
    }
    if (index_map.size() != indexes_in.size()) return plan;
    std::set<uint64_t> norm;
    for (uint64_t idx : indexes_in) norm.insert(idx - (idx & 1));
    std::vector<uint64_t> indexes(norm.begin(), norm.end());
    if (indexes.size() != nodes.size()) return plan;

    std::map<uint64_t, uint32_t> v;                              // node index -> pool slot of its computed hash
    std::vector<uint64_t> next;
    std::vector<size_t> ptrs;
    plan.level_start.push_back(0);
    for (size_t i = 0; i < indexes.size(); i++) {
        const uint64_t index = indexes[i];
        auto i1 = index_map.find(index), i2 = index_map.find(index + 1);
        uint32_t left, right;
        if (i1 != index_map.end()) {
            if (n_values <= i1->second) return plan;
            left = values_base + (uint32_t)i1->second;
            if (i2 != index_map.end()) {
                if (n_values <= i2->second) return plan;
                right = values_base + (uint32_t)i2->second;
                ptrs.push_back(0);
            } else {
                if (nodes[i].size() < 1) return plan;
                right = nodes_base[i];
                ptrs.push_back(1);
            }
        } else {
            if (nodes[i].size() < 1) return plan;
            left = nodes_base[i];
            if (i2 == index_map.end()) return plan;
            if (n_values <= i2->second) return plan;
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
                if (s == v.end()) return plan;
                sibling = s->second;
                i += 1;
            } else {
                // the reference indexes proof.nodes and the pointers with the position inside the CURRENT level's list
                if (i >= ptrs.size() || i >= nodes.size()) return plan;
                const size_t pointer = ptrs[i];
                if (nodes[i].size() <= pointer) return plan;
                sibling = nodes_base[i] + (uint32_t)pointer;
                ptrs[i] += 1;
            }
            auto nd = v.find(node_index);
            if (nd == v.end()) return plan;
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
    if (rt == v.end()) return plan;
    plan.root_slot = rt->second;
    plan.ok = true;
    return plan;
}

struct TreeDesc { uint32_t ops_base, n_levels, levels_base, pad; };

// one block per tree: ops of a level in parallel, levels separated by barriers
__global__ void __launch_bounds__(128) merkle_verify_kernel(uint4 *pool, const uint32_t *__restrict__ ops, const uint32_t *__restrict__ level_start,
                                                            const TreeDesc *__restrict__ trees) {
    const TreeDesc t = trees[blockIdx.x];
    for (uint32_t l = 0; l < t.n_levels; l++) {
        const uint32_t a = level_start[t.levels_base + l], b = level_start[t.levels_base + l + 1];
        for (uint32_t o = a + threadIdx.x; o < b; o += blockDim.x) {
            const uint32_t *op = ops + 3 * (size_t)(t.ops_base + o);
            uint32_t m[16], cv[8];
            const uint4 l0 = pool[2 * (size_t)op[0]], l1 = pool[2 * (size_t)op[0] + 1], r0 = pool[2 * (size_t)op[1]], r1 = pool[2 * (size_t)op[1] + 1];
            m[0] = l0.x; m[1] = l0.y; m[2] = l0.z; m[3] = l0.w; m[4] = l1.x; m[5] = l1.y; m[6] = l1.z; m[7] = l1.w;
            m[8] = r0.x; m[9] = r0.y; m[10] = r0.z; m[11] = r0.w; m[12] = r1.x; m[13] = r1.y; m[14] = r1.z; m[15] = r1.w;
            b3::hash64(m, cv);
            pool[2 * (size_t)op[2]] = make_uint4(cv[0], cv[1], cv[2], cv[3]);
            pool[2 * (size_t)op[2] + 1] = make_uint4(cv[4], cv[5], cv[6], cv[7]);
        }
        __syncthreads();
    }
}

// Per-proof descriptors of the batched kernels below.  Every pointer is into the group's one device allocation.
struct AtZDesc {                        // constraint value at z of one proof (verifier.rs:79-97, evaluator.rs:181-326)
    const fe *z1;                       // the deep values: z1 (w), then z2 (w)
    const fe *bcoef;                    // boundary coefficients bAi | bBi | bAf | bBf, nb each
    const fe *t_at_z;                   // the transition combination at z (row 0 of the constraint kernel's output)
    fe *slab;                           // 128-step stand-in trace of the constraint kernel, [w][128]
    fe KiA, KiB, KfA, KfB, z, x_last;
    unsigned long long n;               // trace length
    int w, nb;
};
struct ComposeDesc {                    // DEEP composition of one proof (verifier.rs:101-162)
    const fe *rows;                     // opened trace rows: column j of query q at rows[j * row_stride + q]
    unsigned long long row_stride;
    const fe *zs;                       // z1 | z2 | cc1 | cc2, w each
    const fe *c_at_z;
    fe z, zg, t1_degree, t2_degree, k_constraints;
    TwiddleRef twN;                     // powers of the LDE root of this proof's domain
    unsigned long long inc;             // get_incremental_trace_degree
    unsigned first;                     // index of this proof's first query in the group
    int w;
};
struct FoldDesc {                       // FRI folds of one proof (fri/verifier.rs:33-75)
    TwiddleRef inv_root;                // powers of the inverse LDE root of this proof's domain
    const fe *alphas;                   // one folding point per layer
};

// the deep values as rows 0 and 1 of each proof's stand-in slab (the slabs are zeroed before): block = proof, thread = register
__global__ void __launch_bounds__(128) deep_rows_to_slab_kernel(const AtZDesc *__restrict__ d) {
    const AtZDesc &D = d[blockIdx.x];
    const int j = threadIdx.x;
    if (j >= D.w) return;
    D.slab[(size_t)j * 128] = D.z1[j];
    D.slab[(size_t)j * 128 + 1] = D.z1[D.w + j];
}

// one thread per proof: boundary numerators at z, then C(z) = I(z) / (z - 1) + F(z) / (z - x_last) + T(z) / ((z^n - 1) / (z - x_last)),
// every division with field::div semantics (inv(0) = 0, field.rs:75-84) and in the order of the reference
__global__ void verify_at_z_kernel(const AtZDesc *__restrict__ d, int count, fe *__restrict__ c_at_z) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= count) return;
    const AtZDesc &D = d[i];
    const fe z = D.z;
    const fe zadj = fe_pow_u64(z, 6 * D.n + 2);
    fe ia = fe_make(0, 0), ib = ia, fa = ia, fb = ia;
    for (int j = 0; j < D.nb; j++) {
        const fe s = D.z1[j];
        ia = fe_add(ia, fe_mul(s, D.bcoef[j])); ib = fe_add(ib, fe_mul(s, D.bcoef[D.nb + j]));
        fa = fe_add(fa, fe_mul(s, D.bcoef[2 * D.nb + j])); fb = fe_add(fb, fe_mul(s, D.bcoef[3 * D.nb + j]));
    }
    const fe i_value = fe_add(fe_sub(ia, D.KiA), fe_mul(zadj, fe_sub(ib, D.KiB)));
    const fe f_value = fe_add(fe_sub(fa, D.KfA), fe_mul(zadj, fe_sub(fb, D.KfB)));
    fe zz = fe_sub(z, fe_make(1, 0));
    fe result = fe_mul(i_value, fe_inv(zz));
    zz = fe_sub(z, D.x_last);
    result = fe_add(result, fe_mul(f_value, fe_inv(zz)));
    zz = fe_mul(fe_sub(fe_pow_u64(z, D.n), fe_make(1, 0)), fe_inv(zz));
    c_at_z[i] = fe_add(result, fe_mul(*D.t_at_z, fe_inv(zz)));
}

// DEEP composition at every query position of every proof: one thread per (proof, query), proof[g] names the descriptor
__global__ void compose_at_queries_batch_kernel(const ComposeDesc *__restrict__ d, const unsigned *__restrict__ proof, unsigned count,
                                                const unsigned long long *__restrict__ positions, const fe *__restrict__ c_evals,
                                                fe *__restrict__ out) {
    const unsigned g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= count) return;
    const ComposeDesc &A = d[proof[g]];
    const unsigned q = g - A.first;
    const unsigned long long pos = positions[g];
    auto pw = [&](unsigned long long e) {
        const unsigned ee = (unsigned)(e & (unsigned long long)A.twN.mask);
        return fe_mul(A.twN.lo[ee & ((1u << A.twN.lo_bits) - 1u)], A.twN.hi[ee >> A.twN.lo_bits]);
    };
    const fe x = pw(pos);
    const fe inv1 = fe_inv(fe_sub(x, A.z)), inv2 = fe_inv(fe_sub(x, A.zg));
    const int w = A.w;
    fe comp = fe_make(0, 0);
    for (int i = 0; i < w; i++) {
        const fe r = A.rows[(size_t)i * A.row_stride + q];
        comp = fe_add(comp, fe_mul(fe_mul(fe_sub(r, A.zs[i]), inv1), A.zs[2 * w + i]));
        comp = fe_add(comp, fe_mul(fe_mul(fe_sub(r, A.zs[w + i]), inv2), A.zs[3 * w + i]));
    }
    const fe xp = pw(pos * A.inc);
    const fe adj = fe_mul(fe_mul(comp, xp), A.t2_degree);
    comp = fe_add(fe_mul(comp, A.t1_degree), adj);
    const fe cv = fe_mul(fe_sub(c_evals[g], *A.c_at_z), inv1);
    out[g] = fe_add(comp, fe_mul(cv, A.k_constraints));
}

// every opened FRI row of every proof folded at its layer's point: rows[t] = 4 values, pos[t] = row index, layer[t] = d (shift 2 d),
// proof[t] names the descriptor with the proof's folding points and inverse-root table
__global__ void fri_fold_rows_batch_kernel(const fe *__restrict__ rows, const unsigned long long *__restrict__ pos, const unsigned *__restrict__ layer,
                                           const unsigned *__restrict__ proof, unsigned count, const FoldDesc *__restrict__ d, fe tau_inv, fe inv4,
                                           fe *__restrict__ out) {
    const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= count) return;
    const FoldDesc &D = d[proof[t]];
    const unsigned l = layer[t];
    const fe y0 = rows[4 * (size_t)t], y1 = rows[4 * (size_t)t + 1], y2 = rows[4 * (size_t)t + 2], y3 = rows[4 * (size_t)t + 3];
    const unsigned ee = (unsigned)((pos[t] << (2 * l)) & (unsigned long long)D.inv_root.mask);
    const fe xinv = fe_mul(D.inv_root.lo[ee & ((1u << D.inv_root.lo_bits) - 1u)], D.inv_root.hi[ee >> D.inv_root.lo_bits]);
    const fe u = fe_mul(D.alphas[l], xinv);
    const fe s02 = fe_add(y0, y2), d02 = fe_sub(y0, y2), s13 = fe_add(y1, y3), d13 = fe_mul(fe_sub(y1, y3), tau_inv);
    const fe a0 = fe_add(s02, s13), a1 = fe_add(d02, d13), a2 = fe_sub(s02, s13), a3 = fe_sub(d02, d13);
    fe acc = fe_add(a2, fe_mul(u, a3));
    acc = fe_add(a1, fe_mul(u, acc));
    acc = fe_add(a0, fe_mul(u, acc));
    out[t] = fe_mul(acc, inv4);
}

// polynom::interpolate (Lagrange, polynom.rs:106-145) followed by polynom::eval, only for the remainder check (<= 256 points)
bool remainder_is_low_degree(const std::vector<fe> &xs_all, const std::vector<fe> &ys_all, size_t degree_plus_1) {
    const size_t m = degree_plus_1;
    std::vector<fe> xs(xs_all.begin(), xs_all.begin() + m), ys(ys_all.begin(), ys_all.begin() + m);
    // barycentric weights w_i = 1 / prod_{j != i} (x_i - x_j); p(x) = sum_i y_i w_i prod_{j != i} (x - x_j)
    std::vector<fe> wgt(m);
    for (size_t i = 0; i < m; i++) {
        fe d = fe_make(1, 0);
        for (size_t j = 0; j < m; j++) if (j != i) d = fe_mul(d, fe_sub(xs[i], xs[j]));
        wgt[i] = fe_mul(ys[i], fe_inv(d));
    }
    for (size_t t = m; t < xs_all.size(); t++) {
        const fe x = xs_all[t];
        // prefix / suffix products of (x - x_j)
        std::vector<fe> pre(m + 1), suf(m + 1);
        pre[0] = fe_make(1, 0);
        for (size_t j = 0; j < m; j++) pre[j + 1] = fe_mul(pre[j], fe_sub(x, xs[j]));
        suf[m] = fe_make(1, 0);
        for (size_t j = m; j-- > 0;) suf[j] = fe_mul(suf[j + 1], fe_sub(x, xs[j]));
        fe val = fe_make(0, 0);
        for (size_t i = 0; i < m; i++) val = fe_add(val, fe_mul(wgt[i], fe_mul(pre[i], suf[i + 1])));
        if (!fe_eq(val, ys_all[t])) return false;
    }
    return true;
}

}  // namespace

// host-only view of the batch-Merkle hashing plan (CPU tests): values occupy pool slots [0, n_values), the nodes of slot i start at
// n_values + sum of the earlier slots' sizes, computed parents follow.  Returns false where verify_batch returns false before hashing.
bool host_plan_verify_batch(const std::vector<uint64_t> &indexes, int depth, size_t n_values, const std::vector<uint32_t> &node_counts,
                            std::vector<uint32_t> &ops, std::vector<uint32_t> &level_start, uint32_t &root_slot) {
    std::vector<std::vector<Digest>> nodes(node_counts.size());
    std::vector<uint32_t> bases;
    uint32_t next = (uint32_t)n_values;
    for (size_t i = 0; i < node_counts.size(); i++) { nodes[i].resize(node_counts[i]); bases.push_back(next); next += node_counts[i]; }
    MerklePlan p = plan_verify_batch(indexes, depth, n_values, 0, nodes, bases, next);
    if (!p.ok) return false;
    ops = p.ops; level_start = p.level_start; root_slot = p.root_slot;
    return true;
}

namespace {

// one proof through the three phases
struct Item {
    VerifyRequest in;
    std::vector<fe> inputs, outputs;
    bool decided = false;               // verdict known without the device phase
    int status = DG_OK;
    std::string message;
    // ---- prepare
    ParsedProof P;
    int w = 0, log_N = 0, nq = 0;
    uint64_t n = 0;
    std::vector<uint64_t> t_positions;
    std::vector<std::vector<uint64_t>> layer_aug;
    std::vector<MerklePlan> plans;      // trace, constraint, then one per FRI layer
    std::vector<Digest> pool;           // local slots: [trace leaves nq | FRI leaves n_fri | constraint values | proof nodes | parents]
    uint32_t n_fri = 0;                 // opened FRI rows over all layers, layer by layer
    std::vector<uint32_t> fri_off;      // first row of each layer
    fe z;
    fs::ConstraintCoefficients cc;
    fs::CompositionCoefficients dc;
    std::vector<fe> per_xpow;           // cycle polynomials at z^(n/16) (23), z^inc of the six degree groups (6)
    std::vector<fe> c_evals, alphas;
    // ---- device results
    std::vector<Digest> roots;          // computed root of every plan
    std::vector<fe> comp, folded;       // composition at the queries, every FRI row folded
};

void reject(Item &it, const std::string &m) { it.decided = true; it.status = DG_ERR_REJECTED; it.message = m; }

// parse, option checks, PoW, positions, every Fiat-Shamir draw and the Merkle plans; decides the proofs that never reach the device
void prepare(Item &it) {
    DG_REQUIRE(it.in.program_hash && it.in.proof, "null argument");
    DG_REQUIRE((it.in.n_inputs == 0 || it.in.inputs16) && (it.in.n_outputs == 0 || it.in.outputs16), "null public inputs / outputs");
    it.inputs.resize(it.in.n_inputs);
    it.outputs.resize(it.in.n_outputs);
    if (it.in.n_inputs) memcpy(it.inputs.data(), it.in.inputs16, (size_t)it.in.n_inputs * 16);
    if (it.in.n_outputs) memcpy(it.outputs.data(), it.in.outputs16, (size_t)it.in.n_outputs * 16);
    ParsedProof &P = it.P;
    if (!parse_proof(it.in.proof, it.in.proof_len, P)) throw Error(DG_ERR_INVALID, "malformed proof bytes (bincode layout of StarkProof, proof.rs:10-37)");
    if (P.hash_id != 0) return reject(it, "unsupported hash function");
    DG_REQUIRE(P.log_ext >= 4 && P.log_ext <= 8, "invalid extension factor in proof options");
    DG_REQUIRE(P.domain_depth >= P.log_ext + 4 && P.domain_depth <= 30, "invalid domain depth");
    DG_REQUIRE(it.inputs.size() <= 8 && it.outputs.size() <= 8, "cannot have more than 8 public inputs / outputs");
    const uint64_t b = 1ULL << P.log_ext, N = 1ULL << P.domain_depth, n = N >> P.log_ext;
    it.n = n;
    it.log_N = P.domain_depth;
    const int w = it.w = 15 + P.ctx_depth + P.loop_depth + P.stack_depth;
    DG_REQUIRE(P.ctx_depth <= 16 && P.loop_depth <= 8 && P.stack_depth >= 1 && P.stack_depth <= 32 && w < 128, "invalid register counts in the proof");

    // ---- 1: PoW, query positions (verifier.rs:19-31)
    std::vector<uint8_t> fri_roots;
    for (auto &l : P.layers) fri_roots.insert(fri_roots.end(), l.root.begin(), l.root.end());
    fri_roots.insert(fri_roots.end(), P.rem_root.begin(), P.rem_root.end());
    DG_REQUIRE(fri_roots.size() <= 1024, "too many FRI layers");
    uint8_t seed[32], pseed[32];
    fs::blake3_short(fri_roots.data(), fri_roots.size(), seed);
    pow_hash(seed, P.pow_nonce, pseed);
    {
        uint64_t o0;
        memcpy(&o0, pseed, 8);
        const unsigned tz = o0 == 0 ? 64u : (unsigned)__builtin_ctzll(o0);
        if (tz < P.grinding) return reject(it, "seed proof-of-work verification failed");
    }
    try { it.t_positions = fs::query_positions(pseed, N, b, P.num_queries); }
    catch (const std::exception &e) { return reject(it, e.what()); }
    const std::vector<uint64_t> c_positions = fs::constraint_positions(it.t_positions);
    const int nq = it.nq = (int)it.t_positions.size();
    // ---- 2: minimum op count (verifier.rs:34-37; MIN_TRACE_LENGTH = 16)
    if (P.op_count < 16) return reject(it, "Verification of minimum operation count failed");
    if ((int)P.trace_evaluations.size() != nq) return reject(it, "verification of trace Merkle proof failed");
    for (auto &row : P.trace_evaluations) DG_REQUIRE((int)row.size() == w, "trace evaluation row has wrong width");
    DG_REQUIRE((int)P.z1.size() == w && (int)P.z2.size() == w, "deep value vector has wrong width");

    // ---- the Merkle plans over the proof's local pool of digests
    std::vector<Digest> &pool = it.pool;
    auto reserve = [&](size_t k) { uint32_t base = (uint32_t)pool.size(); pool.resize(pool.size() + k); return base; };
    auto put_nodes = [&](const std::vector<std::vector<Digest>> &nodes) {
        std::vector<uint32_t> bases;
        for (auto &slot : nodes) { bases.push_back((uint32_t)pool.size()); pool.insert(pool.end(), slot.begin(), slot.end()); }
        return bases;
    };
    const uint32_t tv_base = reserve(nq);
    std::vector<uint32_t> fv_base;
    for (auto &l : P.layers) { it.fri_off.push_back(it.n_fri); fv_base.push_back(reserve(l.values.size())); it.n_fri += (uint32_t)l.values.size(); }
    const uint32_t cv_base = (uint32_t)pool.size();
    pool.insert(pool.end(), P.c_values.begin(), P.c_values.end());
    const std::vector<uint32_t> tn_bases = put_nodes(P.trace_nodes), cn_bases = put_nodes(P.c_nodes);
    std::vector<std::vector<uint32_t>> fn_bases;
    for (auto &l : P.layers) fn_bases.push_back(put_nodes(l.nodes));
    uint32_t next_slot = (uint32_t)pool.size();

    // FRI positions per layer (fri/verifier.rs:24-31)
    it.layer_aug.resize(P.layers.size());
    {
        std::vector<uint64_t> pos = it.t_positions;
        uint64_t domain = N;
        for (size_t d = 0; d < P.layers.size(); d++) {
            it.layer_aug[d] = fs::augmented_positions(pos, domain);
            pos = it.layer_aug[d];
            domain /= 4;
        }
    }
    it.plans.push_back(plan_verify_batch(it.t_positions, P.domain_depth, nq, tv_base, P.trace_nodes, tn_bases, next_slot));
    it.plans.push_back(plan_verify_batch(c_positions, P.c_depth, P.c_values.size(), cv_base, P.c_nodes, cn_bases, next_slot));
    for (size_t d = 0; d < P.layers.size(); d++)
        it.plans.push_back(plan_verify_batch(it.layer_aug[d], P.layers[d].depth, P.layers[d].values.size(), fv_base[d], P.layers[d].nodes, fn_bases[d], next_slot));
    pool.resize(next_slot);

    // ---- 4: constraints at z (verifier.rs:47-52, 79-97)
    it.z = fs::prng_vector(P.constraint_root.data(), 1)[0];
    fe program_hash_fe[2];
    memcpy(program_hash_fe, it.in.program_hash, 32);
    it.cc = fs::draw_constraint_coefficients(P.trace_root.data(), P.ctx_depth, P.loop_depth, P.stack_depth, it.inputs, it.outputs,
                                             fe_make(P.op_count, 0), program_hash_fe);
    static const int GROUP_DEG[6] = {2, 3, 4, 6, 7, 8};
    it.per_xpow = fs::periodic_at(fe_pow_u64(it.z, n / 16));
    for (int gi = 0; gi < 6; gi++) it.per_xpow.push_back(fe_pow_u64(it.z, (8 * n - 1) - (n - 1) * GROUP_DEG[gi]));

    // ---- 5: DEEP composition coefficients and the constraint evaluation opened at each trace position (verifier.rs:54-69)
    it.dc = fs::draw_composition_coefficients(P.constraint_root.data(), w);
    it.c_evals.resize(nq);
    for (int q = 0; q < nq; q++) {
        const uint64_t position = it.t_positions[q];
        const size_t leaf_idx = std::find(c_positions.begin(), c_positions.end(), position / 2) - c_positions.begin();
        // the reference fails here, before any root is compared: this verdict wins over every later check
        if (leaf_idx >= P.c_values.size()) return reject(it, "verification of constraint Merkle proof failed");
        memcpy(&it.c_evals[q], P.c_values[leaf_idx].data() + (position % 2) * 16, 16);
    }

    // ---- 6: FRI folding points (fri/verifier.rs:33-75)
    for (auto &l : P.layers) it.alphas.push_back(fs::prng_vector(l.root.data(), 1)[0]);
}

// the reference's checks in its order, on the device results; returns "" when the proof is accepted
std::string finish(const Item &it) {
    const ParsedProof &P = it.P;
    const uint64_t b = 1ULL << P.log_ext;
    auto root_ok = [&](size_t t, const Digest &root) { return it.plans[t].ok && it.roots[t] == root; };
    if (!root_ok(0, P.trace_root)) return "verification of trace Merkle proof failed";
    if (!root_ok(1, P.constraint_root)) return "verification of constraint Merkle proof failed";

    std::string fri_err;
    {
        if (P.layers.empty()) return "verification of low-degree proof failed: no FRI layers";
        std::vector<fe> evaluations = it.comp;
        std::vector<uint64_t> positions = it.t_positions;
        uint64_t domain_size = (1ULL << P.layers[0].depth) * 4;
        uint64_t max_degree_plus_1 = (7 * it.n - 1) + 1;          // get_composition_degree(n) + 1
        fe domain_root = host_root_of_unity(P.layers[0].depth + 2);
        for (size_t d = 0; d < P.layers.size() && fri_err.empty(); d++) {
            const FriLayerProof &layer = P.layers[d];
            const std::vector<uint64_t> aug = fs::augmented_positions(positions, domain_size);
            const uint64_t row_length = domain_size / 4;
            std::vector<fe> column_values;
            for (uint64_t p : positions) {
                const size_t idx = std::find(aug.begin(), aug.end(), p % row_length) - aug.begin();
                if (idx >= layer.values.size()) { fri_err = "layer values too short"; break; }
                column_values.push_back(layer.values[idx][p / row_length]);
            }
            if (!fri_err.empty()) break;
            bool same = evaluations.size() == column_values.size();
            for (size_t i = 0; same && i < evaluations.size(); i++) same = fe_eq(evaluations[i], column_values[i]);
            if (!same) { fri_err = "evaluations did not match column value at depth " + std::to_string(d); break; }
            if (!root_ok(2 + d, layer.root)) { fri_err = "verification of Merkle proof failed at layer " + std::to_string(d); break; }
            if (layer.values.size() < aug.size()) { fri_err = "layer values too short"; break; }
            evaluations.assign(it.folded.begin() + it.fri_off[d], it.folded.begin() + it.fri_off[d] + aug.size());
            for (int s = 0; s < 2; s++) domain_root = fe_sqr(domain_root);
            max_degree_plus_1 /= 4;
            domain_size /= 4;
            positions = aug;
        }
        if (fri_err.empty()) {
            for (size_t i = 0; i < positions.size(); i++)
                if (positions[i] >= P.rem_values.size() || !fe_eq(P.rem_values[positions[i]], evaluations[i])) {
                    fri_err = "remainder values are inconsistent with values of the last column";
                    break;
                }
        }
        if (fri_err.empty()) {                                      // verify_remainder (fri/verifier.rs:97-131)
            const std::vector<fe> &rem = P.rem_values;
            if (max_degree_plus_1 > rem.size()) fri_err = "remainder degree is greater than number of remainder values";
            else {
                std::vector<fe> xs, ys;
                fe xpow = fe_make(1, 0);
                for (size_t i = 0; i < rem.size(); i++) {
                    if (i % b != 0) { xs.push_back(xpow); ys.push_back(rem[i]); }
                    xpow = fe_mul(xpow, domain_root);
                }
                if (max_degree_plus_1 > xs.size()) fri_err = "remainder degree is greater than number of remainder values";
                else if (!remainder_is_low_degree(xs, ys, (size_t)max_degree_plus_1))
                    fri_err = "remainder is not a valid degree " + std::to_string(max_degree_plus_1 - 1) + " polynomial";
            }
        }
    }
    if (!fri_err.empty()) return "verification of low-degree proof failed: " + fri_err;
    return "";
}

// Host image of everything a group uploads: sections 256-byte aligned, so that any of them can be read as fe / uint4 / structs.
struct Blob {
    std::vector<uint8_t> b;
    size_t reserve(size_t bytes) { const size_t o = (b.size() + 255) & ~(size_t)255; b.resize(o + bytes); return o; }
    size_t put(const void *p, size_t bytes) { const size_t o = reserve(bytes); if (bytes) memcpy(b.data() + o, p, bytes); return o; }
    template <typename T> size_t put(const std::vector<T> &v) { return put(v.data(), v.size() * sizeof(T)); }
};

size_t aligned(size_t x) { return (x + 255) & ~(size_t)255; }

// device bytes of one prepared proof in a group (the sections of run_group, without their alignment)
size_t item_bytes(const Item &it) {
    size_t ops = 0, levels = 0;
    for (auto &pl : it.plans) { ops += pl.ops.size(); levels += pl.level_start.size() + 1; }
    const size_t nq = it.nq, w = it.w, T = it.cc.coefA.size(), nb = it.cc.n_boundary_regs;
    return w * nq * 16 + (size_t)it.n_fri * (64 + 8 + 4 + 4 + 16) + (it.pool.size() + it.plans.size()) * 32 + ops * 4 + levels * 4 +
           it.plans.size() * sizeof(TreeDesc) + nq * (8 + 4 + 16 + 16) + 4 * w * 16 + 2 * T * 16 + 29 * 16 + 4 * nb * 16 +
           it.alphas.size() * 16 + sizeof(AtZDesc) + sizeof(ComposeDesc) + sizeof(FoldDesc) + 128 * w * 16 + 128 * 16 + 16;
}

// the device phase of one group: one upload, one launch per stage for the whole group, one download, one synchronise
void run_group(Context &c, const std::vector<Item *> &g, float *ms) {
    const int K = (int)g.size();
    // register shapes (ctx, loop, stack depth) and widths, in order of first appearance
    std::vector<std::array<int, 3>> shapes;
    std::vector<int> shape_of(K), widths;
    for (int i = 0; i < K; i++) {
        const std::array<int, 3> s{g[i]->P.ctx_depth, g[i]->P.loop_depth, g[i]->P.stack_depth};
        shape_of[i] = (int)(std::find(shapes.begin(), shapes.end(), s) - shapes.begin());
        if (shape_of[i] == (int)shapes.size()) shapes.push_back(s);
        if (std::find(widths.begin(), widths.end(), g[i]->w) == widths.end()) widths.push_back(g[i]->w);
    }
    // global pool of digests: [trace leaves, width by width | FRI leaves | per proof: the rest of its local pool | one root per plan]
    std::vector<uint32_t> tleaf(K), fleaf(K), rest(K), root0(K), qfirst(K), ffirst(K);
    std::vector<uint32_t> width_leaf0, width_rows;
    uint32_t slots = 0, Q = 0, F = 0, n_trees = 0;
    for (int wv : widths) {
        width_leaf0.push_back(slots);
        for (int i = 0; i < K; i++) if (g[i]->w == wv) { tleaf[i] = slots; slots += g[i]->nq; }
        width_rows.push_back(slots - width_leaf0.back());
    }
    for (int i = 0; i < K; i++) { fleaf[i] = slots; ffirst[i] = F; slots += g[i]->n_fri; F += g[i]->n_fri; qfirst[i] = Q; Q += g[i]->nq; }
    for (int i = 0; i < K; i++) { rest[i] = slots; slots += (uint32_t)g[i]->pool.size() - g[i]->nq - g[i]->n_fri; }
    const uint32_t roots_slot = slots;
    for (int i = 0; i < K; i++) { root0[i] = roots_slot + n_trees; n_trees += (uint32_t)g[i]->plans.size(); }

    Blob up;
    // opened trace rows, column-major per width: column j of width group v holds the rows of all its proofs, proof after proof
    std::vector<size_t> rows_off;
    for (size_t v = 0; v < widths.size(); v++) {
        const int wv = widths[v];
        const size_t R = width_rows[v];
        rows_off.push_back(up.reserve((size_t)wv * R * 16));
        fe *rows = (fe *)(up.b.data() + rows_off.back());
        for (int i = 0; i < K; i++) {
            if (g[i]->w != wv) continue;
            const size_t q0 = tleaf[i] - width_leaf0[v];
            for (int q = 0; q < g[i]->nq; q++)
                for (int j = 0; j < wv; j++) rows[(size_t)j * R + q0 + q] = g[i]->P.trace_evaluations[q][j];
        }
    }
    // opened FRI rows and what their folds need
    const size_t fri_rows_off = up.reserve((size_t)F * 64), fri_pos_off = up.reserve((size_t)F * 8), fri_layer_off = up.reserve((size_t)F * 4),
                 fri_proof_off = up.reserve((size_t)F * 4);
    {
        fe *rows = (fe *)(up.b.data() + fri_rows_off);
        unsigned long long *pos = (unsigned long long *)(up.b.data() + fri_pos_off);
        unsigned *layer = (unsigned *)(up.b.data() + fri_layer_off), *proof = (unsigned *)(up.b.data() + fri_proof_off);
        for (int i = 0; i < K; i++) {
            size_t t = ffirst[i];
            for (size_t d = 0; d < g[i]->P.layers.size(); d++)
                for (size_t j = 0; j < g[i]->P.layers[d].values.size(); j++, t++) {
                    for (int k = 0; k < 4; k++) rows[4 * t + k] = g[i]->P.layers[d].values[j][k];
                    pos[t] = j < g[i]->layer_aug[d].size() ? g[i]->layer_aug[d][j] : 0;
                    layer[t] = (unsigned)d;
                    proof[t] = (unsigned)i;
                }
        }
    }
    // per query: position, proof, opened constraint evaluation; per proof: z1 | z2 | cc1 | cc2, boundary coefficients, folding points
    std::vector<unsigned long long> positions;
    std::vector<unsigned> qproof;
    std::vector<fe> c_evals;
    std::vector<size_t> zs_off(K), bc_off(K), alpha_off(K);
    for (int i = 0; i < K; i++) {
        positions.insert(positions.end(), g[i]->t_positions.begin(), g[i]->t_positions.end());
        qproof.insert(qproof.end(), g[i]->nq, (unsigned)i);
        c_evals.insert(c_evals.end(), g[i]->c_evals.begin(), g[i]->c_evals.end());
    }
    const size_t pos_off = up.put(positions), qproof_off = up.put(qproof), cev_off = up.put(c_evals);
    for (int i = 0; i < K; i++) {
        const Item &it = *g[i];
        std::vector<fe> v(it.P.z1);
        v.insert(v.end(), it.P.z2.begin(), it.P.z2.end());
        v.insert(v.end(), it.dc.trace1.begin(), it.dc.trace1.end());
        v.insert(v.end(), it.dc.trace2.begin(), it.dc.trace2.end());
        zs_off[i] = up.put(v);
        v.assign(it.cc.bAi.begin(), it.cc.bAi.end());
        v.insert(v.end(), it.cc.bBi.begin(), it.cc.bBi.end());
        v.insert(v.end(), it.cc.bAf.begin(), it.cc.bAf.end());
        v.insert(v.end(), it.cc.bBf.begin(), it.cc.bBf.end());
        bc_off[i] = up.put(v);
        alpha_off[i] = up.put(it.alphas);
    }
    // constraint kernel inputs per shape, proof after proof: coefA | coefB (coef_stride 2 T), periodic | xpow (override_stride 29)
    std::vector<size_t> coef_off, px_off;
    std::vector<int> shape_count(shapes.size(), 0), shape_pos(K);
    for (size_t s = 0; s < shapes.size(); s++) {
        std::vector<fe> coef, px;
        for (int i = 0; i < K; i++) {
            if (shape_of[i] != (int)s) continue;
            shape_pos[i] = shape_count[s]++;
            coef.insert(coef.end(), g[i]->cc.coefA.begin(), g[i]->cc.coefA.end());
            coef.insert(coef.end(), g[i]->cc.coefB.begin(), g[i]->cc.coefB.end());
            px.insert(px.end(), g[i]->per_xpow.begin(), g[i]->per_xpow.end());
        }
        coef_off.push_back(up.put(coef));
        px_off.push_back(up.put(px));
    }
    // Merkle plans, remapped from each proof's local pool to the global one; each root goes to its slot after the pool
    std::vector<uint32_t> ops, level_start;
    std::vector<TreeDesc> trees;
    for (int i = 0; i < K; i++) {
        const Item &it = *g[i];
        const uint32_t nq = it.nq, nf = it.n_fri;
        auto slot = [&](uint32_t s) { return s < nq ? tleaf[i] + s : s < nq + nf ? fleaf[i] + (s - nq) : rest[i] + (s - nq - nf); };
        for (size_t t = 0; t < it.plans.size(); t++) {
            const MerklePlan &pl = it.plans[t];
            TreeDesc td{(uint32_t)(ops.size() / 3), 0, (uint32_t)level_start.size(), 0};
            if (pl.ok) {
                td.n_levels = (uint32_t)pl.level_start.size() - 1;
                for (size_t o = 0; o < pl.ops.size(); o++)
                    ops.push_back(o % 3 == 2 && pl.ops[o] == pl.root_slot ? root0[i] + (uint32_t)t : slot(pl.ops[o]));
                level_start.insert(level_start.end(), pl.level_start.begin(), pl.level_start.end());
            } else {
                level_start.push_back(0);
            }
            trees.push_back(td);
        }
    }
    const size_t ops_off = up.put(ops), ls_off = up.put(level_start), trees_off = up.put(trees);

    // the device allocation: [upload: sections above | descriptors | pool up to its roots] [download: roots | composition | folds] [work]
    const size_t atz_off = up.reserve(K * sizeof(AtZDesc)), cd_off = up.reserve(K * sizeof(ComposeDesc)), fd_off = up.reserve(K * sizeof(FoldDesc));
    const size_t pool_off = up.reserve((size_t)roots_slot * 32);
    const size_t up_bytes = up.b.size();
    const size_t down_bytes = (size_t)n_trees * 32 + (size_t)Q * 16 + (size_t)F * 16;
    size_t slab_elems = 0;
    std::vector<size_t> slab0(shapes.size()), tev0(shapes.size());
    for (size_t s = 0; s < shapes.size(); s++) { slab0[s] = slab_elems; slab_elems += (size_t)shape_count[s] * 128 * (15 + shapes[s][0] + shapes[s][1] + shapes[s][2]); }
    for (size_t s = 0, e = 0; s < shapes.size(); s++) { tev0[s] = e; e += (size_t)shape_count[s] * 128; }
    const size_t work_off = aligned(up_bytes + down_bytes);
    const size_t slab_off = work_off, tev_off = aligned(slab_off + slab_elems * 16), cz_off = aligned(tev_off + (size_t)K * 128 * 16);
    DevBuf dev(cz_off + (size_t)K * 16);
    uint8_t *base = dev.as<uint8_t>();
    fe *slab = (fe *)(base + slab_off), *tev = (fe *)(base + tev_off), *c_at_z = (fe *)(base + cz_off);
    uint4 *pool = (uint4 *)(base + pool_off);
    fe *comp = (fe *)(base + up_bytes + (size_t)n_trees * 32), *folded = comp + Q;

    // descriptors: the pointers are into `dev`
    {
        AtZDesc *atz = (AtZDesc *)(up.b.data() + atz_off);
        ComposeDesc *cd = (ComposeDesc *)(up.b.data() + cd_off);
        FoldDesc *fd = (FoldDesc *)(up.b.data() + fd_off);
        for (int i = 0; i < K; i++) {
            const Item &it = *g[i];
            const int s = shape_of[i];
            const size_t v = std::find(widths.begin(), widths.end(), it.w) - widths.begin();
            const fe *zs = (const fe *)(base + zs_off[i]);
            const fe root_n = host_root_of_unity(it.log_N - it.P.log_ext);
            AtZDesc &a = atz[i];
            a.z1 = zs; a.bcoef = (const fe *)(base + bc_off[i]);
            a.t_at_z = tev + tev0[s] + (size_t)shape_pos[i] * 128;
            a.slab = slab + slab0[s] + (size_t)shape_pos[i] * 128 * it.w;
            a.KiA = it.cc.KiA; a.KiB = it.cc.KiB; a.KfA = it.cc.KfA; a.KfB = it.cc.KfB;
            a.z = it.z; a.x_last = host_inv(root_n);
            a.n = it.n; a.w = it.w; a.nb = it.cc.n_boundary_regs;
            ComposeDesc &d = cd[i];
            d.rows = (const fe *)(base + rows_off[v]) + (tleaf[i] - width_leaf0[v]);
            d.row_stride = width_rows[v];
            d.zs = zs;
            d.c_at_z = c_at_z + i;
            d.z = it.z; d.zg = fe_mul(it.z, root_n);
            d.t1_degree = it.dc.t1_degree; d.t2_degree = it.dc.t2_degree; d.k_constraints = it.dc.constraints;
            d.twN = c.twiddle(it.log_N, false);
            d.inc = (8 * it.n - 1 - it.n) - (it.n - 2);               // get_incremental_trace_degree: composition degree - (n - 2), composition degree = 7n - 1
            d.first = qfirst[i];
            d.w = it.w;
            fd[i].inv_root = c.twiddle(it.log_N, true);
            fd[i].alphas = (const fe *)(base + alpha_off[i]);
        }
        // the pool below the roots: leaves are computed on the device, the rest of each proof's local pool comes from the proof
        uint8_t *pl = up.b.data() + pool_off;
        for (int i = 0; i < K; i++) {
            const Item &it = *g[i];
            const size_t skip = (size_t)it.nq + it.n_fri;
            memcpy(pl + (size_t)rest[i] * 32, it.pool.data() + skip, (it.pool.size() - skip) * 32);
        }
    }

    EventTimer timer(c.stream, ms);
    c.staging.ensure(up_bytes + down_bytes);
    uint8_t *pinned = (uint8_t *)c.staging.p;
    memcpy(pinned, up.b.data(), up_bytes);
    DG_CUDA(cudaMemcpyAsync(base, pinned, up_bytes, cudaMemcpyHostToDevice, c.stream));
    DG_CUDA(cudaMemsetAsync(slab, 0, slab_elems * 16, c.stream));
    const AtZDesc *atz_dev = (const AtZDesc *)(base + atz_off);

    // ---- leaves: trace rows (one launch per width), FRI rows (one launch)
    for (size_t v = 0; v < widths.size(); v++)
        if (width_rows[v]) hash_rows_plain(c, (const fe *)(base + rows_off[v]), pool + 2 * (size_t)width_leaf0[v], widths[v], width_rows[v]);
    if (F) hash64_contiguous(c, base + fri_rows_off, pool + 2 * (size_t)fleaf[0], F);
    // ---- all Merkle plans of all proofs, one block per tree
    merkle_verify_kernel<<<n_trees, 128, 0, c.stream>>>(pool, (const uint32_t *)(base + ops_off), (const uint32_t *)(base + ls_off),
                                                        (const TreeDesc *)(base + trees_off)); c.launches++;
    DG_CUDA(cudaGetLastError());
    // ---- transition constraints at z: the deep values as a 128-step stand-in trace, one constraint launch per register shape
    deep_rows_to_slab_kernel<<<K, 128, 0, c.stream>>>(atz_dev); c.launches++;
    DG_CUDA(cudaGetLastError());
    for (size_t s = 0; s < shapes.size(); s++) {
        const int ctx_depth = shapes[s][0], loop_depth = shapes[s][1], stack_depth = shapes[s][2], w = 15 + ctx_depth + loop_depth + stack_depth;
        const int i0 = (int)(std::find(shape_of.begin(), shape_of.end(), (int)s) - shape_of.begin());
        const size_t T = g[i0]->cc.coefA.size();
        AirParams A;
        memset(&A, 0, sizeof A);
        A.w = w; A.ctx_depth = ctx_depth; A.loop_depth = loop_depth; A.stack_depth = stack_depth;
        A.cl = std::max(ctx_depth, 1); A.ll = std::max(loop_depth, 1); A.sl = std::max(stack_depth, 8);
        A.log_n = 7; A.log_blowup = 3;
        A.ext = slab + slab0[s]; A.col_stride = 128; A.ext_stride = 128ULL * w;
        A.c8_base = 0; A.num_c8 = 1;
        A.t_ev = tev + tev0[s]; A.t_ev_stride = 128;
        const fe *coef = (const fe *)(base + coef_off[s]), *px = (const fe *)(base + px_off[s]);
        A.periodic = px;                                            // unused in verify mode (per_override is set)
        A.coefA = coef; A.coefB = coef + T; A.coef_stride = 2 * T;
        A.twN = c.twiddle(10, false);
        A.violation = nullptr;
        A.verify_mode = 1;
        A.per_override = px; A.xpow_override = px + 23; A.override_stride = 29;
        launch_constraint_eval(c, A, shape_count[s]);
    }
    // ---- C(z) per proof, then the DEEP composition at every query and every FRI row folded
    verify_at_z_kernel<<<(K + 127) / 128, 128, 0, c.stream>>>(atz_dev, K, c_at_z); c.launches++;
    DG_CUDA(cudaGetLastError());
    if (Q) {
        compose_at_queries_batch_kernel<<<(Q + 63) / 64, 64, 0, c.stream>>>((const ComposeDesc *)(base + cd_off), (const unsigned *)(base + qproof_off), Q,
                                                                            (const unsigned long long *)(base + pos_off), (const fe *)(base + cev_off), comp);
        c.launches++;
        DG_CUDA(cudaGetLastError());
    }
    if (F) {
        fri_fold_rows_batch_kernel<<<(F + 127) / 128, 128, 0, c.stream>>>(
            (const fe *)(base + fri_rows_off), (const unsigned long long *)(base + fri_pos_off), (const unsigned *)(base + fri_layer_off),
            (const unsigned *)(base + fri_proof_off), F, (const FoldDesc *)(base + fd_off), host_inv(host_root_of_unity(2)), host_inv(fe_make(4, 0)), folded);
        c.launches++;
        DG_CUDA(cudaGetLastError());
    }

    // ---- results back: the roots, the composition values and the folds
    uint8_t *down = pinned + up_bytes;
    DG_CUDA(cudaMemcpyAsync(down, base + up_bytes, down_bytes, cudaMemcpyDeviceToHost, c.stream));
    timer.stop();
    DG_CUDA(cudaStreamSynchronize(c.stream));
    const Digest *roots = (const Digest *)down;
    const fe *cv = (const fe *)(down + (size_t)n_trees * 32), *fv = cv + Q;
    for (int i = 0; i < K; i++) {
        Item &it = *g[i];
        it.roots.assign(roots + (root0[i] - roots_slot), roots + (root0[i] - roots_slot) + it.plans.size());
        it.comp.assign(cv + qfirst[i], cv + qfirst[i] + it.nq);
        it.folded.assign(fv + ffirst[i], fv + ffirst[i] + it.n_fri);
    }
}

// Proofs per group: a fixed device-memory budget, at most 65535 proofs of one shape (the constraint launch puts them on the grid's y
// dimension) and $DG_BATCH_GROUP.
const size_t GROUP_BYTES = (size_t)512 << 20;

}  // namespace

void verify_proofs(Context &c, const std::vector<VerifyRequest> &req, std::vector<int> &status, std::vector<std::string> &messages,
                   dg_verify_stats_t *stats) {
    const unsigned long long launches0 = c.launches;
    size_t cap = (size_t)-1;
    if (const char *e = getenv("DG_BATCH_GROUP")) {
        const long long v = atoll(e);
        DG_REQUIRE(v >= 1, "DG_BATCH_GROUP must be a positive integer");
        cap = (size_t)v;
    }
    std::vector<Item> items(req.size());
    // ---- prepare, proof by proof in input order (the Fiat-Shamir callbacks see the proofs one after the other)
    for (size_t i = 0; i < req.size(); i++) {
        Item &it = items[i];
        it.in = req[i];
        try { prepare(it); }
        catch (const Error &e) { it.decided = true; it.status = e.code; it.message = e.what(); }
        catch (const std::exception &e) { it.decided = true; it.status = DG_ERR_INVALID; it.message = e.what(); }
    }
    // ---- device, group by group
    float total_ms = 0;
    uint32_t groups = 0;
    std::vector<Item *> g;
    std::map<std::array<int, 3>, size_t> per_shape;
    size_t bytes = 0;
    auto flush = [&]() {
        if (g.empty()) return;
        ArenaScope arena_scope;
        float ms = 0;
        run_group(c, g, stats ? &ms : nullptr);
        total_ms += ms;
        groups++;
        g.clear(); per_shape.clear(); bytes = 0;
    };
    for (Item &it : items) {
        if (it.decided) continue;
        const size_t b = item_bytes(it);
        const std::array<int, 3> shape{it.P.ctx_depth, it.P.loop_depth, it.P.stack_depth};
        if (!g.empty() && (bytes + b > GROUP_BYTES || g.size() >= cap || per_shape[shape] >= 65535)) flush();
        g.push_back(&it);
        per_shape[shape]++;
        bytes += b;
    }
    flush();
    // ---- finish, proof by proof
    status.assign(req.size(), DG_OK);
    messages.assign(req.size(), std::string());
    for (size_t i = 0; i < items.size(); i++) {
        Item &it = items[i];
        if (!it.decided) {
            it.message = finish(it);
            it.status = it.message.empty() ? DG_OK : DG_ERR_REJECTED;
        }
        status[i] = it.status;
        messages[i] = it.message;
    }
    if (stats) { stats->total_ms = total_ms; stats->kernel_launches = c.launches - launches0; stats->groups = groups; }
}

}  // namespace dg
