// ORACLE -- TEST INFRASTRUCTURE ONLY.  Never linked into or called by the product path.
//
// CPU restatement (single thread) of the reference's STARK prover and verifier:
//   TraceTable        /root/reference/src/stark/trace/trace_table.rs:23-261
//   ConstraintTable   /root/reference/src/stark/constraints/constraint_table.rs:18-88
//   ConstraintPoly    /root/reference/src/stark/constraints/constraint_poly.rs:13-60
//   prove()           /root/reference/src/stark/prover.rs:17-201
//   fri::reduce / build_proof   /root/reference/src/stark/fri/prover.rs:11-95, fri/utils.rs:4-21
//   PoW / positions   /root/reference/src/stark/utils/proof_of_work.rs:4-56, utils/mod.rs:13-53
//   StarkProof + bincode layout   /root/reference/src/stark/proof.rs:10-77, fri/mod.rs:17-30, options.rs:15-23,97-125
//                      (bincode 1.3.1 defaults restated: LE fixed ints, u64 length prefixes; byte layout is
//                       PARITY UNPINNED by the reference -- no test pins proof bytes)
//   verify()          /root/reference/src/stark/verifier.rs:11-162, fri/verifier.rs:11-155
#ifndef ORACLE_STARK_H
#define ORACLE_STARK_H

#include "air.h"
#include <string>

namespace oracle {

struct ProofOptions {  // options.rs:16-23 (hash_fn fixed to blake3 = id 0 unless overridden for tests)
    size_t extension_factor = 32, num_queries = 50;
    uint32_t grinding_factor = 20;
    HashFn hash_fn = blake3;
};

struct FriLayer { Digest root; std::vector<quartic::Q> values; std::vector<std::vector<Digest>> nodes; uint8_t depth; };
struct FriProof { std::vector<FriLayer> layers; Digest rem_root; std::vector<u128> rem_values; };

struct StarkProof {
    Digest trace_root;
    uint8_t domain_depth, ctx_depth, loop_depth, stack_depth; uint32_t op_count;   // TraceInfo
    std::vector<std::vector<Digest>> trace_nodes;
    std::vector<std::vector<u128>> trace_evaluations;
    Digest constraint_root;
    BatchMerkleProof constraint_proof;
    std::vector<u128> trace_at_z1, trace_at_z2;    // DeepValues
    FriProof degree_proof;
    uint64_t pow_nonce;
    uint8_t opt_ext_log2, opt_num_queries, opt_grinding, opt_hash_id;

    size_t domain_size() const { return (size_t)1 << domain_depth; }
    size_t extension_factor() const { return (size_t)1 << opt_ext_log2; }
    size_t trace_length() const { return domain_size() / extension_factor(); }
};

// ---- bincode 1.3.1 default-config writer / reader -------------------------------------------------------------
struct Writer {
    std::vector<uint8_t> b;
    void u8(uint8_t v) { b.push_back(v); }
    void u32(uint32_t v) { for (int i = 0; i < 4; i++) b.push_back((uint8_t)(v >> (8 * i))); }
    void u64v(uint64_t v) { for (int i = 0; i < 8; i++) b.push_back((uint8_t)(v >> (8 * i))); }
    void f(u128 v) { for (int i = 0; i < 16; i++) b.push_back((uint8_t)(v >> (8 * i))); }
    void d(const Digest &x) { b.insert(b.end(), x.begin(), x.end()); }
    void dvec(const std::vector<Digest> &v) { u64v(v.size()); for (auto &x : v) d(x); }
    void dvv(const std::vector<std::vector<Digest>> &v) { u64v(v.size()); for (auto &x : v) dvec(x); }
    void fvec(const std::vector<u128> &v) { u64v(v.size()); for (auto x : v) f(x); }
};
static inline std::vector<uint8_t> serialize(const StarkProof &p) {
    Writer w;
    w.d(p.trace_root);
    w.u8(p.domain_depth); w.u8(p.ctx_depth); w.u8(p.loop_depth); w.u8(p.stack_depth); w.u32(p.op_count);
    w.dvv(p.trace_nodes);
    w.u64v(p.trace_evaluations.size()); for (auto &r : p.trace_evaluations) w.fvec(r);
    w.d(p.constraint_root);
    w.dvec(p.constraint_proof.values); w.dvv(p.constraint_proof.nodes); w.u8(p.constraint_proof.depth);
    w.fvec(p.trace_at_z1); w.fvec(p.trace_at_z2);
    w.u64v(p.degree_proof.layers.size());
    for (auto &l : p.degree_proof.layers) {
        w.d(l.root);
        w.u64v(l.values.size()); for (auto &q : l.values) for (int k = 0; k < 4; k++) w.f(q.v[k]);
        w.dvv(l.nodes); w.u8(l.depth);
    }
    w.d(p.degree_proof.rem_root); w.fvec(p.degree_proof.rem_values);
    w.u64v(p.pow_nonce);
    w.u8(p.opt_ext_log2); w.u8(p.opt_num_queries); w.u8(p.opt_grinding); w.u8(p.opt_hash_id);
    return w.b;
}
struct Reader {
    const uint8_t *p, *end;
    Reader(const uint8_t *b, size_t n) : p(b), end(b + n) {}
    void need(size_t n) { if ((size_t)(end - p) < n) throw std::runtime_error("proof truncated"); }
    uint8_t u8() { need(1); return *p++; }
    uint32_t u32() { need(4); uint32_t v = 0; for (int i = 0; i < 4; i++) v |= (uint32_t)p[i] << (8 * i); p += 4; return v; }
    uint64_t u64v() { need(8); uint64_t v = 0; for (int i = 0; i < 8; i++) v |= (uint64_t)p[i] << (8 * i); p += 8; return v; }
    u128 f() { need(16); u128 v = 0; for (int i = 0; i < 16; i++) v |= (u128)p[i] << (8 * i); p += 16; return v; }
    Digest d() { need(32); Digest x; memcpy(x.data(), p, 32); p += 32; return x; }
    size_t len() { uint64_t n = u64v(); if (n > (1u << 26)) throw std::runtime_error("bad length"); return (size_t)n; }
    std::vector<Digest> dvec() { size_t n = len(); std::vector<Digest> v(n); for (auto &x : v) x = d(); return v; }
    std::vector<std::vector<Digest>> dvv() { size_t n = len(); std::vector<std::vector<Digest>> v(n); for (auto &x : v) x = dvec(); return v; }
    std::vector<u128> fvec() { size_t n = len(); std::vector<u128> v(n); for (auto &x : v) x = f(); return v; }
};
static inline StarkProof deserialize(const uint8_t *bytes, size_t n) {
    Reader r(bytes, n);
    StarkProof p;
    p.trace_root = r.d();
    p.domain_depth = r.u8(); p.ctx_depth = r.u8(); p.loop_depth = r.u8(); p.stack_depth = r.u8(); p.op_count = r.u32();
    p.trace_nodes = r.dvv();
    { size_t k = r.len(); p.trace_evaluations.resize(k); for (auto &row : p.trace_evaluations) row = r.fvec(); }
    p.constraint_root = r.d();
    p.constraint_proof.values = r.dvec(); p.constraint_proof.nodes = r.dvv(); p.constraint_proof.depth = r.u8();
    p.trace_at_z1 = r.fvec(); p.trace_at_z2 = r.fvec();
    size_t nl = r.len();
    p.degree_proof.layers.resize(nl);
    for (auto &l : p.degree_proof.layers) {
        l.root = r.d();
        size_t nv = r.len(); l.values.resize(nv);
        for (auto &q : l.values) for (int k = 0; k < 4; k++) q.v[k] = r.f();
        l.nodes = r.dvv(); l.depth = r.u8();
    }
    p.degree_proof.rem_root = r.d(); p.degree_proof.rem_values = r.fvec();
    p.pow_nonce = r.u64v();
    p.opt_ext_log2 = r.u8(); p.opt_num_queries = r.u8(); p.opt_grinding = r.u8(); p.opt_hash_id = r.u8();
    if (r.p != r.end) throw std::runtime_error("trailing bytes in proof");
    return p;
}

// ---- stark/utils ----------------------------------------------------------------------------------------------
static inline size_t get_composition_degree(size_t n) { return (MAX_CONSTRAINT_DEGREE - 1) * n - 1; }
static inline size_t get_incremental_trace_degree(size_t n) { return get_composition_degree(n) - (n - 2); }

// utils/mod.rs:25-44
static inline std::vector<size_t> compute_query_positions(const uint8_t seed[32], size_t domain_size, size_t ext, size_t num_queries) {
    ChaChaRng rng(seed);
    std::vector<size_t> result;
    for (int t = 0; t < 1000; t++) {
        size_t value = (size_t)sample_usize(rng, domain_size);
        if (value % ext == 0) continue;
        if (std::find(result.begin(), result.end(), value) != result.end()) continue;
        result.push_back(value);
        if (result.size() >= num_queries) break;
    }
    if (result.size() < num_queries) throw std::runtime_error("could not generate enough query positions");
    return result;
}
// utils/mod.rs:46-53
static inline std::vector<size_t> map_trace_to_constraint_positions(const std::vector<size_t> &positions) {
    std::vector<size_t> r;
    for (size_t p : positions) { size_t cp = p / 2; if (std::find(r.begin(), r.end(), cp) == r.end()) r.push_back(cp); }
    return r;
}
// proof_of_work.rs:4-32 ; `after` > 0 (forged proofs only) returns the first valid nonce above it
static inline uint64_t find_pow_nonce(const uint8_t seed[32], uint32_t grinding, HashFn hash, uint8_t out_seed[32], uint64_t after = 0) {
    uint8_t in[64];
    memset(in, 0, 64);
    memcpy(in, seed, 32);
    uint64_t nonce = after;
    for (;;) {
        nonce += 1;
        for (int i = 0; i < 8; i++) in[32 + i] = (uint8_t)(nonce >> (8 * i));
        hash(in, 64, out_seed);
        uint64_t o0 = 0;
        for (int i = 0; i < 8; i++) o0 |= (uint64_t)out_seed[i] << (8 * i);
        uint32_t tz = o0 == 0 ? 64 : (uint32_t)__builtin_ctzll(o0);
        if (tz >= grinding) break;
    }
    return nonce;
}
// proof_of_work.rs:34-56
static inline bool verify_pow_nonce(const uint8_t seed[32], uint64_t nonce, uint32_t grinding, HashFn hash, uint8_t out_seed[32]) {
    uint8_t in[64];
    memset(in, 0, 64);
    memcpy(in, seed, 32);
    for (int i = 0; i < 8; i++) in[32 + i] = (uint8_t)(nonce >> (8 * i));
    hash(in, 64, out_seed);
    uint64_t o0 = 0;
    for (int i = 0; i < 8; i++) o0 |= (uint64_t)out_seed[i] << (8 * i);
    uint32_t tz = o0 == 0 ? 64 : (uint32_t)__builtin_ctzll(o0);
    return tz >= grinding;
}

// ---- forged proofs (tests only; the reference has no such switch) ----------------------------------------------
// One value is changed before it is committed.  Every root, Fiat-Shamir draw, PoW nonce, query position and opening after it is
// derived from the changed value, so the proof passes the Merkle and PoW checks and only the verifier's algebraic checks can reject it.
struct Forgery {
    enum Kind {
        none = 0,
        transition,         // a: trace row whose top user-stack value gets +1, breaking the transitions into and out of it; stage 3's
                            //    assertion and stage 4's degree check are skipped
        op_count,           // a: the op count in the proof and in the boundary constraint at the last step (stage 4 check skipped)
        constraint_offset,  // a: added to the combined constraint polynomial before its LDE and tree
        deep_value,         // a: register, b: 0 = its value at z, 1 = at z * g; gets +1 and is used so in the DEEP composition
        fri_offset,         // a: FRI layer whose values all get +1 before its tree; a = number of layers: the remainder
        fri_alpha,          // a: FRI layer folded at prng(root) + 1
        remainder_point,    // +1 on the last non-skipped remainder value that no query opens (retried downwards until one is found)
        layers,             // a: folds beyond (> 0) or short of (< 0) the prover's count; everything stays honest
        remainder_cut,      // only the first (degree bound + a) remainder values are sent; the nonce is the first valid one whose
                            //    queries open none of the cut values (the verifier hashes the remainder root only into the PoW seed)
    } kind = none;
    int64_t a = 0, b = 0;
};

// ---- FRI (fri/prover.rs, fri/utils.rs) -----------------------------------------------------------------------
static const size_t MAX_REMAINDER_LENGTH = 256;

static inline std::vector<Digest> hash_values(const std::vector<quartic::Q> &values, HashFn hash) {
    std::vector<Digest> r(values.size());
    const int T = fft::host_threads();
    #pragma omp parallel for num_threads(T) if (T > 1 && values.size() >= 4096)
    for (size_t i = 0; i < values.size(); i++) hash((const uint8_t *)values[i].v, 64, r[i].data());
    return r;
}
static inline std::vector<size_t> get_augmented_positions(const std::vector<size_t> &positions, size_t column_length) {
    size_t row_length = column_length / 4;
    std::vector<size_t> r;
    for (size_t p : positions) { size_t ap = p % row_length; if (std::find(r.begin(), r.end(), ap) == r.end()) r.push_back(ap); }
    return r;
}
// number of folds fri_reduce makes on a domain of this size: while (p_tree.leaves().len() * 4 > MAX_REMAINDER_LENGTH)
static inline size_t fri_fold_count(size_t domain_size) {
    size_t k = 0;
    for (; domain_size > MAX_REMAINDER_LENGTH; domain_size /= 4) k++;
    return k;
}
static inline void fri_reduce(const std::vector<u128> &evaluations, const std::vector<u128> &domain, HashFn hash,
                              std::vector<MerkleTree> &trees, std::vector<std::vector<quartic::Q>> &values,
                              const Forgery &forge = Forgery()) {
    const size_t folds = fri_fold_count(evaluations.size()) + (forge.kind == Forgery::layers ? forge.a : 0);
    auto commit = [&](std::vector<quartic::Q> &v) {         // the tree of layer trees.size() (the remainder after the last fold)
        if (forge.kind == Forgery::fri_offset && (size_t)forge.a == trees.size())
            for (auto &q : v) for (auto &x : q.v) x = field::add(x, 1);
        return MerkleTree(hash_values(v, hash), hash);
    };
    std::vector<quartic::Q> p_values = quartic::transpose(evaluations.data(), evaluations.size(), 1);
    MerkleTree p_tree = commit(p_values);
    while (trees.size() < folds) {
        size_t depth = trees.size();
        size_t stride = (size_t)1 << (2 * depth);
        std::vector<quartic::Q> xs = quartic::transpose(domain.data(), domain.size(), stride);
        std::vector<quartic::Q> polys = quartic::interpolate_batch(xs, p_values);
        u128 special_x = prng(p_tree.root().data());
        if (forge.kind == Forgery::fri_alpha && (size_t)forge.a == depth) special_x = field::add(special_x, 1);
        std::vector<u128> column = quartic::evaluate_batch(polys, special_x);
        trees.push_back(std::move(p_tree));
        values.push_back(std::move(p_values));
        p_values = quartic::transpose(column.data(), column.size(), 1);
        p_tree = commit(p_values);
    }
    trees.push_back(std::move(p_tree));
    values.push_back(std::move(p_values));
}
static inline FriProof fri_build_proof(const std::vector<MerkleTree> &trees, const std::vector<std::vector<quartic::Q>> &values,
                                       const std::vector<size_t> &positions_in) {
    std::vector<size_t> positions = positions_in;
    size_t domain_size = trees[0].values.size() * 4;
    FriProof fp;
    for (size_t i = 0; i + 1 < trees.size(); i++) {
        positions = get_augmented_positions(positions, domain_size);
        BatchMerkleProof proof = trees[i].prove_batch(positions);
        FriLayer l;
        l.root = trees[i].root();
        for (size_t p : positions) l.values.push_back(values[i][p]);
        l.nodes = proof.nodes;
        l.depth = proof.depth;
        fp.layers.push_back(std::move(l));
        domain_size /= 4;
    }
    const std::vector<quartic::Q> &last = values.back();
    size_t n = last.size();
    fp.rem_values.assign(n * 4, 0);
    for (size_t i = 0; i < n; i++)
        for (int k = 0; k < 4; k++) fp.rem_values[i + n * k] = last[i].v[k];
    fp.rem_root = trees.back().root();
    return fp;
}

// ---- prover ---------------------------------------------------------------------------------------------------
// Optional capture of intermediate values (used by GPU stage-parity tests).
struct ProverTrace {
    bool keep_large = false;                          // keep extended trace etc. (small traces only)
    std::vector<std::vector<u128>> polys, extended;   // [w][n], [w][N]
    Digest trace_root, constraint_root;
    std::vector<u128> i_evals, f_evals, t_evals;      // constraint accumulators over E points
    std::vector<u128> constraint_poly;                // combined, E coefficients
    std::vector<u128> constraint_evals;               // N evaluations
    std::vector<u128> composition_poly;               // 8n coefficients
    std::vector<u128> composed_evals;                 // N evaluations
    u128 z = 0;
    std::vector<Digest> fri_roots;
    std::vector<u128> fri_alphas;
    uint64_t pow_nonce = 0;
    Digest pow_seed;
    std::vector<size_t> positions;
    double stage_ms[9] = {0};
};

static inline double now_ms();

static inline StarkProof prove(const std::vector<std::vector<u128>> &registers, size_t ctx_depth, size_t loop_depth,
                               const std::vector<u128> &inputs, const std::vector<u128> &outputs,
                               const ProofOptions &opt, ProverTrace *dbg = nullptr, const Forgery &forge = Forgery()) {
    const size_t w = registers.size();
    const size_t n = registers[0].size();
    const size_t b = opt.extension_factor;
    const size_t N = n * b;
    const HashFn hash = opt.hash_fn;
    if (b < 16 || b > 256 || (b & (b - 1))) throw std::runtime_error("invalid extension factor");
    if (n < 16 || (n & (n - 1))) throw std::runtime_error("trace length must be a power of two >= 16");
    const size_t decoder_width = 15 + ctx_depth + loop_depth;
    if (w <= decoder_width || w >= MAX_REGISTER_COUNT) throw std::runtime_error("invalid register count");
    const size_t stack_depth = w - decoder_width;
    const bool lax = forge.kind == Forgery::transition || forge.kind == Forgery::op_count;   // a false statement: skip the prover's checks
    double t0 = now_ms();

    // 1 ----- extend execution trace (prover.rs:22-27, trace_table.rs:143-169) --------------------
    u128 lde_root = field::get_root_of_unity(N);
    std::vector<u128> lde_domain = field::get_power_series(lde_root, N);
    std::vector<u128> lde_twiddles(lde_domain.begin(), lde_domain.begin() + N / 2);
    fft::permute(lde_twiddles.data(), lde_twiddles.size());

    u128 trace_root_w = field::get_root_of_unity(n);
    std::vector<u128> inv_twiddles = fft::get_inv_twiddles(trace_root_w, n);
    std::vector<std::vector<u128>> polys(registers);
    if (forge.kind == Forgery::transition) polys.at(decoder_width).at(forge.a) = field::add(polys[decoder_width][forge.a], 1);
    std::vector<std::vector<u128>> ext(w);
    const int T = fft::host_threads();
    if (T <= 1 || (size_t)T >= 2 * w) {                  // many more threads than columns: parallelism inside each transform instead
        for (size_t j = 0; j < w; j++) {
            polynom::interpolate_fft_twiddles(polys[j].data(), n, inv_twiddles.data(), true);
            ext[j].assign(N, 0);
            std::copy(polys[j].begin(), polys[j].end(), ext[j].begin());
            polynom::eval_fft_twiddles(ext[j].data(), N, lde_twiddles.data(), true);
        }
    } else {                                                 // one column per thread, each transform sequential as in the reference
        #pragma omp parallel for schedule(dynamic) num_threads(T)
        for (size_t j = 0; j < w; j++) {
            fft::fft_in_place(polys[j].data(), n, inv_twiddles.data(), 1, 1, 0);
            const u128 inv_len = field::inv((u128)n);
            for (size_t i = 0; i < n; i++) polys[j][i] = field::mul(polys[j][i], inv_len);
            fft::permute(polys[j].data(), n);
            ext[j].assign(N, 0);
            std::copy(polys[j].begin(), polys[j].end(), ext[j].begin());
            fft::fft_in_place(ext[j].data(), N, lde_twiddles.data(), 1, 1, 0);
            fft::permute(ext[j].data(), N);
        }
    }
    double t1 = now_ms(); if (dbg) dbg->stage_ms[0] = t1 - t0;

    // 2 ----- trace Merkle tree (trace_table.rs:174-185) ------------------------------------------
    std::vector<Digest> hashed_states(N);
    #pragma omp parallel num_threads(T) if (T > 1)
    {
        std::vector<u128> row(w);
        #pragma omp for
        for (size_t i = 0; i < N; i++) {
            for (size_t j = 0; j < w; j++) row[j] = ext[j][i];
            hash((const uint8_t *)row.data(), w * 16, hashed_states[i].data());
        }
    }
    MerkleTree trace_tree(std::move(hashed_states), hash);
    double t2 = now_ms(); if (dbg) dbg->stage_ms[1] = t2 - t1;

    // 3 ----- evaluate constraints (prover.rs:43-64) ----------------------------------------------
    TraceState last_state(ctx_depth, loop_depth, stack_depth);
    last_state.from_columns(ext, N - b);
    const size_t E = n * MAX_CONSTRAINT_DEGREE;
    const u128 op_count = forge.kind == Forgery::op_count ? (u128)forge.a : last_state.op_counter;
    Evaluator evaluator(n, MAX_CONSTRAINT_DEGREE, E, ctx_depth, loop_depth, stack_depth, trace_tree.root().data(),
                        last_state.sponge, op_count, inputs, outputs);
    std::vector<u128> i_ev(E), f_ev(E), t_ev(E);
    {
        const size_t stride = b / MAX_CONSTRAINT_DEGREE;
        std::string failure;                                 // first (lowest-step) failure, reported as the sequential loop would
        size_t failure_step = ~(size_t)0;
        #pragma omp parallel num_threads(T) if (T > 1)
        {
            TraceState cur(ctx_depth, loop_depth, stack_depth), nxt(ctx_depth, loop_depth, stack_depth);
            #pragma omp for schedule(static)
            for (size_t step = 0; step < E; step++) {
                const size_t i = step * stride;
                try {
                    cur.from_columns(ext, i);
                    nxt.from_columns(ext, (i + b) % N);
                    evaluator.evaluate_boundaries(cur, lde_domain[i], i_ev[step], f_ev[step]);
                    t_ev[step] = evaluator.evaluate_transition(cur, nxt, lde_domain[i], step, nullptr, !lax);
                } catch (const std::exception &e) {
                    #pragma omp critical
                    if (step < failure_step) { failure_step = step; failure = e.what(); }
                }
            }
        }
        if (failure_step != ~(size_t)0) throw std::runtime_error(failure);
    }
    if (dbg) { dbg->i_evals = i_ev; dbg->f_evals = f_ev; dbg->t_evals = t_ev; }
    double t3 = now_ms(); if (dbg) dbg->stage_ms[2] = t3 - t2;

    // 4 ----- combine into one constraint polynomial (constraint_table.rs:54-88) -------------------
    std::vector<u128> combined(E);
    {
        u128 comb_root = field::get_root_of_unity(E);
        std::vector<u128> inv_tw = fft::get_inv_twiddles(comb_root, E);
        polynom::interpolate_fft_twiddles(i_ev.data(), E, inv_tw.data(), true);
        polynom::syn_div_in_place(i_ev.data(), E, 1);
        combined = i_ev;
        polynom::interpolate_fft_twiddles(f_ev.data(), E, inv_tw.data(), true);
        u128 x_last = evaluator.get_x_at_last_step();
        polynom::syn_div_in_place(f_ev.data(), E, x_last);
        for (size_t k = 0; k < E; k++) combined[k] = field::add(combined[k], f_ev[k]);
        polynom::interpolate_fft_twiddles(t_ev.data(), E, inv_tw.data(), true);
        polynom::syn_div_expanded_in_place(t_ev.data(), E, n, &x_last, 1);
        for (size_t k = 0; k < E; k++) combined[k] = field::add(combined[k], t_ev[k]);
        // constraint_poly.rs:16-19 (debug assertion in the reference; a hard check here)
        if (!lax && polynom::degree_of(combined.data(), E) != E - n)
            throw std::runtime_error("combined constraint polynomial has unexpected degree");
    }
    if (forge.kind == Forgery::constraint_offset) combined[0] = field::add(combined[0], (u128)forge.a);
    if (dbg) dbg->constraint_poly = combined;
    double t4 = now_ms(); if (dbg) dbg->stage_ms[3] = t4 - t3;

    // 5 ----- constraint evaluations + tree (prover.rs:82-86) -------------------------------------
    std::vector<u128> c_evals(N, 0);
    std::copy(combined.begin(), combined.end(), c_evals.begin());
    polynom::eval_fft_twiddles(c_evals.data(), N, lde_twiddles.data(), true);
    std::vector<Digest> c_leaves(N / 2);
    memcpy(c_leaves.data(), c_evals.data(), N * 16);
    MerkleTree constraint_tree(std::move(c_leaves), hash);
    if (dbg && dbg->keep_large) dbg->constraint_evals = c_evals;
    double t5 = now_ms(); if (dbg) dbg->stage_ms[4] = t5 - t4;

    // 6 ----- DEEP composition polynomial (prover.rs:189-201, trace_table.rs:206-261, constraint_poly.rs:39-52)
    const uint8_t *cseed = constraint_tree.root().data();
    u128 z = prng(cseed);
    CompositionCoefficients cc(cseed);
    u128 next_z = field::mul(z, trace_root_w);
    std::vector<u128> state1(w), state2(w);
    for (size_t j = 0; j < w; j++) { state1[j] = polynom::eval(polys[j], z); }
    for (size_t j = 0; j < w; j++) { state2[j] = polynom::eval(polys[j], next_z); }
    if (forge.kind == Forgery::deep_value) { u128 &v = (forge.b ? state2 : state1).at(forge.a); v = field::add(v, 1); }
    std::vector<u128> t1c(n, 0), t2c(n, 0);
    for (size_t j = 0; j < w; j++) {
        field::mul_acc(t1c.data(), polys[j].data(), cc.trace1[j], n);
        t1c[0] = field::sub(t1c[0], field::mul(state1[j], cc.trace1[j]));
        field::mul_acc(t2c.data(), polys[j].data(), cc.trace2[j], n);
        t2c[0] = field::sub(t2c[0], field::mul(state2[j], cc.trace2[j]));
    }
    polynom::syn_div_in_place(t1c.data(), n, z);
    polynom::syn_div_in_place(t2c.data(), n, next_z);
    for (size_t k = 0; k < n; k++) t1c[k] = field::add(t1c[k], t2c[k]);
    size_t poly_size = 1; while (poly_size < get_composition_degree(n)) poly_size <<= 1;   // next_power_of_two
    std::vector<u128> comp(poly_size, 0);
    size_t inc = get_incremental_trace_degree(n);
    field::mul_acc(comp.data(), t1c.data(), cc.t1_degree, n);
    field::mul_acc(comp.data() + inc, t1c.data(), cc.t2_degree, n);
    {   // merge_into
        std::vector<u128> cp(combined);
        u128 z_value = polynom::eval(cp, z);
        cp[0] = field::sub(cp[0], z_value);
        polynom::syn_div_in_place(cp.data(), cp.size(), z);
        field::mul_acc(comp.data(), cp.data(), cc.constraints, comp.size());
    }
    if (dbg) { dbg->composition_poly = comp; dbg->z = z; }
    std::vector<u128> composed(N, 0);
    std::copy(comp.begin(), comp.end(), composed.begin());
    polynom::eval_fft_twiddles(composed.data(), N, lde_twiddles.data(), true);
    if (dbg && dbg->keep_large) dbg->composed_evals = composed;
    double t6 = now_ms(); if (dbg) dbg->stage_ms[5] = t6 - t5;

    // 7 ----- FRI layers (prover.rs:109-114) ------------------------------------------------------
    std::vector<MerkleTree> fri_trees;
    std::vector<std::vector<quartic::Q>> fri_values;
    fri_reduce(composed, lde_domain, hash, fri_trees, fri_values, forge);
    double t7 = now_ms(); if (dbg) dbg->stage_ms[6] = t7 - t6;

    // 8 ----- query positions (prover.rs:119-133) -------------------------------------------------
    uint8_t seed[32], pow_seed[32];
    uint64_t pow_nonce = 0;
    std::vector<size_t> positions;
    auto draw_positions = [&]() {
        std::vector<uint8_t> fri_roots;
        for (auto &t : fri_trees) fri_roots.insert(fri_roots.end(), t.root().begin(), t.root().end());
        hash(fri_roots.data(), fri_roots.size(), seed);
        pow_nonce = find_pow_nonce(seed, opt.grinding_factor, hash, pow_seed);
        positions = compute_query_positions(pow_seed, N, b, opt.num_queries);
    };
    draw_positions();
    // forged remainders: the remainder positions the queries open (fri/verifier.rs:33-80) and the degree bound the verifier applies
    const size_t n_layers = fri_trees.size() - 1;
    auto remainder_positions = [&]() {
        std::vector<size_t> p = positions;
        for (size_t d = 0, D = N; d < n_layers; d++, D /= 4) p = get_augmented_positions(p, D);
        return p;
    };
    size_t rem_bound = get_composition_degree(n) + 1;
    for (size_t d = 0; d < n_layers; d++) rem_bound /= 4;
    if (forge.kind == Forgery::remainder_point) {
        std::vector<quartic::Q> &last = fri_values.back();
        const std::vector<quartic::Q> honest = last;
        const size_t rows = last.size();
        for (size_t r = rows * 4; ; ) {
            do { if (r-- == 0) throw std::runtime_error("every remainder value is opened"); } while (r % b == 0);
            last = honest;
            last[r % rows].v[r / rows] = field::add(last[r % rows].v[r / rows], 1);
            fri_trees.back() = MerkleTree(hash_values(last, hash), hash);
            draw_positions();
            std::vector<size_t> opened = remainder_positions();
            if (std::find(opened.begin(), opened.end(), r) == opened.end()) break;
        }
    }
    if (forge.kind == Forgery::remainder_cut) {
        const size_t kept = (size_t)((int64_t)rem_bound + forge.a);
        for (int t = 0;; t++) {
            std::vector<size_t> opened = remainder_positions();
            if (*std::max_element(opened.begin(), opened.end()) < kept) break;
            if (t == 100000) throw std::runtime_error("no nonce opens only the kept remainder values");
            pow_nonce = find_pow_nonce(seed, opt.grinding_factor, hash, pow_seed, pow_nonce);
            positions = compute_query_positions(pow_seed, N, b, opt.num_queries);
        }
    }
    if (dbg) {
        for (auto &t : fri_trees) dbg->fri_roots.push_back(t.root());
        dbg->pow_nonce = pow_nonce; memcpy(dbg->pow_seed.data(), pow_seed, 32); dbg->positions = positions;
        dbg->trace_root = trace_tree.root(); dbg->constraint_root = constraint_tree.root();
    }
    double t8 = now_ms(); if (dbg) dbg->stage_ms[7] = t8 - t7;

    // 9 ----- proof object (prover.rs:143-165) ----------------------------------------------------
    StarkProof proof;
    proof.degree_proof = fri_build_proof(fri_trees, fri_values, positions);
    if (forge.kind == Forgery::remainder_cut) proof.degree_proof.rem_values.resize((size_t)((int64_t)rem_bound + forge.a));
    for (size_t p : positions) {
        std::vector<u128> row(w);
        for (size_t j = 0; j < w; j++) row[j] = ext[j][p];
        proof.trace_evaluations.push_back(row);
    }
    std::vector<size_t> c_positions = map_trace_to_constraint_positions(positions);
    BatchMerkleProof tproof = trace_tree.prove_batch(positions);
    proof.trace_root = trace_tree.root();
    proof.domain_depth = tproof.depth;
    proof.ctx_depth = (uint8_t)ctx_depth; proof.loop_depth = (uint8_t)loop_depth; proof.stack_depth = (uint8_t)stack_depth;
    proof.op_count = (uint32_t)op_count;
    proof.trace_nodes = tproof.nodes;
    proof.constraint_root = constraint_tree.root();
    proof.constraint_proof = constraint_tree.prove_batch(c_positions);
    proof.trace_at_z1 = state1; proof.trace_at_z2 = state2;
    proof.pow_nonce = pow_nonce;
    proof.opt_ext_log2 = (uint8_t)__builtin_ctzll(b); proof.opt_num_queries = (uint8_t)opt.num_queries;
    proof.opt_grinding = (uint8_t)opt.grinding_factor; proof.opt_hash_id = 0;
    if (dbg) {
        dbg->stage_ms[8] = now_ms() - t8;
        if (dbg->keep_large) { dbg->polys = polys; dbg->extended = ext; }
    }
    return proof;
}

// ---- verifier (verifier.rs, fri/verifier.rs) --------------------------------------------------------------------
static inline void state_from_vec(TraceState &s, const std::vector<u128> &v) {
    if (v.size() != s.width()) throw std::runtime_error("deep value vector has wrong width");
    s.from_row(v.data());
}

static inline std::string fri_verify(const FriProof &proof, std::vector<u128> evaluations, std::vector<size_t> positions,
                                     size_t max_degree, const ProofOptions &opt) {
    if (proof.layers.empty()) return "no FRI layers";
    size_t domain_size = ((size_t)1 << proof.layers[0].depth) * 4;
    u128 domain_root = field::get_root_of_unity(domain_size);
    u128 qr[4] = { 1, field::exp(domain_root, (u128)(domain_size / 4)), field::exp(domain_root, (u128)(domain_size / 2)),
                   field::exp(domain_root, (u128)(domain_size * 3 / 4)) };
    size_t max_degree_plus_1 = max_degree + 1;
    for (size_t depth = 0; depth < proof.layers.size(); depth++) {
        const FriLayer &layer = proof.layers[depth];
        std::vector<size_t> aug = get_augmented_positions(positions, domain_size);
        // get_column_values  fri/verifier.rs:136-147
        size_t row_length = domain_size / 4;
        std::vector<u128> column_values;
        for (size_t p : positions) {
            size_t idx = std::find(aug.begin(), aug.end(), p % row_length) - aug.begin();
            if (idx >= layer.values.size()) return "layer values too short";
            column_values.push_back(layer.values[idx].v[p / row_length]);
        }
        if (evaluations != column_values) return "evaluations did not match column value at depth " + std::to_string(depth);
        BatchMerkleProof mp;
        mp.values = hash_values(layer.values, opt.hash_fn); mp.nodes = layer.nodes; mp.depth = layer.depth;
        if (!MerkleTree::verify_batch(layer.root, aug, mp, opt.hash_fn)) return "verification of Merkle proof failed at layer " + std::to_string(depth);
        std::vector<quartic::Q> xs;
        for (size_t i : aug) {
            u128 xe = field::exp(domain_root, (u128)i);
            xs.push_back({{ field::mul(qr[0], xe), field::mul(qr[1], xe), field::mul(qr[2], xe), field::mul(qr[3], xe) }});
        }
        std::vector<quartic::Q> row_polys = quartic::interpolate_batch(xs, layer.values);
        u128 special_x = prng(layer.root.data());
        evaluations = quartic::evaluate_batch(row_polys, special_x);
        domain_root = field::exp(domain_root, 4);
        max_degree_plus_1 /= 4;
        domain_size /= 4;
        positions = aug;
    }
    for (size_t i = 0; i < positions.size(); i++) {
        if (positions[i] >= proof.rem_values.size() || proof.rem_values[positions[i]] != evaluations[i])
            return "remainder values are inconsistent with values of the last column";
    }
    // verify_remainder  fri/verifier.rs:97-131
    const std::vector<u128> &rem = proof.rem_values;
    if (max_degree_plus_1 > rem.size()) return "remainder degree is greater than number of remainder values";
    std::vector<size_t> pos;
    for (size_t i = 0; i < rem.size(); i++) if (i % opt.extension_factor != 0) pos.push_back(i);
    std::vector<u128> domain = field::get_power_series(domain_root, rem.size());
    std::vector<u128> xs, ys;
    // fri/verifier.rs:108-110 indexes positions[i] past its end when the bound exceeds the non-skipped points, and panics
    if (max_degree_plus_1 > pos.size())
        throw std::runtime_error("index out of bounds: the len is " + std::to_string(pos.size()) + " but the index is " + std::to_string(pos.size()));
    for (size_t i = 0; i < max_degree_plus_1; i++) { xs.push_back(domain[pos[i]]); ys.push_back(rem[pos[i]]); }
    std::vector<u128> poly = polynom::interpolate(xs, ys);
    for (size_t i = max_degree_plus_1; i < pos.size(); i++)
        if (polynom::eval(poly, domain[pos[i]]) != rem[pos[i]])
            return "remainder is not a valid degree " + std::to_string(max_degree_plus_1 - 1) + " polynomial";
    return "";
}

// returns "" on success, error message otherwise  (verifier.rs:11-75)
static inline std::string verify(const uint8_t program_hash[32], const std::vector<u128> &inputs, const std::vector<u128> &outputs,
                                 const StarkProof &proof) {
    ProofOptions opt;
    opt.extension_factor = proof.extension_factor(); opt.num_queries = proof.opt_num_queries; opt.grinding_factor = proof.opt_grinding;
    if (proof.opt_hash_id != 0) return "unsupported hash function";
    HashFn hash = opt.hash_fn;
    // 1
    std::vector<uint8_t> fri_roots;
    for (auto &l : proof.degree_proof.layers) fri_roots.insert(fri_roots.end(), l.root.begin(), l.root.end());
    fri_roots.insert(fri_roots.end(), proof.degree_proof.rem_root.begin(), proof.degree_proof.rem_root.end());
    uint8_t seed[32], pseed[32];
    hash(fri_roots.data(), fri_roots.size(), seed);
    if (!verify_pow_nonce(seed, proof.pow_nonce, opt.grinding_factor, hash, pseed)) return "seed proof-of-work verification failed";
    std::vector<size_t> t_positions, c_positions;
    try { t_positions = compute_query_positions(pseed, proof.domain_size(), opt.extension_factor, opt.num_queries); }
    catch (std::exception &e) { return e.what(); }
    c_positions = map_trace_to_constraint_positions(t_positions);
    // 2
    if (proof.op_count < MIN_TRACE_LENGTH) return "Verification of minimum operation count failed";
    // 3
    BatchMerkleProof tp;
    tp.nodes = proof.trace_nodes; tp.depth = proof.domain_depth;
    for (auto &row : proof.trace_evaluations) { Digest d; hash((const uint8_t *)row.data(), row.size() * 16, d.data()); tp.values.push_back(d); }
    if (!MerkleTree::verify_batch(proof.trace_root, t_positions, tp, hash)) return "verification of trace Merkle proof failed";
    if (!MerkleTree::verify_batch(proof.constraint_root, c_positions, proof.constraint_proof, hash)) return "verification of constraint Merkle proof failed";
    // 4
    u128 z = prng(proof.constraint_root.data());
    size_t n = proof.trace_length();
    u128 ph[2];
    memcpy(ph, program_hash, 32);
    Evaluator ev(n, opt.extension_factor, proof.domain_size(), proof.ctx_depth, proof.loop_depth, proof.stack_depth,
                 proof.trace_root.data(), ph, (u128)proof.op_count, inputs, outputs);
    TraceState s1(proof.ctx_depth, proof.loop_depth, proof.stack_depth), s2(proof.ctx_depth, proof.loop_depth, proof.stack_depth);
    try { state_from_vec(s1, proof.trace_at_z1); state_from_vec(s2, proof.trace_at_z2); }
    catch (std::exception &e) { return e.what(); }
    u128 constraint_at_z;
    {   // evaluate_constraints  verifier.rs:79-97
        u128 i_value, f_value;
        ev.evaluate_boundaries(s1, z, i_value, f_value);
        u128 t_value = ev.evaluate_transition_at(s1, s2, z);
        u128 zz = field::sub(z, 1);
        u128 result = field::div(i_value, zz);
        zz = field::sub(z, ev.get_x_at_last_step());
        result = field::add(result, field::div(f_value, zz));
        zz = field::div(field::sub(field::exp(z, (u128)n), 1), zz);
        result = field::add(result, field::div(t_value, zz));
        constraint_at_z = result;
    }
    // 5
    CompositionCoefficients cc(proof.constraint_root.data());
    u128 lde_root = field::get_root_of_unity(proof.domain_size());
    u128 next_z = field::mul(z, field::get_root_of_unity(n));
    u128 inc = (u128)get_incremental_trace_degree(n);
    std::vector<u128> evaluations;
    if (proof.trace_evaluations.size() != t_positions.size()) return "wrong number of trace evaluations";
    for (size_t q = 0; q < t_positions.size(); q++) {
        size_t position = t_positions[q];
        u128 x = field::exp(lde_root, (u128)position);
        const std::vector<u128> &regs = proof.trace_evaluations[q];
        if (regs.size() != proof.trace_at_z1.size()) return "trace evaluation row has wrong width";
        u128 comp = 0;
        for (size_t i = 0; i < regs.size(); i++) {
            u128 t1 = field::div(field::sub(regs[i], proof.trace_at_z1[i]), field::sub(x, z));
            comp = field::add(comp, field::mul(t1, cc.trace1[i]));
            u128 t2 = field::div(field::sub(regs[i], proof.trace_at_z2[i]), field::sub(x, next_z));
            comp = field::add(comp, field::mul(t2, cc.trace2[i]));
        }
        u128 xp = field::exp(x, inc);
        u128 adj = field::mul(field::mul(comp, xp), cc.t2_degree);
        comp = field::add(field::mul(comp, cc.t1_degree), adj);
        // compose_constraints  verifier.rs:139-162
        size_t leaf_idx = std::find(c_positions.begin(), c_positions.end(), position / 2) - c_positions.begin();
        if (leaf_idx >= proof.constraint_proof.values.size()) return "constraint proof values too short";
        u128 evaluation;
        memcpy(&evaluation, proof.constraint_proof.values[leaf_idx].data() + (position % 2) * 16, 16);
        u128 c = field::div(field::sub(evaluation, constraint_at_z), field::sub(x, z));
        evaluations.push_back(field::add(comp, field::mul(c, cc.constraints)));
    }
    // 6
    std::string err = fri_verify(proof.degree_proof, evaluations, t_positions, get_composition_degree(n), opt);
    if (!err.empty()) return "verification of low-degree proof failed: " + err;
    return "";
}

} // namespace oracle

#include <chrono>
namespace oracle {
static inline double now_ms() {
    return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
}
#endif
