// ORACLE -- TEST INFRASTRUCTURE ONLY.  C-ABI over the CPU restatement (math.h, crypto.h, air.h, stark.h) so that
// tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs can call it through ctypes.
// Nothing in distaff_b200/ links or loads this library.
#include "stark.h"

using namespace oracle;

static HashFn hash_by_id(int id) {
    switch (id) {
        case 0: return blake3;
        case 1: return rescue;
        case 2: return poseidon;
        case 3: return gmimc;
        default: throw std::runtime_error("unknown hash id");
    }
}
static inline u128 ld(const uint8_t *p) { u128 v; memcpy(&v, p, 16); return v; }
static inline void st(uint8_t *p, u128 v) { memcpy(p, &v, 16); }

struct ProveResult {
    std::vector<uint8_t> bytes;
    ProverTrace trace;
    std::string error;
};

extern "C" {

// host threads used by the prover / FFTs (1 = the reference's behaviour; see fft::host_threads).  Returns the value in effect.
int or_set_threads(int t) { if (t >= 1) fft::host_threads() = t; return fft::host_threads(); }

// ---- field -------------------------------------------------------------------------------------------------
void or_field_op(int op, const uint8_t *a, const uint8_t *b, uint8_t *out) {
    u128 x = ld(a), y = b ? ld(b) : 0, r = 0;
    switch (op) {
        case 0: r = field::add(x, y); break;
        case 1: r = field::sub(x, y); break;
        case 2: r = field::mul(x, y); break;
        case 3: r = field::inv(x); break;
        case 4: r = field::exp(x, y); break;
        case 5: r = field::neg(x); break;
    }
    st(out, r);
}
void or_root_of_unity(uint64_t order, uint8_t *out) { st(out, field::get_root_of_unity(order)); }
void or_inv_many(const uint8_t *in, uint8_t *out, uint64_t n) {
    std::vector<u128> v(n), r(n);
    memcpy(v.data(), in, n * 16);
    field::inv_many_fill(v.data(), r.data(), n);
    memcpy(out, r.data(), n * 16);
}
// natural-order forward / inverse DFT over the subgroup of size n (polynom::eval_fft / interpolate_fft), in place
void or_fft(uint8_t *values, uint64_t n, int inverse) {
    std::vector<u128> v(n);
    memcpy(v.data(), values, n * 16);
    if (inverse) polynom::interpolate_fft(v); else polynom::eval_fft(v);
    memcpy(values, v.data(), n * 16);
}
// raw fft_in_place + optional permute, with caller twiddles (fft.rs test contract)
void or_fft_in_place(uint8_t *values, uint64_t n, const uint8_t *twiddles, int permute) {
    std::vector<u128> v(n), tw(n / 2);
    memcpy(v.data(), values, n * 16); memcpy(tw.data(), twiddles, n / 2 * 16);
    fft::fft_in_place(v.data(), n, tw.data(), 1, 1, 0);
    if (permute) fft::permute(v.data(), n);
    memcpy(values, v.data(), n * 16);
}
void or_get_twiddles(const uint8_t *root, uint64_t size, int inverse, uint8_t *out) {
    std::vector<u128> tw = inverse ? fft::get_inv_twiddles(ld(root), size) : fft::get_twiddles(ld(root), size);
    memcpy(out, tw.data(), tw.size() * 16);
}
void or_poly_eval(const uint8_t *p, uint64_t n, const uint8_t *x, uint8_t *out) {
    std::vector<u128> v(n); memcpy(v.data(), p, n * 16);
    st(out, polynom::eval(v, ld(x)));
}
void or_syn_div(uint8_t *p, uint64_t n, const uint8_t *b) {
    std::vector<u128> v(n); memcpy(v.data(), p, n * 16);
    polynom::syn_div_in_place(v.data(), n, ld(b));
    memcpy(p, v.data(), n * 16);
}
void or_syn_div_expanded(uint8_t *p, uint64_t n, uint64_t degree, const uint8_t *exc, uint64_t n_exc) {
    std::vector<u128> v(n), e(n_exc); memcpy(v.data(), p, n * 16); memcpy(e.data(), exc, n_exc * 16);
    polynom::syn_div_expanded_in_place(v.data(), n, degree, e.data(), n_exc);
    memcpy(p, v.data(), n * 16);
}
// long division a / b -> out (len = deg a - deg b + 1 returned)
uint64_t or_poly_div(const uint8_t *a, uint64_t na, const uint8_t *b, uint64_t nb, uint8_t *out) {
    std::vector<u128> va(na), vb(nb); memcpy(va.data(), a, na * 16); memcpy(vb.data(), b, nb * 16);
    std::vector<u128> r = polynom::div(va, vb);
    memcpy(out, r.data(), r.size() * 16);
    return r.size();
}
void or_lagrange(const uint8_t *xs, const uint8_t *ys, uint64_t n, uint8_t *out) {
    std::vector<u128> vx(n), vy(n); memcpy(vx.data(), xs, n * 16); memcpy(vy.data(), ys, n * 16);
    std::vector<u128> r = polynom::interpolate(vx, vy);
    memcpy(out, r.data(), n * 16);
}
// quartic: xs, ys are n rows of 4 ; out = n rows of 4 coefficients
void or_quartic_interpolate_batch(const uint8_t *xs, const uint8_t *ys, uint64_t n, uint8_t *out) {
    std::vector<quartic::Q> vx(n), vy(n);
    memcpy(vx.data(), xs, n * 64); memcpy(vy.data(), ys, n * 64);
    std::vector<quartic::Q> r = quartic::interpolate_batch(vx, vy);
    memcpy(out, r.data(), n * 64);
}
void or_quartic_transpose(const uint8_t *v, uint64_t len, uint64_t stride, uint8_t *out) {
    std::vector<u128> in(len); memcpy(in.data(), v, len * 16);
    std::vector<quartic::Q> r = quartic::transpose(in.data(), len, stride);
    memcpy(out, r.data(), r.size() * 64);
}
// n cubics (rows of 4 coefficients) evaluated at x
void or_quartic_evaluate_batch(const uint8_t *polys, uint64_t n, const uint8_t *x, uint8_t *out) {
    std::vector<quartic::Q> p(n); memcpy(p.data(), polys, n * 64);
    std::vector<u128> r = quartic::evaluate_batch(p, ld(x));
    memcpy(out, r.data(), n * 16);
}
// field::get_power_series: b^0 .. b^(length - 1)
void or_power_series(const uint8_t *b, uint64_t length, uint8_t *out) {
    std::vector<u128> r = field::get_power_series(ld(b), length);
    memcpy(out, r.data(), length * 16);
}

// ---- hashing / merkle -------------------------------------------------------------------------------------------
int or_hash(int id, const uint8_t *in, uint64_t len, uint8_t *out32) {
    try { hash_by_id(id)(in, len, out32); return 0; } catch (...) { return -1; }
}
// blake3 of every row of a column-major [w][rows] matrix, as the prover's trace commitment hashes the rows of the extension
void or_hash_rows(const uint8_t *cols, uint64_t w, uint64_t rows, uint8_t *out32) {
    const int T = fft::host_threads();
    #pragma omp parallel num_threads(T) if (T > 1)
    {
        std::vector<u128> row(w);
        #pragma omp for
        for (uint64_t i = 0; i < rows; i++) {
            for (uint64_t j = 0; j < w; j++) memcpy(&row[j], cols + 16 * (j * rows + i), 16);
            blake3((const uint8_t *)row.data(), w * 16, out32 + 32 * i);
        }
    }
}
// nodes_out: n_leaves * 32 bytes (heap layout, nodes[0] = 0, root = nodes[1])
int or_merkle_nodes(int id, const uint8_t *leaves, uint64_t n, uint8_t *nodes_out) {
    try {
        std::vector<Digest> l(n); memcpy(l.data(), leaves, n * 32);
        std::vector<Digest> nodes = build_merkle_nodes(l, hash_by_id(id));
        memcpy(nodes_out, nodes.data(), n * 32);
        return 0;
    } catch (...) { return -1; }
}
// batch proof, flattened: out = [n_values u64][values..][n_node_vecs u64]([len u64][nodes..])*[depth u8]; returns byte count
int64_t or_merkle_prove_batch(int id, const uint8_t *leaves, uint64_t n, const uint64_t *indexes, uint64_t n_idx, uint8_t *out, uint64_t cap) {
    try {
        std::vector<Digest> l(n); memcpy(l.data(), leaves, n * 32);
        MerkleTree t(l, hash_by_id(id));
        std::vector<size_t> idx(indexes, indexes + n_idx);
        BatchMerkleProof p = t.prove_batch(idx);
        Writer w; w.dvec(p.values); w.dvv(p.nodes); w.u8(p.depth);
        if (w.b.size() > cap) return -2;
        memcpy(out, w.b.data(), w.b.size());
        return (int64_t)w.b.size();
    } catch (...) { return -1; }
}
int or_merkle_verify_batch(int id, const uint8_t *root, const uint64_t *indexes, uint64_t n_idx, const uint8_t *proof, uint64_t proof_len) {
    try {
        Reader r(proof, proof_len);
        BatchMerkleProof p; p.values = r.dvec(); p.nodes = r.dvv(); p.depth = r.u8();
        Digest rt; memcpy(rt.data(), root, 32);
        std::vector<size_t> idx(indexes, indexes + n_idx);
        return MerkleTree::verify_batch(rt, idx, p, hash_by_id(id)) ? 1 : 0;
    } catch (...) { return -1; }
}

// ---- Fiat-Shamir pieces ----------------------------------------------------------------------------------------------
void or_prng_vector(const uint8_t *seed32, uint64_t n, uint8_t *out) {
    std::vector<u128> v = prng_vector(seed32, n);
    memcpy(out, v.data(), n * 16);
}
void or_chacha_words(const uint8_t *seed32, uint64_t n_words, uint32_t *out) {
    ChaChaRng g(seed32);
    for (uint64_t i = 0; i < n_words; i++) out[i] = g.next_u32();
}
int or_query_positions(const uint8_t *seed32, uint64_t domain, uint64_t ext, uint64_t nq, uint64_t *out) {
    try {
        std::vector<size_t> p = compute_query_positions(seed32, domain, ext, nq);
        for (size_t i = 0; i < p.size(); i++) out[i] = p[i];
        return (int)p.size();
    } catch (...) { return -1; }
}
uint64_t or_find_pow_nonce(const uint8_t *seed32, uint32_t grinding, uint8_t *out_seed32) {
    return find_pow_nonce(seed32, grinding, blake3, out_seed32);
}
// constraint coefficients, flattened as the 2*NUM_CONSTRAINTS raw draws are not needed; this returns the compacted
// transition vector length and copies [i_boundary(94)][f_boundary(94)][transition(...)]
uint64_t or_constraint_coefficients(const uint8_t *seed32, uint32_t cd, uint32_t ldp, uint32_t sd, uint8_t *out) {
    ConstraintCoefficients c(seed32, cd, ldp, sd);
    memcpy(out, &c.i_boundary, sizeof(BoundaryCoefficients));
    memcpy(out + sizeof(BoundaryCoefficients), &c.f_boundary, sizeof(BoundaryCoefficients));
    memcpy(out + 2 * sizeof(BoundaryCoefficients), c.transition.data(), c.transition.size() * 16);
    return c.transition.size();
}

// ---- in-VM hash helpers (examples/merkle.rs needs hasher::digest) -----------------------------------------------------
void or_hasher_digest(const uint8_t *values, uint32_t n, uint8_t *out32) {
    u128 v[4] = {0, 0, 0, 0}, o[2];
    memcpy(v, values, (size_t)n * 16);
    hasher6::digest(v, n, o);
    memcpy(out32, o, 32);
}

// ---- prover / verifier ---------------------------------------------------------------------------------------------------
// cols: column-major w x n field elements.  Returns a handle (never null); query with or_result_*.
void *or_prove_forged(const uint8_t *cols, uint32_t w, uint64_t n, uint32_t ctx_depth, uint32_t loop_depth,
                      const uint8_t *inputs, uint32_t n_in, const uint8_t *outputs, uint32_t n_out,
                      uint32_t ext, uint32_t num_queries, uint32_t grinding, int keep_large, int forge_kind, int64_t forge_a, int64_t forge_b);
void *or_prove(const uint8_t *cols, uint32_t w, uint64_t n, uint32_t ctx_depth, uint32_t loop_depth,
               const uint8_t *inputs, uint32_t n_in, const uint8_t *outputs, uint32_t n_out,
               uint32_t ext, uint32_t num_queries, uint32_t grinding, int keep_large) {
    return or_prove_forged(cols, w, n, ctx_depth, loop_depth, inputs, n_in, outputs, n_out, ext, num_queries, grinding, keep_large,
                           Forgery::none, 0, 0);
}
// or_prove with one value changed before it is committed (stark.h Forgery: kind, a, b); a proof of a false statement whose
// commitments are all consistent, for testing what the verifiers reject
void *or_prove_forged(const uint8_t *cols, uint32_t w, uint64_t n, uint32_t ctx_depth, uint32_t loop_depth,
                      const uint8_t *inputs, uint32_t n_in, const uint8_t *outputs, uint32_t n_out,
                      uint32_t ext, uint32_t num_queries, uint32_t grinding, int keep_large, int forge_kind, int64_t forge_a, int64_t forge_b) {
    ProveResult *r = new ProveResult();
    try {
        Forgery forge;
        if (forge_kind < Forgery::none || forge_kind > Forgery::remainder_cut) throw std::runtime_error("unknown forgery");
        forge.kind = (Forgery::Kind)forge_kind; forge.a = forge_a; forge.b = forge_b;
        std::vector<std::vector<u128>> regs(w, std::vector<u128>(n));
        for (uint32_t j = 0; j < w; j++) memcpy(regs[j].data(), cols + (size_t)j * n * 16, n * 16);
        std::vector<u128> in(n_in), out(n_out);
        if (n_in) memcpy(in.data(), inputs, n_in * 16);
        if (n_out) memcpy(out.data(), outputs, n_out * 16);
        ProofOptions opt; opt.extension_factor = ext; opt.num_queries = num_queries; opt.grinding_factor = grinding;
        r->trace.keep_large = keep_large != 0;
        StarkProof p = prove(regs, ctx_depth, loop_depth, in, out, opt, &r->trace, forge);
        r->bytes = serialize(p);
    } catch (std::exception &e) { r->error = e.what(); }
    return r;
}
const char *or_result_error(void *h) { auto *r = (ProveResult *)h; return r->error.empty() ? nullptr : r->error.c_str(); }
uint64_t or_result_proof_len(void *h) { return ((ProveResult *)h)->bytes.size(); }
void or_result_proof(void *h, uint8_t *out) { auto *r = (ProveResult *)h; memcpy(out, r->bytes.data(), r->bytes.size()); }
void or_result_stage_ms(void *h, double *out9) { memcpy(out9, ((ProveResult *)h)->trace.stage_ms, 9 * sizeof(double)); }
// named intermediate vectors; returns element count (16-byte elements unless noted), copies when out != null
uint64_t or_result_vector(void *h, const char *name, uint32_t index, uint8_t *out) {
    ProverTrace &t = ((ProveResult *)h)->trace;
    std::string s(name);
    const std::vector<u128> *v = nullptr;
    if (s == "i_evals") v = &t.i_evals; else if (s == "f_evals") v = &t.f_evals; else if (s == "t_evals") v = &t.t_evals;
    else if (s == "constraint_poly") v = &t.constraint_poly; else if (s == "constraint_evals") v = &t.constraint_evals;
    else if (s == "composition_poly") v = &t.composition_poly; else if (s == "composed_evals") v = &t.composed_evals;
    else if (s == "poly") { if (index < t.polys.size()) v = &t.polys[index]; }
    else if (s == "extended") { if (index < t.extended.size()) v = &t.extended[index]; }
    else if (s == "z") { if (out) st(out, t.z); return 1; }
    else if (s == "trace_root") { if (out) memcpy(out, t.trace_root.data(), 32); return 2; }
    else if (s == "constraint_root") { if (out) memcpy(out, t.constraint_root.data(), 32); return 2; }
    else if (s == "pow_seed") { if (out) memcpy(out, t.pow_seed.data(), 32); return 2; }
    else if (s == "fri_roots") { if (out) memcpy(out, t.fri_roots.data(), t.fri_roots.size() * 32); return t.fri_roots.size() * 2; }
    else if (s == "positions") { if (out) for (size_t i = 0; i < t.positions.size(); i++) ((uint64_t *)out)[i] = t.positions[i]; return t.positions.size(); }
    else if (s == "pow_nonce") { if (out) *(uint64_t *)out = t.pow_nonce; return 1; }
    if (!v) return 0;
    if (out) memcpy(out, v->data(), v->size() * 16);
    return v->size();
}
void or_result_free(void *h) { delete (ProveResult *)h; }

// returns 0 when the proof verifies; otherwise copies the error message into err (NUL-terminated) and returns 1
int or_verify(const uint8_t *program_hash32, const uint8_t *inputs, uint32_t n_in, const uint8_t *outputs, uint32_t n_out,
              const uint8_t *proof, uint64_t proof_len, char *err, uint32_t err_cap) {
    std::string msg;
    try {
        std::vector<u128> in(n_in), out(n_out);
        if (n_in) memcpy(in.data(), inputs, n_in * 16);
        if (n_out) memcpy(out.data(), outputs, n_out * 16);
        StarkProof p = deserialize(proof, proof_len);
        msg = verify(program_hash32, in, out, p);
    } catch (std::exception &e) { msg = std::string("exception: ") + e.what(); }
    if (msg.empty()) return 0;
    if (err && err_cap) { strncpy(err, msg.c_str(), err_cap - 1); err[err_cap - 1] = 0; }
    return 1;
}

// evaluates all transition constraints of the AIR for a (current,next) row pair on the 8x evaluation domain `step`
// (used to pin decoder/stack constraint tests from the reference's unit tests); rows are `width` elements
uint32_t or_eval_transition_raw(const uint8_t *cur_row, const uint8_t *next_row, uint32_t cd, uint32_t ldp, uint32_t sd,
                                uint64_t trace_length, uint64_t step, uint8_t *out) {
    TraceState c(cd, ldp, sd), n(cd, ldp, sd);
    std::vector<u128> rc(c.width()), rn(c.width());
    memcpy(rc.data(), cur_row, rc.size() * 16); memcpy(rn.data(), next_row, rn.size() * 16);
    c.from_row(rc.data()); n.from_row(rn.data());
    DecoderAir dec(trace_length, 8, cd, ldp);
    StackAir stk(trace_length, 8, sd);
    std::vector<u128> ev(dec.constraint_count() + stk.degrees.size(), 0);
    dec.evaluate(c, n, step, ev.data());
    stk.evaluate(c, n, step, ev.data() + dec.constraint_count());
    memcpy(out, ev.data(), ev.size() * 16);
    return (uint32_t)ev.size();
}
// the prover's stage-3 transition loop (stark.h prove, prover.rs:52-64) over a supplied extended trace: ext = w columns of n * blowup
// elements in LDE order; the Evaluator's coefficients come from seed32, with no public inputs or outputs.  check = 1: the prover's loop,
// which returns 1 with its error message (lowest failing step) in err when a trace-domain step does not vanish, else 0 and
// evaluate_transition at every step; check = 0: combine_transition_constraints at every step, without the trace-domain assertion.
// out: 8n values in step order.
int or_eval_transitions(const uint8_t *ext16, uint32_t cd, uint32_t ldp, uint32_t sd, uint64_t n, uint32_t blowup, const uint8_t *seed32,
                        int check, uint8_t *out16, char *err, uint32_t err_cap) {
    try {
        const size_t w = 15 + cd + ldp + sd, N = n * blowup, E = n * MAX_CONSTRAINT_DEGREE, stride = blowup / MAX_CONSTRAINT_DEGREE;
        std::vector<std::vector<u128>> ext(w, std::vector<u128>(N));
        for (size_t j = 0; j < w; j++) memcpy(ext[j].data(), ext16 + j * N * 16, N * 16);
        const u128 no_hash[2] = {0, 0};
        Evaluator evaluator(n, MAX_CONSTRAINT_DEGREE, E, cd, ldp, sd, seed32, no_hash, 0, {}, {});
        std::vector<u128> lde_domain = field::get_power_series(field::get_root_of_unity(N), N);
        TraceState cur(cd, ldp, sd), nxt(cd, ldp, sd);
        std::vector<u128> ev(evaluator.t_constraint_num);
        for (size_t step = 0; step < E; step++) {
            const size_t i = step * stride;
            cur.from_columns(ext, i);
            nxt.from_columns(ext, (i + blowup) % N);
            u128 t;
            if (check) {
                t = evaluator.evaluate_transition(cur, nxt, lde_domain[i], step);
            } else {
                std::fill(ev.begin(), ev.end(), 0);
                evaluator.decoder.evaluate(cur, nxt, step, ev.data());
                evaluator.stack.evaluate(cur, nxt, step, ev.data() + evaluator.decoder.constraint_count());
                t = evaluator.combine_transition_constraints(ev, lde_domain[i]);
            }
            st(out16 + step * 16, t);
        }
        return 0;
    } catch (const std::exception &e) {
        if (err && err_cap) { strncpy(err, e.what(), err_cap - 1); err[err_cap - 1] = 0; }
        return 1;
    }
}
// Decoder::evaluate with explicit periodic values (ark[8], masks[3]) instead of a step: what the reference's unit tests of
// enforce_op_bits / enforce_hacc pass in (decoder/op_bits.rs, decoder/sponge.rs mod tests)
uint32_t or_decoder_run_raw(const uint8_t *cur_row, const uint8_t *next_row, uint32_t cd, uint32_t ldp, uint32_t sd,
                            const uint8_t *ark8, const uint8_t *masks3, uint8_t *out) {
    TraceState c(cd, ldp, sd), n(cd, ldp, sd);
    std::vector<u128> rc(c.width()), rn(c.width());
    memcpy(rc.data(), cur_row, rc.size() * 16); memcpy(rn.data(), next_row, rn.size() * 16);
    c.from_row(rc.data()); n.from_row(rn.data());
    DecoderAir dec(16, 8, cd, ldp);
    u128 ark[8], masks[3];
    memcpy(ark, ark8, sizeof ark); memcpy(masks, masks3, sizeof masks);
    std::vector<u128> ev(dec.constraint_count(), 0);
    dec.run(c, n, ark, masks, ev.data());
    memcpy(out, ev.data(), ev.size() * 16);
    return (uint32_t)ev.size();
}
// constraints::utils::enforce_left_shift (utils.rs:64-83) on plain vectors of length len
void or_enforce_left_shift(const uint8_t *old_stack, const uint8_t *new_stack, uint64_t len, uint64_t from, uint64_t num, const uint8_t *flag, uint8_t *result) {
    std::vector<u128> o(len), n(len), r(len, 0);
    u128 f;
    memcpy(o.data(), old_stack, len * 16); memcpy(n.data(), new_stack, len * 16); memcpy(&f, flag, 16);
    cu::left_shift(r.data(), len, o.data(), n.data(), from, num, f);
    memcpy(result, r.data(), len * 16);
}
// TraceState::from_vec decoded (trace_state.rs:88-118): out = op_counter, sponge[4], cf[3], ld[5], hd[2], ctx[ctx_len], loop[loop_len],
// user[stack_len], op_code; returns the number of elements written
uint32_t or_trace_state_fields(const uint8_t *row, uint32_t cd, uint32_t ldp, uint32_t sd, uint8_t *out) {
    TraceState c(cd, ldp, sd);
    std::vector<u128> r(c.width());
    memcpy(r.data(), row, r.size() * 16);
    c.from_row(r.data());
    std::vector<u128> v;
    v.push_back(c.op_counter);
    v.insert(v.end(), c.sponge, c.sponge + 4); v.insert(v.end(), c.cf_bits, c.cf_bits + 3);
    v.insert(v.end(), c.ld_bits, c.ld_bits + 5); v.insert(v.end(), c.hd_bits, c.hd_bits + 2);
    v.insert(v.end(), c.ctx_stack, c.ctx_stack + c.ctx_len); v.insert(v.end(), c.loop_stack, c.loop_stack + c.loop_len);
    v.insert(v.end(), c.user_stack, c.user_stack + c.stack_len);
    v.push_back(c.op_code());
    memcpy(out, v.data(), v.size() * 16);
    return (uint32_t)v.size();
}
// stand-alone FRI round trip as in fri/mod.rs mod tests: reduce + build_proof over `evaluations` (domain = powers of the root of unity of
// that size, default ProofOptions), then verify against max_degree with the first `drop` sampled evaluations removed.
// Returns 0 and writes "" on success, else writes the verifier's error message (NUL terminated) into msg.
int or_fri_roundtrip(const uint8_t *evaluations, uint64_t domain_size, uint64_t max_degree, uint32_t drop, char *msg, uint64_t cap) {
    try {
        std::vector<u128> ev(domain_size);
        memcpy(ev.data(), evaluations, domain_size * 16);
        std::vector<u128> domain = field::get_power_series(field::get_root_of_unity(domain_size), domain_size);
        ProofOptions opt;
        std::vector<MerkleTree> trees; std::vector<std::vector<quartic::Q>> values;
        fri_reduce(ev, domain, hash_by_id(0), trees, values);
        std::vector<size_t> positions = compute_query_positions(trees.back().root().data(), domain_size, opt.extension_factor, opt.num_queries);
        FriProof proof = fri_build_proof(trees, values, positions);
        std::vector<u128> sampled;
        for (size_t p : positions) sampled.push_back(ev[p]);
        sampled.erase(sampled.begin(), sampled.begin() + std::min<size_t>(drop, sampled.size()));
        std::string err = fri_verify(proof, sampled, positions, max_degree, opt);
        snprintf(msg, cap, "%s", err.c_str());
        return err.empty() ? 0 : 1;
    } catch (const std::exception &e) { snprintf(msg, cap, "exception: %s", e.what()); return -1; }
}
// utils::sponge::apply_round (sponge.rs:13-30) on a 4-element state, in place
void or_sponge_round(uint8_t *state4, const uint8_t *op_code, const uint8_t *op_value, uint64_t step) {
    u128 s[4], c, v;
    memcpy(s, state4, 64); memcpy(&c, op_code, 16); memcpy(&v, op_value, 16);
    sponge4::apply_round(s, c, v, step);
    memcpy(state4, s, 64);
}
// op flags of a row: out = cf[8] ld[32] hd[4] begin noop  (46 elements)
void or_op_flags(const uint8_t *row, uint32_t cd, uint32_t ldp, uint32_t sd, uint8_t *out) {
    TraceState c(cd, ldp, sd);
    std::vector<u128> r(c.width());
    memcpy(r.data(), row, r.size() * 16);
    c.from_row(r.data());
    u128 o[46];
    memcpy(o, c.cf_flags, sizeof c.cf_flags); memcpy(o + 8, c.ld_flags, sizeof c.ld_flags); memcpy(o + 40, c.hd_flags, sizeof c.hd_flags);
    o[44] = c.begin_flag; o[45] = c.noop_flag;
    memcpy(out, o, sizeof o);
}

}  // extern "C"
