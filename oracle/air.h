// ORACLE -- TEST INFRASTRUCTURE ONLY.  Never linked into or called by the product path.
//
// CPU restatement of the Distaff AIR (constraint system) as the reference evaluates it:
//   TraceState            /root/reference/src/stark/trace/trace_state.rs:50-350   (row decode, op flags incl. quirk :301)
//   ConstraintCoefficients/CompositionCoefficients   /root/reference/src/stark/utils/coefficients.rs:63-185
//   Decoder constraints   /root/reference/src/stark/constraints/decoder/{mod.rs:75-223, op_bits.rs:10-79, sponge.rs:10-43, flow_ops.rs:10-165}
//   Stack constraints     /root/reference/src/stark/constraints/stack/{mod.rs:57-206, arithmetic.rs, comparison.rs, conditional.rs,
//                                                                       hash.rs, input.rs, manipulation.rs (quirk :63-64)}
//   Evaluator             /root/reference/src/stark/constraints/evaluator.rs:35-443
//   in-VM Rescue helpers  /root/reference/src/utils/sponge.rs:38-79, /root/reference/src/utils/hasher.rs:43-91
#ifndef ORACLE_AIR_H
#define ORACLE_AIR_H

#include "crypto.h"

namespace oracle {

// lib.rs:79-138
static const size_t MAX_CONTEXT_DEPTH = 16, MAX_LOOP_DEPTH = 8, MAX_STACK_DEPTH = 32, MAX_PUBLIC_INPUTS = 8;
static const size_t MIN_TRACE_LENGTH = 16, MAX_REGISTER_COUNT = 128, BASE_CYCLE_LENGTH = 16;
static const size_t MIN_STACK_DEPTH = 8, MIN_CONTEXT_DEPTH = 1, MIN_LOOP_DEPTH = 1;
static const size_t SPONGE_WIDTH = 4, HASH_STATE_WIDTH = 6, PROGRAM_DIGEST_SIZE = 2;
static const size_t NUM_CF_OP_BITS = 3, NUM_LD_OP_BITS = 5, NUM_HD_OP_BITS = 2, NUM_OP_BITS = 10;
static const size_t MAX_CONSTRAINT_DEGREE = 8;  // stark/mod.rs:25

// processor/opcodes.rs:5-14,46-92
enum FlowOp { F_HACC = 0, F_BEGIN = 1, F_TEND = 2, F_FEND = 3, F_LOOP = 4, F_WRAP = 5, F_BREAK = 6, F_VOID = 7 };
enum UserOp {
    OP_ASSERT = 0x60, OP_ASSERTEQ = 0x61, OP_EQ = 0x62, OP_DROP = 0x63, OP_DROP4 = 0x64, OP_CHOOSE = 0x65, OP_CHOOSE2 = 0x66, OP_CSWAP2 = 0x67,
    OP_ADD = 0x68, OP_MUL = 0x69, OP_AND = 0x6a, OP_OR = 0x6b, OP_INV = 0x6c, OP_NEG = 0x6d, OP_NOT = 0x6e,
    OP_READ = 0x70, OP_READ2 = 0x71, OP_DUP = 0x72, OP_DUP2 = 0x73, OP_DUP4 = 0x74, OP_PAD2 = 0x75,
    OP_SWAP = 0x78, OP_SWAP2 = 0x79, OP_SWAP4 = 0x7a, OP_ROLL4 = 0x7b, OP_ROLL8 = 0x7c, OP_BINACC = 0x7d,
    OP_PUSH = 0x1f, OP_CMP = 0x3f, OP_RESCR = 0x5f,
    OP_BEGIN = 0x00, OP_NOOP = 0x7f,
};
static inline size_t ld_index(int op) { return op & 0x1f; }
static inline size_t hd_index(int op) { return (op >> 5) & 3; }

// ---- in-VM Rescue permutation pieces (utils/sponge.rs: 4 wide; utils/hasher.rs: 6 wide) ----------------
namespace sponge4 {
static inline void apply_sbox(u128 *s) { for (int i = 0; i < 4; i++) s[i] = field::exp(s[i], 3); }
static inline void apply_inv_sbox(u128 *s) { u128 ia = cst(REF_INV_ALPHA); for (int i = 0; i < 4; i++) s[i] = field::exp(s[i], ia); }
static inline void matmul(u128 *s, const unsigned long long (*m)[2]) {
    u128 r[4];
    for (int i = 0; i < 4; i++) { r[i] = 0; for (int j = 0; j < 4; j++) r[i] = field::add(r[i], field::mul(cst(m[i * 4 + j]), s[j])); }
    memcpy(s, r, sizeof r);
}
static inline void apply_mds(u128 *s) { matmul(s, REF_SPONGE_MDS); }
static inline void apply_inv_mds(u128 *s) { matmul(s, REF_SPONGE_INV_MDS); }
static inline u128 ark(size_t reg, size_t round) { return cst(REF_SPONGE_ARK[reg * 16 + round]); }
// sponge.rs:13-30
static inline void apply_round(u128 *s, u128 op_code, u128 op_value, size_t step) {
    size_t idx = step % 16;
    for (int i = 0; i < 4; i++) s[i] = field::add(s[i], ark(i, idx));
    apply_sbox(s); apply_mds(s);
    s[0] = field::add(s[0], op_code);
    s[1] = field::add(s[1], op_value);
    for (int i = 0; i < 4; i++) s[i] = field::add(s[i], ark(4 + i, idx));
    apply_inv_sbox(s); apply_mds(s);
}
} // namespace sponge4

namespace hasher6 {
static inline void apply_sbox(u128 *s) { for (int i = 0; i < 6; i++) s[i] = field::exp(s[i], 3); }
static inline void apply_inv_sbox(u128 *s) { u128 ia = cst(REF_INV_ALPHA); for (int i = 0; i < 6; i++) s[i] = field::exp(s[i], ia); }
static inline void matmul(u128 *s, const unsigned long long (*m)[2]) {
    u128 r[6];
    for (int i = 0; i < 6; i++) { r[i] = 0; for (int j = 0; j < 6; j++) r[i] = field::add(r[i], field::mul(cst(m[i * 6 + j]), s[j])); }
    memcpy(s, r, sizeof r);
}
static inline void apply_mds(u128 *s) { matmul(s, REF_HASHER_MDS); }
static inline void apply_inv_mds(u128 *s) { matmul(s, REF_HASHER_INV_MDS); }
static inline u128 ark(size_t reg, size_t round) { return cst(REF_HASHER_ARK[reg * 16 + round]); }
// hasher.rs:28-40
static inline void apply_round(u128 *s, size_t step) {
    size_t idx = step % 16;
    for (int i = 0; i < 6; i++) s[i] = field::add(s[i], ark(i, idx));
    apply_sbox(s); apply_mds(s);
    for (int i = 0; i < 6; i++) s[i] = field::add(s[i], ark(6 + i, idx));
    apply_inv_sbox(s); apply_mds(s);
}
// hasher.rs:12-26
static inline void digest(const u128 *values, size_t n, u128 out[2]) {
    u128 st[6] = {0, 0, 0, 0, 0, 0};
    for (size_t i = 0; i < n; i++) st[i] = values[i];
    std::reverse(st, st + 6);
    for (int i = 0; i < 10; i++) apply_round(st, i);
    std::reverse(st, st + 6);
    out[0] = st[0]; out[1] = st[1];
}
} // namespace hasher6

// ---- TraceState ------------------------------------------------------------------------------------------
struct TraceState {
    u128 op_counter;
    u128 sponge[4], cf_bits[3], ld_bits[5], hd_bits[2];
    u128 ctx_stack[MAX_CONTEXT_DEPTH], loop_stack[MAX_LOOP_DEPTH], user_stack[MAX_STACK_DEPTH];
    size_t ctx_depth, loop_depth, stack_depth;
    size_t ctx_len, loop_len, stack_len;  // padded lengths: max(depth, MIN_*)   (trace_state.rs:58-60)
    u128 cf_flags[8], ld_flags[32], hd_flags[4], begin_flag, noop_flag;

    TraceState(size_t cd, size_t ld, size_t sd) : ctx_depth(cd), loop_depth(ld), stack_depth(sd) {
        ctx_len = std::max(cd, MIN_CONTEXT_DEPTH); loop_len = std::max(ld, MIN_LOOP_DEPTH); stack_len = std::max(sd, MIN_STACK_DEPTH);
        op_counter = 0;
        memset(sponge, 0, sizeof sponge); memset(cf_bits, 0, sizeof cf_bits); memset(ld_bits, 0, sizeof ld_bits); memset(hd_bits, 0, sizeof hd_bits);
        memset(ctx_stack, 0, sizeof ctx_stack); memset(loop_stack, 0, sizeof loop_stack); memset(user_stack, 0, sizeof user_stack);
        set_op_flags();
    }
    size_t width() const { return 15 + ctx_depth + loop_depth + stack_depth; }

    // trace_state.rs:77-117 / :251-277
    void from_row(const u128 *row) {
        op_counter = row[0];
        for (int i = 0; i < 4; i++) sponge[i] = row[1 + i];
        for (int i = 0; i < 3; i++) cf_bits[i] = row[5 + i];
        for (int i = 0; i < 5; i++) ld_bits[i] = row[8 + i];
        for (int i = 0; i < 2; i++) hd_bits[i] = row[13 + i];
        size_t o = 15;
        for (size_t i = 0; i < ctx_depth; i++) ctx_stack[i] = row[o + i];
        o += ctx_depth;
        for (size_t i = 0; i < loop_depth; i++) loop_stack[i] = row[o + i];
        o += loop_depth;
        for (size_t i = 0; i < stack_depth; i++) user_stack[i] = row[o + i];
        set_op_flags();
    }
    void from_columns(const std::vector<std::vector<u128>> &trace, size_t step) {
        u128 row[MAX_REGISTER_COUNT];
        for (size_t j = 0; j < width(); j++) row[j] = trace[j][step];
        from_row(row);
    }
    // trace_state.rs:169-178
    u128 op_code() const {
        u128 r = ld_bits[0];
        r = field::add(r, field::mul(ld_bits[1], 2)); r = field::add(r, field::mul(ld_bits[2], 4));
        r = field::add(r, field::mul(ld_bits[3], 8)); r = field::add(r, field::mul(ld_bits[4], 16));
        r = field::add(r, field::mul(hd_bits[0], 32)); r = field::add(r, field::mul(hd_bits[1], 64));
        return r;
    }
    // trace_state.rs:281-350
    void set_op_flags() {
        using field::mul; using field::sub;
        u128 not_0 = sub(1, cf_bits[0]), not_1 = sub(1, cf_bits[1]);
        cf_flags[0] = mul(not_0, not_1); cf_flags[1] = mul(cf_bits[0], not_1);
        cf_flags[2] = mul(not_0, cf_bits[1]); cf_flags[3] = mul(cf_bits[0], cf_bits[1]);
        for (int i = 0; i < 4; i++) cf_flags[4 + i] = cf_flags[i];
        u128 not_2 = sub(1, cf_bits[2]);
        for (int i = 0; i < 4; i++) cf_flags[i] = mul(cf_flags[i], not_2);
        for (int i = 4; i < 8; i++) cf_flags[i] = mul(cf_flags[i], cf_bits[2]);

        not_0 = sub(1, ld_bits[0]); not_1 = sub(1, ld_bits[1]);
        ld_flags[0] = mul(not_0, not_1); ld_flags[1] = mul(ld_bits[0], not_1);
        ld_flags[2] = mul(not_0, cf_bits[1]);  // sic: trace_state.rs:301 uses cf_op_bits[1]
        ld_flags[3] = mul(ld_bits[0], ld_bits[1]);
        for (int i = 0; i < 4; i++) ld_flags[4 + i] = ld_flags[i];
        not_2 = sub(1, ld_bits[2]);
        for (int i = 0; i < 4; i++) ld_flags[i] = mul(ld_flags[i], not_2);
        for (int i = 4; i < 8; i++) ld_flags[i] = mul(ld_flags[i], ld_bits[2]);
        for (int i = 0; i < 8; i++) ld_flags[8 + i] = ld_flags[i];
        u128 not_3 = sub(1, ld_bits[3]);
        for (int i = 0; i < 8; i++) ld_flags[i] = mul(ld_flags[i], not_3);
        for (int i = 8; i < 16; i++) ld_flags[i] = mul(ld_flags[i], ld_bits[3]);
        for (int i = 0; i < 16; i++) ld_flags[16 + i] = ld_flags[i];
        u128 not_4 = sub(1, ld_bits[4]);
        for (int i = 0; i < 16; i++) ld_flags[i] = mul(ld_flags[i], not_4);
        for (int i = 16; i < 32; i++) ld_flags[i] = mul(ld_flags[i], ld_bits[4]);

        not_0 = sub(1, hd_bits[0]); not_1 = sub(1, hd_bits[1]);
        hd_flags[0] = mul(not_0, not_1); hd_flags[1] = mul(hd_bits[0], not_1);
        hd_flags[2] = mul(not_0, hd_bits[1]); hd_flags[3] = mul(hd_bits[0], hd_bits[1]);

        begin_flag = mul(ld_flags[ld_index(OP_BEGIN)], hd_flags[hd_index(OP_BEGIN)]);
        noop_flag = mul(ld_flags[ld_index(OP_NOOP)], hd_flags[hd_index(OP_NOOP)]);
        hd_flags[0] = mul(hd_flags[0], ld_bits[0]);   // PUSH adjust
        ld_flags[0] = mul(ld_flags[0], hd_bits[0]);   // ASSERT adjust
    }
};

// ---- coefficients (coefficients.rs) ----------------------------------------------------------------------
struct BoundaryCoefficients {
    u128 op_counter[2], sponge[8], op_bits[20], ctx_stack[32], loop_stack[16], user_stack[16];
};
static const size_t NUM_BOUNDARY_CONSTRAINTS = 1 + 4 + 10 + 16 + 8 + 8;            // 47
static const size_t NUM_STATIC_DECODER_CONSTRAINTS = 15 + 4 + 1;                   // 20
static const size_t NUM_AUX_STACK_CONSTRAINTS = 2;
static const size_t NUM_TRANSITION_CONSTRAINTS = NUM_STATIC_DECODER_CONSTRAINTS + 16 + 8 + 32 + NUM_AUX_STACK_CONSTRAINTS;  // 78
static const size_t NUM_CONSTRAINTS = NUM_TRANSITION_CONSTRAINTS + 2 * NUM_BOUNDARY_CONSTRAINTS;                            // 172

struct ConstraintCoefficients {
    BoundaryCoefficients i_boundary, f_boundary;
    std::vector<u128> transition;
    ConstraintCoefficients() {}
    ConstraintCoefficients(const uint8_t seed[32], size_t ctx_depth, size_t loop_depth, size_t stack_depth) {
        std::vector<u128> c = prng_vector(seed, 2 * NUM_CONSTRAINTS);
        size_t i = fill_boundary(i_boundary, c.data());
        i += fill_boundary(f_boundary, c.data() + i);
        const u128 *t = c.data() + i;
        size_t cd = std::max(ctx_depth, MIN_CONTEXT_DEPTH), ld = std::max(loop_depth, MIN_LOOP_DEPTH), sd = std::max(stack_depth, MIN_STACK_DEPTH);
        // coefficients.rs:140-185: source laid out for MAX depths, target compacted
        size_t s = 0;
        auto take = [&](size_t src, size_t n) { for (size_t k = 0; k < n; k++) transition.push_back(t[src + k]); };
        take(s, NUM_STATIC_DECODER_CONSTRAINTS * 2); s += NUM_STATIC_DECODER_CONSTRAINTS * 2;
        take(s, cd * 2);                             s += MAX_CONTEXT_DEPTH * 2;
        take(s, ld * 2);                             s += MAX_LOOP_DEPTH * 2;
        take(s, NUM_AUX_STACK_CONSTRAINTS * 2);      s += NUM_AUX_STACK_CONSTRAINTS * 2;
        take(s, sd * 2);
    }
    static size_t fill_boundary(BoundaryCoefficients &b, const u128 *c) {
        size_t o = 0;
        memcpy(b.op_counter, c + o, sizeof b.op_counter); o += 2;
        memcpy(b.sponge, c + o, sizeof b.sponge); o += 8;
        memcpy(b.op_bits, c + o, sizeof b.op_bits); o += 20;
        memcpy(b.ctx_stack, c + o, sizeof b.ctx_stack); o += 32;
        memcpy(b.loop_stack, c + o, sizeof b.loop_stack); o += 16;
        memcpy(b.user_stack, c + o, sizeof b.user_stack); o += 16;
        return o;
    }
};

struct CompositionCoefficients {
    u128 trace1[2 * MAX_REGISTER_COUNT], trace2[2 * MAX_REGISTER_COUNT], t1_degree, t2_degree, constraints;
    explicit CompositionCoefficients(const uint8_t seed[32]) {
        std::vector<u128> c = prng_vector(seed, 1 + 4 * MAX_REGISTER_COUNT + 3);
        memcpy(trace1, c.data() + 1, sizeof trace1);
        memcpy(trace2, c.data() + 1 + 2 * MAX_REGISTER_COUNT, sizeof trace2);
        size_t idx = 1 + 4 * MAX_REGISTER_COUNT;
        t1_degree = c[idx]; t2_degree = c[idx + 1]; constraints = c[idx + 2];
    }
};

// ---- shared constraint helpers (constraints/utils.rs) -------------------------------------------------------
namespace cu {
static inline u128 is_binary(u128 v) { return field::sub(field::mul(v, v), v); }
static inline u128 binary_not(u128 v) { return field::sub(1, v); }
static inline u128 are_equal(u128 a, u128 b) { return field::sub(a, b); }
static inline void agg(u128 *r, size_t i, u128 flag, u128 value) { r[i] = field::add(r[i], field::mul(flag, value)); }
static inline void stack_copy(u128 *r, size_t rlen, const u128 *o, const u128 *n, size_t from, u128 flag) {
    for (size_t i = from; i < rlen; i++) agg(r, i, flag, are_equal(o[i], n[i]));
}
static inline void right_shift(u128 *r, size_t rlen, const u128 *o, const u128 *n, size_t num, u128 flag) {
    for (size_t i = num; i < rlen; i++) agg(r, i, flag, are_equal(o[i - num], n[i]));
}
static inline void left_shift(u128 *r, size_t rlen, const u128 *o, const u128 *n, size_t from, size_t num, u128 flag) {
    size_t start = from - num, rem = rlen - num;
    for (size_t i = start; i < rem; i++) agg(r, i, flag, are_equal(o[i + num], n[i]));
    for (size_t i = rem; i < rlen; i++) agg(r, i, flag, n[i]);
}
// constraints/utils.rs:87-113 : interpolate 16 values, zero-pad, evaluate on 16*ext points
static inline void extend_constants(const unsigned long long (*table)[2], size_t ncols, size_t ext,
                                    std::vector<std::vector<u128>> &polys, std::vector<std::vector<u128>> &evals,
                                    const u128 *direct = nullptr) {
    u128 root = field::get_root_of_unity(BASE_CYCLE_LENGTH);
    std::vector<u128> inv_tw = fft::get_inv_twiddles(root, BASE_CYCLE_LENGTH);
    size_t domain = BASE_CYCLE_LENGTH * ext;
    std::vector<u128> tw = fft::get_twiddles(field::get_root_of_unity(domain), domain);
    for (size_t c = 0; c < ncols; c++) {
        std::vector<u128> e(BASE_CYCLE_LENGTH);
        for (size_t k = 0; k < BASE_CYCLE_LENGTH; k++) e[k] = direct ? direct[c * BASE_CYCLE_LENGTH + k] : cst(table[c * BASE_CYCLE_LENGTH + k]);
        polynom::interpolate_fft_twiddles(e.data(), e.size(), inv_tw.data(), true);
        polys.push_back(e);
        e.resize(domain, 0);
        polynom::eval_fft_twiddles(e.data(), e.size(), tw.data(), true);
        evals.push_back(e);
    }
}
} // namespace cu

// ---- Decoder constraints -------------------------------------------------------------------------------------
struct DecoderAir {
    size_t ctx_depth, loop_depth, trace_length, cycle_length;
    std::vector<std::vector<u128>> ark_polys, ark_evals, mask_polys, mask_evals;
    std::vector<size_t> degrees;

    DecoderAir() {}
    DecoderAir(size_t n, size_t ext, size_t cd, size_t ld) : ctx_depth(cd), loop_depth(ld), trace_length(n) {
        static const size_t OP_DEG[15] = { 2, 2, 2, 2, 2, 2, 2, 2, 2, 2, 3, 8, 8, 6, 4 };
        static const size_t SPONGE_DEG[4] = { 6, 7, 6, 6 };
        degrees.assign(OP_DEG, OP_DEG + 15);
        degrees.insert(degrees.end(), SPONGE_DEG, SPONGE_DEG + 4);
        degrees.push_back(4);
        degrees.resize(degrees.size() + std::max(cd, MIN_CONTEXT_DEPTH) + std::max(ld, MIN_LOOP_DEPTH), 4);
        cycle_length = BASE_CYCLE_LENGTH * ext;
        cu::extend_constants(REF_SPONGE_ARK, 8, ext, ark_polys, ark_evals);
        static const u128 MASKS[3 * 16] = {  // decoder/mod.rs:219-223
            0, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1,
            1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0,
            0, 1, 1, 1, 1, 1, 1, 1, 0, 1, 1, 1, 1, 1, 1, 1 };
        cu::extend_constants(nullptr, 3, ext, mask_polys, mask_evals, MASKS);
    }
    size_t constraint_count() const { return degrees.size(); }

    void evaluate(const TraceState &cur, const TraceState &nxt, size_t step, u128 *result) const {
        u128 ark[8], masks[3];
        for (int j = 0; j < 8; j++) ark[j] = ark_evals[j][step % cycle_length];
        for (int j = 0; j < 3; j++) masks[j] = mask_evals[j][step % cycle_length];
        run(cur, nxt, ark, masks, result);
    }
    void evaluate_at(const TraceState &cur, const TraceState &nxt, u128 x, u128 *result) const {
        u128 xc = field::exp(x, (u128)(trace_length / BASE_CYCLE_LENGTH));
        u128 ark[8], masks[3];
        for (int j = 0; j < 8; j++) ark[j] = polynom::eval(ark_polys[j], xc);
        for (int j = 0; j < 3; j++) masks[j] = polynom::eval(mask_polys[j], xc);
        run(cur, nxt, ark, masks, result);
    }

    void run(const TraceState &cur, const TraceState &nxt, const u128 *ark, const u128 *masks, u128 *result) const {
        using namespace cu; using field::add; using field::mul; using field::sub;
        // ---- op_bits.rs:10-79
        size_t i = 0;
        u128 cf_bit_sum = 0, ld_bit_prod = 1, hd_bit_prod = 1;
        for (int k = 0; k < 3; k++) { result[i++] = is_binary(cur.cf_bits[k]); cf_bit_sum = add(cf_bit_sum, cur.cf_bits[k]); }
        for (int k = 0; k < 5; k++) { result[i++] = is_binary(cur.ld_bits[k]); ld_bit_prod = mul(ld_bit_prod, cur.ld_bits[k]); }
        for (int k = 0; k < 2; k++) { result[i++] = is_binary(cur.hd_bits[k]); hd_bit_prod = mul(hd_bit_prod, cur.hd_bits[k]); }
        u128 is_hacc = cur.cf_flags[F_HACC];
        u128 hacc_transition = mul(add(cur.op_counter, 1), is_hacc);
        u128 rest_transition = mul(cur.op_counter, binary_not(is_hacc));
        result[i++] = are_equal(add(hacc_transition, rest_transition), nxt.op_counter);
        result[i++] = mul(cur.op_counter, mul(binary_not(ld_bit_prod), binary_not(hd_bit_prod)));
        result[i++] = mul(cf_bit_sum, binary_not(mul(ld_bit_prod, hd_bit_prod)));
        result[i++] = mul(cur.cf_flags[F_VOID], binary_not(nxt.cf_flags[F_VOID]));
        // alignment constraint (index 14) aggregates several flags
        agg(result, i, cur.cf_flags[F_BEGIN], masks[1]); agg(result, i, cur.cf_flags[F_LOOP], masks[1]);
        agg(result, i, cur.cf_flags[F_WRAP], masks[1]);  agg(result, i, cur.cf_flags[F_BREAK], masks[1]);
        agg(result, i, cur.cf_flags[F_TEND], masks[0]);  agg(result, i, cur.cf_flags[F_FEND], masks[0]);
        agg(result, i, cur.hd_flags[hd_index(OP_PUSH)], masks[2]);

        u128 *r = result + 15;
        const size_t cl = cur.ctx_len, ll = cur.loop_len;
        u128 *ctx_r = r + SPONGE_WIDTH + 1, *loop_r = ctx_r + cl;
        const u128 *os = cur.sponge, *ns = nxt.sponge;

        // ---- HACC  sponge.rs:10-43
        {
            u128 f = cur.cf_flags[F_HACC];
            u128 op_value = mul(nxt.user_stack[0], cur.hd_flags[hd_index(OP_PUSH)]);
            u128 old_s[4], new_s[4];
            for (int k = 0; k < 4; k++) old_s[k] = add(os[k], ark[k]);
            sponge4::apply_sbox(old_s); sponge4::apply_mds(old_s);
            old_s[0] = add(old_s[0], cur.op_code());
            old_s[1] = add(old_s[1], op_value);
            for (int k = 0; k < 4; k++) new_s[k] = ns[k];
            sponge4::apply_inv_mds(new_s); sponge4::apply_sbox(new_s);
            for (int k = 0; k < 4; k++) new_s[k] = sub(new_s[k], ark[4 + k]);
            for (int k = 0; k < 4; k++) agg(r, k, f, are_equal(old_s[k], new_s[k]));
        }
        // ---- BEGIN  flow_ops.rs:10-31
        {
            u128 f = cur.cf_flags[F_BEGIN];
            for (int k = 0; k < 4; k++) agg(r, k, f, ns[k]);
            agg(ctx_r, 0, f, are_equal(os[0], nxt.ctx_stack[0]));
            right_shift(ctx_r, cl, cur.ctx_stack, nxt.ctx_stack, 1, f);
            stack_copy(loop_r, ll, cur.loop_stack, nxt.loop_stack, 0, f);
        }
        // ---- TEND  flow_ops.rs:33-54
        {
            u128 f = cur.cf_flags[F_TEND];
            agg(r, 0, f, are_equal(cur.ctx_stack[0], ns[0]));
            agg(r, 1, f, are_equal(os[0], ns[1]));
            agg(r, 3, f, ns[3]);
            left_shift(ctx_r, cl, cur.ctx_stack, nxt.ctx_stack, 1, 1, f);
            stack_copy(loop_r, ll, cur.loop_stack, nxt.loop_stack, 0, f);
        }
        // ---- FEND  flow_ops.rs:56-77
        {
            u128 f = cur.cf_flags[F_FEND];
            agg(r, 0, f, are_equal(cur.ctx_stack[0], ns[0]));
            agg(r, 2, f, are_equal(os[0], ns[2]));
            agg(r, 3, f, ns[3]);
            left_shift(ctx_r, cl, cur.ctx_stack, nxt.ctx_stack, 1, 1, f);
            stack_copy(loop_r, ll, cur.loop_stack, nxt.loop_stack, 0, f);
        }
        // ---- LOOP  flow_ops.rs:79-101
        {
            u128 f = cur.cf_flags[F_LOOP];
            for (int k = 0; k < 4; k++) agg(r, k, f, ns[k]);
            agg(ctx_r, 0, f, are_equal(os[0], nxt.ctx_stack[0]));
            right_shift(ctx_r, cl, cur.ctx_stack, nxt.ctx_stack, 1, f);
            right_shift(loop_r, ll, cur.loop_stack, nxt.loop_stack, 1, f);
        }
        // ---- WRAP  flow_ops.rs:103-125
        {
            u128 f = cur.cf_flags[F_WRAP];
            for (int k = 0; k < 4; k++) agg(r, k, f, ns[k]);
            agg(r, SPONGE_WIDTH, f, are_equal(os[0], cur.loop_stack[0]));
            stack_copy(ctx_r, cl, cur.ctx_stack, nxt.ctx_stack, 0, f);
            stack_copy(loop_r, ll, cur.loop_stack, nxt.loop_stack, 0, f);
        }
        // ---- BREAK  flow_ops.rs:127-148
        {
            u128 f = cur.cf_flags[F_BREAK];
            for (int k = 0; k < 4; k++) agg(r, k, f, are_equal(os[k], ns[k]));
            agg(r, SPONGE_WIDTH, f, are_equal(os[0], cur.loop_stack[0]));
            stack_copy(ctx_r, cl, cur.ctx_stack, nxt.ctx_stack, 0, f);
            left_shift(loop_r, ll, cur.loop_stack, nxt.loop_stack, 1, 1, f);
        }
        // ---- VOID  flow_ops.rs:150-165
        {
            u128 f = cur.cf_flags[F_VOID];
            for (int k = 0; k < 4; k++) agg(r, k, f, are_equal(os[k], ns[k]));
            stack_copy(ctx_r, cl, cur.ctx_stack, nxt.ctx_stack, 0, f);
            stack_copy(loop_r, ll, cur.loop_stack, nxt.loop_stack, 0, f);
        }
    }
};

// ---- Stack constraints -----------------------------------------------------------------------------------------
struct StackAir {
    size_t trace_length, cycle_length, stack_depth;
    std::vector<std::vector<u128>> ark_polys, ark_evals;
    std::vector<size_t> degrees;
    StackAir() {}
    StackAir(size_t n, size_t ext, size_t sd) : trace_length(n), stack_depth(sd) {
        degrees.assign(2, 7);
        degrees.resize(sd + NUM_AUX_STACK_CONSTRAINTS, 7);
        cycle_length = BASE_CYCLE_LENGTH * ext;
        cu::extend_constants(REF_HASHER_ARK, 12, ext, ark_polys, ark_evals);
    }
    void evaluate(const TraceState &cur, const TraceState &nxt, size_t step, u128 *result) const {
        u128 ark[12];
        for (int j = 0; j < 12; j++) ark[j] = ark_evals[j][step % cycle_length];
        run(cur, nxt, ark, result);
    }
    void evaluate_at(const TraceState &cur, const TraceState &nxt, u128 x, u128 *result) const {
        u128 xc = field::exp(x, (u128)(trace_length / BASE_CYCLE_LENGTH));
        u128 ark[12];
        for (int j = 0; j < 12; j++) ark[j] = polynom::eval(ark_polys[j], xc);
        run(cur, nxt, ark, result);
    }
    // stack/mod.rs:117-195
    void run(const TraceState &cur, const TraceState &nxt, const u128 *ark, u128 *result) const {
        using namespace cu; using field::add; using field::mul; using field::sub;
        u128 *aux = result;
        u128 *out = result + NUM_AUX_STACK_CONSTRAINTS;
        const u128 *o = cur.user_stack, *n = nxt.user_stack;
        const size_t L = cur.stack_len;
        u128 ev[MAX_STACK_DEPTH];
        for (size_t i = 0; i < L; i++) ev[i] = 0;
        const u128 *ldf = cur.ld_flags;
        u128 f;

        // assert / asserteq   comparison.rs:25-38
        f = ldf[ld_index(OP_ASSERT)];   left_shift(ev, L, o, n, 1, 1, f); agg(aux, 0, f, are_equal(1, o[0]));
        f = ldf[ld_index(OP_ASSERTEQ)]; left_shift(ev, L, o, n, 2, 2, f); agg(aux, 0, f, are_equal(o[0], o[1]));
        // read / read2   input.rs
        f = ldf[ld_index(OP_READ)];  right_shift(ev, L, o, n, 1, f);
        f = ldf[ld_index(OP_READ2)]; right_shift(ev, L, o, n, 2, f);
        // dup / dup2 / dup4 / pad2   manipulation.rs:12-48
        f = ldf[ld_index(OP_DUP)];  agg(ev, 0, f, are_equal(n[0], o[0])); right_shift(ev, L, o, n, 1, f);
        f = ldf[ld_index(OP_DUP2)]; for (int k = 0; k < 2; k++) agg(ev, k, f, are_equal(n[k], o[k])); right_shift(ev, L, o, n, 2, f);
        f = ldf[ld_index(OP_DUP4)]; for (int k = 0; k < 4; k++) agg(ev, k, f, are_equal(n[k], o[k])); right_shift(ev, L, o, n, 4, f);
        f = ldf[ld_index(OP_PAD2)]; agg(ev, 0, f, n[0]); agg(ev, 1, f, n[1]); right_shift(ev, L, o, n, 2, f);
        // drop / drop4
        f = ldf[ld_index(OP_DROP)];  left_shift(ev, L, o, n, 1, 1, f);
        f = ldf[ld_index(OP_DROP4)]; left_shift(ev, L, o, n, 4, 4, f);
        // swap (both constraints land on index 0: manipulation.rs:63-64) / swap2 / swap4
        f = ldf[ld_index(OP_SWAP)];
        agg(ev, 0, f, are_equal(n[0], o[1])); agg(ev, 0, f, are_equal(n[1], o[0])); stack_copy(ev, L, o, n, 2, f);
        f = ldf[ld_index(OP_SWAP2)];
        agg(ev, 0, f, are_equal(n[0], o[2])); agg(ev, 1, f, are_equal(n[1], o[3]));
        agg(ev, 2, f, are_equal(n[2], o[0])); agg(ev, 3, f, are_equal(n[3], o[1])); stack_copy(ev, L, o, n, 4, f);
        f = ldf[ld_index(OP_SWAP4)];
        for (int k = 0; k < 4; k++) agg(ev, k, f, are_equal(n[k], o[4 + k]));
        for (int k = 0; k < 4; k++) agg(ev, 4 + k, f, are_equal(n[4 + k], o[k]));
        stack_copy(ev, L, o, n, 8, f);
        // roll4 / roll8
        f = ldf[ld_index(OP_ROLL4)];
        agg(ev, 0, f, are_equal(n[0], o[3])); for (int k = 1; k < 4; k++) agg(ev, k, f, are_equal(n[k], o[k - 1])); stack_copy(ev, L, o, n, 4, f);
        f = ldf[ld_index(OP_ROLL8)];
        agg(ev, 0, f, are_equal(n[0], o[7])); for (int k = 1; k < 8; k++) agg(ev, k, f, are_equal(n[k], o[k - 1])); stack_copy(ev, L, o, n, 8, f);
        // arithmetic.rs
        f = ldf[ld_index(OP_ADD)]; agg(ev, 0, f, are_equal(n[0], add(o[0], o[1]))); left_shift(ev, L, o, n, 2, 1, f);
        f = ldf[ld_index(OP_MUL)]; agg(ev, 0, f, are_equal(n[0], mul(o[0], o[1]))); left_shift(ev, L, o, n, 2, 1, f);
        f = ldf[ld_index(OP_INV)]; agg(ev, 0, f, are_equal(1, mul(n[0], o[0]))); stack_copy(ev, L, o, n, 1, f);
        f = ldf[ld_index(OP_NEG)]; agg(ev, 0, f, add(n[0], o[0])); stack_copy(ev, L, o, n, 1, f);
        f = ldf[ld_index(OP_NOT)]; agg(ev, 0, f, are_equal(n[0], binary_not(o[0]))); stack_copy(ev, L, o, n, 1, f); agg(aux, 0, f, is_binary(o[0]));
        f = ldf[ld_index(OP_AND)]; agg(ev, 0, f, are_equal(n[0], mul(o[0], o[1]))); left_shift(ev, L, o, n, 2, 1, f);
        agg(aux, 0, f, is_binary(o[0])); agg(aux, 1, f, is_binary(o[1]));
        f = ldf[ld_index(OP_OR)];  agg(ev, 0, f, are_equal(n[0], binary_not(mul(binary_not(o[0]), binary_not(o[1]))))); left_shift(ev, L, o, n, 2, 1, f);
        agg(aux, 0, f, is_binary(o[0])); agg(aux, 1, f, is_binary(o[1]));
        // eq   comparison.rs:45-65
        f = ldf[ld_index(OP_EQ)];
        {
            u128 diff = sub(o[1], o[2]);
            agg(ev, 0, f, are_equal(n[0], binary_not(mul(diff, o[0]))));
            left_shift(ev, L, o, n, 3, 2, f);
            agg(aux, 0, f, mul(n[0], diff));
        }
        // binacc   comparison.rs:111-133
        f = ldf[ld_index(OP_BINACC)];
        {
            u128 bit = n[0];
            agg(ev, 0, f, is_binary(bit));
            agg(ev, 1, f, n[1]);
            agg(ev, 2, f, are_equal(n[2], mul(o[2], 2)));
            agg(ev, 3, f, are_equal(n[3], add(o[3], mul(bit, o[2]))));
            stack_copy(ev, L, o, n, 4, f);
        }
        // choose / choose2 / cswap2   conditional.rs
        f = ldf[ld_index(OP_CHOOSE)];
        {
            u128 c = o[2], nc = binary_not(c);
            agg(ev, 0, f, are_equal(n[0], add(mul(c, o[0]), mul(nc, o[1]))));
            left_shift(ev, L, o, n, 3, 2, f);
            agg(aux, 0, f, is_binary(c));
        }
        f = ldf[ld_index(OP_CHOOSE2)];
        {
            u128 c = o[4], nc = binary_not(c);
            agg(ev, 0, f, are_equal(n[0], add(mul(c, o[0]), mul(nc, o[2]))));
            agg(ev, 1, f, are_equal(n[1], add(mul(c, o[1]), mul(nc, o[3]))));
            left_shift(ev, L, o, n, 6, 4, f);
            agg(aux, 0, f, is_binary(c));
        }
        f = ldf[ld_index(OP_CSWAP2)];
        {
            u128 c = o[4], nc = binary_not(c);
            agg(ev, 0, f, are_equal(n[0], add(mul(c, o[2]), mul(nc, o[0]))));
            agg(ev, 1, f, are_equal(n[1], add(mul(c, o[3]), mul(nc, o[1]))));
            agg(ev, 2, f, are_equal(n[2], add(mul(c, o[0]), mul(nc, o[2]))));
            agg(ev, 3, f, are_equal(n[3], add(mul(c, o[1]), mul(nc, o[3]))));
            left_shift(ev, L, o, n, 6, 2, f);
            agg(aux, 0, f, is_binary(c));
        }
        // ---- high-degree ops
        const u128 *hdf = cur.hd_flags;
        f = hdf[hd_index(OP_PUSH)]; right_shift(ev, L, o, n, 1, f);
        // cmp   comparison.rs:71-108   layout [pow, bit_a, bit_b, not_set, gt, lt, acc_b, acc_a]
        f = hdf[hd_index(OP_CMP)];
        {
            u128 x_bit = n[1], y_bit = n[2];
            agg(ev, 0, f, is_binary(x_bit)); agg(ev, 1, f, is_binary(y_bit));
            u128 not_set = n[3];
            u128 bit_gt = mul(x_bit, binary_not(y_bit)), bit_lt = mul(y_bit, binary_not(x_bit));
            u128 gt = add(o[4], mul(bit_gt, not_set)), lt = add(o[5], mul(bit_lt, not_set));
            agg(ev, 2, f, are_equal(n[4], gt)); agg(ev, 3, f, are_equal(n[5], lt));
            u128 p2 = o[0];
            u128 x_acc = add(o[7], mul(x_bit, p2)), y_acc = add(o[6], mul(y_bit, p2));
            agg(ev, 4, f, are_equal(n[6], y_acc)); agg(ev, 5, f, are_equal(n[7], x_acc));
            u128 not_set_check = mul(binary_not(o[5]), binary_not(o[4]));
            agg(ev, 6, f, are_equal(not_set, not_set_check));
            agg(ev, 7, f, are_equal(mul(n[0], 2), p2));
            stack_copy(ev, L, o, n, 8, f);
        }
        // rescr   hash.rs:9-35
        f = hdf[hd_index(OP_RESCR)];
        {
            u128 old_s[6], new_s[6];
            for (int k = 0; k < 6; k++) old_s[k] = add(o[k], ark[k]);
            hasher6::apply_sbox(old_s); hasher6::apply_mds(old_s);
            for (int k = 0; k < 6; k++) new_s[k] = n[k];
            hasher6::apply_inv_mds(new_s); hasher6::apply_sbox(new_s);
            for (int k = 0; k < 6; k++) new_s[k] = sub(new_s[k], ark[6 + k]);
            for (int k = 0; k < 6; k++) agg(ev, k, f, are_equal(new_s[k], old_s[k]));
            stack_copy(ev, L, o, n, 6, f);
        }
        // ---- composite ops: BEGIN and NOOP copy the stack
        stack_copy(ev, L, o, n, 0, cur.begin_flag);
        stack_copy(ev, L, o, n, 0, cur.noop_flag);
        for (size_t i = 0; i < stack_depth; i++) out[i] = ev[i];
    }
};

// ---- Evaluator (evaluator.rs) ---------------------------------------------------------------------------------
struct Evaluator {
    DecoderAir decoder;
    StackAir stack;
    ConstraintCoefficients coefficients;
    size_t domain_size, extension_factor, t_constraint_num;
    std::vector<std::pair<u128, std::vector<size_t>>> t_degree_groups;
    u128 program_hash[2], op_count, b_degree_adj;
    std::vector<u128> inputs, outputs;

    // from_trace (:35-79) when ext == MAX_CONSTRAINT_DEGREE ; from_proof (:81-112) passes the proof's extension factor
    Evaluator(size_t trace_length, size_t ext, size_t domain, size_t cd, size_t ld, size_t sd, const uint8_t trace_root[32],
              const u128 prog_hash[2], u128 opc, const std::vector<u128> &in, const std::vector<u128> &out)
        : decoder(trace_length, ext, cd, ld), stack(trace_length, ext, sd), coefficients(trace_root, cd, ld, sd),
          domain_size(domain), extension_factor(ext), inputs(in), outputs(out) {
        std::vector<size_t> deg = decoder.degrees;
        deg.insert(deg.end(), stack.degrees.begin(), stack.degrees.end());
        t_constraint_num = deg.size();
        // group_transition_constraints :385-406
        std::vector<std::vector<size_t>> groups(9);
        for (size_t i = 0; i < deg.size(); i++) groups[deg[i]].push_back(i);
        size_t target = (MAX_CONSTRAINT_DEGREE - 1) * trace_length + (trace_length - 1);
        for (size_t d = 0; d < groups.size(); d++) {
            if (groups[d].empty()) continue;
            t_degree_groups.push_back({ (u128)(target - (trace_length - 1) * d), groups[d] });
        }
        program_hash[0] = prog_hash[0]; program_hash[1] = prog_hash[1];
        op_count = opc;
        b_degree_adj = (u128)((MAX_CONSTRAINT_DEGREE - 1) * trace_length + 1 - (trace_length - 1));
    }
    size_t trace_length() const { return domain_size / extension_factor; }
    u128 get_x_at_last_step() const {
        return field::exp(field::get_root_of_unity(trace_length()), (u128)(trace_length() - 1));
    }
    bool should_evaluate_to_zero_at(size_t step) const {
        return (step & (extension_factor - 1)) == 0 && step != domain_size - extension_factor;
    }
    // :335-358
    u128 combine_transition_constraints(const std::vector<u128> &ev, u128 x) const {
        const std::vector<u128> &cc = coefficients.transition;
        u128 result = 0;
        size_t i = 0;
        for (auto &grp : t_degree_groups) {
            u128 result_adj = 0;
            for (size_t idx : grp.second) {
                result = field::add(result, field::mul(ev[idx], cc[i * 2]));
                result_adj = field::add(result_adj, field::mul(ev[idx], cc[i * 2 + 1]));
                i++;
            }
            u128 xp = field::exp(x, grp.first);
            result = field::add(result, field::mul(result_adj, xp));
        }
        return result;
    }
    // :139-162 ; `raw` (optional) receives the individual constraint evaluations.  check = false (forged proofs only) skips the
    // assertion and combines the constraints at trace steps as at every other step.
    u128 evaluate_transition(const TraceState &cur, const TraceState &nxt, u128 x, size_t step, std::vector<u128> *raw = nullptr,
                             bool check = true) const {
        std::vector<u128> ev(t_constraint_num, 0);
        decoder.evaluate(cur, nxt, step, ev.data());
        stack.evaluate(cur, nxt, step, ev.data() + decoder.constraint_count());
        if (raw) *raw = ev;
        if (check && should_evaluate_to_zero_at(step)) {
            for (size_t i = 0; i < ev.size(); i++)
                if (ev[i] != 0) throw std::runtime_error("transition constraint at step " + std::to_string(step / extension_factor) + " were not satisfied (constraint " + std::to_string(i) + ")");
            return 0;
        }
        return combine_transition_constraints(ev, x);
    }
    // :167-175
    u128 evaluate_transition_at(const TraceState &cur, const TraceState &nxt, u128 x) const {
        std::vector<u128> ev(t_constraint_num, 0);
        decoder.evaluate_at(cur, nxt, x, ev.data());
        stack.evaluate_at(cur, nxt, x, ev.data() + decoder.constraint_count());
        return combine_transition_constraints(ev, x);
    }
    // :181-326
    void evaluate_boundaries(const TraceState &cur, u128 x, u128 &i_result, u128 &f_result) const {
        using field::add; using field::mul; using field::sub;
        u128 xp = field::exp(x, b_degree_adj);
        {
            const BoundaryCoefficients &cc = coefficients.i_boundary;
            u128 res = 0, adj = 0;
            auto acc = [&](u128 v, u128 c0, u128 c1) { res = add(res, mul(v, c0)); adj = add(adj, mul(v, c1)); };
            acc(cur.op_counter, cc.op_counter[0], cc.op_counter[1]);
            for (int i = 0; i < 4; i++) acc(cur.sponge[i], cc.sponge[i * 2], cc.sponge[i * 2 + 1]);
            size_t k = 0;
            for (int i = 0; i < 3; i++, k += 2) acc(cur.cf_bits[i], cc.op_bits[k], cc.op_bits[k + 1]);
            for (int i = 0; i < 5; i++, k += 2) acc(cur.ld_bits[i], cc.op_bits[k], cc.op_bits[k + 1]);
            for (int i = 0; i < 2; i++, k += 2) acc(cur.hd_bits[i], cc.op_bits[k], cc.op_bits[k + 1]);
            for (size_t i = 0; i < cur.ctx_len; i++) acc(cur.ctx_stack[i], cc.ctx_stack[i * 2], cc.ctx_stack[i * 2 + 1]);
            for (size_t i = 0; i < cur.loop_len; i++) acc(cur.loop_stack[i], cc.loop_stack[i * 2], cc.loop_stack[i * 2 + 1]);
            for (size_t i = 0; i < inputs.size(); i++) acc(sub(cur.user_stack[i], inputs[i]), cc.user_stack[i * 2], cc.user_stack[i * 2 + 1]);
            i_result = add(res, mul(adj, xp));
        }
        {
            const BoundaryCoefficients &cc = coefficients.f_boundary;
            u128 res = 0, adj = 0;
            auto acc = [&](u128 v, u128 c0, u128 c1) { res = add(res, mul(v, c0)); adj = add(adj, mul(v, c1)); };
            acc(sub(cur.op_counter, op_count), cc.op_counter[0], cc.op_counter[1]);
            for (size_t i = 0; i < PROGRAM_DIGEST_SIZE; i++) acc(sub(cur.sponge[i], program_hash[i]), cc.sponge[i * 2], cc.sponge[i * 2 + 1]);
            size_t k = 0;
            for (int i = 0; i < 3; i++, k += 2) acc(sub(cur.cf_bits[i], 1), cc.op_bits[k], cc.op_bits[k + 1]);
            for (int i = 0; i < 5; i++, k += 2) acc(sub(cur.ld_bits[i], 1), cc.op_bits[k], cc.op_bits[k + 1]);
            for (int i = 0; i < 2; i++, k += 2) acc(sub(cur.hd_bits[i], 1), cc.op_bits[k], cc.op_bits[k + 1]);
            for (size_t i = 0; i < cur.ctx_len; i++) acc(cur.ctx_stack[i], cc.ctx_stack[i * 2], cc.ctx_stack[i * 2 + 1]);
            for (size_t i = 0; i < cur.loop_len; i++) acc(cur.loop_stack[i], cc.loop_stack[i * 2], cc.loop_stack[i * 2 + 1]);
            for (size_t i = 0; i < outputs.size(); i++) acc(sub(cur.user_stack[i], outputs[i]), cc.user_stack[i * 2], cc.user_stack[i * 2 + 1]);
            f_result = add(res, mul(adj, xp));
        }
    }
};

} // namespace oracle
#endif
