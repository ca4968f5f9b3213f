// Parameters of the constraint-evaluation kernel (air.cu).
#pragma once
#include "common.cuh"

namespace dg {

struct AirParams {
    int w, ctx_depth, loop_depth, stack_depth;
    int cl, ll, sl;                     // padded stack lengths: max(depth, 1 / 1 / 8)   (trace_state.rs:58-60)
    int log_n, log_blowup;
    const fe *ext;                      // extended trace slab of this rank: [w][local cosets][n], column stride col_stride
    unsigned long long col_stride;
    int c8_base, num_c8;                // evaluation-domain cosets handled here: c8 in [c8_base, c8_base + num_c8)  (c8 = step mod 8)
    fe *t_ev;                           // output (combined transition constraints), coset-major: [c8 - c8_base][k]  (step s = 8k + c8)
    const fe *periodic;                 // [128][23] = sponge ARK (8) | masks (3) | hasher ARK (12), row = step % 128
    const fe *coefA, *coefB;            // per transition constraint (evaluation order): cc[2i], cc[2i+1] of its flattened slot
    TwiddleRef twN;                     // powers of the LDE root w_N
    unsigned long long inc[6];          // incremental degrees of the groups 2,3,4,6,7,8  (evaluator.rs:395-402)
    unsigned *violation;                // the lowest violating trace step, encoded by violation_word (0 = none)
    // verifier mode (verifier.cu): evaluate the transition combination at ONE out-of-domain point z -- the rows are (trace(z), trace(z g)),
    // the periodic values are the cycle polynomials at z^(n/16) and the degree-adjustment powers z^inc_g come from the host
    int verify_mode;
    const fe *per_override;             // 23 values, or null
    const fe *xpow_override;            // 6 values, or null
    // batched proving: proof q of the batch reads ext + q * ext_stride and coefA / coefB + q * coef_stride, writes t_ev + q * t_ev_stride
    // and violation[q]
    unsigned long long ext_stride, t_ev_stride, coef_stride;
    // batched verification: proof q reads per_override / xpow_override + q * override_stride
    unsigned long long override_stride;
    // trace check (launch_constraint_check): per trace step k of proof q, masks[(q n + k) * 3 + j] bit i = constraint 32 j + i is nonzero
    unsigned *masks;
};

// The register layout of a trace (trace_state.rs:58-60): 15 decoder registers, the context stack, the loop stack, then the user stack.
struct TraceShape {
    int w, ctx_depth, loop_depth, stack_depth;
    int cl, ll, sl;                     // padded stack lengths: max(depth, 1 / 1 / 8)
    int T;                              // transition constraints: 20 decoder, cl context, ll loop, 2 stack auxiliary, stack_depth stack
    int stack_reg;                      // first user-stack register
    // the layout of depths known to be in range
    TraceShape(int ctx_depth, int loop_depth, int stack_depth);
    // what dg_prove accepts: at most 16 context, 8 loop and 32 user-stack registers, at least one of the last
    static bool in_range(uint32_t ctx_depth, uint32_t loop_depth, uint32_t stack_depth);
    // the shape of a trace of `width` registers (trace_table.rs:23-58); throws DG_ERR_INVALID with the prover's message when out of range
    static TraceShape of_trace(uint32_t width, uint32_t ctx_depth, uint32_t loop_depth);
    // AirParams with this shape's part filled in for traces of n steps (depths, padded lengths, log_n, inc[]), every other field zero
    AirParams air_params(uint64_t n) const;
};

// exponent of the degree adjustment of degree group g (degrees 2, 3, 4, 6, 7, 8) for traces of n steps (evaluator.rs:395-402)
unsigned long long group_increment(int g, uint64_t n);

// the periodic AIR tables on c's device, uploaded the first time
const fe *periodic_table(Context &c);

// A trace step k that violates a transition constraint is recorded as atomicMax(violation, 0xFFFFFFFF - k), so the lowest violating
// step wins, as in the reference's sequential loop (prover.rs:52-64), and a max-reduce over ranks keeps it.  0 means no violation.
__host__ __device__ inline unsigned violation_word(unsigned long long step) { return 0xFFFFFFFFu - (unsigned)step; }
inline unsigned long long violation_step(unsigned word) { return 0xFFFFFFFFu - word; }

// evaluates the transition constraints of `batch` proofs of one shape (proof q at the strides of P) in one launch (blockIdx.y = proof);
// traces of at least 16 steps
void launch_constraint_eval(Context &c, const AirParams &P, int batch = 1);

// the trace check: the same kernel on the register traces themselves (coset 0 of the extension is the trace: num_c8 = 1, log_blowup = 3,
// col_stride = n, ext_stride = w n), recording per trace step which constraints do not vanish (P.masks, 3 words per step; the exempt
// last step n - 1 gets 0) instead of combining them.  No coefficient, power of x or violation word is read or written.
void launch_constraint_check(Context &c, const AirParams &P, int batch);
// masks of `batch` traces of n steps -> per trace q, at stats + q * CHECK_STATS: [0, 96) violating steps per constraint, [96] steps with
// any violation, then at + 97 the lowest such step (UINT64_MAX if none), in the same order
constexpr int CHECK_SLOTS = 97, CHECK_STATS = 2 * CHECK_SLOTS;
void launch_check_reduce(Context &c, const unsigned *masks, unsigned long long n, int T, int batch, unsigned long long *stats);

}  // namespace dg
