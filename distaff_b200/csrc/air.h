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
};

// A trace step k that violates a transition constraint is recorded as atomicMax(violation, 0xFFFFFFFF - k), so the lowest violating
// step wins, as in the reference's sequential loop (prover.rs:52-64), and a max-reduce over ranks keeps it.  0 means no violation.
__host__ __device__ inline unsigned violation_word(unsigned long long step) { return 0xFFFFFFFFu - (unsigned)step; }
inline unsigned long long violation_step(unsigned word) { return 0xFFFFFFFFu - word; }

// evaluates the transition constraints of `batch` proofs of one shape (proof q at the strides of P) in one launch (blockIdx.y = proof);
// traces of at least 16 steps
void launch_constraint_eval(Context &c, const AirParams &P, int batch = 1);

}  // namespace dg
