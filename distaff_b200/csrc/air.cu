// Constraint evaluation kernel: one thread per point of the 8n-point constraint evaluation domain.
//
// Replaces the serial loop of /root/reference/src/stark/prover.rs:52-64 and everything it calls:
//   TraceState::update_from_trace / set_op_flags   /root/reference/src/stark/trace/trace_state.rs:251-350
//   Evaluator::evaluate_boundaries                 /root/reference/src/stark/constraints/evaluator.rs:181-326
//   Evaluator::evaluate_transition + combine       /root/reference/src/stark/constraints/evaluator.rs:139-162,335-358
//   Decoder constraints                            /root/reference/src/stark/constraints/decoder/{mod.rs:129-150, op_bits.rs, sponge.rs, flow_ops.rs}
//   Stack constraints                              /root/reference/src/stark/constraints/stack/{mod.rs:117-195, *.rs}
//
// All arithmetic is exact in F_M, so sums are regrouped freely (flags of operations that impose the same shift on a
// stack slot are added before the multiplication, the boundary combination is one dot product per row, exp(x, d) is a
// table lookup because x is a power of the LDE root) -- the values written are bit-identical to the reference's.
// Both documented quirks are reproduced: ld_op_flags[2] uses cf_op_bits[1] (trace_state.rs:301) and SWAP accumulates both
// of its constraints into stack slot 0 (stack/manipulation.rs:63-64).
//
// Layout: the extended trace is coset-major ([column][c][k], LDE index = k*blowup + c).  Evaluation-domain step
// s = 8k + c8 uses LDE index s*(blowup/8) => coset c = c8*(blowup/8), element k; the "next" row (LDE index + blowup) is
// element k+1 of the same coset, so both rows are unit-stride reads across a warp.  One kernel, constraint_eval_smem_kernel, serves every
// trace length (n >= 16), the prover and the verifier: it stages a block's rows in shared memory, where each step's "next" row is the
// slot after its own.
// The kernel is tens of thousands of straight-line instructions.  With every field multiplication inlined it is many times the
// size of the instruction cache and the warps starve on instruction fetch, so it calls one shared out-of-line multiply body.
#define DG_MUL_CALL 1
#include "air.h"
#include "air_constants.h"
#include "host_fs.h"

namespace dg {

__constant__ fe c_sponge_mds[16], c_sponge_inv_mds[16], c_hasher_mds[36], c_hasher_inv_mds[36];

void air_upload_constants(Context &c) {
    if (c.air_consts) return;
    auto conv = [](const unsigned long long (*t)[2], int n, std::vector<fe> &out) {
        out.resize(n);
        for (int i = 0; i < n; i++) out[i] = fe_make(t[i][0], t[i][1]);
    };
    std::vector<fe> v;
    conv(DG_SPONGE_MDS, 16, v);      DG_CUDA(cudaMemcpyToSymbol(c_sponge_mds, v.data(), 16 * sizeof(fe)));
    conv(DG_SPONGE_INV_MDS, 16, v);  DG_CUDA(cudaMemcpyToSymbol(c_sponge_inv_mds, v.data(), 16 * sizeof(fe)));
    conv(DG_HASHER_MDS, 36, v);      DG_CUDA(cudaMemcpyToSymbol(c_hasher_mds, v.data(), 36 * sizeof(fe)));
    conv(DG_HASHER_INV_MDS, 36, v);  DG_CUDA(cudaMemcpyToSymbol(c_hasher_inv_mds, v.data(), 36 * sizeof(fe)));
    c.air_consts = true;
}

__device__ __forceinline__ fe tw_pow(const TwiddleRef &t, unsigned long long e) {
    unsigned ee = (unsigned)(e & (unsigned long long)t.mask);
    return fe_mul(t.lo[ee & ((1u << t.lo_bits) - 1u)], t.hi[ee >> t.lo_bits]);
}

// DG_STEP() is a block barrier every few hundred instructions: the warps of a block walk the code together, so that an instruction
// line is fetched once per block instead of once per warp.
#define DG_STEP() __syncthreads()

template <int W>
__device__ __forceinline__ void matvec(const fe *m, fe *s) {
    fe r[W];
#pragma unroll
    for (int i = 0; i < W; i++) {
        r[i] = fe_dot<W>(m + i * W, s);          // one reduction per row: the W products are accumulated unreduced
        DG_STEP();
    }
#pragma unroll
    for (int i = 0; i < W; i++) s[i] = r[i];
}

#define ONE fe_make(1, 0)
#define ZERO fe_make(0, 0)
__device__ __forceinline__ fe bnot(fe v) { return fe_sub(ONE, v); }
__device__ __forceinline__ fe is_bin(fe v) { return fe_sub(fe_sqr(v), v); }

// degree groups in ascending order of constraint degree: 2, 3, 4, 6, 7, 8  (evaluator.rs:385-406)
enum { G2 = 0, G3 = 1, G4 = 2, G6 = 3, G7 = 4, G8 = 5 };

// sums of products accumulated unreduced (fe_wide: fewer than 128 products of canonical operands)
__device__ __forceinline__ void wide_first(fe_wide &w, fe a, fe b) { wide_set(w, DG_MUL_WIDE(a, b)); }
__device__ __forceinline__ void wide_mac(fe_wide &w, fe a, fe b) { wide_add(w, DG_MUL_WIDE(a, b)); }

// The combination  sum_i v_i * cA_i + sum_g (sum_{i in g} v_i * cB_i) * x^inc_g  (evaluator.rs:335-358).  The constraints are evaluated
// group by group, so each degree group is one run: its cB side is accumulated unreduced in `run`, reduced once when the run closes and
// multiplied by x^inc_g into `res`, which is reduced once at the end.  Bounds (products per accumulator, all operands canonical):
//   res: one per constraint (at most 20 + 16 + 8 + 2 + 32 = 78) + one per group (6) = 84;
//   run: the longest runs are G7 (sponge 1, 2 aux, at most 32 stack slots: 35) and G4 (align, image, at most 16 context and 8 loop
//   entries: 26).  launch_constraint_eval checks cl <= 16, ll <= 8, sl <= 32.
struct Acc {
    fe_wide res, run;
    bool nonzero, first, run_first;
    __device__ __forceinline__ void fold(fe v, fe a, fe b) {
        if (first) { wide_first(res, v, a); first = false; }
        else wide_mac(res, v, a);
        if (run_first) { wide_first(run, v, b); run_first = false; }
        else wide_mac(run, v, b);
        nonzero = nonzero || !fe_is_zero(v);
    }
    __device__ __forceinline__ void close(fe xpow) {
        wide_mac(res, DG_REDUCE_WIDE(run), xpow);
        run_first = true;
    }
};

// The rows of a block's BLOCK consecutive steps are staged once in shared memory, column-major, so that the "next" row of every thread
// is the slot after its own:
//   n >= BLOCK: the block lies inside one coset.  Pitch BLOCK + 1; slot t holds the row of thread t, and the extra slot BLOCK the
//     "next" row of the block's last thread.
//   n < BLOCK (SHORT, n >= 16): the block covers BLOCK / n whole cosets.  Thread t stores its row at slot t + t / n, which leaves a
//     spare slot after each coset's n rows; the coset's k = 0 thread stores its row there too, as the wrap-around "next" row of the
//     coset's last step.  Pitch BLOCK + BLOCK / 16.
// Context / loop / user-stack registers are then addressed dynamically in shared memory instead of in per-thread arrays, which the
// runtime loop bounds would force into local memory; stack slots >= 8 are folded into the accumulators as soon as they are evaluated.
// The 15 decoder registers are staged as well (read from shared memory at every use) instead of being held in registers.
// blockIdx.y is the proof of a batch (AirParams strides).
// CHECK: the trace check (launch_constraint_check).  fold records which constraints are nonzero in three mask words instead of combining
// them, close does nothing, and each step writes its mask words.
template <int BLOCK, int MIN_BLOCKS, bool SHORT = false, bool CHECK = false>
__global__ void __launch_bounds__(BLOCK, MIN_BLOCKS) constraint_eval_smem_kernel(const AirParams P) {
    extern __shared__ __align__(16) unsigned char air_smem[];
    fe *s_rows = reinterpret_cast<fe *>(air_smem);
    constexpr int PITCH = SHORT ? BLOCK + BLOCK / 16 : BLOCK + 1;
    const int tid = threadIdx.x;
    const int slot = SHORT ? tid + (tid >> P.log_n) : tid;
    const unsigned long long n = 1ULL << P.log_n;
    const unsigned long long total = n * (unsigned long long)P.num_c8;
    unsigned long long gid = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = gid < total;            // no early exit: every thread takes part in the barriers
    if (!live) gid = total - 1;
    const unsigned long long c8_local = gid >> P.log_n, k = gid & (n - 1);
    const unsigned long long c8 = c8_local + P.c8_base;
    const unsigned long long s = (k << 3) + c8;                       // evaluation-domain step
    const int stride = 1 << (P.log_blowup - 3);
    const unsigned long long N = P.col_stride;                         // column stride of the local slab
    const unsigned long long lde_index = s * (unsigned long long)stride;   // = k*blowup + c8*stride
    const fe *const ext = P.ext + blockIdx.y * P.ext_stride;
    const fe *cur_p = ext + (c8_local * stride) * n + k;              // the slab starts at coset c8_base*stride
    const unsigned long long out_idx = (c8_local << P.log_n) + k;

    const int cl = P.cl, ll = P.ll, sl = P.sl;
    const int ctx_off = 15, loop_off = 15 + P.ctx_depth, stk_off = 15 + P.ctx_depth + P.loop_depth;

    // ---- the two rows.  Boundary constraints are not evaluated here: their numerators are assembled in coefficient form from the
    //      trace polynomials (poly.cu: boundary_coeffs), which is 8x less work than evaluating them on this domain.
    {
        const int w = P.w;
        // the k = 0 test is on tid, so that threads past the end of the domain (clamped to its last step) fill their spare slots too
        const bool wrap_row = SHORT && (tid & (n - 1)) == 0;
        for (int j = 0; j < w; j++) {
            const fe v = cur_p[(unsigned long long)j * N];
            s_rows[j * PITCH + slot] = v;
            if (wrap_row) s_rows[j * PITCH + slot + (int)n] = v;
        }
        // the extra row: "next" of the block's last thread (k + 1 wraps to 0 of the same coset at the end of the coset)
        if (!SHORT && tid < w) {
            const unsigned long long gl = (unsigned long long)blockIdx.x * BLOCK + (BLOCK - 1);
            const unsigned long long cl8 = gl >> P.log_n, kl = gl & (n - 1);
            s_rows[tid * PITCH + BLOCK] = ext[(unsigned long long)tid * N + (cl8 * stride) * n + ((kl + 1) & (n - 1))];
        }
    }
    __syncthreads();
#define SCOL(col, nx) s_rows[(col) * PITCH + slot + (nx)]
#define DCUR(j) s_rows[(j) * PITCH + slot]
#define DNXT(j) s_rows[(j) * PITCH + slot + 1]
#define C_CTX(i) (((i) < P.ctx_depth) ? SCOL(ctx_off + (i), 0) : ZERO)
#define N_CTX(i) (((i) < P.ctx_depth) ? SCOL(ctx_off + (i), 1) : ZERO)
#define C_LOOP(i) (((i) < P.loop_depth) ? SCOL(loop_off + (i), 0) : ZERO)
#define N_LOOP(i) (((i) < P.loop_depth) ? SCOL(loop_off + (i), 1) : ZERO)
#define O(i) (((i) < P.stack_depth) ? SCOL(stk_off + (i), 0) : ZERO)
#define NW(i) (((i) < P.stack_depth) ? SCOL(stk_off + (i), 1) : ZERO)

    DG_STEP();
    // ---- op flags (trace_state.rs:281-350) ----------------------------------------------------------------------------------
    const fe op_counter = DCUR(0);
#define sp(i) DCUR(1 + (i))
#define cf(i) DCUR(5 + (i))
#define ld(i) DCUR(8 + (i))
#define hd(i) DCUR(13 + (i))
#define nsp(i) DNXT(1 + (i))
#define ncf(i) DNXT(5 + (i))
    fe cff[8], ldf[32], hdf[4];
    {
        // products of bits and negated bits; f*(1 - x) is computed as f - f*x (one multiplication per pair of flags)
        fe a3 = fe_mul(cf(0), cf(1));
        fe a1 = fe_sub(cf(0), a3), a2 = fe_sub(cf(1), a3), a0 = fe_sub(bnot(cf(0)), a2);
        cff[4] = fe_mul(a0, cf(2)); cff[5] = fe_mul(a1, cf(2)); cff[6] = fe_mul(a2, cf(2)); cff[7] = fe_mul(a3, cf(2));
        cff[0] = fe_sub(a0, cff[4]); cff[1] = fe_sub(a1, cff[5]); cff[2] = fe_sub(a2, cff[6]); cff[3] = fe_sub(a3, cff[7]);
    }
    fe hdf_raw0;
    {
        hdf[3] = fe_mul(hd(0), hd(1));
        hdf[1] = fe_sub(hd(0), hdf[3]); hdf[2] = fe_sub(hd(1), hdf[3]); hdf[0] = fe_sub(bnot(hd(0)), hdf[2]);
        hdf_raw0 = hdf[0];
        hdf[0] = fe_mul(hdf[0], ld(0));      // PUSH flag adjustment
    }
    fe next_void;
    {
        fe a3 = fe_mul(ncf(0), ncf(1));
        next_void = fe_mul(a3, ncf(2));
    }

    Acc acc;
    acc.first = true;
    acc.run_first = true;
    acc.nonzero = false;
    // CHECK: bit idx of (m2 m1 m0) is set when constraint idx is nonzero (T <= 78); scalars, since a runtime-indexed array would live in
    // local memory
    unsigned m0 = 0, m1 = 0, m2 = 0;
    // the proof's coefficients are read at each use: pointers to them held across the body would add live registers
    auto fold = [&](int idx, fe v) {
        if constexpr (CHECK) {
            const unsigned bit = fe_is_zero(v) ? 0u : 1u;
            if (idx < 32) m0 |= bit << idx;
            else if (idx < 64) m1 |= bit << (idx - 32);
            else m2 |= bit << (idx - 64);
        } else {
            const unsigned long long at = idx + blockIdx.y * P.coef_stride;
            acc.fold(v, P.coefA[at], P.coefB[at]);
        }
    };
    // closes the run of degree group g: x^inc_g is the host's value at the verifier's point, else a power of the LDE root
    auto close = [&](int g) {
        if constexpr (!CHECK)
            acc.close(P.xpow_override ? P.xpow_override[blockIdx.y * P.override_stride + g] : tw_pow(P.twN, lde_index * P.inc[g]));
    };

    const fe *per = P.per_override ? P.per_override + blockIdx.y * P.override_stride
                                   : P.periodic + (s & 127ULL) * 23;     // [ark_sponge 8][masks 3][ark_hasher 12]

    DG_STEP();
    // ---- decoder: op bits (decoder/op_bits.rs:10-79), constraints 0..13 -------------------------------------------------------
    {
        fe cf_sum = ZERO, ld_prod = ONE, hd_prod = ONE;
#pragma unroll
        for (int i = 0; i < 3; i++) { fold(i, is_bin(cf(i))); cf_sum = fe_add(cf_sum, cf(i)); }
#pragma unroll
        for (int i = 0; i < 5; i++) { fold(3 + i, is_bin(ld(i))); ld_prod = fe_mul(ld_prod, ld(i)); }
#pragma unroll
        for (int i = 0; i < 2; i++) { fold(8 + i, is_bin(hd(i))); hd_prod = fe_mul(hd_prod, hd(i)); }
        close(G2);
        // (op_counter + 1) * hacc + op_counter * (1 - hacc) = op_counter + hacc
        fold(10, fe_sub(fe_add(op_counter, cff[0]), DNXT(0)));
        close(G3);
        fold(11, fe_mul(op_counter, fe_mul(bnot(ld_prod), bnot(hd_prod))));
        fold(12, fe_mul(cf_sum, bnot(fe_mul(ld_prod, hd_prod))));
        close(G8);
    }

    DG_STEP();
    // ---- decoder: sponge / flow ops (decoder/sponge.rs, flow_ops.rs) --------------------------------------------------------------
    fe r_sp1;                                   // sponge 1 is a degree-7 constraint: folded with the stack's run
    {
        fold(13, fe_mul(cff[7], bnot(next_void)));
        // HACC
        {
            fe f = cff[0];
            fe op_value = fe_mul(NW(0), hdf[0]);
            fe os[4], ns[4];
#pragma unroll
            for (int i = 0; i < 4; i++) os[i] = fe_cube(fe_add(sp(i), per[i]));
            DG_STEP();
            matvec<4>(c_sponge_mds, os);
            // op_code = sum ld(i)*2^i + hd(i)*2^(5+i)
            fe opc = ld(0);
            opc = fe_add(opc, fe_mul_small(ld(1), 2)); opc = fe_add(opc, fe_mul_small(ld(2), 4));
            opc = fe_add(opc, fe_mul_small(ld(3), 8)); opc = fe_add(opc, fe_mul_small(ld(4), 16));
            opc = fe_add(opc, fe_mul_small(hd(0), 32)); opc = fe_add(opc, fe_mul_small(hd(1), 64));
            os[0] = fe_add(os[0], opc);
            os[1] = fe_add(os[1], op_value);
#pragma unroll
            for (int i = 0; i < 4; i++) ns[i] = nsp(i);
            matvec<4>(c_sponge_inv_mds, ns);
#pragma unroll
            for (int i = 0; i < 4; i++) ns[i] = fe_sub(fe_cube(ns[i]), per[4 + i]);
            DG_STEP();
            // sponge register i: HACC f * (os[i] - ns[i]); BEGIN, LOOP, WRAP clear the sponge (flag sum * new_sponge[i]); TEND / FEND;
            // BREAK / VOID keep the sponge.  One unreduced sum of four products per register
            const fe fclr = fe_add(fe_add(cff[1], cff[4]), cff[5]);
            const fe ft = cff[2], ff = cff[3], fb = fe_add(ft, ff), fk = fe_add(cff[6], cff[7]);
            auto sponge = [&](const int i) -> fe {
                fe_wide w;
                wide_first(w, f, fe_sub(os[i], ns[i]));
                wide_mac(w, fclr, nsp(i));
                if (i == 0) wide_mac(w, fb, fe_sub(C_CTX(0), nsp(0)));
                if (i == 1) wide_mac(w, ft, fe_sub(sp(0), nsp(1)));
                if (i == 2) wide_mac(w, ff, fe_sub(sp(0), nsp(2)));
                if (i == 3) wide_mac(w, fb, nsp(3));
                wide_mac(w, fk, fe_sub(sp(i), nsp(i)));
                return DG_REDUCE_WIDE(w);
            };
            fold(15, sponge(0));
            fold(17, sponge(2));
            fold(18, sponge(3));
            close(G6);
            r_sp1 = sponge(1);
        }
    }

    DG_STEP();
    // ---- decoder: alignment, loop image, context and loop stacks: the degree-4 run ------------------------------------------------
    {
        {
            fe_wide w;
            wide_first(w, fe_add(fe_add(cff[1], cff[4]), fe_add(cff[5], cff[6])), per[8 + 1]);     // BEGIN, LOOP, WRAP, BREAK
            wide_mac(w, fe_add(cff[2], cff[3]), per[8 + 0]);                                       // TEND, FEND
            wide_mac(w, hdf[0], per[8 + 2]);                                                       // PUSH
            fold(14, DG_REDUCE_WIDE(w));
        }
        // loop image (WRAP, BREAK)
        fold(19, fe_mul(fe_add(cff[5], cff[6]), fe_sub(sp(0), C_LOOP(0))));

        DG_STEP();
        // context stack: BEGIN/LOOP push (right shift 1, slot 0 = parent hash), TEND/FEND pop (left shift 1), WRAP/BREAK/VOID copy
        {
            fe f_push = fe_add(cff[1], cff[4]), f_pop = fe_add(cff[2], cff[3]), f_copy = fe_add(fe_add(cff[5], cff[6]), cff[7]);
            for (int i = 0; i < cl; i++) {
                fe_wide w;
                wide_first(w, f_copy, fe_sub(C_CTX(i), N_CTX(i)));
                wide_mac(w, f_push, fe_sub(i == 0 ? sp(0) : C_CTX(i - 1), N_CTX(i)));
                wide_mac(w, f_pop, i < cl - 1 ? fe_sub(C_CTX(i + 1), N_CTX(i)) : N_CTX(i));
                fold(20 + i, DG_REDUCE_WIDE(w));
            }
        }
        DG_STEP();
        // loop stack: BEGIN/TEND/FEND/WRAP/VOID copy, LOOP right shift 1 (slot 0 unconstrained), BREAK left shift 1
        {
            fe f_copy = fe_add(fe_add(fe_add(cff[1], cff[2]), fe_add(cff[3], cff[5])), cff[7]);
            fe f_rs = cff[4], f_ls = cff[6];
            for (int i = 0; i < ll; i++) {
                fe_wide w;
                wide_first(w, f_copy, fe_sub(C_LOOP(i), N_LOOP(i)));
                if (i >= 1) wide_mac(w, f_rs, fe_sub(C_LOOP(i - 1), N_LOOP(i)));
                wide_mac(w, f_ls, i < ll - 1 ? fe_sub(C_LOOP(i + 1), N_LOOP(i)) : N_LOOP(i));
                fold(20 + cl + i, DG_REDUCE_WIDE(w));
            }
        }
        close(G4);
    }

    {
        fe n0 = bnot(ld(0));
        ldf[3] = fe_mul(ld(0), ld(1));
        ldf[1] = fe_sub(ld(0), ldf[3]);                               // ld0 (1 - ld1)
        ldf[0] = fe_sub(n0, fe_sub(ld(1), ldf[3]));                   // (1 - ld0)(1 - ld1)
        ldf[2] = fe_mul(n0, cf(1));                                   // sic (trace_state.rs:301)
#pragma unroll
        for (int i = 0; i < 4; i++) { ldf[4 + i] = fe_mul(ldf[i], ld(2)); ldf[i] = fe_sub(ldf[i], ldf[4 + i]); }
#pragma unroll
        for (int i = 0; i < 8; i++) { ldf[8 + i] = fe_mul(ldf[i], ld(3)); ldf[i] = fe_sub(ldf[i], ldf[8 + i]); }
        DG_STEP();
#pragma unroll
        for (int i = 0; i < 16; i++) { ldf[16 + i] = fe_mul(ldf[i], ld(4)); ldf[i] = fe_sub(ldf[i], ldf[16 + i]); }
        DG_STEP();
    }
    DG_STEP();
    fe begin_flag, noop_flag;
    {
        begin_flag = fe_mul(ldf[0], hdf_raw0);
        noop_flag = fe_mul(ldf[31], hdf[3]);
        ldf[0] = fe_mul(ldf[0], hd(0));      // ASSERT flag adjustment
    }
    DG_STEP();
    // ---- stack constraints (stack/mod.rs:117-195) -----------------------------------------------------------------------------------
    {
        const int base = 20 + cl + ll;       // aux constraints at base, base+1; stack slots from base+2
        const int L = sl;
        // op flags by name (processor/opcodes.rs:46-92: ld index = opcode & 31)
        const fe f_assert = ldf[0], f_asserteq = ldf[1], f_eq = ldf[2], f_drop = ldf[3], f_drop4 = ldf[4], f_choose = ldf[5],
                 f_choose2 = ldf[6], f_cswap2 = ldf[7], f_add = ldf[8], f_mul = ldf[9], f_and = ldf[10], f_or = ldf[11], f_inv = ldf[12],
                 f_neg = ldf[13], f_not = ldf[14], f_read = ldf[16], f_read2 = ldf[17], f_dup = ldf[18], f_dup2 = ldf[19],
                 f_dup4 = ldf[20], f_pad2 = ldf[21], f_swap = ldf[24], f_swap2 = ldf[25], f_swap4 = ldf[26], f_roll4 = ldf[27],
                 f_roll8 = ldf[28], f_binacc = ldf[29];
        const fe f_push = hdf[0], f_cmp = hdf[1], f_rescr = hdf[2];

        DG_STEP();
        // the degree-7 run: sponge 1, the auxiliary constraints, every stack slot
        fold(16, r_sp1);
        // --- auxiliary constraints
        {
            const fe f_ao = fe_add(f_and, f_or);
            fe_wide w;
            wide_first(w, f_assert, fe_sub(ONE, O(0)));
            wide_mac(w, f_asserteq, fe_sub(O(0), O(1)));
            wide_mac(w, fe_add(f_not, f_ao), is_bin(O(0)));
            wide_mac(w, f_eq, fe_mul(NW(0), fe_sub(O(1), O(2))));
            wide_mac(w, f_choose, is_bin(O(2)));
            wide_mac(w, fe_add(f_choose2, f_cswap2), is_bin(O(4)));
            fold(base, DG_REDUCE_WIDE(w));
            fold(base + 1, fe_mul(f_ao, is_bin(O(1))));
        }

        DG_STEP();
        // --- per-slot shift structure.  For slot i the generic contribution of an operation is
        //        copy:         f * (O(i)   - n[i])                    when i >= from
        //        right shift s: f * (O(i-s) - n[i])                   when i >= s
        //        left shift s from slot `from`: f * (O(i+s) - n[i])   when from-s <= i < L-s, and f * n[i] when i >= L-s
        //     flags with the same shape are summed first.
        const fe f_copy0 = fe_add(begin_flag, noop_flag);                                   // from 0
        const fe f_copy1 = fe_add(fe_add(f_inv, f_neg), f_not);                              // from 1
        const fe f_copy2 = f_swap;                                                           // from 2
        const fe f_copy4 = fe_add(fe_add(f_swap2, f_roll4), f_binacc);                       // from 4
        const fe f_copy6 = f_rescr;                                                          // from 6
        const fe f_copy8 = fe_add(fe_add(f_swap4, f_roll8), f_cmp);                          // from 8
        const fe f_rs1 = fe_add(fe_add(f_read, f_dup), f_push);
        const fe f_rs2 = fe_add(fe_add(f_read2, f_dup2), f_pad2);
        const fe f_rs4 = f_dup4;
        const fe f_ls1_0 = fe_add(f_assert, f_drop);                                         // left 1, start slot 0
        const fe f_ls1_1 = fe_add(fe_add(f_add, f_mul), fe_add(f_and, f_or));                // left 1, start slot 1
        const fe f_ls2_0 = f_asserteq;                                                       // left 2, start slot 0
        const fe f_ls2_1 = fe_add(f_eq, f_choose);                                           // left 2, start slot 1
        const fe f_ls2_4 = f_cswap2;                                                         // left 2, start slot 4
        const fe f_ls4_0 = f_drop4;                                                          // left 4, start slot 0
        const fe f_ls4_2 = f_choose2;                                                        // left 4, start slot 2
        // slot i's seven shift products open its unreduced sum; fc / fl1 / fl2 / fl4 are the copy and left-shift flag sums that apply
        // to this slot
        auto slot_shifts = [&](fe_wide &w, const int i, const fe fc, const fe fl1, const fe fl2, const fe fl4) {
            const fe nwi = NW(i);
            wide_first(w, fc, fe_sub(O(i), nwi));
            if (i >= 1) wide_mac(w, f_rs1, fe_sub(O(i - 1), nwi));
            if (i >= 2) wide_mac(w, f_rs2, fe_sub(O(i - 2), nwi));
            if (i >= 4) wide_mac(w, f_rs4, fe_sub(O(i - 4), nwi));
            wide_mac(w, fl1, (i < L - 1) ? fe_sub(O(i + 1), nwi) : nwi);
            wide_mac(w, fl2, (i < L - 2) ? fe_sub(O(i + 2), nwi) : nwi);
            wide_mac(w, fl4, (i < L - 4) ? fe_sub(O(i + 4), nwi) : nwi);
        };
        auto slot_fold = [&](const int i, const fe_wide &w) {
            if (i < P.stack_depth) fold(base + 2 + i, DG_REDUCE_WIDE(w));
        };

        // slots >= 8 carry no operation-specific terms (every shape applies)
        {
            const fe fc_hi = fe_add(fe_add(fe_add(f_copy0, f_copy1), fe_add(f_copy2, f_copy4)), fe_add(f_copy6, f_copy8));
            const fe fl1_hi = fe_add(f_ls1_0, f_ls1_1), fl2_hi = fe_add(fe_add(f_ls2_0, f_ls2_1), f_ls2_4), fl4_hi = fe_add(f_ls4_0, f_ls4_2);
            for (int i = 8; i < L; i++) {
                fe_wide w;
                slot_shifts(w, i, fc_hi, fl1_hi, fl2_hi, fl4_hi);
                slot_fold(i, w);
                DG_STEP();
            }
        }
        // --- low slots 0..7, slot by slot: the shift products, then every operation-specific product of the slot, in one unreduced sum
        //     (slot 0: 7 + 20 products).  Terms shared between slots are computed once, in reduced form.
        // rescr (stack/hash.rs:9-35): slot q gets f_rescr * (ns[q] - os[q])
        fe rs[6];
        {
            fe os[6], ns[6];
#pragma unroll
            for (int q = 0; q < 6; q++) os[q] = fe_cube(fe_add(O(q), per[11 + q]));
            matvec<6>(c_hasher_mds, os);
#pragma unroll
            for (int q = 0; q < 6; q++) ns[q] = NW(q);
            matvec<6>(c_hasher_inv_mds, ns);
#pragma unroll
            for (int q = 0; q < 6; q++) rs[q] = fe_sub(fe_sub(fe_cube(ns[q]), per[11 + 6 + q]), os[q]);
        }
        DG_STEP();
        // choose2 / cswap2 with c = O(4): c O(j) + (1 - c) O(j+2) = O(j+2) + c (O(j) - O(j+2)); the swapped selection
        // c O(j+2) + (1 - c) O(j) is O(j) + O(j+2) minus it
        auto sel = [&](const int j) { return fe_add(O(j + 2), fe_mul(O(4), fe_sub(O(j), O(j + 2)))); };
        // roll4 and roll8 shift slots 1..3 alike
        const fe f_roll48 = fe_add(f_roll4, f_roll8);
        fe fc = f_copy0, fl1 = f_ls1_0, fl2 = f_ls2_0, fl4 = f_ls4_0;
        {
            fe_wide w;
            slot_shifts(w, 0, fc, fl1, fl2, fl4);
            wide_mac(w, fe_add(fe_add(f_dup, f_dup2), f_dup4), fe_sub(NW(0), O(0)));        // dup / dup2 / dup4: new[k] == old[k]
            wide_mac(w, f_pad2, NW(0));
            wide_mac(w, f_swap, fe_add(fe_sub(NW(0), O(1)), fe_sub(NW(1), O(0))));          // swap: both constraints in slot 0
                                                                                            // (stack/manipulation.rs:63-64)
            wide_mac(w, f_swap2, fe_sub(NW(0), O(2)));
            wide_mac(w, f_swap4, fe_sub(NW(0), O(4)));
            wide_mac(w, f_roll4, fe_sub(NW(0), O(3)));
            wide_mac(w, f_roll8, fe_sub(NW(0), O(7)));
            // arithmetic / boolean
            const fe prod = fe_mul(O(0), O(1));
            wide_mac(w, f_add, fe_sub(NW(0), fe_add(O(0), O(1))));
            wide_mac(w, fe_add(f_mul, f_and), fe_sub(NW(0), prod));
            wide_mac(w, f_inv, fe_sub(ONE, fe_mul(NW(0), O(0))));
            wide_mac(w, f_neg, fe_add(NW(0), O(0)));
            wide_mac(w, f_not, fe_sub(NW(0), bnot(O(0))));
            wide_mac(w, f_or, fe_sub(NW(0), fe_sub(fe_add(O(0), O(1)), prod)));             // 1 - (1 - O(0)) (1 - O(1))
            wide_mac(w, f_eq, fe_sub(NW(0), bnot(fe_mul(fe_sub(O(1), O(2)), O(0)))));       // eq: new[0] == 1 - (O(1)-O(2)) * O(0)
            wide_mac(w, f_choose, fe_sub(NW(0), fe_add(O(1), fe_mul(O(2), fe_sub(O(0), O(1))))));   // c O(0) + (1 - c) O(1), c = O(2)
            {
                const fe s0 = sel(0);
                wide_mac(w, f_choose2, fe_sub(NW(0), s0));
                wide_mac(w, f_cswap2, fe_sub(NW(0), fe_sub(fe_add(O(0), O(2)), s0)));
            }
            wide_mac(w, f_binacc, is_bin(NW(0)));                                            // binacc (comparison.rs:111-133)
            wide_mac(w, f_cmp, is_bin(NW(1)));      // cmp (comparison.rs:71-108): [pow, bit_a, bit_b, not_set, gt, lt, acc_b, acc_a]
            wide_mac(w, f_rescr, rs[0]);
            slot_fold(0, w);
        }
        DG_STEP();
        fc = fe_add(fc, f_copy1); fl1 = fe_add(fl1, f_ls1_1); fl2 = fe_add(fl2, f_ls2_1);
        {
            fe_wide w;
            slot_shifts(w, 1, fc, fl1, fl2, fl4);
            wide_mac(w, fe_add(f_dup2, f_dup4), fe_sub(NW(1), O(1)));
            wide_mac(w, f_pad2, NW(1));
            wide_mac(w, f_swap2, fe_sub(NW(1), O(3)));
            wide_mac(w, f_swap4, fe_sub(NW(1), O(5)));
            wide_mac(w, f_roll48, fe_sub(NW(1), O(0)));
            {
                const fe s1 = sel(1);
                wide_mac(w, f_choose2, fe_sub(NW(1), s1));
                wide_mac(w, f_cswap2, fe_sub(NW(1), fe_sub(fe_add(O(1), O(3)), s1)));
            }
            wide_mac(w, f_binacc, NW(1));
            wide_mac(w, f_cmp, is_bin(NW(2)));
            wide_mac(w, f_rescr, rs[1]);
            slot_fold(1, w);
        }
        DG_STEP();
        fc = fe_add(fc, f_copy2); fl4 = fe_add(fl4, f_ls4_2);
        // cmp: gt = O(4) + bit_a (1 - bit_b) not_set, lt = O(5) + bit_b (1 - bit_a) not_set
        const fe xy = fe_mul(NW(1), NW(2));
        {
            fe_wide w;
            slot_shifts(w, 2, fc, fl1, fl2, fl4);
            wide_mac(w, f_dup4, fe_sub(NW(2), O(2)));
            wide_mac(w, f_swap2, fe_sub(NW(2), O(0)));
            wide_mac(w, f_swap4, fe_sub(NW(2), O(6)));
            wide_mac(w, f_roll48, fe_sub(NW(2), O(1)));
            wide_mac(w, f_cswap2, fe_sub(NW(2), sel(0)));
            wide_mac(w, f_binacc, fe_sub(NW(2), fe_mul_small(O(2), 2)));
            wide_mac(w, f_cmp, fe_sub(NW(4), fe_add(O(4), fe_mul(fe_sub(NW(1), xy), NW(3)))));
            wide_mac(w, f_rescr, rs[2]);
            slot_fold(2, w);
        }
        DG_STEP();
        {
            fe_wide w;
            slot_shifts(w, 3, fc, fl1, fl2, fl4);
            wide_mac(w, f_dup4, fe_sub(NW(3), O(3)));
            wide_mac(w, f_swap2, fe_sub(NW(3), O(1)));
            wide_mac(w, f_swap4, fe_sub(NW(3), O(7)));
            wide_mac(w, f_roll48, fe_sub(NW(3), O(2)));
            wide_mac(w, f_cswap2, fe_sub(NW(3), sel(1)));
            wide_mac(w, f_binacc, fe_sub(NW(3), fe_add(O(3), fe_mul(NW(0), O(2)))));
            wide_mac(w, f_cmp, fe_sub(NW(5), fe_add(O(5), fe_mul(fe_sub(NW(2), xy), NW(3)))));
            wide_mac(w, f_rescr, rs[3]);
            slot_fold(3, w);
        }
        DG_STEP();
        fc = fe_add(fc, f_copy4); fl2 = fe_add(fl2, f_ls2_4);
#pragma unroll
        for (int q = 4; q < 8; q++) {
            if (q == 6) fc = fe_add(fc, f_copy6);
            fe_wide w;
            slot_shifts(w, q, fc, fl1, fl2, fl4);
            wide_mac(w, f_swap4, fe_sub(NW(q), O(q - 4)));
            wide_mac(w, f_roll8, fe_sub(NW(q), O(q - 1)));
            if (q == 4) wide_mac(w, f_cmp, fe_sub(NW(6), fe_add(O(6), fe_mul(NW(2), O(0)))));     // acc_b
            if (q == 5) wide_mac(w, f_cmp, fe_sub(NW(7), fe_add(O(7), fe_mul(NW(1), O(0)))));     // acc_a
            if (q == 6) wide_mac(w, f_cmp, fe_sub(NW(3), fe_mul(bnot(O(5)), bnot(O(4)))));        // not_set
            if (q == 7) wide_mac(w, f_cmp, fe_sub(fe_mul_small(NW(0), 2), O(0)));                 // pow
            if (q < 6) wide_mac(w, f_rescr, rs[q]);
            slot_fold(q, w);
            if (q & 1) DG_STEP();
        }
        close(G7);
    }

    DG_STEP();
    if constexpr (CHECK) {
        // the wrap-around transition n - 1 -> 0 is exempt (evaluator.rs:330-333: should_evaluate_to_zero_at)
        if (live) {
            unsigned *m = P.masks + (blockIdx.y * n + k) * 3;
            const bool exempt = k == n - 1;
            m[0] = exempt ? 0u : m0;
            m[1] = exempt ? 0u : m1;
            m[2] = exempt ? 0u : m2;
        }
        return;
    }
    // ---- combine (evaluator.rs:335-358): result + sum_g adj_g * x^inc_g, every group already closed into acc.res ---------------------------
    fe t_res = DG_REDUCE_WIDE(acc.res);
    // on the trace domain (except its last step) every constraint must vanish (evaluator.rs:149-158)
    if (!P.verify_mode && c8 == 0 && k != n - 1) {
        if (acc.nonzero && live) atomicMax(P.violation + blockIdx.y, violation_word(k));
        t_res = ZERO;
    }
    if (live) P.t_ev[blockIdx.y * P.t_ev_stride + out_idx] = t_res;
}

#undef DCUR
#undef DNXT
#undef SCOL
#undef C_CTX
#undef N_CTX
#undef C_LOOP
#undef N_LOOP
#undef O
#undef NW
#undef sp
#undef cf
#undef ld
#undef hd
#undef nsp
#undef ncf

void launch_constraint_eval(Context &c, const AirParams &P, int batch) {
    air_upload_constants(c);
    DG_REQUIRE(batch >= 1 && batch <= 65535, "constraint evaluation batch out of range");
    // the kernel's unreduced sums are bounded for at most 16 context, 8 loop and 32 stack registers (Acc)
    DG_REQUIRE(P.cl >= 1 && P.cl <= 16 && P.ll >= 1 && P.ll <= 8 && P.sl >= 8 && P.sl <= 32, "constraint evaluation register shape out of range");
    const unsigned long long E = (unsigned long long)P.num_c8 << P.log_n;
    // H100 SXM (700 W), stage 3 of the 2^20-step proof x 26 registers: per-thread arrays 24.8 ms; shared-memory rows, stack-like columns
    // only 23.7; all columns 23.2; all columns + unreduced per-slot sums (constraint_eval_smem_kernel) 22.2.  The other forms were removed
    // after this measurement.
    // H100 80GB HBM3 (700 W), same proof: constraint_eval_smem_kernel with one unreduced sum per constraint and per degree group 18.27 ms,
    // 21.08 ms with one reduction per product outside the per-slot shift sums (mean of 4 alternating runs each).
    // All proofs of a batch run in one launch.  Traces shorter than a block take the SHORT layout; with several ranks their domain slice
    // can be shorter than one block, and the clamped threads of the partial block write nothing.
    const bool short_n = P.log_n < 7;
    const size_t smem = (size_t)P.w * (short_n ? 128 + 128 / 16 : 128 + 1) * sizeof(fe);
    // widths are bounded by the prover's and verifier's argument checks (w <= 15 + 16 + 8 + 32 = 71, 154,496 B in the SHORT layout)
    DG_REQUIRE(P.log_n >= 4 && smem <= 200 * 1024, "constraint evaluation needs at least 16 steps and at most 200 KB of rows per block");
    auto k = short_n ? constraint_eval_smem_kernel<128, 4, true> : constraint_eval_smem_kernel<128, 4>;
    set_func_smem(c, (const void *)k, smem);
    k<<<dim3((unsigned)((E + 127) / 128), (unsigned)batch), 128, smem, c.stream>>>(P);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

void launch_constraint_check(Context &c, const AirParams &P, int batch) {
    air_upload_constants(c);
    DG_REQUIRE(batch >= 1 && batch <= 65535, "trace check batch out of range");
    DG_REQUIRE(P.cl >= 1 && P.cl <= 16 && P.ll >= 1 && P.ll <= 8 && P.sl >= 8 && P.sl <= 32, "trace check register shape out of range");
    DG_REQUIRE(P.num_c8 == 1 && P.c8_base == 0 && P.log_blowup == 3 && P.masks, "the trace check runs on the trace domain");
    const bool short_n = P.log_n < 7;
    const size_t smem = (size_t)P.w * (short_n ? 128 + 128 / 16 : 128 + 1) * sizeof(fe);
    DG_REQUIRE(P.log_n >= 4 && smem <= 200 * 1024, "the trace check needs at least 16 steps and at most 200 KB of rows per block");
    auto k = short_n ? constraint_eval_smem_kernel<128, 4, true, true> : constraint_eval_smem_kernel<128, 4, false, true>;
    set_func_smem(c, (const void *)k, smem);
    k<<<dim3((unsigned)(((1ULL << P.log_n) + 127) / 128), (unsigned)batch), 128, smem, c.stream>>>(P);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

// One atomic per block and constraint: each warp turns a constraint's bits into a ballot (popc = violating steps, ffs = the lowest), the
// warps of a block combine in shared memory, and the block adds its counts to the trace's totals.  Random rows violate every constraint at
// every step, where one atomic per step and constraint would serialise.
__global__ void check_reduce_kernel(const unsigned *__restrict__ masks, unsigned long long n, int T, unsigned long long *stats) {
    __shared__ unsigned s_cnt[CHECK_SLOTS];
    __shared__ unsigned long long s_first[CHECK_SLOTS];
    for (int i = threadIdx.x; i < CHECK_SLOTS; i += blockDim.x) { s_cnt[i] = 0; s_first[i] = ~0ULL; }
    __syncthreads();
    const unsigned *m = masks + (unsigned long long)blockIdx.y * n * 3;
    const int lane = threadIdx.x & 31;
    for (unsigned long long base = (unsigned long long)blockIdx.x * blockDim.x; base < n; base += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long k = base + threadIdx.x;
        const unsigned long long warp0 = k - lane;
        unsigned w[3] = {0, 0, 0};
        if (k < n) { w[0] = m[k * 3]; w[1] = m[k * 3 + 1]; w[2] = m[k * 3 + 2]; }
        const unsigned any = __ballot_sync(0xFFFFFFFFu, (w[0] | w[1] | w[2]) != 0);
        if (!any) continue;                                                     // warp-uniform
        if (lane == 0) {
            atomicAdd(&s_cnt[CHECK_SLOTS - 1], __popc(any));
            atomicMin(&s_first[CHECK_SLOTS - 1], warp0 + __ffs(any) - 1);
        }
#pragma unroll
        for (int j = 0; j < 3; j++) {
            if (!__any_sync(0xFFFFFFFFu, w[j] != 0)) continue;
            for (int b = 0; b < 32 && 32 * j + b < T; b++) {
                const unsigned ballot = __ballot_sync(0xFFFFFFFFu, (w[j] >> b) & 1u);
                if (lane == 0 && ballot) {
                    atomicAdd(&s_cnt[32 * j + b], __popc(ballot));
                    atomicMin(&s_first[32 * j + b], warp0 + __ffs(ballot) - 1);
                }
            }
        }
    }
    __syncthreads();
    unsigned long long *st = stats + (unsigned long long)blockIdx.y * CHECK_STATS;
    for (int i = threadIdx.x; i < CHECK_SLOTS; i += blockDim.x)
        if (s_cnt[i]) {
            atomicAdd(&st[i], (unsigned long long)s_cnt[i]);
            atomicMin(&st[CHECK_SLOTS + i], s_first[i]);
        }
}

void launch_check_reduce(Context &c, const unsigned *masks, unsigned long long n, int T, int batch, unsigned long long *stats) {
    DG_REQUIRE(batch >= 1 && batch <= 65535 && T >= 1 && T < CHECK_SLOTS, "trace check reduction out of range");
    // counts 0, lowest steps UINT64_MAX
    DG_CUDA(cudaMemsetAsync(stats, 0, (size_t)batch * CHECK_STATS * 8, c.stream));
    DG_CUDA(cudaMemset2DAsync(stats + CHECK_SLOTS, CHECK_STATS * 8, 0xFF, CHECK_SLOTS * 8, batch, c.stream));
    // enough blocks to fill the GPU, each walking several 256-step tiles: fewer blocks, fewer global atomics
    const unsigned long long tiles = (n + 255) / 256;
    const unsigned gx = (unsigned)std::max<unsigned long long>(1, std::min<unsigned long long>(tiles, (unsigned long long)(4 * c.num_sms + batch - 1) / batch));
    check_reduce_kernel<<<dim3(gx, (unsigned)batch), 256, 0, c.stream>>>(masks, n, T, stats);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

// ---- host side: the register shape ---------------------------------------------------------------------------------------------

static int first_stack_register(uint32_t ctx_depth, uint32_t loop_depth) { return 15 + (int)ctx_depth + (int)loop_depth; }

TraceShape::TraceShape(int ctx, int loop, int stack)
    : w(first_stack_register(ctx, loop) + stack), ctx_depth(ctx), loop_depth(loop), stack_depth(stack), cl(std::max(ctx, 1)),
      ll(std::max(loop, 1)), sl(std::max(stack, 8)), T(20 + cl + ll + 2 + stack), stack_reg(first_stack_register(ctx, loop)) {}

bool TraceShape::in_range(uint32_t ctx_depth, uint32_t loop_depth, uint32_t stack_depth) {
    return ctx_depth <= 16 && loop_depth <= 8 && stack_depth >= 1 && stack_depth <= 32;
}

TraceShape TraceShape::of_trace(uint32_t width, uint32_t ctx_depth, uint32_t loop_depth) {
    DG_REQUIRE(ctx_depth <= 16, "context depth cannot be greater than 16");
    DG_REQUIRE(loop_depth <= 8, "loop depth cannot be greater than 8");
    DG_REQUIRE(width < 128, "execution trace cannot have more than 128 registers");
    const int stack_depth = (int)width - first_stack_register(ctx_depth, loop_depth);
    DG_REQUIRE(stack_depth >= 1, "user stack must consist of at least one register");
    DG_REQUIRE(stack_depth <= 32, "stack depth cannot be greater than 32");
    return TraceShape((int)ctx_depth, (int)loop_depth, stack_depth);
}

AirParams TraceShape::air_params(uint64_t n) const {
    AirParams P;
    memset(&P, 0, sizeof P);
    P.w = w; P.ctx_depth = ctx_depth; P.loop_depth = loop_depth; P.stack_depth = stack_depth;
    P.cl = cl; P.ll = ll; P.sl = sl;
    P.log_n = ceil_log2(n);
    for (int g = 0; g < 6; g++) P.inc[g] = group_increment(g, n);
    return P;
}

unsigned long long group_increment(int g, uint64_t n) {
    static const int GROUP_DEG[6] = {2, 3, 4, 6, 7, 8};
    return (8 * n - 1) - (n - 1) * GROUP_DEG[g];
}

const fe *periodic_table(Context &c) {
    if (!c.d_periodic.p) {
        const std::vector<fe> per = fs::periodic_tables();
        c.d_periodic.alloc(per.size() * 16, true);
        DG_CUDA(cudaMemcpyAsync(c.d_periodic.p, per.data(), per.size() * 16, cudaMemcpyHostToDevice, c.stream));
        DG_CUDA(cudaStreamSynchronize(c.stream));
    }
    return c.d_periodic.as<fe>();
}

}  // namespace dg
