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

struct Acc {
    fe_wide res;                        // sum_i v_i * cA_i, unreduced (at most 78 constraints < 128 products)
    fe adj[6];
    bool nonzero, first;
    __device__ __forceinline__ void fold(int group, fe v, fe a, fe b) {
        if (first) { wide_set(res, DG_MUL_WIDE(v, a)); first = false; }
        else wide_add(res, DG_MUL_WIDE(v, a));
        adj[group] = fe_add(adj[group], fe_mul(v, b));
        nonzero = nonzero || !fe_is_zero(v);
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
template <int BLOCK, int MIN_BLOCKS, bool SHORT = false>
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
#pragma unroll
    for (int g = 0; g < 6; g++) acc.adj[g] = ZERO;
    acc.nonzero = false;
    // the proof's coefficients are read at each use: pointers to them held across the body would add live registers
    auto fold = [&](int idx, int group, fe v) {
        const unsigned long long at = idx + blockIdx.y * P.coef_stride;
        acc.fold(group, v, P.coefA[at], P.coefB[at]);
    };

    const fe *per = P.per_override ? P.per_override + blockIdx.y * P.override_stride
                                   : P.periodic + (s & 127ULL) * 23;     // [ark_sponge 8][masks 3][ark_hasher 12]

    DG_STEP();
    // ---- decoder: op bits (decoder/op_bits.rs:10-79), constraints 0..14 -------------------------------------------------------
    {
        fe cf_sum = ZERO, ld_prod = ONE, hd_prod = ONE;
#pragma unroll
        for (int i = 0; i < 3; i++) { fold(i, G2, is_bin(cf(i))); cf_sum = fe_add(cf_sum, cf(i)); }
#pragma unroll
        for (int i = 0; i < 5; i++) { fold(3 + i, G2, is_bin(ld(i))); ld_prod = fe_mul(ld_prod, ld(i)); }
#pragma unroll
        for (int i = 0; i < 2; i++) { fold(8 + i, G2, is_bin(hd(i))); hd_prod = fe_mul(hd_prod, hd(i)); }
        fe is_hacc = cff[0];
        fe hacc_t = fe_mul(fe_add(op_counter, ONE), is_hacc);
        fe rest_t = fe_mul(op_counter, bnot(is_hacc));
        fold(10, G3, fe_sub(fe_add(hacc_t, rest_t), DNXT(0)));
        fold(11, G8, fe_mul(op_counter, fe_mul(bnot(ld_prod), bnot(hd_prod))));
        fold(12, G8, fe_mul(cf_sum, bnot(fe_mul(ld_prod, hd_prod))));
        fold(13, G6, fe_mul(cff[7], bnot(next_void)));
        fe prefix = fe_add(fe_add(cff[1], cff[4]), fe_add(cff[5], cff[6]));      // BEGIN, LOOP, WRAP, BREAK
        fe align = fe_mul(prefix, per[8 + 1]);
        align = fe_add(align, fe_mul(fe_add(cff[2], cff[3]), per[8 + 0]));       // TEND, FEND
        align = fe_add(align, fe_mul(hdf[0], per[8 + 2]));                        // PUSH
        fold(14, G4, align);
    }

    DG_STEP();
    // ---- decoder: sponge / flow ops (decoder/sponge.rs, flow_ops.rs) --------------------------------------------------------------
    {
        fe r_sp[4], r_img;
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
#pragma unroll
            for (int i = 0; i < 4; i++) r_sp[i] = fe_mul(f, fe_sub(os[i], ns[i]));
        }
        DG_STEP();
        // BEGIN, LOOP, WRAP clear the sponge: flag sum * new_sponge[i]
        {
            fe fclr = fe_add(fe_add(cff[1], cff[4]), cff[5]);
#pragma unroll
            for (int i = 0; i < 4; i++) r_sp[i] = fe_add(r_sp[i], fe_mul(fclr, nsp(i)));
        }
        DG_STEP();
        // TEND / FEND
        {
            fe ft = cff[2], ff = cff[3], fb = fe_add(ft, ff);
            r_sp[0] = fe_add(r_sp[0], fe_mul(fb, fe_sub(C_CTX(0), nsp(0))));
            r_sp[1] = fe_add(r_sp[1], fe_mul(ft, fe_sub(sp(0), nsp(1))));
            r_sp[2] = fe_add(r_sp[2], fe_mul(ff, fe_sub(sp(0), nsp(2))));
            r_sp[3] = fe_add(r_sp[3], fe_mul(fb, nsp(3)));
        }
        // BREAK / VOID keep the sponge
        {
            fe fk = fe_add(cff[6], cff[7]);
#pragma unroll
            for (int i = 0; i < 4; i++) r_sp[i] = fe_add(r_sp[i], fe_mul(fk, fe_sub(sp(i), nsp(i))));
        }
        fold(15, G6, r_sp[0]); fold(16, G7, r_sp[1]); fold(17, G6, r_sp[2]); fold(18, G6, r_sp[3]);
        // loop image (WRAP, BREAK)
        r_img = fe_mul(fe_add(cff[5], cff[6]), fe_sub(sp(0), C_LOOP(0)));
        fold(19, G4, r_img);

        DG_STEP();
        // context stack: BEGIN/LOOP push (right shift 1, slot 0 = parent hash), TEND/FEND pop (left shift 1), WRAP/BREAK/VOID copy
        {
            fe f_push = fe_add(cff[1], cff[4]), f_pop = fe_add(cff[2], cff[3]), f_copy = fe_add(fe_add(cff[5], cff[6]), cff[7]);
            for (int i = 0; i < cl; i++) {
                fe v = fe_mul(f_copy, fe_sub(C_CTX(i), N_CTX(i)));
                if (i == 0) v = fe_add(v, fe_mul(f_push, fe_sub(sp(0), N_CTX(0))));
                else v = fe_add(v, fe_mul(f_push, fe_sub(C_CTX(i - 1), N_CTX(i))));
                if (i < cl - 1) v = fe_add(v, fe_mul(f_pop, fe_sub(C_CTX(i + 1), N_CTX(i))));
                else v = fe_add(v, fe_mul(f_pop, N_CTX(i)));
                fold(20 + i, G4, v);
            }
        }
        DG_STEP();
        // loop stack: BEGIN/TEND/FEND/WRAP/VOID copy, LOOP right shift 1 (slot 0 unconstrained), BREAK left shift 1
        {
            fe f_copy = fe_add(fe_add(fe_add(cff[1], cff[2]), fe_add(cff[3], cff[5])), cff[7]);
            fe f_rs = cff[4], f_ls = cff[6];
            for (int i = 0; i < ll; i++) {
                fe v = fe_mul(f_copy, fe_sub(C_LOOP(i), N_LOOP(i)));
                if (i >= 1) v = fe_add(v, fe_mul(f_rs, fe_sub(C_LOOP(i - 1), N_LOOP(i))));
                if (i < ll - 1) v = fe_add(v, fe_mul(f_ls, fe_sub(C_LOOP(i + 1), N_LOOP(i))));
                else v = fe_add(v, fe_mul(f_ls, N_LOOP(i)));
                fold(20 + cl + i, G4, v);
            }
        }
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
        // --- auxiliary constraints
        fe aux0, aux1;
        {
            aux0 = fe_mul(f_assert, fe_sub(ONE, O(0)));
            aux0 = fe_add(aux0, fe_mul(f_asserteq, fe_sub(O(0), O(1))));
            fe b0 = is_bin(O(0)), b1 = is_bin(O(1));
            fe f_ao = fe_add(f_and, f_or);
            aux0 = fe_add(aux0, fe_mul(fe_add(f_not, f_ao), b0));
            aux1 = fe_mul(f_ao, b1);
            fe diff = fe_sub(O(1), O(2));
            aux0 = fe_add(aux0, fe_mul(f_eq, fe_mul(NW(0), diff)));
            aux0 = fe_add(aux0, fe_mul(f_choose, is_bin(O(2))));
            aux0 = fe_add(aux0, fe_mul(fe_add(f_choose2, f_cswap2), is_bin(O(4))));
        }
        fold(base, G7, aux0);
        fold(base + 1, G7, aux1);

        DG_STEP();
        // --- per-slot shift structure.  For slot i the generic contribution of an operation is
        //        copy:         f * (O(i)   - n[i])                    when i >= from
        //        right shift s: f * (O(i-s) - n[i])                   when i >= s
        //        left shift s from slot `from`: f * (O(i+s) - n[i])   when from-s <= i < L-s, and f * n[i] when i >= L-s
        //     flags with the same shape are summed first.
        fe ev[8];
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
        // generic part of slot i; fc / fl1 / fl2 / fl4 are the copy and left-shift flag sums that apply to this slot
        auto slot_value = [&](const int i, const fe fc, const fe fl1, const fe fl2, const fe fl4) -> fe {
            const fe nwi = NW(i);
            // the seven products of a slot are accumulated unreduced (288 bits) and reduced once: 7 x (product + 9-limb add) + 1 reduction
            // instead of 7 x (modular product + modular add)
            fe_wide acc7;
            wide_set(acc7, DG_MUL_WIDE(fc, fe_sub(O(i), nwi)));
            if (i >= 1) wide_add(acc7, DG_MUL_WIDE(f_rs1, fe_sub(O(i - 1), nwi)));
            if (i >= 2) wide_add(acc7, DG_MUL_WIDE(f_rs2, fe_sub(O(i - 2), nwi)));
            if (i >= 4) wide_add(acc7, DG_MUL_WIDE(f_rs4, fe_sub(O(i - 4), nwi)));
            wide_add(acc7, DG_MUL_WIDE(fl1, (i < L - 1) ? fe_sub(O(i + 1), nwi) : nwi));
            wide_add(acc7, DG_MUL_WIDE(fl2, (i < L - 2) ? fe_sub(O(i + 2), nwi) : nwi));
            wide_add(acc7, DG_MUL_WIDE(fl4, (i < L - 4) ? fe_sub(O(i + 4), nwi) : nwi));
            return DG_REDUCE_WIDE(acc7);
        };
        fe fc_hi, fl1_hi, fl2_hi, fl4_hi;                  // the sums for slots >= 8 (every shape applies)
        {
            fe fc = f_copy0, fl1 = f_ls1_0, fl2 = f_ls2_0, fl4 = f_ls4_0;
#pragma unroll
            for (int i = 0; i < 8; i++) {
                if (i == 1) { fc = fe_add(fc, f_copy1); fl1 = fe_add(fl1, f_ls1_1); fl2 = fe_add(fl2, f_ls2_1); }
                if (i == 2) { fc = fe_add(fc, f_copy2); fl4 = fe_add(fl4, f_ls4_2); }
                if (i == 4) { fc = fe_add(fc, f_copy4); fl2 = fe_add(fl2, f_ls2_4); }
                if (i == 6) fc = fe_add(fc, f_copy6);
                ev[i] = slot_value(i, fc, fl1, fl2, fl4);
                if (i & 1) DG_STEP();
            }
            fc_hi = fe_add(fc, f_copy8); fl1_hi = fl1; fl2_hi = fl2; fl4_hi = fl4;
        }
        // slots >= 8 carry no operation-specific terms: evaluate and fold them straight away (no per-thread array)
        for (int i = 8; i < L; i++) {
            fold(base + 2 + i, G7, slot_value(i, fc_hi, fl1_hi, fl2_hi, fl4_hi));
            DG_STEP();
        }
        DG_STEP();
        // --- operation-specific constraints on the low slots
        // dup / dup2 / dup4: new[k] == old[k]
        ev[0] = fe_add(ev[0], fe_mul(fe_add(fe_add(f_dup, f_dup2), f_dup4), fe_sub(NW(0), O(0))));
        ev[1] = fe_add(ev[1], fe_mul(fe_add(f_dup2, f_dup4), fe_sub(NW(1), O(1))));
        ev[2] = fe_add(ev[2], fe_mul(f_dup4, fe_sub(NW(2), O(2))));
        ev[3] = fe_add(ev[3], fe_mul(f_dup4, fe_sub(NW(3), O(3))));
        // pad2
        ev[0] = fe_add(ev[0], fe_mul(f_pad2, NW(0)));
        ev[1] = fe_add(ev[1], fe_mul(f_pad2, NW(1)));
        // swap: both constraints accumulate into slot 0 (stack/manipulation.rs:63-64)
        ev[0] = fe_add(ev[0], fe_mul(f_swap, fe_add(fe_sub(NW(0), O(1)), fe_sub(NW(1), O(0)))));
        DG_STEP();
        // swap2
        ev[0] = fe_add(ev[0], fe_mul(f_swap2, fe_sub(NW(0), O(2)))); ev[1] = fe_add(ev[1], fe_mul(f_swap2, fe_sub(NW(1), O(3))));
        ev[2] = fe_add(ev[2], fe_mul(f_swap2, fe_sub(NW(2), O(0)))); ev[3] = fe_add(ev[3], fe_mul(f_swap2, fe_sub(NW(3), O(1))));
        // swap4
#pragma unroll
        for (int q = 0; q < 4; q++) {
            ev[q] = fe_add(ev[q], fe_mul(f_swap4, fe_sub(NW(q), O(4 + q))));
            ev[4 + q] = fe_add(ev[4 + q], fe_mul(f_swap4, fe_sub(NW(4 + q), O(q))));
        }
        DG_STEP();
        // roll4 / roll8
        ev[0] = fe_add(ev[0], fe_mul(f_roll4, fe_sub(NW(0), O(3))));
#pragma unroll
        for (int q = 1; q < 4; q++) ev[q] = fe_add(ev[q], fe_mul(f_roll4, fe_sub(NW(q), O(q - 1))));
        ev[0] = fe_add(ev[0], fe_mul(f_roll8, fe_sub(NW(0), O(7))));
#pragma unroll
        for (int q = 1; q < 8; q++) ev[q] = fe_add(ev[q], fe_mul(f_roll8, fe_sub(NW(q), O(q - 1))));
        DG_STEP();
        // arithmetic / boolean: slot 0
        {
            fe prod = fe_mul(O(0), O(1));
            fe v = fe_mul(f_add, fe_sub(NW(0), fe_add(O(0), O(1))));
            v = fe_add(v, fe_mul(fe_add(f_mul, f_and), fe_sub(NW(0), prod)));
            v = fe_add(v, fe_mul(f_inv, fe_sub(ONE, fe_mul(NW(0), O(0)))));
            v = fe_add(v, fe_mul(f_neg, fe_add(NW(0), O(0))));
            v = fe_add(v, fe_mul(f_not, fe_sub(NW(0), bnot(O(0)))));
            v = fe_add(v, fe_mul(f_or, fe_sub(NW(0), bnot(fe_mul(bnot(O(0)), bnot(O(1)))))));
            // eq: new[0] == 1 - (O(1)-O(2)) * O(0)
            v = fe_add(v, fe_mul(f_eq, fe_sub(NW(0), bnot(fe_mul(fe_sub(O(1), O(2)), O(0))))));
            // choose
            {
                fe c = O(2);
                v = fe_add(v, fe_mul(f_choose, fe_sub(NW(0), fe_add(fe_mul(c, O(0)), fe_mul(bnot(c), O(1))))));
            }
            ev[0] = fe_add(ev[0], v);
        }
        DG_STEP();
        // choose2 / cswap2
        {
            fe c = O(4), nc = bnot(c);
            ev[0] = fe_add(ev[0], fe_mul(f_choose2, fe_sub(NW(0), fe_add(fe_mul(c, O(0)), fe_mul(nc, O(2))))));
            ev[1] = fe_add(ev[1], fe_mul(f_choose2, fe_sub(NW(1), fe_add(fe_mul(c, O(1)), fe_mul(nc, O(3))))));
            ev[0] = fe_add(ev[0], fe_mul(f_cswap2, fe_sub(NW(0), fe_add(fe_mul(c, O(2)), fe_mul(nc, O(0))))));
            ev[1] = fe_add(ev[1], fe_mul(f_cswap2, fe_sub(NW(1), fe_add(fe_mul(c, O(3)), fe_mul(nc, O(1))))));
            ev[2] = fe_add(ev[2], fe_mul(f_cswap2, fe_sub(NW(2), fe_add(fe_mul(c, O(0)), fe_mul(nc, O(2))))));
            ev[3] = fe_add(ev[3], fe_mul(f_cswap2, fe_sub(NW(3), fe_add(fe_mul(c, O(1)), fe_mul(nc, O(3))))));
        }
        DG_STEP();
        // binacc (comparison.rs:111-133)
        {
            fe bit = NW(0);
            ev[0] = fe_add(ev[0], fe_mul(f_binacc, is_bin(bit)));
            ev[1] = fe_add(ev[1], fe_mul(f_binacc, NW(1)));
            ev[2] = fe_add(ev[2], fe_mul(f_binacc, fe_sub(NW(2), fe_mul_small(O(2), 2))));
            ev[3] = fe_add(ev[3], fe_mul(f_binacc, fe_sub(NW(3), fe_add(O(3), fe_mul(bit, O(2))))));
        }
        DG_STEP();
        // cmp (comparison.rs:71-108): [pow, bit_a, bit_b, not_set, gt, lt, acc_b, acc_a]
        {
            fe xb = NW(1), yb = NW(2), not_set = NW(3);
            fe bit_gt = fe_mul(xb, bnot(yb)), bit_lt = fe_mul(yb, bnot(xb));
            fe gt = fe_add(O(4), fe_mul(bit_gt, not_set)), lt = fe_add(O(5), fe_mul(bit_lt, not_set));
            fe p2 = O(0);
            fe x_acc = fe_add(O(7), fe_mul(xb, p2)), y_acc = fe_add(O(6), fe_mul(yb, p2));
            fe nsc = fe_mul(bnot(O(5)), bnot(O(4)));
            ev[0] = fe_add(ev[0], fe_mul(f_cmp, is_bin(xb)));
            ev[1] = fe_add(ev[1], fe_mul(f_cmp, is_bin(yb)));
            ev[2] = fe_add(ev[2], fe_mul(f_cmp, fe_sub(NW(4), gt)));
            ev[3] = fe_add(ev[3], fe_mul(f_cmp, fe_sub(NW(5), lt)));
            ev[4] = fe_add(ev[4], fe_mul(f_cmp, fe_sub(NW(6), y_acc)));
            ev[5] = fe_add(ev[5], fe_mul(f_cmp, fe_sub(NW(7), x_acc)));
            ev[6] = fe_add(ev[6], fe_mul(f_cmp, fe_sub(not_set, nsc)));
            ev[7] = fe_add(ev[7], fe_mul(f_cmp, fe_sub(fe_mul_small(NW(0), 2), p2)));
        }
        DG_STEP();
        // rescr (stack/hash.rs:9-35)
        {
            fe os[6], ns[6];
#pragma unroll
            for (int q = 0; q < 6; q++) os[q] = fe_cube(fe_add(O(q), per[11 + q]));
            matvec<6>(c_hasher_mds, os);
#pragma unroll
            for (int q = 0; q < 6; q++) ns[q] = NW(q);
            matvec<6>(c_hasher_inv_mds, ns);
#pragma unroll
            for (int q = 0; q < 6; q++) ns[q] = fe_sub(fe_cube(ns[q]), per[11 + 6 + q]);
#pragma unroll
            for (int q = 0; q < 6; q++) ev[q] = fe_add(ev[q], fe_mul(f_rescr, fe_sub(ns[q], os[q])));
        }
#pragma unroll
        for (int i = 0; i < 8; i++)
            if (i < P.stack_depth) fold(base + 2 + i, G7, ev[i]);
    }

    DG_STEP();
    // ---- combine (evaluator.rs:335-358): result + sum_g adj_g * x^inc_g ------------------------------------------------------------------
    fe t_res = DG_REDUCE_WIDE(acc.res);
    const fe *const xpow_override = P.xpow_override ? P.xpow_override + blockIdx.y * P.override_stride : nullptr;
#pragma unroll
    for (int g = 0; g < 6; g++) t_res = fe_add(t_res, fe_mul(acc.adj[g], xpow_override ? xpow_override[g] : tw_pow(P.twN, lde_index * P.inc[g])));
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
    const unsigned long long E = (unsigned long long)P.num_c8 << P.log_n;
    // H100 SXM (700 W), stage 3 of the 2^20-step proof x 26 registers: per-thread arrays 24.8 ms; shared-memory rows, stack-like columns
    // only 23.7; all columns 23.2; all columns + unreduced per-slot sums (constraint_eval_smem_kernel) 22.2.  The other forms were removed
    // after this measurement.
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

}  // namespace dg
