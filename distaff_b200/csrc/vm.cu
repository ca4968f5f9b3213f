// The Distaff VM on the GPU: processor::execute (processor/mod.rs:23-182, decoder/mod.rs, stack/mod.rs) of many programs for many
// inputs, one thread per execution.  It restates the Machine of the host VM (hostvm/vm.cpp) as a loop: run_blocks / close_block /
// run_span become an explicit frame stack, and the decoder and stack operations keep their order, checks and messages.  The programs of
// a call share one set of tables; each program's executions start on a warp boundary, so that a warp runs one instruction stream.
//
// Two passes, each one launch for many executions:
//   shape pass  no sponge and no register writes: the step count, the ctx / loop / stack depths, the peak tape lengths, the final stack
//               and the first failure.  Control flow and the stack never read the sponge, so this is the whole execution but the hash.
//   write pass  the same execution with the sponge, writing every register of every row up to the last step into its own place and
//               shape (one launch covers executions of any mix of shapes); it also checks the loop images and the program hash, which
//               need the sponge.  A second, coalesced kernel writes the padding rows of Machine::finalize, one launch per shape.
// Executions from sponge tables (dg_trace_many / dg_execute_many, and dg_trace_one / dg_execute_one as their one-execution case) run
// three more kernels instead:
//   table       the sponge chain of every block list of every program, level by level (vm.h); the sponge never reads data, so with
//               consistent hashes the state after every step is a table lookup
//   sequential  each execution on one lane, as the write pass but with the sponge from the table and no register writes: it records a
//               checkpoint (the whole machine state) at the first top of the frame loop at or after every S steps, and logs every value
//               popped from the tapes (hints push onto them mid-execution, so a segment cannot read the tapes itself)
//   segment     one thread per checkpoint of every execution of a wave: replays from it to the next one with the sponge from the table
//               and the tape values from the log, writes those rows, and checks that it ends in the state the next checkpoint holds
// The per-thread stack, context stack, loop stack and frame stack are indexed at run time and live in local memory by design.
#define DG_MUL_CALL 1
#include "common.cuh"
#include "air_constants.h"
#include "alg_sbox.cuh"
#include "vm.h"

namespace dg {

__constant__ fe c_vm_sponge_ark[128];     // utils/sponge.rs ARK: 8 rows of 16
__constant__ fe c_vm_sponge_mds[16];
__constant__ fe c_vm_hasher_ark[192];     // utils/hasher.rs ARK: 12 rows of 16
__constant__ fe c_vm_hasher_mds[36];

void vm_upload_constants(Context &c) {
    if (c.vm_consts) return;
    std::vector<fe> v(192);
    for (int i = 0; i < 128; i++) v[i] = fe_make(DG_SPONGE_ARK[i][0], DG_SPONGE_ARK[i][1]);
    DG_CUDA(cudaMemcpyToSymbol(c_vm_sponge_ark, v.data(), 128 * sizeof(fe)));
    for (int i = 0; i < 16; i++) v[i] = fe_make(DG_SPONGE_MDS[i][0], DG_SPONGE_MDS[i][1]);
    DG_CUDA(cudaMemcpyToSymbol(c_vm_sponge_mds, v.data(), 16 * sizeof(fe)));
    for (int i = 0; i < 192; i++) v[i] = fe_make(DG_HASHER_ARK[i][0], DG_HASHER_ARK[i][1]);
    DG_CUDA(cudaMemcpyToSymbol(c_vm_hasher_ark, v.data(), 192 * sizeof(fe)));
    for (int i = 0; i < 36; i++) v[i] = fe_make(DG_HASHER_MDS[i][0], DG_HASHER_MDS[i][1]);
    DG_CUDA(cudaMemcpyToSymbol(c_vm_hasher_mds, v.data(), 36 * sizeof(fe)));
    c.vm_consts = true;
}

std::string vm_message(unsigned code, unsigned long long step, unsigned long long max_steps) {
    static const char *const MSG[VM_NO_STEP] = {
        "", "ASSERT failed", "ASSERTEQ failed", "stack underflow", "stack overflow", "invalid value for PUSH", "attempt to read from empty tape A",
        "invalid hint for READ", "too few items on tapes for pmpath macro", "attempt to read from empty tape", "invalid hint for READ2",
        "CHOOSE on a non-binary condition", "CHOOSE2 on a non-binary condition", "CSWAP2 on a non-binary condition", "cannot compute INV of 0",
        "NOT of a non-binary value", "AND of a non-binary value", "OR of a non-binary value", "invalid AUX value for EQ", "invalid hint for CMP",
        "expected binary input", "expected top of the stack to be a power of 2", "invalid hint for BINACC",
        "expected 3rd value from the top of the stack to be a power of 2", "unknown opcode", "op_value is non-zero for a non-PUSH operation",
        "invalid PUSH operation alignment", "context stack overflow", "context stack underflow", "loop stack overflow", "loop stack underflow",
        "cannot start context block: invalid alignment", "cannot exit context block: invalid alignment", "cannot start a loop: invalid alignment",
        "cannot wrap a loop: invalid alignment", "cannot break a loop: invalid alignment", "hash of the last iteration doesn't match loop image",
        "cannot select a branch based on a non-binary condition", "cannot exit loop based on a non-binary condition",
        "cannot enter loop based on a non-binary condition"};
    if (code < VM_NO_STEP) return std::string(MSG[code]) + " at step " + std::to_string(step);
    switch (code) {
        case VM_SEGMENT: return "internal error: a trace segment did not end in the state the sequential pass recorded, at step " + std::to_string(step);
        case VM_CAP: return "execution exceeds " + std::to_string(max_steps) + " steps";
        case VM_MIN_OPS: return "a program must consist of at least 16 operations";
        case VM_HASH: return "program hash does not match trace hash";
        case VM_DIVERGED: return "internal error: the write pass left the path of the shape pass at step " + std::to_string(step);
        default: return "tape scratch exhausted";
    }
}

namespace {

// op codes (processor/opcodes.rs) and decoder flow ops, as hostvm/vm.cpp names them
enum : unsigned {
    OP_BEGIN = 0x00, OP_PUSH = 0x1f, OP_CMP = 0x3f, OP_RESCR = 0x5f, OP_ASSERT = 0x60, OP_ASSERTEQ = 0x61, OP_EQ = 0x62, OP_DROP = 0x63,
    OP_DROP4 = 0x64, OP_CHOOSE = 0x65, OP_CHOOSE2 = 0x66, OP_CSWAP2 = 0x67, OP_ADD = 0x68, OP_MUL = 0x69, OP_AND = 0x6a, OP_OR = 0x6b,
    OP_INV = 0x6c, OP_NEG = 0x6d, OP_NOT = 0x6e, OP_READ = 0x70, OP_READ2 = 0x71, OP_DUP = 0x72, OP_DUP2 = 0x73, OP_DUP4 = 0x74, OP_PAD2 = 0x75,
    OP_SWAP = 0x78, OP_SWAP2 = 0x79, OP_SWAP4 = 0x7a, OP_ROLL4 = 0x7b, OP_ROLL8 = 0x7c, OP_BINACC = 0x7d, OP_NOOP = 0x7f,
};
enum : unsigned { F_HACC = 0, F_BEGIN = 1, F_TEND = 2, F_FEND = 3, F_LOOP = 4, F_WRAP = 5, F_BREAK = 6 };
enum : unsigned { H_NONE = DG_HINT_NONE, H_PUSH = DG_HINT_PUSH, H_EQ = DG_HINT_EQ_START, H_RC = DG_HINT_RC_START, H_CMP = DG_HINT_CMP_START,
                  H_PMPATH = DG_HINT_PMPATH_START };
// continuation of a block list when it ends (what hostvm's run_blocks does after its recursive call returns)
enum : unsigned { C_ROOT, C_GROUP, C_SWITCH_TRUE, C_SWITCH_FALSE, C_LOOP_SKIP, C_LOOP_BODY };

__device__ __forceinline__ fe fe_small(unsigned long long v) { return fe_make(v, 0); }
__device__ __forceinline__ bool is_bin(fe v) { return v.hi == 0 && v.lo <= 1; }
__device__ __forceinline__ bool is_one(fe v) { return v.hi == 0 && v.lo == 1; }
__device__ __forceinline__ bool is_pow2(fe v) {
    return v.hi == 0 ? (v.lo != 0 && (v.lo & (v.lo - 1)) == 0) : (v.lo == 0 && (v.hi & (v.hi - 1)) == 0);
}
// bit k (< 256) of a 128-bit value; 0 above bit 127
__device__ __forceinline__ unsigned long long bit_of(fe v, unsigned k) { return k < 64 ? (v.lo >> k) & 1 : k < 128 ? (v.hi >> (k - 64)) & 1 : 0; }

template <int W>
__device__ __forceinline__ void vm_mds(fe *s, const fe *m) {
    fe r[W];
#pragma unroll
    for (int i = 0; i < W; i++) {
        fe acc = fe_mul(m[i * W], s[0]);
#pragma unroll
        for (int j = 1; j < W; j++) acc = fe_add(acc, fe_mul(m[i * W + j], s[j]));
        r[i] = acc;
    }
#pragma unroll
    for (int i = 0; i < W; i++) s[i] = r[i];
}
// utils/sponge.rs:13-30
__device__ void sponge_round(fe s[4], unsigned op, fe op_value, unsigned long long step) {
    const unsigned idx = (unsigned)(step & 15);
#pragma unroll
    for (int i = 0; i < 4; i++) s[i] = fe_cube(fe_add(s[i], c_vm_sponge_ark[i * 16 + idx]));
    vm_mds<4>(s, c_vm_sponge_mds);
    s[0] = fe_add(s[0], fe_small(op));
    s[1] = fe_add(s[1], op_value);
#pragma unroll 1
    for (int i = 0; i < 4; i++) s[i] = alg_inv_sbox(fe_add(s[i], c_vm_sponge_ark[(4 + i) * 16 + idx]));
    vm_mds<4>(s, c_vm_sponge_mds);
}
// utils/hasher.rs:28-40
__device__ void hasher_round(fe s[6], unsigned long long step) {
    const unsigned idx = (unsigned)(step & 15);
#pragma unroll
    for (int i = 0; i < 6; i++) s[i] = fe_cube(fe_add(s[i], c_vm_hasher_ark[i * 16 + idx]));
    vm_mds<6>(s, c_vm_hasher_mds);
#pragma unroll 1
    for (int i = 0; i < 6; i++) s[i] = alg_inv_sbox(fe_add(s[i], c_vm_hasher_ark[(6 + i) * 16 + idx]));
    vm_mds<6>(s, c_vm_hasher_mds);
}

struct Frame { unsigned first, count, k, block, cont; };

// what a Machine runs: the shape and write passes, or the sequential and segment passes of one execution, which take the sponge from the
// table (vm.h)
enum : int { M_SHAPE, M_WRITE, M_SEQUENTIAL, M_SEGMENT };

// the whole state of an execution at the top of the frame loop: what the sequential pass records and a segment starts from
struct VmCheckpoint {
    unsigned long long step, opc, na, nb, lpos, at, tpos[16];
    unsigned depth, max_depth, ctx_depth, loop_depth, ctx_cols, loop_cols;
    int top;
    unsigned pad;
    Frame fr[16];
    fe sponge[4], S[32], ctx[16], lp[8];
};

// the members only the tabled passes have (an empty base of the shape and write passes)
template <bool TABLED> struct TableState {};
template <> struct TableState<true> {
    const VmSponge *tab;
    const VmChainRef *chains;
    unsigned long long at, parent_at;                 // the next entry of the running frame's chain; the entry end_block resumes at
    fe *log;
    unsigned long long lpos, lcap;                    // values popped so far (the next one to log or read)
    VmCheckpoint *cp;                                 // sequential pass: checkpoints recorded and room for them, where the next is due
    unsigned long long ncp, cp_cap, next_cp, seg;
    const VmCheckpoint *expect;                       // segment pass: the state it must end in, at the first boundary at or after `stop`
    unsigned long long stop;
};

// One execution.  The decoder and the stack advance in lock-step, so `step` serves both; the registers of row `step` are the fields
// below (S[i] = 0 at and above the stack depth, ctx / lp = 0 at and above their depths, as the host VM's columns are).
template <int MODE>
struct Machine : TableState<(MODE >= M_SEQUENTIAL)> {
    static constexpr bool WRITE = MODE == M_WRITE || MODE == M_SEGMENT;       // writes registers
    static constexpr bool SPONGE = MODE != M_SHAPE;                           // knows the sponge (rounds or the table)
    static constexpr bool TABLED = MODE >= M_SEQUENTIAL;
    const VmLaunch &L;
    unsigned long long step = 0, opc = 0, max_steps;
    unsigned code = VM_OK;
    unsigned long long fail_step = 0;
    unsigned ctx_depth = 1, loop_depth = 0, ctx_cols = 1, loop_cols = 0, depth, max_depth;
    fe sponge[4];
    fe ctx[16], lp[8], S[32];
    fe *ta, *tb;
    unsigned long long na, nb, cap_a, cap_b, peak_a, peak_b;
    fe *out;                      // write pass: this execution's registers, column stride `length`
    unsigned long long length;
    unsigned ctx_out, loop_out, stack_out;

    __device__ Machine(const VmLaunch &l) : L(l), max_steps(l.max_steps) {}

    __device__ __forceinline__ bool fail(unsigned c) { code = c; fail_step = step; return false; }
    __device__ __forceinline__ bool failed() const { return code != VM_OK; }

    // ---- registers of the write pass
    __device__ __forceinline__ void put(unsigned col, unsigned long long row, fe v) { out[(size_t)col * length + row] = v; }
    __device__ void commit_state() {
        if (!WRITE) return;
        const unsigned long long s = step;
        put(0, s, fe_small(opc));
        for (int i = 0; i < 4; i++) put(1 + i, s, sponge[i]);
        unsigned col = 15;
        for (unsigned i = 0; i < ctx_out; i++) put(col++, s, ctx[i]);
        for (unsigned i = 0; i < loop_out; i++) put(col++, s, lp[i]);
        for (unsigned i = 0; i < stack_out; i++) put(col++, s, i < 32 ? S[i] : fe_small(0));
    }
    __device__ void commit_bits(unsigned flow, unsigned user) {    // the op bits of the step that led to row `step` sit in row step - 1
        if (!WRITE) return;
        const unsigned long long s = step - 1;
        for (int i = 0; i < 3; i++) put(5 + i, s, fe_small((flow >> i) & 1));
        for (int i = 0; i < 5; i++) put(8 + i, s, fe_small((user >> i) & 1));
        for (int i = 0; i < 2; i++) put(13 + i, s, fe_small((user >> (i + 5)) & 1));
    }

    // ---- tapes (stacks: the next value to read is the last one)
    __device__ __forceinline__ bool push_a(fe v) {
        if constexpr (MODE == M_SEGMENT) { na++; return true; }          // a segment counts the tapes and reads popped values from the log
        if (na == cap_a) return fail(VM_TAPE_SCRATCH);
        ta[na++] = v;
        peak_a = max(peak_a, na);
        return true;
    }
    __device__ __forceinline__ bool push_b(fe v) {
        if constexpr (MODE == M_SEGMENT) { nb++; return true; }
        if (nb == cap_b) return fail(VM_TAPE_SCRATCH);
        tb[nb++] = v;
        peak_b = max(peak_b, nb);
        return true;
    }
    __device__ __forceinline__ fe pop_a() {
        if constexpr (MODE == M_SEGMENT) { --na; return this->log[this->lpos++]; }
        const fe v = ta[--na];
        if constexpr (MODE == M_SEQUENTIAL) logged(v);
        return v;
    }
    __device__ __forceinline__ fe pop_b() {
        if constexpr (MODE == M_SEGMENT) { --nb; return this->log[this->lpos++]; }
        const fe v = tb[--nb];
        if constexpr (MODE == M_SEQUENTIAL) logged(v);
        return v;
    }
    __device__ __forceinline__ void logged(fe v) {     // a log too small for the execution is counted on; the host runs it again
        if (this->lpos < this->lcap) this->log[this->lpos] = v;
        this->lpos++;
    }
    // the tabled passes: the state after this step is the running frame's next chain entry
    __device__ __forceinline__ void take() {
        const VmSponge &e = this->tab[this->at++];
        for (int i = 0; i < 4; i++) sponge[i] = e.s[i];
    }

    __device__ bool advance(bool user_op) {
        if (step + 1 >= max_steps) { code = VM_CAP; fail_step = step; return false; }
        if (WRITE && step + 1 >= length) return fail(VM_DIVERGED);        // never past the rows the shape pass measured
        step += 1;
        if (user_op) opc += 1;
        return true;
    }
    __device__ bool save_context() {
        ctx_depth += 1;
        if (ctx_depth > 16) return fail(VM_CTX_OVERFLOW);
        ctx_cols = max(ctx_cols, ctx_depth);
        for (int i = 15; i > 0; i--) ctx[i] = ctx[i - 1];
        ctx[0] = sponge[0];
        return true;
    }
    __device__ bool pop_context(fe &h) {
        if (ctx_depth == 0) return fail(VM_CTX_UNDERFLOW);
        h = ctx[0];
        for (int i = 1; i < 16; i++) ctx[i - 1] = ctx[i];
        ctx[15] = fe_small(0);
        ctx_depth -= 1;
        return true;
    }
    __device__ bool save_loop_image(fe image) {
        loop_depth += 1;
        if (loop_depth > 8) return fail(VM_LOOP_OVERFLOW);
        loop_cols = max(loop_cols, loop_depth);
        for (int i = 7; i > 0; i--) lp[i] = lp[i - 1];
        lp[0] = image;
        return true;
    }
    __device__ bool pop_loop_image(fe &img) {
        if (loop_depth == 0) return fail(VM_LOOP_UNDERFLOW);
        img = lp[0];
        for (int i = 1; i < 8; i++) lp[i - 1] = lp[i];
        lp[7] = fe_small(0);
        loop_depth -= 1;
        return true;
    }
    __device__ __forceinline__ void set_sponge(fe a, fe b, fe c, fe d) { sponge[0] = a; sponge[1] = b; sponge[2] = c; sponge[3] = d; }

    // ---- decoder ops (decoder/mod.rs), each followed by a NOOP of the stack
    __device__ bool start_block() {
        if (step % 16 != 15) return fail(VM_START_ALIGN);
        if (!advance(false) || !save_context()) return false;
        const fe z = fe_small(0);
        set_sponge(z, z, z, z);
        commit_bits(F_BEGIN, OP_NOOP); commit_state();
        return true;
    }
    __device__ bool end_block(fe sibling, bool true_branch) {
        if (step % 16 != 0) return fail(VM_END_ALIGN);
        fe h;
        if (!advance(false) || !pop_context(h)) return false;
        const fe bh = sponge[0], z = fe_small(0);
        if (true_branch) set_sponge(h, bh, sibling, z); else set_sponge(h, sibling, bh, z);
        if constexpr (TABLED) this->at++;               // computed as the write pass does; the table holds the same state
        commit_bits(true_branch ? F_TEND : F_FEND, OP_NOOP); commit_state();
        return true;
    }
    __device__ bool start_loop(fe image) {
        if (step % 16 != 15) return fail(VM_LOOP_ALIGN);
        if (!advance(false) || !save_context() || !save_loop_image(image)) return false;
        const fe z = fe_small(0);
        set_sponge(z, z, z, z);
        commit_bits(F_LOOP, OP_NOOP); commit_state();
        return true;
    }
    __device__ bool wrap_loop() {
        if (step % 16 != 15) return fail(VM_WRAP_ALIGN);
        if (!advance(false)) return false;
        if (loop_depth == 0) return fail(VM_LOOP_UNDERFLOW);
        if (SPONGE && !fe_eq(sponge[0], lp[0])) return fail(VM_LOOP_IMAGE);
        const fe z = fe_small(0);
        set_sponge(z, z, z, z);
        commit_bits(F_WRAP, OP_NOOP); commit_state();
        return true;
    }
    __device__ bool break_loop() {
        if (step % 16 != 15) return fail(VM_BREAK_ALIGN);
        fe img;
        if (!advance(false) || !pop_loop_image(img)) return false;
        if (SPONGE && !fe_eq(sponge[0], img)) return fail(VM_LOOP_IMAGE);
        commit_bits(F_BREAK, OP_NOOP); commit_state();
        return true;
    }
    __device__ bool exec(unsigned op, const VmHint &hint) {
        const fe op_value = hint.kind == H_PUSH ? hint.value : fe_small(0);
        if (!fe_is_zero(op_value)) {
            if (op != OP_PUSH) return fail(VM_OPVALUE);
            if (step % 8 != 0) return fail(VM_PUSH_ALIGN);
        }
        if (!advance(true)) return false;
        if constexpr (TABLED) take();
        else if (WRITE) sponge_round(sponge, op, op_value, step - 1);
        if (!stack_op(op, hint)) return false;
        commit_bits(F_HACC, op); commit_state();
        return true;
    }
    __device__ bool noop() { VmHint h; h.kind = H_NONE; h.n = 0; h.value = fe_small(0); return exec(OP_NOOP, h); }

    // ---- stack (stack/mod.rs) on row `step`, already advanced
    __device__ __forceinline__ bool need(unsigned d) { return depth < d ? fail(VM_STACK_UNDERFLOW) : true; }
    __device__ bool shift_left(unsigned start, unsigned cnt) {
        if (depth < cnt) return fail(VM_STACK_UNDERFLOW);
        for (unsigned i = start; i < depth; i++) S[i - cnt] = S[i];
        for (unsigned i = depth - cnt; i < depth; i++) S[i] = fe_small(0);
        depth -= cnt;
        return true;
    }
    __device__ bool shift_right(unsigned cnt) {
        depth += cnt;
        if (depth > 32) return fail(VM_STACK_OVERFLOW);
        if (depth > max_depth) max_depth += cnt;         // as the host VM counts it (stack/mod.rs)
        for (unsigned i = depth - 1; i >= cnt; i--) S[i] = S[i - cnt];
        return true;
    }
    __device__ bool stack_op(unsigned op, const VmHint &hint) {
        switch (op) {
        case OP_BEGIN: case OP_NOOP: return true;
        case OP_ASSERT: if (!need(1)) return false; if (!is_one(S[0])) return fail(VM_ASSERT); return shift_left(1, 1);
        case OP_ASSERTEQ: if (!need(2)) return false; if (!fe_eq(S[0], S[1])) return fail(VM_ASSERTEQ); return shift_left(2, 2);
        case OP_PUSH:
            if (hint.kind != H_PUSH) return fail(VM_PUSH_VALUE);
            if (!shift_right(1)) return false;
            S[0] = hint.value;
            return true;
        case OP_READ:
            if (hint.kind == H_EQ) {
                if (!need(2)) return false;
                const fe x = S[0], y = S[1];
                if (!push_a(fe_eq(x, y) ? fe_small(1) : fe_inv(fe_sub(x, y)))) return false;
            } else if (hint.kind == H_NONE) { if (na == 0) return fail(VM_EMPTY_TAPE_A); }
            else return fail(VM_HINT_READ);
            if (!shift_right(1)) return false;
            S[0] = pop_a();
            return true;
        case OP_READ2:
            if (hint.kind == H_PMPATH) {
                if (!need(3)) return false;
                const unsigned n = hint.n - 1;
                if (na < n || nb < n) return fail(VM_PMPATH_TAPES);
                if (na + n > cap_a) return fail(VM_TAPE_SCRATCH);
                // the last n values of A become (bit, value) pairs; backwards, so that no value is overwritten before it is read
                const fe idx = S[2];
                const unsigned long long base = na - n;
                if constexpr (MODE != M_SEGMENT)
                    for (int i = (int)n - 1; i >= 0; i--) {
                        const fe v = ta[base + i];
                        ta[base + 2 * i] = fe_small(bit_of(idx, n - i - 1));
                        ta[base + 2 * i + 1] = v;
                    }
                na += n;
                peak_a = max(peak_a, na);
            } else if (hint.kind == H_NONE) { if (na == 0 || nb == 0) return fail(VM_EMPTY_TAPE); }
            else return fail(VM_HINT_READ2);
            if (!shift_right(2)) return false;
            S[1] = pop_a();
            S[0] = pop_b();
            return true;
        case OP_DUP: return need(1) && shift_right(1);
        case OP_DUP2: return need(2) && shift_right(2);
        case OP_DUP4: return need(4) && shift_right(4);
        case OP_PAD2: if (!shift_right(2)) return false; S[0] = S[1] = fe_small(0); return true;
        case OP_DROP: return need(1) && shift_left(1, 1);
        case OP_DROP4: return need(4) && shift_left(4, 4);
        case OP_SWAP: { if (!need(2)) return false; const fe t = S[0]; S[0] = S[1]; S[1] = t; return true; }
        case OP_SWAP2: {
            if (!need(4)) return false;
            for (int i = 0; i < 2; i++) { const fe t = S[i]; S[i] = S[i + 2]; S[i + 2] = t; }
            return true; }
        case OP_SWAP4: {
            if (!need(8)) return false;
            for (int i = 0; i < 4; i++) { const fe t = S[i]; S[i] = S[i + 4]; S[i + 4] = t; }
            return true; }
        case OP_ROLL4: { if (!need(4)) return false; const fe t = S[3]; for (int i = 3; i > 0; i--) S[i] = S[i - 1]; S[0] = t; return true; }
        case OP_ROLL8: { if (!need(8)) return false; const fe t = S[7]; for (int i = 7; i > 0; i--) S[i] = S[i - 1]; S[0] = t; return true; }
        case OP_CHOOSE: {
            if (!need(3)) return false;
            const fe c = S[2];
            if (!is_bin(c)) return fail(VM_CHOOSE);
            if (c.lo == 0) S[0] = S[1];
            return shift_left(3, 2); }
        case OP_CHOOSE2: {
            if (!need(6)) return false;
            const fe c = S[4];
            if (!is_bin(c)) return fail(VM_CHOOSE2);
            if (c.lo == 0) { S[0] = S[2]; S[1] = S[3]; }
            return shift_left(6, 4); }
        case OP_CSWAP2: {
            if (!need(6)) return false;
            const fe c = S[4];
            if (!is_bin(c)) return fail(VM_CSWAP2);
            if (c.lo == 1) for (int i = 0; i < 2; i++) { const fe t = S[i]; S[i] = S[i + 2]; S[i + 2] = t; }
            return shift_left(6, 2); }
        case OP_ADD: if (!need(2)) return false; S[0] = fe_add(S[0], S[1]); return shift_left(2, 1);
        case OP_MUL: if (!need(2)) return false; S[0] = fe_mul(S[0], S[1]); return shift_left(2, 1);
        case OP_INV: if (!need(1)) return false; if (fe_is_zero(S[0])) return fail(VM_INV_ZERO); S[0] = fe_inv(S[0]); return true;
        case OP_NEG: if (!need(1)) return false; S[0] = fe_sub(fe_small(0), S[0]); return true;
        case OP_NOT: if (!need(1)) return false; if (!is_bin(S[0])) return fail(VM_NOT); S[0] = fe_small(1 - S[0].lo); return true;
        case OP_AND: case OP_OR: {
            if (!need(2)) return false;
            if (!is_bin(S[0]) || !is_bin(S[1])) return fail(op == OP_AND ? VM_AND : VM_OR);
            S[0] = fe_small(op == OP_AND ? (S[0].lo & S[1].lo) : (S[0].lo | S[1].lo));
            return shift_left(2, 1); }
        case OP_EQ: {
            if (!need(3)) return false;
            const fe aux = S[0], x = S[1], y = S[2];
            if (fe_eq(x, y)) S[0] = fe_small(1);
            else { if (!fe_eq(aux, fe_inv(fe_sub(x, y)))) return fail(VM_EQ_AUX); S[0] = fe_small(0); }
            return shift_left(3, 2); }
        case OP_CMP: {
            if (hint.kind == H_CMP) {
                if (!need(10)) return false;
                const fe a = S[8], b = S[9];
                for (unsigned i = 0; i < hint.n; i++)
                    if (!push_a(fe_small(bit_of(a, i))) || !push_b(fe_small(bit_of(b, i)))) return false;
            } else if (hint.kind == H_NONE) { if (!need(8)) return false; if (na == 0 || nb == 0) return fail(VM_EMPTY_TAPE); }
            else return fail(VM_HINT_CMP);
            // (spelt so that the shape and write passes compile exactly as they did before the tabled passes)
            const fe a_bit = TABLED ? pop_a() : ta[--na], b_bit = TABLED ? pop_b() : tb[--nb];
            if (!is_bin(a_bit) || !is_bin(b_bit)) return fail(VM_BINARY);
            const fe p2 = S[0];
            if (!is_pow2(p2)) return fail(VM_CMP_POW2);
            const unsigned long long ab = a_bit.lo, bb = b_bit.lo;
            const fe np2 = (p2.hi == 0 && p2.lo == 1) ? fe_inv(fe_small(2)) : fe_make((p2.lo >> 1) | (p2.hi << 63), p2.hi >> 1);
            const fe gt = S[4], lt = S[5];
            const fe not_set = fe_mul(fe_sub(fe_small(1), gt), fe_sub(fe_small(1), lt));
            S[0] = np2; S[1] = a_bit; S[2] = b_bit; S[3] = not_set;
            if (ab & (1 - bb)) S[4] = fe_add(gt, not_set);
            if (bb & (1 - ab)) S[5] = fe_add(lt, not_set);
            if (bb) S[6] = fe_add(S[6], p2);
            if (ab) S[7] = fe_add(S[7], p2);
            return true; }
        case OP_BINACC: {
            if (hint.kind == H_RC) {
                if (!need(5)) return false;
                const fe v = S[4];
                for (unsigned i = 0; i < hint.n; i++) if (!push_a(fe_small(bit_of(v, hint.n - i - 1)))) return false;
            } else if (hint.kind == H_NONE) { if (!need(4)) return false; if (na == 0) return fail(VM_EMPTY_TAPE_A); }
            else return fail(VM_HINT_BINACC);
            const fe bit = pop_a();
            if (!is_bin(bit)) return fail(VM_BINARY);
            const fe p2 = S[2];
            if (!is_pow2(p2)) return fail(VM_BINACC_POW2);
            S[0] = bit; S[1] = fe_small(0); S[2] = fe_add(p2, p2);
            if (bit.lo) S[3] = fe_add(S[3], p2);
            return true; }
        case OP_RESCR: {
            if (!need(6)) return false;
            fe st[6];
            for (int i = 0; i < 6; i++) st[i] = S[i];
            hasher_round(st, step - 1);
            for (int i = 0; i < 6; i++) S[i] = st[i];
            return true; }
        default: return fail(VM_UNKNOWN_OP);
        }
    }

    // ---- processor/mod.rs:50-182
    __device__ bool close_block(fe sibling, bool true_branch) {
        if (!noop()) return false;                      // the last step of the closed list's frame
        if constexpr (TABLED) this->at = this->parent_at;
        if (!end_block(sibling, true_branch)) return false;
        for (int i = 0; i < 14; i++) if (!noop()) return false;
        return true;
    }
    __device__ bool run_span(const VmBlock &b, bool is_first) {
        if (!is_first && !noop()) return false;
        for (unsigned i = 0; i < b.count; i++) if (!exec(L.ops[b.first + i], L.hints[b.first + i])) return false;
        return true;
    }
    // ---- checkpoints of the tabled passes: the state at the top of the frame loop, the frames and where each resumes in its chain
    __device__ void save(VmCheckpoint &c, const Frame *fr, int top, const unsigned long long *tpos) const {
        c.step = step; c.opc = opc; c.na = na; c.nb = nb; c.lpos = this->lpos; c.at = this->at;
        c.depth = depth; c.max_depth = max_depth; c.ctx_depth = ctx_depth; c.loop_depth = loop_depth; c.ctx_cols = ctx_cols;
        c.loop_cols = loop_cols; c.top = top; c.pad = 0;
        for (int i = 0; i < 16; i++) {
            c.tpos[i] = i < top ? tpos[i] : 0;
            c.fr[i] = i <= top ? fr[i] : Frame{0, 0, 0, 0, 0};
            c.ctx[i] = ctx[i];
        }
        for (int i = 0; i < 4; i++) c.sponge[i] = sponge[i];
        for (int i = 0; i < 32; i++) c.S[i] = S[i];
        for (int i = 0; i < 8; i++) c.lp[i] = lp[i];
    }
    __device__ void load(const VmCheckpoint &c) {
        step = c.step; opc = c.opc; na = c.na; nb = c.nb; this->lpos = c.lpos; this->at = c.at;
        depth = c.depth; max_depth = c.max_depth; ctx_depth = c.ctx_depth; loop_depth = c.loop_depth; ctx_cols = c.ctx_cols;
        loop_cols = c.loop_cols;
        for (int i = 0; i < 4; i++) sponge[i] = c.sponge[i];
        for (int i = 0; i < 32; i++) S[i] = c.S[i];
        for (int i = 0; i < 16; i++) ctx[i] = c.ctx[i];
        for (int i = 0; i < 8; i++) lp[i] = c.lp[i];
    }
    __device__ bool same(const VmCheckpoint &c, const Frame *fr, int top, const unsigned long long *tpos) const {
        bool ok = c.step == step && c.opc == opc && c.na == na && c.nb == nb && c.lpos == this->lpos && c.at == this->at && c.depth == depth &&
                  c.max_depth == max_depth && c.ctx_depth == ctx_depth && c.loop_depth == loop_depth && c.ctx_cols == ctx_cols &&
                  c.loop_cols == loop_cols && c.top == top;
        for (int i = 0; ok && i <= top; i++)
            ok = c.fr[i].first == fr[i].first && c.fr[i].count == fr[i].count && c.fr[i].k == fr[i].k && c.fr[i].block == fr[i].block &&
                 c.fr[i].cont == fr[i].cont && (i == top || c.tpos[i] == tpos[i]);
        for (int i = 0; i < 4; i++) ok = ok && fe_eq(c.sponge[i], sponge[i]);
        for (int i = 0; i < 32; i++) ok = ok && fe_eq(c.S[i], S[i]);
        for (int i = 0; i < 16; i++) ok = ok && fe_eq(c.ctx[i], ctx[i]);
        for (int i = 0; i < 8; i++) ok = ok && fe_eq(c.lp[i], lp[i]);
        return ok;
    }
    // the top of the frame loop: the sequential pass records a checkpoint at the first one at or after every `seg` steps (a buffer too
    // small is counted on, as the log); a segment stops at the first one at or after `stop`, which must hold the next checkpoint's state
    __device__ bool boundary(const Frame *fr, int top, const unsigned long long *tpos) {
        if constexpr (MODE == M_SEQUENTIAL) {
            if (step >= this->next_cp) {
                if (this->ncp < this->cp_cap) save(this->cp[this->ncp], fr, top, tpos);
                this->ncp++;
                this->next_cp = (step / this->seg + 1) * this->seg;
            }
            return false;
        } else {
            if (step < this->stop) return false;
            if (!same(*this->expect, fr, top, tpos)) fail(VM_SEGMENT);
            return true;
        }
    }
    // the root is closed: the final state goes after the checkpoints (sequential pass), and the last segment must end in it
    __device__ void ended(const Frame *fr, int top, const unsigned long long *tpos) {
        if constexpr (MODE == M_SEQUENTIAL) {
            if (this->ncp < this->cp_cap) save(this->cp[this->ncp], fr, top, tpos);
        } else if (!same(*this->expect, fr, top, tpos)) {
            fail(VM_SEGMENT);
        }
    }

    // run_blocks(root body), then close_block(0, true), with the recursion as a frame stack: a frame is a block list being run, `k` the
    // next block of it, `cont` what its block does when the list ends.  The host checked that lists nest at most 15 deep.  The tabled
    // passes also keep where each frame below the top resumes in its own chain; a segment starts from the frames of its checkpoint.
    __device__ void run(unsigned root_first, unsigned root_count) {
        Frame fr[16];
        unsigned long long tpos[TABLED ? 16 : 1];
        int top = 0;
        if constexpr (MODE == M_SEGMENT) {
            const VmCheckpoint &c = *(this->expect - 1);
            top = c.top;
            for (int i = 0; i <= top; i++) { fr[i] = c.fr[i]; tpos[i] = c.tpos[i]; }
        } else {
            fr[0] = Frame{root_first, root_count, 0, 0, C_ROOT};
        }
        const fe z = fe_small(0);
        for (;;) {
            if constexpr (TABLED) { if (boundary(fr, top, tpos)) return; }
            Frame &f = fr[top];
            if (f.k < f.count) {
                const unsigned bi = L.children[f.first + f.k];
                const VmBlock &b = L.blocks[bi];
                const bool first = f.k == 0;
                f.k++;
                if (b.kind == DG_BLOCK_SPAN) { if (!run_span(b, first)) return; continue; }
                Frame nf{b.first, b.count, 0, bi, C_GROUP};
                if (b.kind == DG_BLOCK_GROUP) {
                    if (!start_block()) return;
                } else if (b.kind == DG_BLOCK_SWITCH) {
                    if (!start_block()) return;
                    if (!is_bin(S[0])) { fail(VM_SWITCH_COND); return; }
                    if (S[0].lo == 0) nf = Frame{b.alt_first, b.alt_count, 0, bi, C_SWITCH_FALSE};
                    else nf.cont = C_SWITCH_TRUE;
                } else {
                    if (!is_bin(S[0])) { fail(VM_LOOP_ENTER_COND); return; }
                    if (S[0].lo == 0) {
                        if (!start_block()) return;
                        nf = Frame{b.alt_first, b.alt_count, 0, bi, C_LOOP_SKIP};
                    } else {
                        if (!start_loop(b.hash[0])) return;
                        nf.cont = C_LOOP_BODY;
                    }
                }
                fr[++top] = nf;
                if constexpr (TABLED) {
                    tpos[top - 1] = this->at;
                    this->at = nf.cont == C_SWITCH_FALSE || nf.cont == C_LOOP_SKIP ? this->chains[bi].alt : this->chains[bi].main;
                }
                continue;
            }
            const VmBlock &b = L.blocks[f.block];
            if constexpr (TABLED) this->parent_at = top > 0 ? tpos[top - 1] : this->at + 1;    // the root's end follows its closing NOOP
            switch (f.cont) {
            case C_ROOT:
                if (!close_block(z, true)) return;
                if constexpr (TABLED) ended(fr, top, tpos);
                return;
            case C_GROUP: if (!close_block(z, true)) return; break;
            case C_SWITCH_TRUE: if (!close_block(b.hash[1], true)) return; break;
            case C_SWITCH_FALSE: if (!close_block(b.hash[0], false)) return; break;
            case C_LOOP_SKIP: if (!close_block(b.hash[1], false)) return; break;
            default:                                          // C_LOOP_BODY: one iteration ended
                if (!is_bin(S[0])) { fail(VM_LOOP_EXIT_COND); return; }
                if (S[0].lo == 1) {
                    if (!wrap_loop()) return;
                    if constexpr (TABLED) this->at = this->chains[f.block].main;
                    f.k = 0;
                    continue;
                }
                if constexpr (TABLED) this->at = this->chains[f.block].brk;
                if (!break_loop() || !run_span(L.blocks[L.children[b.alt_first]], true) || !close_block(b.hash[2], true)) return;
                break;
            }
            top--;
        }
    }
};

template <bool WRITE>
__global__ void __launch_bounds__(32) vm_kernel(const VmLaunch L) {
    const unsigned q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= L.count) return;
    const unsigned e = L.ids[q];
    if (e == VM_NO_EXECUTION) return;
    const VmInput in = L.in[e];
    const VmProgram &P = L.programs[in.program];
    Machine<WRITE ? M_WRITE : M_SHAPE> m(L);
    m.ta = L.tapes + L.tape_off[e];
    m.cap_a = L.cap[2 * e];
    m.tb = m.ta + m.cap_a;
    m.cap_b = L.cap[2 * e + 1];
    m.na = m.peak_a = in.n_a;
    m.nb = m.peak_b = in.n_b;
    for (unsigned long long i = 0; i < in.n_a; i++) m.ta[i] = L.data[in.a + i];
    for (unsigned long long i = 0; i < in.n_b; i++) m.tb[i] = L.data[in.b + i];
    const fe z = fe_small(0);
    m.set_sponge(z, z, z, z);
    for (int i = 0; i < 16; i++) m.ctx[i] = z;
    for (int i = 0; i < 8; i++) m.lp[i] = z;
    for (int i = 0; i < 32; i++) m.S[i] = (unsigned)i < in.n_pub ? L.data[in.pub + i] : z;
    m.depth = m.max_depth = in.n_pub;
    if (WRITE) {
        const VmOut o = L.outs[e];
        m.out = L.out + o.offset;
        m.length = o.length;
        m.ctx_out = o.ctx_out; m.loop_out = o.loop_out; m.stack_out = o.stack_out;
        m.commit_state();
    }
    m.run(P.root_first, P.root_count);
    VmResult &r = L.res[e];
    if (!m.failed()) {
        if (m.opc < 16) m.fail(VM_MIN_OPS);                                      // lib.rs:48-52
        else if (WRITE && !(fe_eq(m.sponge[0], P.hash[0]) && fe_eq(m.sponge[1], P.hash[1]))) m.fail(VM_HASH);    // lib.rs:55-59
    }
    // the write pass must retrace the shape pass (control flow never reads the sponge); anything else would mean the shape is wrong
    if (WRITE && !m.failed() && (m.step != r.steps || m.ctx_cols != r.ctx_cols || m.loop_cols != r.loop_cols || m.max_depth != r.max_depth))
        m.fail(VM_DIVERGED);
    r.code = m.code;
    r.fail_step = m.fail_step;
    if (WRITE) return;
    r.steps = m.step;
    r.op_count = m.opc;
    r.peak_a = m.peak_a;
    r.peak_b = m.peak_b;
    r.ctx_cols = m.ctx_cols;
    r.loop_cols = m.loop_cols;
    r.max_depth = m.max_depth;
    for (int i = 0; i < 8; i++) r.top[i] = m.S[i];
}

// Machine::finalize: rows after the last step repeat it (the op counter, sponge, stacks), and the op bits are 1 from the last step on.
// One thread per (row, column, execution); executions that failed are left alone.
__global__ void vm_pad_kernel(fe *out, const VmResult *res, const unsigned *ids, unsigned width, unsigned long long length) {
    const unsigned long long row = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned col = blockIdx.y, q = blockIdx.z;
    const VmResult &r = res[ids[q]];
    if (row >= length || r.code != VM_OK) return;
    fe *c = out + ((size_t)q * width + col) * length;
    const bool op_bit = col >= 5 && col < 15;
    if (op_bit ? row < r.steps : row <= r.steps) return;
    c[row] = op_bit ? fe_small(1) : c[r.steps];
}

// ---- one execution from the sponge table ------------------------------------------------------------------------------------------------
// One thread per chain of a level (vm.h): the rounds of Machine<M_WRITE>, each at the cycle position its step has (every flow op is aligned
// to the 16-step cycle, so a step's round constants depend only on its place in its frame).  A child's end_block state is [h, x, y, 0]
// with h the state before the child: a group's x is its body's result; a switch's (x, y) are its two branch hashes and a loop's its body
// and skip hashes, which every path through the block must reproduce -- the item's program's bad word is set where one does not, or
// where a loop body does not end on its image.  The items of a launch may belong to any programs of the call.
__global__ void __launch_bounds__(64) vm_table_kernel(const VmLaunch L, const VmChainItem *items, unsigned count, const VmChainRef *chains,
                                                      VmSponge *tab, unsigned *bad) {
    const unsigned q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= count) return;
    const VmChainItem it = items[q];
    const fe z = fe_small(0);
    unsigned long long pos = it.out;
    fe s[4];
    auto put = [&] {
        for (int i = 0; i < 4; i++) tab[pos].s[i] = s[i];
        pos++;
    };
    auto span = [&](const VmBlock &b) {
        for (unsigned i = 0; i < b.count; i++) {
            const VmHint &h = L.hints[b.first + i];
            sponge_round(s, L.ops[b.first + i], h.kind == H_PUSH ? h.value : z, i);
            put();
        }
    };
    auto noop = [&](unsigned cycle) { sponge_round(s, OP_NOOP, z, cycle); put(); };
    if (it.kind == VM_CHAIN_BREAK) {                 // from the body's last state: the skip's first span, then close_block's NOOP
        const VmBlock &b = L.blocks[it.block];
        const VmSponge &last = tab[chains[it.block].main_close - 1];
        for (int i = 0; i < 4; i++) s[i] = last.s[i];
        span(L.blocks[L.children[b.alt_first]]);
        noop(15);
        return;
    }
    for (int i = 0; i < 4; i++) s[i] = z;
    bool ok = true;
    for (unsigned k = 0; k < it.count; k++) {
        const unsigned bi = L.children[it.first + k];
        const VmBlock &b = L.blocks[bi];
        if (b.kind == DG_BLOCK_SPAN) {
            if (k > 0) noop(15);
            span(b);
            continue;
        }
        const VmChainRef r = chains[bi];
        if (b.kind == DG_BLOCK_GROUP) {
            s[1] = tab[r.main_close].s[0];
            s[2] = z;
        } else if (b.kind == DG_BLOCK_SWITCH) {
            ok = ok && fe_eq(tab[r.main_close].s[0], b.hash[0]) && fe_eq(tab[r.alt_close].s[0], b.hash[1]);
            s[1] = b.hash[0];
            s[2] = b.hash[1];
        } else {
            ok = ok && fe_eq(tab[r.main_close - 1].s[0], b.hash[0]) && fe_eq(tab[r.brk_close].s[0], b.hash[1]) &&
                 fe_eq(tab[r.alt_close].s[0], b.hash[2]);
            s[1] = b.hash[1];
            s[2] = b.hash[2];
        }
        s[3] = z;
        put();
        for (unsigned i = 1; i <= 14; i++) noop(i);
    }
    noop(15);
    if (it.tail) {                                   // the root's close_block(0, true): [ctx 0 = 0, root result, 0, 0], then 14 NOOPs
        s[1] = s[0];
        s[0] = s[2] = s[3] = z;
        put();
        for (unsigned i = 1; i <= 14; i++) noop(i);
    }
    if (!ok) atomicOr(bad + it.program, 1u);
}

// the start of execution e, as vm_kernel sets it up
template <int MODE>
__device__ void start(Machine<MODE> &m, const VmLaunch &L, const VmInput &in, unsigned e) {
    m.ta = L.tapes + L.tape_off[e];
    m.cap_a = L.cap[2 * e];
    m.tb = m.ta + m.cap_a;
    m.cap_b = L.cap[2 * e + 1];
    m.na = m.peak_a = in.n_a;
    m.nb = m.peak_b = in.n_b;
    for (unsigned long long i = 0; i < in.n_a; i++) m.ta[i] = L.data[in.a + i];
    for (unsigned long long i = 0; i < in.n_b; i++) m.tb[i] = L.data[in.b + i];
    const fe z = fe_small(0);
    m.set_sponge(z, z, z, z);
    for (int i = 0; i < 16; i++) m.ctx[i] = z;
    for (int i = 0; i < 8; i++) m.lp[i] = z;
    for (int i = 0; i < 32; i++) m.S[i] = (unsigned)i < in.n_pub ? L.data[in.pub + i] : z;
    m.depth = m.max_depth = in.n_pub;
}

// The sequential pass of every execution L.ids[q], one per lane: the write pass's checks, codes and steps, the sponge from the tables, no
// register writes; VmResult as the shape pass fills it, the checkpoints and the read log in T[e], their counts in out[e]
__global__ void __launch_bounds__(32) vm_sequential_kernel(const VmLaunch L, const VmTables G, const VmTabled *T, VmSequential *out) {
    const unsigned q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= L.count) return;
    const unsigned e = L.ids[q];
    if (e == VM_NO_EXECUTION) return;
    const VmInput in = L.in[e];
    const VmProgram &P = L.programs[in.program];
    const VmTabled t = T[e];
    Machine<M_SEQUENTIAL> m(L);
    start(m, L, in, e);
    m.tab = G.tab; m.chains = G.chains; m.at = t.root; m.parent_at = 0;
    m.log = t.log; m.lpos = 0; m.lcap = t.log_cap;
    m.cp = (VmCheckpoint *)t.checkpoints; m.ncp = 0; m.cp_cap = t.cp_cap; m.next_cp = 0; m.seg = G.segment_steps;
    m.run(P.root_first, P.root_count);
    if (!m.failed()) {
        if (m.opc < 16) m.fail(VM_MIN_OPS);
        else if (!(fe_eq(m.sponge[0], P.hash[0]) && fe_eq(m.sponge[1], P.hash[1]))) m.fail(VM_HASH);
    }
    VmResult &r = L.res[e];
    r.code = m.code;
    r.fail_step = m.fail_step;
    r.steps = m.step;
    r.op_count = m.opc;
    r.peak_a = m.peak_a;
    r.peak_b = m.peak_b;
    r.ctx_cols = m.ctx_cols;
    r.loop_cols = m.loop_cols;
    r.max_depth = m.max_depth;
    for (int i = 0; i < 8; i++) r.top[i] = m.S[i];
    out[e].checkpoints = m.ncp;
    out[e].logged = m.lpos;
}

// Global segment g is segment q of execution e = execs[j] (first[j] <= g < first[j + 1]): from its checkpoint q to the first frame-loop
// boundary at or after checkpoint q + 1's step (its last segment to the end), rows written as the write pass writes them (segment 0 also
// row 0); codes[2g] = VM_OK, VM_SEGMENT when it does not end in the recorded state, or the failure it met (both internal errors: the
// sequential pass ran the same execution to the end), and codes[2g + 1] the step it stopped at
__global__ void __launch_bounds__(32) vm_segment_kernel(const VmLaunch L, const VmTables G, const VmTabled *T, const unsigned *execs,
                                                        const unsigned long long *first, unsigned n, unsigned long long segments,
                                                        unsigned long long *codes) {
    const unsigned long long g = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= segments) return;
    unsigned lo = 0, hi = n;                          // the last j with first[j] <= g
    while (hi - lo > 1) {
        const unsigned mid = (lo + hi) / 2;
        if (first[mid] <= g) lo = mid; else hi = mid;
    }
    const unsigned e = execs[lo];
    const unsigned long long q = g - first[lo], count = first[lo + 1] - first[lo];
    const VmTabled t = T[e];
    const VmCheckpoint *cp = (const VmCheckpoint *)t.checkpoints;
    Machine<M_SEGMENT> m(L);
    m.ta = m.tb = nullptr;
    m.cap_a = m.cap_b = ~0ULL;
    m.peak_a = m.peak_b = 0;
    m.tab = G.tab; m.chains = G.chains; m.log = t.log;
    m.expect = cp + q + 1;
    m.stop = q + 1 < count ? cp[q + 1].step : ~0ULL;
    m.load(cp[q]);
    const VmOut o = L.outs[e];
    m.out = L.out + o.offset;
    m.length = o.length;
    m.ctx_out = o.ctx_out; m.loop_out = o.loop_out; m.stack_out = o.stack_out;
    if (q == 0) m.commit_state();
    m.run(0, 0);
    codes[2 * g] = m.code;
    codes[2 * g + 1] = m.fail_step;
}

}  // namespace

size_t vm_checkpoint_bytes() { return sizeof(VmCheckpoint); }

void vm_table_level(Context &c, const VmLaunch &L, const VmChainItem *items, unsigned count, const VmChainRef *chains, VmSponge *tab,
                    unsigned *bad) {
    if (count == 0) return;
    vm_upload_constants(c);
    vm_table_kernel<<<(count + 63) / 64, 64, 0, c.stream>>>(L, items, count, chains, tab, bad);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

void vm_sequential_pass(Context &c, const VmLaunch &L, const VmTables &G, const VmTabled *T, VmSequential *out) {
    if (L.count == 0) return;
    vm_upload_constants(c);            // RESCR's hasher round
    vm_sequential_kernel<<<(L.count + 31) / 32, 32, 0, c.stream>>>(L, G, T, out);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

void vm_segment_pass(Context &c, const VmLaunch &L, const VmTables &G, const VmTabled *T, const unsigned *execs, const unsigned long long *first,
                     unsigned n, unsigned long long segments, unsigned long long *codes) {
    if (segments == 0) return;
    vm_upload_constants(c);
    vm_segment_kernel<<<(unsigned)((segments + 31) / 32), 32, 0, c.stream>>>(L, G, T, execs, first, n, segments, codes);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

void vm_shape_pass(Context &c, const VmLaunch &L) {
    if (L.count == 0) return;
    vm_upload_constants(c);            // RESCR's hasher round runs in this pass too
    vm_kernel<false><<<(L.count + 31) / 32, 32, 0, c.stream>>>(L);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

void vm_write_pass(Context &c, const VmLaunch &L) {
    if (L.count == 0) return;
    vm_upload_constants(c);
    vm_kernel<true><<<(L.count + 31) / 32, 32, 0, c.stream>>>(L);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

void vm_pad_rows(Context &c, fe *out, const VmResult *res, const unsigned *ids, unsigned count, unsigned width, unsigned long long length) {
    if (count == 0) return;
    DG_REQUIRE(count <= 65535 && width <= 65535, "too many executions or registers for one padding launch");
    vm_pad_kernel<<<dim3((unsigned)((length + 255) / 256), width, count), 256, 0, c.stream>>>(out, res, ids, width, length);
    c.launches++;
    DG_CUDA(cudaGetLastError());
}

}  // namespace dg
