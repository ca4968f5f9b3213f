// The VM interpreter (vm.cu) and what the host orchestration of the execution calls (execute.cu) passes to it.
#pragma once
#include "../../include/distaff_gpu.h"
#include "common.cuh"

namespace dg {

// the program encoding of dg_program_t in device form (field elements aligned for the device)
struct VmHint { unsigned kind, n; fe value; };
struct VmBlock { unsigned kind, first, count, alt_first, alt_count, pad[3]; fe hash[3]; };

// The programs of a call share the ops / hints / blocks / children tables (their ranges rebased on the host); per program only the root
// body and Program::hash() differ
struct VmProgram { unsigned root_first, root_count; fe hash[2]; };

// per execution: public inputs at data[pub], tape A (reversed: its first element last) at data[a], tape B (reversed) at data[b], and the
// index of its program in VmLaunch::programs
struct VmInput { unsigned long long pub, a, b, n_a, n_b; unsigned n_pub, program; };

// write pass, per execution: its registers at VmLaunch::out + offset, `width` columns of `length` rows, of which the context, loop and
// stack columns number ctx_out, loop_out and stack_out
struct VmOut { unsigned long long offset, length; unsigned width, ctx_out, loop_out, stack_out; };

// launch slots that run no execution (the lanes after a program's last execution in its last warp)
constexpr unsigned VM_NO_EXECUTION = 0xffffffffu;

// Why an execution stopped.  Codes below VM_NO_STEP are the VM's own failures, reported as "<message> at step <fail_step>" (hostvm's
// Machine::fail); the others carry no step.  VM_TAPE_SCRATCH is internal: the shape pass ran out of tape scratch and is repeated with more.
enum VmCode : unsigned {
    VM_OK = 0, VM_ASSERT, VM_ASSERTEQ, VM_STACK_UNDERFLOW, VM_STACK_OVERFLOW, VM_PUSH_VALUE, VM_EMPTY_TAPE_A, VM_HINT_READ, VM_PMPATH_TAPES,
    VM_EMPTY_TAPE, VM_HINT_READ2, VM_CHOOSE, VM_CHOOSE2, VM_CSWAP2, VM_INV_ZERO, VM_NOT, VM_AND, VM_OR, VM_EQ_AUX, VM_HINT_CMP, VM_BINARY,
    VM_CMP_POW2, VM_HINT_BINACC, VM_BINACC_POW2, VM_UNKNOWN_OP, VM_OPVALUE, VM_PUSH_ALIGN, VM_CTX_OVERFLOW, VM_CTX_UNDERFLOW, VM_LOOP_OVERFLOW,
    VM_LOOP_UNDERFLOW, VM_START_ALIGN, VM_END_ALIGN, VM_LOOP_ALIGN, VM_WRAP_ALIGN, VM_BREAK_ALIGN, VM_LOOP_IMAGE, VM_SWITCH_COND, VM_LOOP_EXIT_COND,
    VM_LOOP_ENTER_COND,
    VM_NO_STEP, VM_CAP = VM_NO_STEP, VM_MIN_OPS, VM_HASH, VM_TAPE_SCRATCH,
    VM_DIVERGED,                          // the write pass did not retrace the shape pass (a guard: control flow never reads the sponge)
};
// the segment pass's guard, beside the VM's codes: a trace segment did not end in the state the sequential pass recorded
constexpr unsigned VM_SEGMENT = VM_DIVERGED + 1;

// what a pass reports per execution (indexed by execution)
struct VmResult {
    unsigned long long steps, fail_step, peak_a, peak_b, op_count;
    unsigned code, ctx_cols, loop_cols, max_depth;
    fe top[8];                            // the stack's top 8 slots at the last step (zero below the depth)
};

struct VmLaunch {
    const uint8_t *ops; const VmHint *hints; const VmBlock *blocks; const unsigned *children;
    const VmProgram *programs;
    const VmInput *in; const fe *data;
    fe *tapes;                            // per execution: tape A at tapes + tape_off[e] (cap[2e] elements), tape B after it (cap[2e + 1])
    const unsigned long long *tape_off, *cap;
    const unsigned *ids;                  // the executions of this launch: each program's from a multiple of 32, VM_NO_EXECUTION between
    unsigned count;
    unsigned long long max_steps;
    VmResult *res;
    // write pass: execution e into out + outs[e].offset, with its own shape
    fe *out;
    const VmOut *outs;
};

// ---- executions from sponge tables (dg_trace_many / dg_execute_many; dg_trace_one / dg_execute_one) ------------------------------------
// The sponge never reads data: with hashes that match their blocks, the state after every step of a block list's frame is a function of
// the program.  The table holds, per block list, its chain -- the state after each step its frame owns: the span ops, the NOOP before a
// non-first span, per child block end_block and the 14 NOOPs after it, then the NOOP close_block runs inside the list -- and, per loop,
// the chain after BREAK (the skip's first span and its closing NOOP, from the body's last state).  The root list's chain continues with
// the root's end_block and 14 NOOPs.  Every program of a call has its chains in one table, indexed through the rebased block tables.
struct VmSponge { fe s[4]; };
// where the chains of a group / switch / loop block start (main: body or true branch; alt: false branch or skip; brk: after BREAK), and the
// index of their closing entries
struct VmChainRef { unsigned long long main, alt, brk, main_close, alt_close, brk_close; };
// one chain to compute: a block list (children[first .. first + count), `tail`: the root's end_block and NOOPs follow its closing NOOP) or
// the chain after BREAK of loop `block`, of program `program`; written from table index `out` on
enum : unsigned { VM_CHAIN_LIST, VM_CHAIN_BREAK };
struct VmChainItem { unsigned kind, first, count, block, tail, program; unsigned long long out; };

// the tables of a call: the chains of every tabled program, the chain references per block, and the segment length S
struct VmTables {
    const VmSponge *tab;
    const VmChainRef *chains;             // per block (spans unused)
    unsigned long long segment_steps;
};
// per execution of the tabled passes
struct VmTabled {
    unsigned long long root;              // where its program's root list chain starts
    fe *log;                              // every value popped from tape A or B, in order
    unsigned long long log_cap;
    void *checkpoints;                    // vm_checkpoint_bytes() each
    unsigned long long cp_cap;
};
// what the sequential pass reports per execution beside VmResult: the checkpoints it recorded (the final state after them: cp_cap must
// exceed this count) and the values it logged (log_cap must reach it); a pass whose buffers were too small reports the sizes it needed
struct VmSequential { unsigned long long checkpoints, logged; };

// one launch per level: every item of a level reads only chains of lower levels; inconsistent hashes set bad[item.program]
void vm_table_level(Context &c, const VmLaunch &L, const VmChainItem *items, unsigned count, const VmChainRef *chains, VmSponge *tab,
                    unsigned *bad);
// every execution L.ids[q] on its lane, sponge from the tables: VmResult as the write pass reports it, T[e]'s checkpoints and read log,
// and out[e]
void vm_sequential_pass(Context &c, const VmLaunch &L, const VmTables &G, const VmTabled *T, VmSequential *out);
// one thread per segment, one segment per checkpoint, for the executions execs[0 .. n): execs[j]'s segments are the global indices
// first[j] .. first[j + 1) (first[n] = segments).  Its segment q replays from checkpoint q to checkpoint q + 1 (the last one to the final
// state) and writes its rows into L.outs[execs[j]] as the write pass does; codes[2g] = VM_OK or why global segment g stopped,
// codes[2g + 1] where
void vm_segment_pass(Context &c, const VmLaunch &L, const VmTables &G, const VmTabled *T, const unsigned *execs, const unsigned long long *first,
                     unsigned n, unsigned long long segments, unsigned long long *codes);
size_t vm_checkpoint_bytes();

void vm_upload_constants(Context &c);
void vm_shape_pass(Context &c, const VmLaunch &L);
void vm_write_pass(Context &c, const VmLaunch &L);
// the padding rows of `count` executions of one shape, ids[q]'s registers at out + q * width * length (after the write pass)
void vm_pad_rows(Context &c, fe *out, const VmResult *res, const unsigned *ids, unsigned count, unsigned width, unsigned long long length);
std::string vm_message(unsigned code, unsigned long long step, unsigned long long max_steps);

}  // namespace dg
