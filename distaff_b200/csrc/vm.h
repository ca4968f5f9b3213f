// The VM interpreter (vm.cu) and what the host orchestration of dg_trace_batch / dg_execute_batch (execute.cu) passes to it.
#pragma once
#include "../../include/distaff_gpu.h"
#include "common.cuh"

namespace dg {

// the program encoding of dg_program_t in device form (field elements aligned for the device)
struct VmHint { unsigned kind, n; fe value; };
struct VmBlock { unsigned kind, first, count, alt_first, alt_count, pad[3]; fe hash[3]; };

// per execution: public inputs at data[pub], tape A (reversed: its first element last) at data[a], tape B (reversed) at data[b]
struct VmInput { unsigned long long pub, a, b, n_a, n_b; unsigned n_pub, pad; };

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

// what a pass reports per execution (indexed by execution)
struct VmResult {
    unsigned long long steps, fail_step, peak_a, peak_b, op_count;
    unsigned code, ctx_cols, loop_cols, max_depth;
    fe top[8];                            // the stack's top 8 slots at the last step (zero below the depth)
};

struct VmLaunch {
    const uint8_t *ops; const VmHint *hints; const VmBlock *blocks; const unsigned *children;
    unsigned root_first, root_count;
    fe hash[2];                           // Program::hash()
    const VmInput *in; const fe *data;
    fe *tapes;                            // per execution: tape A at tapes + tape_off[e] (cap[2e] elements), tape B after it (cap[2e + 1])
    const unsigned long long *tape_off, *cap;
    const unsigned *ids;                  // the executions of this launch
    unsigned count;
    unsigned long long max_steps;
    VmResult *res;
    // write pass: execution ids[q] into out + q * width * length, columns of one shape
    fe *out;
    unsigned long long length;
    unsigned width, ctx_out, loop_out, stack_out;
};

void vm_upload_constants(Context &c);
void vm_shape_pass(Context &c, const VmLaunch &L);
void vm_write_pass(Context &c, const VmLaunch &L);     // the write pass, then the padding rows
std::string vm_message(unsigned code, unsigned long long step, unsigned long long max_steps);

}  // namespace dg
