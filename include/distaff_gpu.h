/* distaff_gpu.h -- C-ABI of the H100 (sm_90a) STARK prover backend for Distaff.
 *
 * The reference has no FFI seam; the seam this library replaces is the single call
 *     stark::prove(&mut trace, inputs, outputs, options) -> StarkProof
 * at /root/reference/src/lib.rs:62  (definition: /root/reference/src/stark/prover.rs:17-169).
 * INTEGRATION.md shows the Rust binding (extern "C" block + replacement body of prover.rs::prove).
 *
 * Conventions
 *   - field elements are 16 little-endian bytes (a Rust u128, /root/reference/src/utils/mod.rs:35-41), canonical < M;
 *   - digests are 32 bytes; all sizes are in elements unless a name says bytes;
 *   - every function returns 0 on success and a negative code on failure; dg_last_error() describes the failure;
 *     nothing unwinds across the boundary;  there is NO CPU fallback: without a CUDA device every call fails with -3;
 *   - the caller owns input buffers (read-only for the duration of the call) and output buffers it passes in;
 *     objects returned through dg_proof_t** are owned by the library until dg_proof_free();
 *   - calls are serialised internally (one context per process, one device: $DG_DEVICE or dg_init()).
 */
#ifndef DISTAFF_GPU_H
#define DISTAFF_GPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DG_OK 0
#define DG_ERR_INVALID (-1)      /* bad argument (mirrors the reference's assert!s, e.g. trace_table.rs:23-58, options.rs:29-50) */
#define DG_ERR_CUDA (-2)         /* CUDA runtime failure */
#define DG_ERR_NO_DEVICE (-3)    /* no CUDA device: this backend has no CPU path */
#define DG_ERR_EXHAUSTED (-4)    /* PoW / query-position search exhausted (utils/mod.rs:39-41 panics in the reference) */
#define DG_ERR_UNSATISFIED (-5)  /* transition constraints do not vanish on the trace (evaluator.rs:152-157 panics) */
#define DG_ERR_REJECTED (-6)     /* dg_verify: the proof was rejected; the message is the reference's Err(String) (verifier.rs:28-73) */

/* ---- lifecycle ------------------------------------------------------------------------------------------------- */
int dg_init(int device);                     /* optional; device < 0 = $DG_DEVICE or 0; an error if the library already runs on another device */
/* Single-process multi-GPU: after dg_init_devices(n) (n = 1, 2, 4 or 8; devices 0 .. n-1) ONE call of dg_prove / dg_prove_device from one
 * host thread shards the proof over the n GPUs -- the library runs one internal host thread and one NCCL communicator per device -- and
 * returns the same bytes as the single-GPU call.  This is the mode the seam at lib.rs:62 (one synchronous call in one process) needs;
 * the one-process-per-GPU mode (dg_comm_init below) remains for hosts that already run one rank per GPU. */
int dg_init_devices(int n_devices);
const char *dg_last_error(void);             /* thread-local message of the last failing call */
int dg_device_info(char *name, size_t cap, int *sm_count, size_t *total_mem);

/* ---- the hot path: replaces stark::prove (prover.rs:17) ----------------------------------------------------------- */
typedef struct {
    const uint8_t *const *columns; /* width pointers, each to length*16 bytes: register traces, column-major (trace_table.rs:10) */
    uint32_t width;                /* 15 + ctx_depth + loop_depth + stack_depth (trace_state.rs:115-118)                    */
    uint64_t length;               /* trace length n, power of two >= 16                                                    */
    uint32_t ctx_depth, loop_depth;/* as returned by processor::execute (processor/mod.rs:23-46)                            */
} dg_trace_t;

typedef struct {                   /* ProofOptions (options.rs:16-23) */
    uint32_t extension_factor;     /* 16..256, power of two (default 32) */
    uint32_t num_queries;          /* 1..128 (default 50)                */
    uint32_t grinding_factor;      /* 0..32 (default 20)                 */
    uint32_t hash_id;              /* 0 = blake3 (the only serialisable hash, options.rs:107) */
} dg_options_t;

typedef struct dg_proof dg_proof_t;

typedef struct {                   /* per-stage device time in ms, the nine steps of prover.rs:19-167 */
    float stage_ms[9];
    float h2d_ms, total_ms;
    uint64_t kernel_launches;
} dg_prove_stats_t;

int dg_prove(const dg_trace_t *trace, const uint8_t *inputs16, uint32_t n_inputs, const uint8_t *outputs16, uint32_t n_outputs,
             const dg_options_t *options, dg_proof_t **proof_out, dg_prove_stats_t *stats /* may be NULL */);
/* same, with the register traces already resident in device memory: one allocation of width*length*16 bytes, column-major */
int dg_prove_device(const void *d_registers, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth,
                    const uint8_t *inputs16, uint32_t n_inputs, const uint8_t *outputs16, uint32_t n_outputs,
                    const dg_options_t *options, dg_proof_t **proof_out, dg_prove_stats_t *stats);

/* Batched proving: `count` traces of ONE shape (same width, length, ctx_depth, loop_depth) proven with the same options in one call; every
 * stage runs once over the whole batch, and every host round trip carries the values of all its proofs.  Public inputs / outputs are
 * per trace (inputs16[i] holds n_inputs[i] elements; the arrays may be NULL when every count is 0).  Per trace: status[i] = DG_OK and
 * proofs_out[i] a proof byte-identical to dg_prove of that trace, or a per-trace failure (DG_ERR_UNSATISFIED, DG_ERR_EXHAUSTED) with
 * proofs_out[i] = NULL; a failing trace does not change any other trace's proof.  Returns DG_OK when the batch ran (even if some traces
 * failed), otherwise the error of the whole call (DG_ERR_INVALID for count == 0, mixed shapes, bad options or a context that spans
 * several GPUs; DG_ERR_CUDA; DG_ERR_NO_DEVICE); on such an error every proofs_out[i] is NULL (nothing to free).  The library splits the
 * batch into groups that fit in device memory and in one launch ($DG_BATCH_GROUP caps the group size further); stats (may be NULL)
 * covers the whole batch.  dg_batch_message(i, ...) copies (NUL-terminated, truncated to message_cap) the message of entry i of the
 * calling thread's last batched call, dg_prove_batch, dg_prove_batch_device, dg_verify_batch, dg_trace_batch, dg_execute_batch,
 * dg_trace_programs, dg_execute_programs, dg_trace_many, dg_execute_many, dg_merkle_verify_paths or dg_merkle_verify_batch: why
 * trace i failed (the message dg_prove gives for that trace), why proof i was not accepted (what dg_verify reports for that proof),
 * why execution i failed, or why path / batch proof i was not accepted, and "" if it was proven / accepted / executed. */
int dg_prove_batch(const dg_trace_t *traces, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                   const uint8_t *const *outputs16, const uint32_t *n_outputs, const dg_options_t *options, dg_proof_t **proofs_out,
                   int *status, dg_prove_stats_t *stats);
/* same, registers already in device memory: one allocation, proof-major [count][width][length] elements */
int dg_prove_batch_device(const void *d_registers, uint32_t count, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth,
                          const uint8_t *const *inputs16, const uint32_t *n_inputs, const uint8_t *const *outputs16, const uint32_t *n_outputs,
                          const dg_options_t *options, dg_proof_t **proofs_out, int *status, dg_prove_stats_t *stats);
int dg_batch_message(uint32_t index, char *message, size_t message_cap);

/* Batched proving across register shapes: `count` traces of any widths, context / loop depths and lengths, proven with the same options in
 * one call.  Per trace the result is exactly dg_prove_batch's: status[i] = DG_OK and proofs_out[i] byte-identical to dg_prove of that
 * trace, or a per-trace DG_ERR_UNSATISFIED / DG_ERR_EXHAUSTED with its message in dg_batch_message(i); a failing trace changes no other
 * proof.  Every trace is checked on the host before the device is touched: a shape, length or public input / output count dg_prove would
 * reject fails the whole call with DG_ERR_INVALID and a message that starts with "trace i: ".  The call is partitioned by trace length;
 * the traces of one length run in groups that fit in device memory and in one launch ($DG_BATCH_GROUP caps them further), and every
 * stage of a group is launched once for all its traces, whatever their shapes, except the constraint evaluation, which is launched once
 * per register shape of the group.  RNG callbacks (dg_set_rng_callbacks) are called length by length, lengths in order of first
 * appearance; inside a length group by group and, in every group, stage by stage in input order.  A context that spans several GPUs is
 * rejected.  Returns and stats as dg_prove_batch. */
int dg_prove_traces(const dg_trace_t *traces, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                    const uint8_t *const *outputs16, const uint32_t *n_outputs, const dg_options_t *options, dg_proof_t **proofs_out,
                    int *status, dg_prove_stats_t *stats);
/* same, registers already in device memory: trace i's width[i] x length[i] elements, column-major, at d_registers[i] */
int dg_prove_traces_device(const void *const *d_registers, const uint32_t *width, const uint64_t *length, const uint32_t *ctx_depth,
                           const uint32_t *loop_depth, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                           const uint8_t *const *outputs16, const uint32_t *n_outputs, const dg_options_t *options, dg_proof_t **proofs_out,
                           int *status, dg_prove_stats_t *stats);
/* Per-trace options: dg_prove_traces / dg_prove_traces_device with `options` an array of `count` entries, trace i proven with options[i];
 * each proof is byte-identical to dg_prove of that trace with its options.  Every options[i] is checked on the host with the trace
 * (DG_ERR_INVALID, "trace i: " before dg_prove's message).  The call is partitioned by (trace length, extension factor), partitions in
 * order of first appearance; inside a partition the groups are cut as dg_prove_traces cuts a length, and the traces of one group may
 * differ in num_queries and grinding_factor (every stage is still one launch per group; the proof-of-work rounds run until the largest
 * grinding factor of the group is met, a proof leaving the rounds once it has its nonce).  RNG callbacks: partition by partition, inside a
 * partition as dg_prove_traces inside a length; with all options equal this is dg_prove_traces' order and result. */
int dg_prove_traces_with_options(const dg_trace_t *traces, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                                 const uint8_t *const *outputs16, const uint32_t *n_outputs, const dg_options_t *options, dg_proof_t **proofs_out,
                                 int *status, dg_prove_stats_t *stats);
int dg_prove_traces_device_with_options(const void *const *d_registers, const uint32_t *width, const uint64_t *length, const uint32_t *ctx_depth,
                                        const uint32_t *loop_depth, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                                        const uint8_t *const *outputs16, const uint32_t *n_outputs, const dg_options_t *options,
                                        dg_proof_t **proofs_out, int *status, dg_prove_stats_t *stats);

/* ---- checking a trace before proving it ------------------------------------------------------------------------------------------
 * dg_prove reports an unsatisfied trace late (after the trace LDE and commitment) and only with its lowest failing step; it does not check
 * the boundary constraints at all (a trace whose first or last row disagrees with the claimed inputs / outputs is proven, and the proof is
 * then rejected by the verifier).  dg_check_traces evaluates every transition constraint at every trace step in one GPU pass over the
 * registers and compares the first and last rows with the boundary assertions (evaluator.rs:181-326):
 *   first row: op counter, sponge, cf / ld / hd op bits, context and loop stacks all 0; user stack[i] = input i;
 *   last row:  cf / ld / hd op bits all 1, context and loop stacks 0; user stack[i] = output i.
 * It also reports what execute (lib.rs:48-60) asserts before proving: the last row's op counter (>= 16) and whether its sponge[0..2]
 * equals the program hash, when one is given.  Transition constraints are numbered in evaluation order, the order of
 * dg_eval_transitions' coefficients; dg_host_constraint_name names them.  The last step (n - 1 -> 0) is exempt, as in the prover.
 * No Fiat-Shamir value is drawn and the RNG callbacks are never called.  Same-shape traces only (as dg_prove_batch; same shape checks as
 * dg_prove), split into groups bounded by device memory, 65535 traces and $DG_BATCH_GROUP; one GPU (DG_ERR_INVALID for a context that
 * spans several). */
typedef struct {
    uint32_t n_constraints;                 /* T, evaluation order = dg_eval_transitions' coefficient order */
    uint64_t violating_steps, first_step;   /* transition violations over steps 0..n-2; first_step = UINT64_MAX if none */
    uint64_t constraint_steps[128];         /* per constraint: steps at which it does not vanish */
    uint64_t constraint_first[128];         /* per constraint: the lowest such step, UINT64_MAX if none */
    uint64_t first_row_registers[2];        /* bit r (of word r / 64): register r of the first row breaks a boundary assertion */
    uint64_t last_row_registers[2];         /* same, last row */
    uint64_t op_count;                      /* op counter of the last row (UINT64_MAX if it does not fit) */
    int32_t op_count_ok;                    /* 1 if that op counter is >= 16 (lib.rs:48-52), else 0 */
    int32_t program_hash_matches;           /* 1, 0, or -1 when no hash was given */
} dg_trace_report_t;
/* traces[i], inputs / outputs as in dg_prove_batch; program_hashes32: NULL or count * 32 bytes; reports: count entries; step_masks: NULL
 * or count * length * 3 words, bit j of word 3 k + j / 32 of trace i = constraint j does not vanish at step k.  Returns DG_OK when every
 * trace was checked, whatever the reports say. */
int dg_check_traces(const dg_trace_t *traces, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                    const uint8_t *const *outputs16, const uint32_t *n_outputs, const uint8_t *program_hashes32, dg_trace_report_t *reports,
                    uint32_t *step_masks);
/* same, registers already in device memory: proof-major [count][width][length] elements; d_step_masks: NULL or device memory */
int dg_check_traces_device(const void *d_registers, uint32_t count, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth,
                           const uint8_t *const *inputs16, const uint32_t *n_inputs, const uint8_t *const *outputs16, const uint32_t *n_outputs,
                           const uint8_t *program_hashes32, dg_trace_report_t *reports, uint32_t *d_step_masks);

/* ---- executing one program on many inputs --------------------------------------------------------------------------------------------
 * processor::execute (processor/mod.rs:23-182) of one compiled program for many ProgramInputs, one GPU thread per execution, and
 * distaff::execute (lib.rs:30-65) on top of it: every trace is proven from device memory where it was generated.  The library has no
 * assembler: the caller passes the compiled block tree of programs/blocks/mod.rs:30-60 in the flat encoding below, hashes included, so
 * the library never hashes program blocks on the host.  Every field can be read from the crate's public Program API (INTEGRATION.md
 * walks program.root() into a dg_program_t).  The encoding is validated on the host before any launch (indices in range, every span as
 * Span::new checks it, every block list as validate_block_list checks it, at most 15 nested blocks and 8 nested loops); a bad encoding
 * fails the call with DG_ERR_INVALID.  Hashes that do not match the blocks are not detected there: the execution then ends with
 * "program hash does not match trace hash" (or a loop image mismatch), as the host VM's does. */
#define DG_HINT_NONE 0           /* OpHint::None                                                    (processor/opcodes.rs:173-180) */
#define DG_HINT_PUSH 1           /* OpHint::PushValue(value16)                                                                       */
#define DG_HINT_EQ_START 2       /* OpHint::EqStart                                                                                  */
#define DG_HINT_RC_START 3       /* OpHint::RcStart(n)                                                                               */
#define DG_HINT_CMP_START 4      /* OpHint::CmpStart(n)                                                                              */
#define DG_HINT_PMPATH_START 5   /* OpHint::PmpathStart(n)                                                                           */
typedef struct {
    uint32_t kind;               /* DG_HINT_* */
    uint32_t n;                  /* RcStart / CmpStart / PmpathStart parameter, else 0 */
    uint8_t value16[16];         /* PushValue, else zero */
} dg_op_hint_t;

#define DG_BLOCK_SPAN 0          /* ProgramBlock::Span:   ops[first .. first + count), one hint per op (Span::op_codes / op_hints)       */
#define DG_BLOCK_GROUP 1         /* ProgramBlock::Group:  body = children[first .. first + count)  (Group::body)                         */
#define DG_BLOCK_SWITCH 2        /* ProgramBlock::Switch: true branch = children[first ..), false branch = children[alt_first ..)         */
#define DG_BLOCK_LOOP 3          /* ProgramBlock::Loop:   body = children[first ..), skip = children[alt_first ..)  (Loop::body / skip)   */
typedef struct {
    uint32_t kind;               /* DG_BLOCK_* */
    uint32_t first, count;       /* span: op range; group / switch / loop: child-list range (true branch, loop body) */
    uint32_t alt_first, alt_count;   /* switch: false branch; loop: skip; else 0 */
    /* hashes the VM needs when it closes the block (blocks/mod.rs:252-318); zero where not listed:
     *   switch: hash0 = true_branch_hash(), hash1 = false_branch_hash()
     *   loop:   hash0 = image(), hash1 = body_hash(), hash2 = skip_hash() */
    uint8_t hash0[16], hash1[16], hash2[16];
} dg_block_t;

typedef struct {                 /* Program (programs/mod.rs) */
    const uint8_t *ops;          /* op codes of every span, n_ops of them (OpCode as u8) */
    const dg_op_hint_t *hints;   /* one hint per op */
    uint64_t n_ops;
    const dg_block_t *blocks;
    uint32_t n_blocks;
    const uint32_t *children;    /* block indices; the child lists of groups, switches and loops and the root body are ranges of it */
    uint32_t n_children;
    uint32_t root_first, root_count;     /* the root Group's body: children[root_first .. root_first + root_count) */
    uint8_t hash32[32];          /* Program::hash() */
} dg_program_t;

/* ProgramInputs::new(public, secret_a, secret_b) (programs/inputs.rs:12).  Every value must be a field element, below M: a public input or
 * tape value in [M, 2^128) fails that execution (DG_ERR_EXECUTION, "public input 2 is not a field element", "tape A value 0 is not a
 * field element", "tape B value 5 ..."; the first one in that order), before it runs, and no other.  The reference accepts such values
 * and leaves what a program computes from them undefined (its field arithmetic assumes canonical operands). */
typedef struct {
    const uint8_t *public16; uint32_t n_public;      /* at most 8 (lib.rs:32), else the execution fails */
    const uint8_t *secret_a16; uint64_t n_secret_a;  /* tape A, read first to last */
    const uint8_t *secret_b16; uint64_t n_secret_b;  /* tape B, not longer than tape A, else the execution fails */
} dg_program_inputs_t;

typedef struct {                 /* the shape of one execution's trace, what execute reports beside it */
    uint32_t width;              /* 15 + ctx_depth + loop_depth + stack_depth */
    uint64_t length;             /* next power of two above the last step, at least 16 */
    uint64_t steps;              /* last step (operations executed) */
    uint32_t ctx_depth, loop_depth, stack_depth;
} dg_execution_info_t;

#define DG_ERR_EXECUTION (-7)    /* the program failed on these inputs (processor::execute / lib.rs:48-60 panic); message as the host VM's */

/* dg_trace_batch: executes the program for inputs[0 .. count): the shape pass, then the write pass in waves (as dg_trace_programs,
 * below).  Per execution: status[i] = DG_OK and info[i], or
 * DG_ERR_EXECUTION with dg_batch_message(i) = the VM's message ("ASSERT failed at step 17", ...; "execution exceeds N steps" when the
 * last step would reach max_steps, which bounds how long a program that never stops keeps the GPU busy).  registers_out: NULL (only the
 * shape pass runs, so that a caller can size its buffers first), or count pointers, each to info[i].width * info[i].length * 16 bytes
 * that receive the column-major registers of a successful execution (entries of failed executions may be NULL).  The shape pass does
 * not compute the sponge, so a shapes-only call reports DG_OK and the shape for the two failures that need it: "program hash does not
 * match trace hash" and "hash of the last iteration doesn't match loop image"; only a call with registers_out reports them.  The trace
 * length is the smallest power of two above the last step (16 at least: a last step of 2^k - 1 gives 2^k), and a last step that would
 * reach max_steps fails the execution: it succeeds with max_steps = last step + 1.  Returns DG_OK when the
 * batch ran, whatever the executions did; DG_ERR_INVALID for a bad encoding or a context that spans several GPUs. */
int dg_trace_batch(const dg_program_t *program, uint32_t count, const dg_program_inputs_t *inputs, uint64_t max_steps,
                   dg_execution_info_t *info, uint8_t *const *registers_out, int *status);
/* dg_execute_batch: dg_trace_batch, then every successful trace proven from the device memory it was generated in, with the same
 * options, grouped by shape and then by device memory ($DG_BATCH_GROUP and dg_set_memory_limit apply).  Per execution: status[i] =
 * DG_OK, proofs_out[i] byte-identical to dg_prove of the trace with the execution's public inputs and outputs, and the num_outputs
 * (<= 8) elements at outputs16 + 16 * num_outputs * i = the top of the last row's stack, zero below its depth (lib.rs:45-46); or a per-execution
 * failure (DG_ERR_EXECUTION, DG_ERR_UNSATISFIED, DG_ERR_EXHAUSTED) with its message in dg_batch_message(i) and proofs_out[i] = NULL.
 * A failing execution changes no other result.  stats (may be NULL) covers the proofs. */
int dg_execute_batch(const dg_program_t *program, uint32_t count, const dg_program_inputs_t *inputs, uint32_t num_outputs, uint64_t max_steps,
                     const dg_options_t *options, dg_proof_t **proofs_out, uint8_t *outputs16, int *status, dg_prove_stats_t *stats);

/* ---- executing many programs -------------------------------------------------------------------------------------------------------
 * dg_trace_programs / dg_execute_programs: dg_trace_batch / dg_execute_batch for executions of different programs in one call (those two
 * are the one-program case).  Execution i runs programs[program_of[i]] on inputs[i]; each program of the table is validated once, and a
 * bad one fails the call with DG_ERR_INVALID and "program p: " before the message when the table holds more than one.  Each program's
 * executions run in warps of their own.  After the shape pass the successful executions are written in waves: one write launch per
 * wave covers every trace shape in it; a wave's traces take at most half of the device memory the library may use (dg_set_memory_limit)
 * and leave room for one proof of the wave's largest shape; $DG_BATCH_GROUP caps the executions of a wave.  dg_execute_programs proves
 * each shape's traces of a wave together, whichever programs they came from, where they were written; the RNG callbacks run shape by
 * shape, in input order inside a shape.  Per execution, results and failures are as in dg_trace_batch / dg_execute_batch, with the
 * messages in dg_batch_message; num_outputs[i] (<= 8) is per execution and outputs16 holds 8 elements per execution (zero past
 * num_outputs[i], and all zero for an execution the VM failed; it may be NULL when every num_outputs[i] is 0).  Bad arguments
 * (n_programs == 0, program_of[i] >= n_programs, more than 2^32 ops in all, num_outputs[i] > 8, a bad encoding) are rejected before the device is touched; a context that spans several GPUs is
 * rejected.  vm_stats (may be NULL) describes the VM passes. */
typedef struct {
    uint32_t shape_launches;     /* shape-pass launches (more than one when an execution outgrows its tape scratch) */
    uint32_t write_launches;     /* write-pass launches, one per wave (each followed by one padding launch per shape) */
    uint32_t waves;
    uint32_t prove_groups;       /* prove groups of dg_execute_programs (0 for dg_trace_programs) */
    uint64_t lanes;              /* threads of the write launches, idle lanes included */
    float shape_ms, write_ms;    /* device time of the shape and write passes (padding included) */
} dg_execution_stats_t;
int dg_trace_programs(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                      const dg_program_inputs_t *inputs, uint64_t max_steps, dg_execution_info_t *info, uint8_t *const *registers_out,
                      int *status, dg_execution_stats_t *vm_stats);
int dg_execute_programs(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                        const dg_program_inputs_t *inputs, const uint32_t *num_outputs, uint64_t max_steps, const dg_options_t *options,
                        dg_proof_t **proofs_out, uint8_t *outputs16, int *status, dg_prove_stats_t *stats, dg_execution_stats_t *vm_stats);
/* dg_execute_programs with `options` an array of `count` entries: execution i is proven with options[i], exactly as dg_execute_programs of
 * it with those options alone.  Every options[i] is checked on the host before the device is touched (DG_ERR_INVALID, "execution i: "
 * before dg_prove's message).  A wave leaves room for one proof of its largest shape and extension factor.  Each shape's traces of a wave
 * are proven by one dg_prove_traces_with_options call: RNG callbacks shape by shape, inside a shape extension factor by extension factor
 * (in order of first appearance), in input order inside those. */
int dg_execute_programs_with_options(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                     const dg_program_inputs_t *inputs, const uint32_t *num_outputs, uint64_t max_steps, const dg_options_t *options,
                                     dg_proof_t **proofs_out, uint8_t *outputs16, int *status, dg_prove_stats_t *stats,
                                     dg_execution_stats_t *vm_stats);

/* ---- executing one long program -------------------------------------------------------------------------------------------------
 * dg_trace_one / dg_execute_one: one execution of one program, split across GPU threads.  The batch calls above run an execution on one
 * thread with the sponge, which costs one sponge round per step.  These calls use that the sponge never reads data: when the encoding's
 * switch and loop hashes match their bodies, the sponge state after every step of a block list is a function of the program, computed
 * once per call into a table (one launch per nesting level).  The execution then runs once on one thread with the sponge looked up
 * (every check, code and step of the batch path's write pass; at the first frame-loop boundary at or after every segment_steps steps it
 * records a checkpoint, and it logs every value read from the tapes), and one thread per checkpoint writes the rows up to the next one.
 * A straight-line program's table is as long as its trace, so it gains nothing.  An encoding whose hashes do not match on some path
 * through a switch or loop runs the batch path instead (dg_trace_batch with one input), so results are identical either way; stats say
 * which path ran.  segment_steps: 0 (the library chooses) or a power of two >= 16.  Arguments are validated as dg_trace_batch /
 * dg_execute_batch validate them (the encoding, num_outputs <= 8, one GPU) before any launch.  A failed execution returns
 * DG_ERR_EXECUTION with the message dg_batch_message would give (dg_last_error).
 * dg_trace_one: info receives the shape; registers_out: NULL (no rows are written) or info->width * info->length * 16 bytes, column-major.
 * Unlike dg_trace_batch's, a call without registers_out also reports the failures that need the sponge (program hash, loop image).
 * dg_execute_one: the trace is proven where it was written (dg_prove's bytes for the trace with the execution's public inputs and the
 * num_outputs elements of the last row's stack top, written to outputs16); prove_stats and info may be NULL. */
typedef struct {
    float table_ms, sequential_ms, segment_ms;   /* device time of the table, the sequential pass and the segment pass (with padding);
                                                    after the fallback, the batch path's shape and write passes */
    uint64_t table_rounds;       /* sponge rounds of the table */
    uint64_t table_entries;      /* states in the table */
    uint32_t table_levels;       /* table launches */
    uint32_t sequential_launches;/* more than one when the tape scratch, the read log or the checkpoint buffer needed more room */
    uint64_t checkpoints;        /* checkpoints recorded (one per segment) */
    uint64_t segments;
    uint64_t logged;             /* tape values logged */
    uint64_t segment_steps;      /* S used */
    int32_t fallback;            /* 1: the encoding's hashes are inconsistent and the batch path ran */
} dg_trace_one_stats_t;
int dg_trace_one(const dg_program_t *program, const dg_program_inputs_t *inputs, uint64_t max_steps, uint64_t segment_steps,
                 dg_execution_info_t *info, uint8_t *registers_out, dg_trace_one_stats_t *stats);
int dg_execute_one(const dg_program_t *program, const dg_program_inputs_t *inputs, uint32_t num_outputs, uint64_t max_steps,
                   uint64_t segment_steps, const dg_options_t *options, dg_proof_t **proof_out, uint8_t *outputs16, dg_execution_info_t *info,
                   dg_prove_stats_t *prove_stats, dg_trace_one_stats_t *stats);

/* ---- executing many long programs -----------------------------------------------------------------------------------------------
 * dg_trace_many / dg_execute_many: dg_trace_programs / dg_execute_programs with every execution run as dg_trace_one runs one (those two
 * are the one-execution case).  The programs' sponge tables are computed in one launch per nesting level for all of them; then one
 * sequential launch runs every execution, one warp each, and the rows are written in waves (cut as dg_trace_programs cuts them), one
 * segment launch per wave covering every checkpoint of every execution in it.  The tables live for the call.  A program whose hashes are
 * inconsistent has all its executions run on the batch path in the same call, before the tabled ones.  Per execution, status[i], info[i],
 * the message in dg_batch_message(i), the registers, the 8 elements of outputs16 (as dg_execute_programs) and the proof are exactly
 * those of dg_trace_programs / dg_execute_programs with registers_out; a failing execution changes no other result.
 * dg_trace_many without registers_out writes no rows, and still reports the failures that need the sponge (program hash, loop image),
 * as dg_trace_one does.  Bad arguments are rejected before the device is touched, as dg_execute_programs rejects them, and segment_steps
 * must be 0 (the library chooses) or a power of two >= 16; a context that spans several GPUs is rejected.
 * RNG callbacks (dg_execute_many): first the fallback executions' proofs, in dg_execute_programs' order; then wave by wave, in every wave
 * shape by shape (shapes ordered by width, length, context depth, loop depth) and in input order inside a shape. */
typedef struct {
    float table_ms, sequential_ms, segment_ms;    /* device time of the tables, the sequential launches and the segment launches (padding
                                                     included) of the tabled executions, all waves */
    uint64_t table_rounds, table_entries;         /* summed over the call's tabled programs */
    uint32_t table_levels;                        /* table launches */
    uint32_t tabled_programs, fallback_programs;  /* programs run from tables / on the batch path (inconsistent hashes) */
    uint32_t sequential_launches;                 /* more than one when an execution needed more tape scratch, read log or checkpoints */
    uint64_t checkpoints, segments, logged;       /* over the successful tabled executions: checkpoints recorded, segments, tape values logged */
    uint64_t segment_steps;                       /* S used */
    uint32_t waves;                               /* segment launches */
    uint32_t prove_groups;                        /* prove groups of the tabled executions (dg_execute_many) */
    dg_execution_stats_t fallback;                /* the batch path's figures for the fallback executions (zero if none) */
} dg_many_stats_t;
int dg_trace_many(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                  const dg_program_inputs_t *inputs, uint64_t max_steps, uint64_t segment_steps, dg_execution_info_t *info,
                  uint8_t *const *registers_out, int *status, dg_many_stats_t *stats);
int dg_execute_many(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                    const dg_program_inputs_t *inputs, const uint32_t *num_outputs, uint64_t max_steps, uint64_t segment_steps,
                    const dg_options_t *options, dg_proof_t **proofs_out, uint8_t *outputs16, int *status, dg_prove_stats_t *prove_stats,
                    dg_many_stats_t *stats);
/* dg_execute_many with `options` an array of `count` entries, as dg_execute_programs_with_options is to dg_execute_programs */
int dg_execute_many_with_options(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                 const dg_program_inputs_t *inputs, const uint32_t *num_outputs, uint64_t max_steps, uint64_t segment_steps,
                                 const dg_options_t *options, dg_proof_t **proofs_out, uint8_t *outputs16, int *status,
                                 dg_prove_stats_t *prove_stats, dg_many_stats_t *stats);

/* ---- program inputs in device memory -------------------------------------------------------------------------------------------------
 * ProgramInputs::new (programs/inputs.rs:12-26) of `count` executions whose values are all in one device buffer: execution i reads its
 * public inputs from d_values[public_first[i] .. + n_public[i]), tape A from d_values[secret_a_first[i] .. + n_secret_a[i]) and tape B
 * from d_values[secret_b_first[i] .. + n_secret_b[i]), each range in reading order (its first value is read first).  Ranges may overlap
 * or be shared between executions (one tape read by many of them): the values are only read.  d_values is device memory on the library's
 * device, 16-byte aligned, n_values field elements of 16 little-endian bytes; it may be NULL when every count is 0.  The six arrays are
 * host arrays of `count` entries each.  Writes to d_values must be complete (or ordered before the call on the library's stream). */
typedef struct {
    const void *d_values;
    uint64_t n_values;
    const uint64_t *public_first; const uint32_t *n_public;          /* at most 8 public inputs (lib.rs:32), else the execution fails */
    const uint64_t *secret_a_first; const uint64_t *n_secret_a;      /* tape A */
    const uint64_t *secret_b_first; const uint64_t *n_secret_b;      /* tape B, not longer than tape A, else the execution fails */
} dg_device_inputs_t;
/* dg_trace_programs, dg_execute_programs_with_options, dg_trace_many and dg_execute_many_with_options with `inputs` in device memory:
 * the same arguments, results, statuses, messages and stats, with the inputs of execution i given by the descriptor.  The execute forms
 * take one options entry per execution (a caller with one set of options replicates it).  Per execution the failures are exactly those of
 * the host form: more than 8 public inputs, tape A shorter than tape B, and the first value >= M in the order public inputs, tape A, tape B
 * ("tape A value 3 is not a field element", the index counted from the start of its range); each fails only its own execution.  Checked
 * on the host before the device is touched (DG_ERR_INVALID, also without a GPU): everything the host forms check, a NULL descriptor or
 * array ("null device inputs"), a NULL or unaligned d_values while any count is non-zero, and a range that overflows or ends past
 * n_values (named by execution and region).  d_values must be device memory (DG_ERR_INVALID otherwise).  One GPU only, as every
 * execution call.  The values are checked and packed for the VM by one kernel; only the public inputs (at most 8 per execution) and the
 * first bad index per region come back to the host. */
int dg_trace_programs_device_inputs(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                    const dg_device_inputs_t *inputs, uint64_t max_steps, dg_execution_info_t *info, uint8_t *const *registers_out,
                                    int *status, dg_execution_stats_t *vm_stats);
int dg_execute_programs_device_inputs(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                      const dg_device_inputs_t *inputs, const uint32_t *num_outputs, uint64_t max_steps, const dg_options_t *options,
                                      dg_proof_t **proofs_out, uint8_t *outputs16, int *status, dg_prove_stats_t *stats,
                                      dg_execution_stats_t *vm_stats);
int dg_trace_many_device_inputs(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                const dg_device_inputs_t *inputs, uint64_t max_steps, uint64_t segment_steps, dg_execution_info_t *info,
                                uint8_t *const *registers_out, int *status, dg_many_stats_t *stats);
int dg_execute_many_device_inputs(const dg_program_t *programs, uint32_t n_programs, uint32_t count, const uint32_t *program_of,
                                  const dg_device_inputs_t *inputs, const uint32_t *num_outputs, uint64_t max_steps, uint64_t segment_steps,
                                  const dg_options_t *options, dg_proof_t **proofs_out, uint8_t *outputs16, int *status,
                                  dg_prove_stats_t *prove_stats, dg_many_stats_t *stats);

/* ---- device memory ----------------------------------------------------------------------------------------------------------------
 * dg_set_memory_limit caps the device memory the library may hold on the current device: the per-proof arena, the stream-ordered pool it
 * allocates from otherwise, and its persistent tables.  0 (the default) means no limit.  The arena is never sized above the limit and the
 * pool keeps no more freed memory than the limit leaves beside the arena.  Every prove call is planned against the limit: a shape whose
 * whole trace extension (16 w n b bytes per proof) fits is proven as without a limit (the full layout); otherwise the prover extends and
 * hashes the extension a chunk of cosets at a time and keeps only the 8 cosets the constraint evaluation reads (the evaluation-coset
 * layout), computing the other opened rows from the trace polynomials.  Both layouts give the same proof bytes.  A call that does not fit
 * in either way fails with DG_ERR_INVALID and a message giving the bytes it needs.  dg_check_traces and dg_verify_batch size their groups
 * within the limit too.  The limit applies to one GPU: a context that spans several (dg_init_devices(n > 1), dg_comm_init) rejects it with
 * DG_ERR_INVALID.
 * dg_memory_usage: device bytes the library holds now (arena + the pool's reservation) and the most it has held since the limit was last
 * set.  dg_plan_prove: what a prove call of `count` traces of this shape would do, without running it.  All three return DG_ERR_NO_DEVICE
 * without a device. */
#define DG_LAYOUT_FULL 0            /* the whole trace extension is kept */
#define DG_LAYOUT_EVAL_COSETS 1     /* a chunk of cosets at a time; the 8 evaluation cosets are kept */
typedef struct {
    int32_t layout;                /* DG_LAYOUT_FULL or DG_LAYOUT_EVAL_COSETS */
    uint32_t group;                /* proofs per group of a batched call (1 for dg_prove) */
    uint32_t coset_chunk;          /* cosets of the trace extension extended at a time (= extension_factor in the full layout) */
    uint32_t retained_cosets;      /* cosets kept for the constraint evaluation and the openings: extension_factor or 8 */
    uint64_t bytes_per_proof;      /* device bytes of one proof of the group */
    uint64_t fixed_bytes;          /* bytes held outside the per-proof buffers: persistent tables, transform scratch, upload buffer */
    uint64_t available_bytes;      /* the budget the group was fitted into */
} dg_prove_plan_t;
int dg_set_memory_limit(size_t bytes);
int dg_memory_usage(size_t *held, size_t *peak);
int dg_plan_prove(uint32_t width, uint64_t length, uint32_t count, const dg_options_t *options, dg_prove_plan_t *plan);

/* Optional: randomness supplied by the host.  The prover derives all of its Fiat-Shamir challenges from two reference functions,
 *   field::prng_vector(seed, n)                            (math/field.rs:264-275: StdRng::from_seed + Uniform(0..M))
 *   utils::compute_query_positions(seed, domain, options)  (stark/utils/mod.rs:25-44: StdRng + Uniform(0..domain), rejections)
 * both built on rand 0.7.3, which is not part of the reference tree.  By default the library uses its own restatement of that
 * generator (ChaCha20, rand's widening-multiply rejection sampling); a Rust host can instead register callbacks that call the real
 * functions, so that no third-party semantics are reproduced on this side of the boundary.  Callbacks return 0 on success; they are
 * called 20-30 times per proof (once per commitment), one at a time: on the thread that calls dg_prove, and after dg_init_devices(n) also
 * from the library's per-device host threads (every rank derives the same challenges; the calls are serialised by a mutex).  draw_field writes `count` canonical field
 * elements (16 LE bytes each); draw_positions writes exactly num_queries distinct positions < domain_size, none a multiple of
 * extension_factor (anything else is rejected with DG_ERR_INVALID; a non-zero return maps to DG_ERR_EXHAUSTED like the reference's panic).
 * Passing NULL restores the built-in generator.  Process-wide; not to be changed while a proof is running. */
typedef struct {
    void *user;
    int (*draw_field)(void *user, const uint8_t seed[32], uint64_t count, uint8_t *out16);
    int (*draw_positions)(void *user, const uint8_t seed[32], uint64_t domain_size, uint32_t extension_factor, uint32_t num_queries,
                          uint64_t *out_positions);
} dg_rng_callbacks_t;
int dg_set_rng_callbacks(const dg_rng_callbacks_t *callbacks);

/* bincode 1.3.1 encoding of StarkProof (proof.rs:10-37), what main.rs:45 serialises */
int dg_proof_serialized_len(const dg_proof_t *proof, size_t *len);
int dg_proof_serialize(const dg_proof_t *proof, uint8_t *buf, size_t cap);
/* intermediate commitments, for differential tests: which = 0 trace root, 1 constraint root, 2 PoW seed */
int dg_proof_digest(const dg_proof_t *proof, int which, uint8_t out32[32]);
int dg_proof_pow_nonce(const dg_proof_t *proof, uint64_t *nonce);
void dg_proof_free(dg_proof_t *proof);

/* ---- the step after the path: stark::verify (verifier.rs:11-75) on the GPU -------------------------------------------------------
 * Checks StarkProof bytes (the bincode encoding dg_proof_serialize emits / main.rs:45 writes) against a program hash and public
 * inputs / outputs.  Returns DG_OK when the reference would return Ok(true); DG_ERR_REJECTED when it would return Err(msg), with msg
 * copied to `message` (NUL-terminated, truncated to message_cap) and available from dg_last_error(); DG_ERR_INVALID for bytes that do
 * not deserialize.  Hashing, Merkle batch verification, the constraint evaluation at z, the DEEP composition at the query positions
 * and the FRI row folds run on the device (verifier.cu); the Fiat-Shamir draws use the same generator / callbacks as dg_prove. */
int dg_verify(const uint8_t program_hash[32], const uint8_t *inputs16, uint32_t n_inputs, const uint8_t *outputs16, uint32_t n_outputs,
              const uint8_t *proof_bytes, size_t proof_len, char *message, size_t message_cap);

/* Batched verification: `count` proofs checked in one call, each verifier stage launched once for a group of proofs.  The proofs may
 * differ in anything: register shape, trace length, extension factor, query count, grinding factor.  Entry i is proof_bytes[i]
 * (proof_lens[i] bytes) against program_hashes[i] (32 bytes) and inputs16[i] / outputs16[i] (n_inputs[i] / n_outputs[i] elements; a
 * pointer may be NULL when its count is 0).  status[i] is exactly what dg_verify returns for that proof alone: DG_OK, DG_ERR_REJECTED
 * (the reference's Err string) or DG_ERR_INVALID (bytes that do not deserialize, a bad argument of that entry); dg_batch_message(i, ...)
 * gives its message, "" for an accepted proof.  A rejected or malformed proof changes no other proof's verdict.  The Fiat-Shamir draws
 * run on the calling thread, proof by proof in input order, so registered RNG callbacks see the concatenation of the calls dg_verify
 * makes for each proof.  Returns DG_OK when the batch ran, otherwise the error of the whole call with every status[i] unset:
 * DG_ERR_INVALID (count == 0, a NULL array), DG_ERR_CUDA, DG_ERR_NO_DEVICE.  Groups are bounded by a device-memory budget and by
 * $DG_BATCH_GROUP; stats (may be NULL) covers the whole call. */
typedef struct {
    float total_ms;                /* device time of the groups (upload to download) */
    uint64_t kernel_launches;
    uint32_t groups;               /* groups that ran on the device (proofs decided on the host take part in none) */
} dg_verify_stats_t;
int dg_verify_batch(uint32_t count, const uint8_t *const *program_hashes, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                    const uint8_t *const *outputs16, const uint32_t *n_outputs, const uint8_t *const *proof_bytes, const size_t *proof_lens,
                    int *status, dg_verify_stats_t *stats);

/* ---- building blocks (micro-benchmarks of BASELINE.json config 5; same kernels the prover uses) ---------------------- */
/* math::fft / polynom::{eval_fft, interpolate_fft} (polynom.rs:23-28,82-86): natural-order DFT of `batch` vectors of 2^log_n
 * elements, in place in host memory */
int dg_ntt(uint8_t *values, uint32_t log_n, uint32_t batch, int inverse);
/* TraceTable::extend (trace_table.rs:143-169) for `batch` columns: n values in, n*blowup evaluations out in LOGICAL order
 * (out[i] = P(w_N^i)), host memory */
int dg_lde(const uint8_t *values, uint8_t *extended, uint32_t log_n, uint32_t log_blowup, uint32_t batch);
/* crypto::build_merkle_nodes (merkle.rs:269-294) with blake3: n_leaves*32 bytes in, n_leaves*32 bytes of nodes out */
int dg_merkle_build(const uint8_t *leaves, uint64_t n_leaves, uint8_t *nodes);
/* TraceTable::build_merkle_tree leaf step (trace_table.rs:176-183): hashes the rows of a column-major width x rows matrix */
int dg_hash_rows(const uint8_t *columns, uint32_t width, uint64_t rows, uint8_t *digests);
/* utils::find_pow_nonce (proof_of_work.rs:4-32) */
int dg_find_pow_nonce(const uint8_t seed[32], uint32_t grinding_factor, uint64_t *nonce, uint8_t new_seed[32]);
/* crypto::hash::{blake3, rescue, poseidon} (hash.rs:119-177,205-209) over n independent 64-byte messages -> n 32-byte digests
 * (benches/hash.rs), and build_merkle_nodes (merkle.rs:269-294) with any of them.  hash: 0 blake3, 1 rescue, 2 poseidon -- ids of
 * THIS interface; a proof can only carry blake3 (options.rs:97-125).  Messages must hold valid field elements for 1 and 2 (field.rs:25).
 *
 * hash 3 is utils::hasher::digest (hasher.rs:12-40), the hash of the VM's RESCR op, so a tree built with it is one that the smpath /
 * pmpath operations of a program verify.  A message is 4 field elements (64 bytes, each a little-endian u128) and its digest 2 elements
 * (32 bytes); a message of 1-3 elements hashes as its zero-padded form.  A leaf is 2 elements, and the heap is nodes[L/2 + i] =
 * digest(leaf[2i] | leaf[2i+1]), nodes[i] = digest(nodes[2i] | nodes[2i+1]), nodes[1] the root, nodes[0] zero.  A tree of L = 2^d
 * leaves has the authentication paths of smpath.n / pmpath.n with n = d + 1, and 2 <= n <= 256 (so 2 <= L <= 2^255).  dg_hash64 and
 * dg_merkle_build_with reject a message or leaf element >= M (DG_ERR_INVALID, naming the first such message or leaf and its element);
 * dg_dev_merkle_build_with expects canonical leaves, as for 1 and 2.  Levels of fewer than 2^16 digests run a kernel that splits each
 * digest over 8 lanes, wider ones a thread per digest. */
#define DG_HASH_BLAKE3 0
#define DG_HASH_RESCUE 1
#define DG_HASH_POSEIDON 2
#define DG_HASH_HASHER 3
int dg_hash64(int hash, const uint8_t *messages64, uint64_t n, uint8_t *digests32);
int dg_merkle_build_with(int hash, const uint8_t *leaves, uint64_t n_leaves, uint8_t *nodes);

/* ---- Merkle trees that stay on the GPU (crypto::MerkleTree, merkle.rs:22-62, kept in device memory) ---------------------------------
 * A dg_tree_t holds L = 2^d leaves and the heap of dg_merkle_build_with (byte for byte) in device memory, on the library's primary device
 * and context; it is owned by the library until dg_tree_free().  Its two buffers (64 L bytes) come from the context's stream-ordered pool,
 * so dg_memory_usage counts a live tree and proofs that run beside it see that memory as taken.  Hash ids as for dg_merkle_build_with.
 * Without a CUDA device every entry point that takes leaves or a tree returns DG_ERR_NO_DEVICE. */
typedef struct dg_tree dg_tree_t;
/* builds a tree of n_leaves x 32 bytes of host leaves.  The checks of dg_merkle_build_with, with its messages, before the device is
 * touched: a hash id of 0-3, L a power of 2 >= 2, and for hash 3 every leaf element < M (the first bad leaf is named). */
int dg_tree_new(int hash, const uint8_t *leaves32, uint64_t n_leaves, dg_tree_t **tree);
/* the same from leaves in device memory, copied into the tree's own buffer; like dg_dev_merkle_build_with it expects canonical leaves */
int dg_tree_new_device(int hash, const void *d_leaves32, uint64_t n_leaves, dg_tree_t **tree);
/* the hash id, the number of leaves and the root (nodes[1]); each may be NULL.  Touches no device: the root is kept on the host. */
int dg_tree_info(const dg_tree_t *tree, int *hash, uint64_t *n_leaves, uint8_t root32[32]);
/* the authentication paths of count leaves (MerkleTree::prove, merkle.rs:47-62) in one launch: paths32 receives count x (d + 1) entries
 * of 32 bytes, path k at k (d + 1), each leaf i, leaf i ^ 1, then nodes[((L + i) >> 1 >> j) ^ 1] for j = 0 .. d - 2.  For hash 3 this is
 * the path of smpath.n / pmpath.n with n = d + 1.  Indexes may repeat and come in any order; one >= L fails the call with DG_ERR_INVALID
 * naming it.  Only the paths are copied to the host. */
int dg_tree_paths(const dg_tree_t *tree, const uint64_t *indexes, uint32_t count, uint8_t *paths32);
/* the leaf at indexes[k] becomes leaves32[k] (a repeated index: its last occurrence), and only the nodes on the changed leaves' paths are
 * hashed again, one pass per level: at most count x d digests instead of L - 1.  When the changed paths hold at least half of the L - 1
 * nodes, the call writes the new leaves and builds the tree again instead, which measured faster there.  Every argument is checked before the device changes
 * (indexes < L, and for hash 3 canonical leaves, named as dg_tree_new names them): a failed call leaves the tree as it was.  root32 (may be
 * NULL) receives the new root; count == 0 changes nothing and gives the current root. */
int dg_tree_update(dg_tree_t *tree, const uint64_t *indexes, const uint8_t *leaves32, uint32_t count, uint8_t root32[32]);
/* copies the L leaves and / or the L heap nodes to the host; either may be NULL */
int dg_tree_read(const dg_tree_t *tree, uint8_t *leaves32, uint8_t *nodes32);
void dg_tree_free(dg_tree_t *tree);

/* ---- membership inputs of a device tree ----------------------------------------------------------------------------------------------
 * dg_tree_membership_inputs: the inputs of smpath.n (DG_PATH_SMPATH, index private) or pmpath.n (DG_PATH_PMPATH, index public), n = d + 1,
 * for the leaves indexes[0 .. count) of a tree of hash 3 (DG_HASH_HASHER), written from the tree's heap straight into d_values in one
 * gather launch; no path reaches the host.  Per index k the values are one run of the layout of the examples' merkle.rs:63-85:
 *   smpath: tape A = leaf[0], then per later path entry e (0, e[0]); tape B = leaf[1], then (index bit, e[1]); no public input.
 *           4 d + 2 values: A at k (4 d + 2), B after it.
 *   pmpath: the index as the one public input, then tape A = e[0] and tape B = e[1] of every path entry.  2 d + 3 values: the index at
 *           k (2 d + 3), A after it, B after A.
 * out->n_values receives count times the values per index.  With d_values NULL that is all (the device is not touched).  Otherwise
 * d_values (device, 16-byte aligned) holds cap values, at least out->n_values; out->d_values becomes d_values and the six arrays of `out`,
 * which the caller points at host arrays of `count` entries, receive the ranges.  Indexes may repeat; one >= L fails the call with
 * DG_ERR_INVALID naming it, as dg_tree_paths does, and so does a tree of another hash. */
#define DG_PATH_SMPATH 0
#define DG_PATH_PMPATH 1
int dg_tree_membership_inputs(const dg_tree_t *tree, int program, const uint64_t *indexes, uint32_t count, void *d_values, uint64_t cap,
                              dg_device_inputs_t *out);

/* ---- batch proofs and their verification (MerkleTree::prove_batch / verify / verify_batch, merkle.rs:64-263) --------------------------
 * The encoding of a BatchMerkleProof {values, nodes, depth} is its bincode: u64 count + 32 B per value; u64 count, then per slot u64 count
 * + 32 B per node; u8 depth.  Hash ids and the hasher's message layout are those of dg_merkle_build_with. */
/* MerkleTree::prove_batch (merkle.rs:64-124) of a device tree: values in request order, node slots per normalised (even) index, and from
 * level 2 up the slot of a sibling is its position in the current level's list (merkle.rs:107-114).  The crate's panics fail the call with
 * DG_ERR_INVALID on the host, in its order, and leave the tree as it was: "invalid index i" for an index > L, "repeating indexes detected",
 * then "invalid index L" for an index of L.  count == 0 gives the empty proof of depth d.  *len receives the proof's length; with
 * proof_out == NULL that is all, from the host plan, and the device is not touched; a cap below *len fails with DG_ERR_INVALID.  Otherwise
 * one gather launch and one copy. */
int dg_tree_prove_batch(const dg_tree_t *tree, const uint64_t *indexes, uint32_t count, uint8_t *proof_out, size_t cap, size_t *len);
/* MerkleTree::verify (merkle.rs:127-151) for `count` paths of `entries` (2..64) 32-byte entries each, path k at paths32 + 32 entries k;
 * n_roots is 1 (every path against roots32) or count (path k against root k).  As in the reference only the low entries - 1 bits of an
 * index are read, so an index >= L = 2^(entries - 1) is checked as index mod L. */
int dg_merkle_verify_paths(int hash, const uint8_t *roots32, uint32_t n_roots, const uint64_t *indexes, const uint8_t *paths32,
                           uint32_t entries, uint32_t count, int *status);
/* MerkleTree::verify_batch (merkle.rs:154-263) for `count` batch proofs: proof i is proofs[i] (proof_lens[i] bytes, the encoding above)
 * against root roots32 + 32 i and the n_indexes[i] indexes at indexes[i] (may be NULL when n_indexes[i] is 0).  Depths 0-63 are planned
 * (a depth above 63 overflows usize::pow in the reference and is treated as its panic).
 *
 * Both verify calls: status[k] is DG_OK where the reference returns true, DG_ERR_REJECTED where it returns false, and DG_ERR_INVALID where
 * it panics ("invalid index i", "repeating indexes detected", "called `Option::unwrap()` on a `None` value") or where the entry's input is
 * malformed: bytes that are not exactly one BatchMerkleProof (read as dg_verify reads a StarkProof), and for hashes 1-3 an entry, value or
 * node element >= M, named in the message (the algebraic kernels take canonical operands; roots are only compared).  Entry k's message is
 * dg_batch_message(k), "" when accepted; one bad entry changes no other verdict.  The whole call fails with DG_ERR_INVALID before the
 * device is touched for a hash id other than 0-3, entries outside 2..64, n_roots other than 1 or count, or a NULL array.  Hashing runs
 * one level at a time over every path or proof of a group (a message launch and one digest launch per level, the hasher's narrow / wide
 * choice by level size); groups fit the device-memory budget of dg_verify_batch (dg_set_memory_limit), and every buffer is the pool's and
 * freed before the call returns. */
int dg_merkle_verify_batch(int hash, uint32_t count, const uint8_t *roots32, const uint64_t *const *indexes, const uint32_t *n_indexes,
                           const uint8_t *const *proofs, const size_t *proof_lens, int *status);

/* element-wise field ops on vectors (op: 0 add, 1 sub, 2 mul, 3 inv, 4 exp(a, b), 6 mul with b as a fixed twiddle: the NTT pass
 * kernels' product with a precomputed companion b * 2^64), for differential tests of the arithmetic;
 * impl: 0 = PTX path used by the kernels, 1 = portable C++ path, 2 / 3 = earlier PTX multiplies (op 2 only) */
int dg_field_op(int op, int impl, const uint8_t *a, const uint8_t *b, uint8_t *out, uint64_t n);
/* out[i] = sum_j a[len*i + j] * b[len*i + j], j < len (1..128), accumulated unreduced in 288 bits and reduced once, as the kernels' dot
 * products and constraint accumulators are; for differential tests of the arithmetic */
int dg_field_dot(const uint8_t *a, const uint8_t *b, uint8_t *out, uint64_t groups, uint32_t len);
/* The prover's constraint-evaluation kernel on a supplied extended trace, for differential tests of the AIR.  ext16 holds count entries
 * of w = 15 + ctx_depth + loop_depth + stack_depth columns of n << log_blowup elements each, in LDE order (what TraceTable::extend gives).
 * Entry i combines its transition constraints with the coefficients the prover draws from seeds32[32 i] (ConstraintCoefficients
 * without public inputs or outputs), or, when coefs16 is not NULL, with coefs16[2T i ..] = [coefA | coefB] of its T constraints in
 * evaluation order.  All entries run in one launch.  out16 receives count x 8n values in step order.  check = 0 evaluates every step
 * (no trace-domain check); check = 1 is the prover's check: trace-domain steps other than the last give 0, and first_violation[i] is
 * 1 + the lowest trace step whose constraints do not all vanish, or 0. */
int dg_eval_transitions(const uint8_t *ext16, uint32_t count, uint32_t ctx_depth, uint32_t loop_depth, uint32_t stack_depth, uint32_t log_n,
                        uint32_t log_blowup, const uint8_t *seeds32, const uint8_t *coefs16, int check, uint8_t *out16, uint32_t *first_violation);

/* ---- device-resident variants (timed with CUDA events on the library's stream; *ms may be NULL) ----------------------- */
int dg_dev_alloc(void **ptr, size_t bytes);
int dg_dev_free(void *ptr);
int dg_dev_upload(void *dst, const void *src, size_t bytes);
int dg_dev_download(void *dst, const void *src, size_t bytes);
int dg_dev_sync(void);
int dg_dev_ntt(void *d_values, uint32_t log_n, uint32_t batch, int inverse, float *ms);
/* d_polys: batch x n coefficients; d_ext: batch x (n << log_blowup) evaluations, coset-major ([c][k] = LDE index k*blowup + c) */
int dg_dev_lde(const void *d_polys, void *d_ext, uint32_t log_n, uint32_t log_blowup, uint32_t batch, float *ms);
int dg_dev_merkle_build(const void *d_leaves, uint64_t n_leaves, void *d_nodes, float *ms);
int dg_dev_merkle_build_with(int hash, const void *d_leaves, uint64_t n_leaves, void *d_nodes, float *ms);
/* d_ext coset-major as produced by dg_dev_lde; d_leaves: (n << log_blowup) digests in logical row order */
int dg_dev_hash_rows(const void *d_ext, uint32_t width, uint32_t log_n, uint32_t log_blowup, void *d_leaves, float *ms);
/* writes > L2-size scratch to evict the L2 between timed iterations */
int dg_dev_flush_l2(void);

/* ---- multi-GPU: one process per GPU, the proof of ONE trace is sharded by LDE coset ranges over `world` ranks ----------------
 * Every rank calls dg_prove / dg_prove_device with the SAME trace and options; every rank returns the same proof bytes.
 * Rank 0 obtains the 128-byte NCCL id, the host distributes it (e.g. torch.distributed broadcast), all ranks call dg_comm_init. */
int dg_comm_unique_id(uint8_t id128[128]);
int dg_comm_init(int rank, int world /* 1, 2, 4 or 8 */, const uint8_t id128[128]);
int dg_comm_finalize(void);
/* index algebra of the sharded Merkle trees, exported for CPU tests: locates level-0 item `index` (is_node = 0) or the internal
 * node with global heap index `index` (is_node = 1) of a tree with n blocks of 2^log_blk items per rank over 2^log_g ranks;
 * out = {owner rank or -1 if replicated, 1 if in the replicated upper heap else 0, local index} */
int dg_host_shard_locate(uint64_t n, int log_blk, int log_g, int is_node, uint64_t index, int64_t out[3]);
/* the grouping of dg_prove_traces, exported for CPU tests: the traces partitioned by length (lengths in order of first appearance, input
 * order inside a length), each length's traces cut into consecutive groups of at most `cap` traces whose footprints[i] sum to at most
 * `budget` (the call uses a budget per length) and whose widths sum to at most 65535.  order_out (count entries) receives the traces in
 * the order the groups run, each group in its device order: grouped by register shape, shapes in order of first appearance, input order
 * inside a shape; group_sizes_out (up to count entries) the sizes of the groups, n_groups their number. */
int dg_host_group_traces(uint32_t count, const uint64_t *lengths, const uint32_t *widths, const uint32_t *ctx_depths, const uint32_t *loop_depths,
                         const uint64_t *footprints, uint64_t budget, uint32_t cap, uint32_t *order_out, uint32_t *group_sizes_out,
                         uint32_t *n_groups);
/* the same for dg_prove_traces_with_options: the traces partitioned by (length, extension_factors[i]), partitions in order of first
 * appearance, each cut and ordered as above */
int dg_host_group_traces_with_options(uint32_t count, const uint64_t *lengths, const uint32_t *extension_factors, const uint32_t *widths,
                                      const uint32_t *ctx_depths, const uint32_t *loop_depths, const uint64_t *footprints, uint64_t budget,
                                      uint32_t cap, uint32_t *order_out, uint32_t *group_sizes_out, uint32_t *n_groups);

/* ---- host-side Fiat-Shamir glue, exported so that it can be unit-tested without a GPU (none of these touch the device) ---- */
/* field::prng_vector (field.rs:271-275): count draws of StdRng::from_seed(seed) through Uniform(0..M) */
int dg_host_prng_vector(const uint8_t seed[32], uint64_t count, uint8_t *out16);
/* utils::compute_query_positions (stark/utils/mod.rs:25-44) */
int dg_host_query_positions(const uint8_t seed[32], uint64_t domain_size, uint32_t extension_factor, uint32_t num_queries, uint64_t *out);
/* blake3 of a message of at most 1024 bytes (the FRI-roots seed of prover.rs:119-127) */
int dg_host_blake3(const uint8_t *data, size_t len, uint8_t out32[32]);
/* MerkleTree::prove_batch planning (merkle.rs:64-124): writes, per normalised slot, the count and then (is_leaf, index) pairs;
 * out layout: [n_slots][depth] then for each slot [count] (is_leaf, index)*count, all uint64 */
int dg_host_plan_batch(const uint64_t *indexes, uint32_t n_indexes, uint64_t n_leaves, uint64_t *out, size_t cap, size_t *written);
/* the plan of dg_tree_update: the indexes deduplicated (last occurrence wins) and sorted, then per level from the leaves' parents in
 * [L/2, L) up to the root the sorted unique changed nodes, each with the position in the level below of its first changed child.
 * out layout, all uint64: [K][d][T = digests hashed] [leaf index]*K [position of its last occurrence in the call]*K, then per level
 * [n] [node id]*n [first changed child]*n */
int dg_host_tree_plan(const uint64_t *indexes, uint32_t count, uint64_t n_leaves, uint64_t *out, size_t cap, size_t *written);
/* MerkleTree::verify_batch (merkle.rs:154-263) as the hashing plan dg_verify executes on the device: digests live in a pool -- the proof's
 * values in slots [0, n_values), the nodes of slot i from n_values + node_counts[0..i) on, computed parents after them; ops = (left, right,
 * out) slot triples, level_start[l] .. level_start[l+1] the ops of level l; the tree is accepted iff pool[root_slot] equals the root.
 * Returns DG_ERR_REJECTED where verify_batch returns false for structural reasons. */
int dg_host_merkle_verify_plan(const uint64_t *indexes, uint32_t n_indexes, uint32_t depth, uint32_t n_values, const uint32_t *node_counts,
                               uint32_t n_slots, uint32_t *ops, size_t ops_cap, uint32_t *n_ops, uint32_t *level_start, size_t levels_cap,
                               uint32_t *n_levels, uint32_t *root_slot);
/* extend_constants tables (constraints/utils.rs:87-113): 128 rows x 23 columns = sponge ARK 8 | masks 3 | hasher ARK 12 */
int dg_host_periodic_tables(uint8_t *out16 /* 128*23 elements */);
/* name of transition constraint `index` (evaluation order) of a register shape: "op bit 3 binary", "op counter", "sponge 1", "ctx stack 0",
 * "stack aux 1", "stack slot 5", ... (NUL-terminated, truncated to cap); DG_ERR_INVALID for a shape dg_prove rejects or index >= T */
int dg_host_constraint_name(uint32_t ctx_depth, uint32_t loop_depth, uint32_t stack_depth, uint32_t index, char *name, size_t cap);

/* ---- test hooks: not user API --------------------------------------------------------------------------------------------------------
 * The prover's coefficient-domain stage kernels one call at a time, on host buffers, for differential tests.  Each hook calls the host
 * function the prover calls, with the power tables, strides and layouts the prover gives it.  Every argument is checked before the
 * device is touched (DG_ERR_INVALID with a message, also without a GPU); every vector element must be < M.  Output buffers are
 * zero-filled on the device before the kernels run, so gaps between strided vectors come back as zeros (or, in place, as the input).
 *
 * dg_test_syn_div: synthetic division by (x - b_q) of `batch` vectors of len (a power of 2) elements, vector q at q in_stride of in16,
 * its quotient out[i] = sum_{j>i} (a[j] - [j == 0] sub0[q]) b_q^(j-i-1) at q out_stride of out16; out16 receives (batch - 1) out_stride
 * + len elements.  in_place: one buffer (in_stride == out_stride).  shared = 0: one point per vector in b16 and a power table per vector
 * (stage 6); shared = 1: one point b16[0] and one table for all vectors (stage 4). */
int dg_test_syn_div(const uint8_t *in16, uint8_t *out16, uint32_t batch, uint64_t len, uint64_t in_stride, uint64_t out_stride, int in_place,
                    const uint8_t *b16, int shared, const uint8_t *sub0_16);
/* division of 8n coefficients by (x^n - 1) / (x - e), plus add0 and add1 (either may be NULL): vector q of a16 / add0_16 / add1_16 at
 * q in_stride, of out16 at q out_stride ((batch - 1) out_stride + 8n elements) */
int dg_test_syn_div_expanded_sum(const uint8_t *a16, const uint8_t *add0_16, const uint8_t *add1_16, uint8_t *out16, uint32_t batch, uint64_t n,
                                 uint64_t in_stride, uint64_t out_stride, const uint8_t *e16);
/* col_proof != NULL: cols columns of n = 2^log_n coefficients, column j at point z[col_proof[j]]: out16[2j] = P_j(z), out16[2j + 1] =
 * P_j(z w_n).  col_proof == NULL: cols == n_z columns of 8n coefficients, out16[2q] = P_q(z_q), out16[2q + 1] = 0.  The powers of every
 * z come from one table of 8n + 1 entries per point. */
int dg_test_eval_polys_at(const uint8_t *polys16, uint32_t cols, uint32_t log_n, const uint8_t *z16, uint32_t n_z, const uint32_t *col_proof,
                          uint8_t *out16);
/* opened trace rows: for each m < count, P_j(w_N^pos[m]) for the width[m] (1..128) columns j from col[m] on, of cols columns of 2^log_n
 * coefficients, N = 2^log_N; out16 receives the values of the rows one after another */
int dg_test_eval_trace_rows(const uint8_t *polys16, uint32_t cols, uint32_t log_n, uint32_t log_N, const uint64_t *pos, const uint32_t *col,
                            const uint32_t *width, uint32_t count, uint8_t *out16);
/* the fold-8 extension of `batch` polynomials of 8n coefficients (8n apart in coeffs16) over the cosets [coset0, coset0 + ncosets) of the
 * domain of 2^(log_n + log_b) points: vector q's coset c at q dst_stride + (c - coset0) n of out16, element k = P(w_N^(k b + c)) */
int dg_test_lde_fold8(const uint8_t *coeffs16, uint8_t *out16, uint32_t log_n, uint32_t log_b, uint32_t coset0, uint32_t ncosets, uint32_t batch,
                      uint64_t dst_stride);
/* interpolation of 8n evaluations given by coset: evals16 holds `batch` vectors of [8][n] (8n apart), e_c[k] = P(w_8n^(8k + c)); out16
 * receives the 8n coefficients of vector q at q out_stride */
int dg_test_coset_interp(const uint8_t *evals16, uint8_t *out16, uint32_t log_n, uint32_t batch, uint64_t out_stride);
/* one FRI layer of `batch` vectors of D = 2^log_d values (values_stride apart), stored natural (log_b = -1) or coset-major with 2^log_b
 * cosets, on the domain of the powers w_N^(4^depth i), N = 2^log_N.  The rows layout is the one the prover chooses.  leaves32: batch x R
 * digests (R = D/4) in logical row order; the folding point of vector q is derived from roots32[32 q] (placed root_stride bytes apart on
 * the device) into alphas16[q], that root copied to root_copies32[32 q]; next16: batch x R folded values in the rows layout's storage
 * order. */
int dg_test_fri_layer(const uint8_t *values16, uint32_t batch, uint64_t values_stride, uint32_t log_d, int32_t log_b, uint32_t log_N,
                      const uint8_t *roots32, uint64_t root_stride, uint8_t *leaves32, uint8_t *alphas16, uint8_t *root_copies32, uint8_t *next16);
/* The evaluation-domain stages the same way.
 * dg_test_trace_lde: stage 1.  `cols` register columns of n = 2^log_n elements (n apart in regs16) are interpolated into polys16 (cols x n
 * coefficients), then extended onto the cosets [coset0, coset0 + ncosets) of the domain of N = n 2^log_b points (log_b 1..16, log_n +
 * log_b <= 30): column j's coset c at j col_stride + (c - coset0) n of ext16, element k = P_j(w_N^(k 2^log_b + c)); ext16 receives (cols -
 * 1) col_stride + ncosets n elements.  copy_coset0 = 1: coset 0 (when in the range) is copied from the registers, as the prover does for a
 * trace on the device; 0: every coset is transformed. */
int dg_test_trace_lde(const uint8_t *regs16, uint32_t cols, uint32_t log_n, uint32_t log_b, uint32_t coset0, uint32_t ncosets, uint64_t col_stride,
                      int copy_coset0, uint8_t *polys16, uint8_t *ext16);
/* stage 2: the rows of the cosets [c0, c0 + nc) of a 2^log_blowup-coset extension, given as total_cols columns of nc n elements
 * ([column][c - c0][k], n = 2^log_n).  col_table (may be NULL): `batch` (first column, width) pairs, one matrix per pair (widths 1..127);
 * NULL: `batch` matrices of total_cols / batch columns one after another.  Matrix q's row of coset c at step k is leaf (k << log_blowup) + c
 * of the q-th run of leaves, leaf_stride digests apart (0: 2^(log_n + log_blowup)); leaves32 receives (batch - 1) stride + 2^(log_n +
 * log_blowup) digests, those of cosets outside the range zero. */
int dg_test_hash_trace_rows(const uint8_t *ext16, uint32_t total_cols, uint32_t log_n, uint32_t log_blowup, uint32_t c0, uint32_t nc, uint32_t batch,
                            const uint32_t *col_table, uint64_t leaf_stride, uint8_t *leaves32);
/* stages 2 and 5: `batch` Merkle trees of L leaves (L a power of 2 in 2..2^30), tree q's leaves and heap (L digests, nodes[0] = 0, root =
 * nodes[1]) at q L digests */
int dg_test_merkle_batch(const uint8_t *leaves32, uint64_t L, uint32_t batch, uint8_t *nodes32);
/* stage 5: the first level of the constraint tree of `batch` slabs of 2^log_nc cosets (log_nc >= 2) of n = 2^log_n evaluations ([c][k],
 * n 2^log_nc elements apart): item (k << (log_nc - 2)) + c4 = blake3(ev[4 c4][k], ..., ev[4 c4 + 3][k]), n 2^(log_nc - 2) digests per slab */
int dg_test_constraint_items(const uint8_t *evals16, uint32_t log_n, uint32_t log_nc, uint32_t batch, uint8_t *items32);

#ifdef __cplusplus
}
#endif
#endif /* DISTAFF_GPU_H */
