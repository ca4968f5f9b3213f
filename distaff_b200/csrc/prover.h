// Host-side orchestration of the prove pipeline (prover.cu) -- the body that replaces
// /root/reference/src/stark/prover.rs:17-169.
#pragma once
#include "../../include/distaff_gpu.h"
#include "common.cuh"
#include "proof.h"
#include <optional>

namespace dg {

// what the caller gives of a trace's register shape (TraceShape::of_trace checks it and derives the rest)
struct RegisterShape {
    uint32_t width, ctx_depth, loop_depth;
    bool operator==(const RegisterShape &o) const { return width == o.width && ctx_depth == o.ctx_depth && loop_depth == o.loop_depth; }
};
// one trace of a prove call: its shape and length, and its registers, either host columns (width pointers) or device memory ([width][length])
struct TraceRef {
    uint32_t width = 0;
    uint64_t length = 0;
    uint32_t ctx_depth = 0, loop_depth = 0;
    const uint8_t *const *host_cols = nullptr;
    const fe *d_regs = nullptr;
    const void *slab = nullptr;        // device traces given as one allocation (a one-shape call): its base; null when not known
    RegisterShape shape() const { return RegisterShape{width, ctx_depth, loop_depth}; }
};
// Proves traces of any shapes and lengths (every trace host, or every trace on the device), trace i with opts[i] and the public inputs /
// outputs inputs16[i] (n_inputs[i] elements) and outputs16[i].  The call is partitioned by (length, extension factor)
// (partition_traces); each partition is planned for its widest shape (plan_prove) and cut into groups (cut_groups) of at most that
// plan's bytes; inside a group the traces are laid out on the device by shape (shape_order), and their num_queries and grinding factors
// may differ.  The Fiat-Shamir draws run partition by partition, group by group, stage by stage, and within a stage in input order.
// batch: a batched call, which runs on one GPU only; otherwise, on several GPUs (dg_prove on every rank), one trace is proven sharded.
// proofs_out[i] / status[i] / messages[i] (why trace i failed, else empty) per trace; when the call throws, no proof is left in
// proofs_out.  groups (may be null) receives the number of groups the traces ran in.
// prove_traces and check_traces take calls that passed check_prove_call (capi.cu) or check_execution_call: they do not check the
// lengths, shapes, registers, public input / output counts or options again.
void prove_traces(Context &c, const std::vector<TraceRef> &traces, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                  const uint8_t *const *outputs16, const uint32_t *n_outputs, const std::vector<dg_options_t> &opts, bool batch,
                  Proof **proofs_out, int *status, std::vector<std::string> &messages, dg_prove_stats_t *stats, uint32_t *groups = nullptr);
// `count` traces of one shape in one device allocation, [count][width][length] at d_regs
std::vector<TraceRef> one_shape_traces(const fe *d_regs, uint32_t count, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth);
// adds a group's stats to a call's
void add_stats(dg_prove_stats_t *sum, const dg_prove_stats_t &s);
// ProofOptions::new's checks (options.rs:29-50) and the hash (only blake3 is serialisable): DG_ERR_INVALID with the reason
void check_options(const dg_options_t &o);
// the traces of each (length, extension factor), partitions in order of first appearance, traces in input order
std::vector<std::vector<uint32_t>> partition_traces(const std::vector<uint64_t> &length, const std::vector<uint32_t> &extension_factor);
// sizes of the consecutive groups the traces (in this order) are cut into: a group holds at most `cap` traces, footprints summing to at
// most `budget` bytes and widths summing to at most 65535 (one launch); a trace that exceeds the budget alone is a group of its own
std::vector<uint32_t> cut_groups(const std::vector<uint32_t> &width, const std::vector<size_t> &footprint, size_t budget, uint32_t cap);
// the device order of a group: positions of the traces grouped by shape, shapes in order of first appearance, input order inside a shape
std::vector<uint32_t> shape_order(const std::vector<RegisterShape> &shape);

// The execution calls (execute.cu).  Execution i runs programs[program_of[i]] on inputs[i]; status / messages per execution.
struct ExecutionCall {
    const dg_program_t *programs;
    uint32_t n_programs, count;
    const uint32_t *program_of;
    const dg_program_inputs_t *inputs;
    uint64_t max_steps;
};
// the output counts of an execute call: num_outputs[i] <= 8 per execution; outputs16 may be null when every count is 0
struct OutputCounts {
    const uint32_t *num_outputs;
    const uint8_t *outputs16;
};
// Every execution entry runs this once before it touches the device: it rejects bad arguments and encodings on the host alone
// (DG_ERR_INVALID), with the output counts of an execute call and the segment_steps of a tabled call (0 or a power of two >= 16) when
// given.  The calls below assume it passed.
void check_execution_call(const ExecutionCall &x, const std::optional<OutputCounts> &outputs = std::nullopt,
                          std::optional<uint64_t> segment_steps = std::nullopt);
// dg_trace_programs / dg_execute_programs (dg_trace_batch / dg_execute_batch with one program): the batch path.  info may be null.
// execute_programs writes 8 output elements per execution (zero past its num_outputs).
void trace_programs(Context &c, const ExecutionCall &x, dg_execution_info_t *info, uint8_t *const *registers_out, int *status,
                    std::vector<std::string> &messages, dg_execution_stats_t *vm_stats);
// opts: the options of every execution (x.count entries)
void execute_programs(Context &c, const ExecutionCall &x, const uint32_t *num_outputs, const dg_options_t *opts, Proof **proofs_out,
                      uint8_t *outputs16, int *status, std::vector<std::string> &messages, dg_prove_stats_t *stats, dg_execution_stats_t *vm_stats);
// dg_trace_many / dg_execute_many (dg_trace_one / dg_execute_one with one execution): trace_programs / execute_programs with the
// executions run from the sponge tables.  info may be null.  stats (may be null) are written also when the tabled passes throw (dg_trace_one
// reports a failed call's).
void trace_many(Context &c, const ExecutionCall &x, uint64_t segment_steps, dg_execution_info_t *info, uint8_t *const *registers_out, int *status,
                std::vector<std::string> &messages, dg_many_stats_t *stats);
void execute_many(Context &c, const ExecutionCall &x, const uint32_t *num_outputs, uint64_t segment_steps, const dg_options_t *opts,
                  Proof **proofs_out, uint8_t *outputs16, dg_execution_info_t *info, int *status, std::vector<std::string> &messages,
                  dg_prove_stats_t *prove_stats, dg_many_stats_t *stats);
// the largest group of a batched call, after $DG_BATCH_GROUP
long long batch_group_cap(long long k);

// What a prove call of one shape does on one GPU (dg_plan_prove): the full layout keeps the whole trace extension; the evaluation-coset
// layout extends and hashes `chunk` cosets at a time, keeps the 8 cosets the constraint evaluation reads and computes the other opened
// rows from the trace polynomials.  Proofs run in groups of `group`; per_proof bytes each (arena) on top of `fixed` bytes outside the
// arena (persistent tables, transform scratch); `available` is the budget the group was fitted into.  Throws DG_ERR_INVALID with the
// bytes needed when not even one proof fits.
struct ProvePlan {
    bool full = true;
    unsigned chunk = 0;
    int group = 1;
    size_t per_proof = 0, fixed = 0, available = 0;
};
ProvePlan plan_prove(Context &c, uint32_t w, uint64_t n, uint32_t b, uint32_t count);
size_t proof_footprint(uint32_t w, uint64_t n, uint32_t b, uint32_t chunk);

// copies `cols` host register columns of n elements each to d_regs (column stride n) by the prover's upload path (pinned columns DMA'd
// directly, pageable ones staged through the library's pinned slots) and orders c.stream after the copies
void upload_trace_columns(Context &c, fe *d_regs, const uint8_t *const *host_cols, int cols, uint64_t n);
// Stage 1's trace LDE of `cols` columns (polynomials `polys`, stride n) onto the cosets [c0, c0 + nc), written to ext (column stride N_loc).
// Coset 0 is P(w_n^k), which is register row k itself (polys = iNTT(regs) exactly): when the range starts at coset 0 and the registers
// are on the device (`regs`, stride n; null if not), slab 0 is copied from them and only the other cosets are transformed.
void extend_trace_columns(Context &c, const fe *polys, const fe *regs, fe *ext, int cols, int log_n, int log_b, uint64_t N_loc, unsigned c0,
                          unsigned nc);

// the trace check (check.cu): per trace, which transition constraints fail at which steps and which boundary registers are wrong.  The
// traces have one shape, host or in one device allocation (one_shape_traces); program_hashes32 (count * 32 bytes) and step_masks (host,
// count * length * 3 words) / d_step_masks (device, same size) may be null
void check_traces(Context &c, const std::vector<TraceRef> &traces, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                  const uint8_t *const *outputs16, const uint32_t *n_outputs, const uint8_t *program_hashes32, dg_trace_report_t *reports,
                  uint32_t *step_masks, uint32_t *d_step_masks);
// name of transition constraint `index` (evaluation order) of a register shape, as the trace check reports it
std::string constraint_name(uint32_t ctx_depth, uint32_t loop_depth, uint32_t stack_depth, uint32_t index);

// GPU verification (verifier.cu).  One proof of dg_verify / dg_verify_batch, with its program hash and public inputs / outputs.
struct VerifyRequest {
    const uint8_t *program_hash;
    const uint8_t *inputs16; uint32_t n_inputs;
    const uint8_t *outputs16; uint32_t n_outputs;
    const uint8_t *proof; size_t proof_len;
};
// Verifies every proof, each stage launched once per group of proofs.  status[i] is what dg_verify returns for proof i alone: DG_OK,
// DG_ERR_REJECTED with the reference's error string in messages[i], or the per-proof error (DG_ERR_INVALID, ...) with its message.
// Throws for errors of the whole call (CUDA failures); then status and messages are left as they were.
void verify_proofs(Context &c, const std::vector<VerifyRequest> &req, std::vector<int> &status, std::vector<std::string> &messages,
                   dg_verify_stats_t *stats);
// the verifier's batch-Merkle hashing plan of one tree, computed on the host alone (verifier.cu)
bool host_plan_verify_batch(const std::vector<uint64_t> &indexes, int depth, size_t n_values, const std::vector<uint32_t> &node_counts,
                            std::vector<uint32_t> &ops, std::vector<uint32_t> &level_start, uint32_t &root_slot);

}  // namespace dg
