// Host-side orchestration of the prove pipeline (prover.cu) -- the body that replaces
// /root/reference/src/stark/prover.rs:17-169.
#pragma once
#include "../../include/distaff_gpu.h"
#include "common.cuh"

namespace dg {

struct Proof {
    std::vector<uint8_t> bytes;          // bincode encoding of StarkProof
    uint8_t trace_root[32], constraint_root[32], pow_seed[32];
    unsigned long long pow_nonce = 0;
};

Proof *prove_host(Context &c, const dg_trace_t &trace, const uint8_t *inputs16, uint32_t n_inputs, const uint8_t *outputs16,
                  uint32_t n_outputs, const dg_options_t &opt, dg_prove_stats_t *stats);
Proof *prove_device(Context &c, const fe *d_registers, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth,
                    const uint8_t *inputs16, uint32_t n_inputs, const uint8_t *outputs16, uint32_t n_outputs, const dg_options_t &opt,
                    dg_prove_stats_t *stats, float h2d_ms);
// batched proving (dg_prove_batch / dg_prove_batch_device): proofs_out[i] / status[i] / messages[i] (why trace i failed, else empty) per
// trace, one GPU only; when the call throws, no proof is left in proofs_out
void prove_batch_host(Context &c, const dg_trace_t *traces, uint32_t count, const uint8_t *const *inputs16, const uint32_t *n_inputs,
                      const uint8_t *const *outputs16, const uint32_t *n_outputs, const dg_options_t &opt, Proof **proofs_out, int *status,
                      std::vector<std::string> &messages, dg_prove_stats_t *stats);
void prove_batch_device(Context &c, const fe *d_regs, uint32_t count, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth,
                        const uint8_t *const *inputs16, const uint32_t *n_inputs, const uint8_t *const *outputs16, const uint32_t *n_outputs,
                        const dg_options_t &opt, Proof **proofs_out, int *status, std::vector<std::string> &messages, dg_prove_stats_t *stats);

// Batched proving of `count` traces of one shape that are generated on the device group by group: generate(first, k, d_regs, failed)
// writes traces [first, first + k) into d_regs ([k][width][length], the buffer the prover then reads) and sets failed[i] to the status and
// message of a trace it could not generate (failed holds k entries of DG_OK on entry).  Otherwise as prove_batch_device.
void prove_batch_generated(Context &c, uint32_t count, uint32_t width, uint64_t length, uint32_t ctx_depth, uint32_t loop_depth,
                           const uint8_t *const *inputs16, const uint32_t *n_inputs, const uint8_t *const *outputs16, const uint32_t *n_outputs,
                           const dg_options_t &opt, Proof **proofs_out, int *status, std::vector<std::string> &messages, dg_prove_stats_t *stats,
                           const std::function<void(uint32_t, int, fe *, std::vector<std::pair<int, std::string>> &)> &generate);
// dg_trace_batch / dg_execute_batch (execute.cu): status / messages per execution.  check_execution_call validates the arguments and the
// program encoding on the host alone (DG_ERR_INVALID); both calls run it again.
void check_execution_call(const dg_program_t *program, uint32_t count, const dg_program_inputs_t *inputs, uint64_t max_steps);
void trace_batch(Context &c, const dg_program_t *program, uint32_t count, const dg_program_inputs_t *inputs, uint64_t max_steps,
                 dg_execution_info_t *info, uint8_t *const *registers_out, int *status, std::vector<std::string> &messages);
void execute_batch(Context &c, const dg_program_t *program, uint32_t count, const dg_program_inputs_t *inputs, uint32_t num_outputs,
                   uint64_t max_steps, const dg_options_t &opt, Proof **proofs_out, uint8_t *outputs16, int *status,
                   std::vector<std::string> &messages, dg_prove_stats_t *stats);
// the largest group of a batched call, after $DG_BATCH_GROUP
int batch_group_cap(long long k);

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

// the trace check (check.cu): per trace, which transition constraints fail at which steps and which boundary registers are wrong.
// d_regs: [count][width][length] on the device, or null with host_cols (count * width column pointers) to upload; program_hashes32
// (count * 32 bytes) and step_masks (host, count * length * 3 words) / d_step_masks (device, same size) may be null
void check_traces(Context &c, const fe *d_regs, const uint8_t *const *host_cols, uint32_t count, uint32_t width, uint64_t length,
                  uint32_t ctx_depth, uint32_t loop_depth, const uint8_t *const *inputs16, const uint32_t *n_inputs,
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
