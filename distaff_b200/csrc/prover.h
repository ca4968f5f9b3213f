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
