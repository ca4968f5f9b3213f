// The proof: the reference's StarkProof and its bincode 1.3.1 encoding, the library's output contract.
//   StarkProof, TraceInfo, DeepValues    /root/reference/src/stark/proof.rs:10-37
//   FriProof, FriLayer                   /root/reference/src/stark/fri/mod.rs:17-30
//   BatchMerkleProof                     /root/reference/src/crypto/merkle.rs:14-18
//   ProofOptions                         /root/reference/src/stark/options.rs:16-23
// The prover fills a StarkProof and writes it (write_proof); the verifier reads one (read_proof).  The field order lives in proof.cu alone.
#pragma once
#include <array>
#include <cstdint>
#include <vector>
#include "common.cuh"

namespace dg {

struct TraceInfo {
    uint8_t domain_depth = 0, ctx_depth = 0, loop_depth = 0, stack_depth = 0;
    uint32_t op_count = 0;                           // the op counter of the last step, truncated (proof.rs:62)
};
struct BatchMerkleProof {
    std::vector<Digest> values;
    std::vector<std::vector<Digest>> nodes;
    uint8_t depth = 0;
};
struct FriLayer {
    Digest root;
    std::vector<std::array<fe, 4>> values;           // one row of 4 values per augmented position
    std::vector<std::vector<Digest>> nodes;
    uint8_t depth = 0;
};
struct FriProof {
    std::vector<FriLayer> layers;
    Digest rem_root;
    std::vector<fe> rem_values;
};
struct ProofOptions {
    uint8_t log_extension_factor = 0, num_queries = 0, grinding_factor = 0, hash_fn = 0;    // hash_fn 0: blake3
};
struct StarkProof {
    Digest trace_root;
    TraceInfo trace_info;
    std::vector<std::vector<Digest>> trace_nodes;
    std::vector<std::vector<fe>> trace_evaluations;  // one row of w values per query
    Digest constraint_root;
    BatchMerkleProof constraint_proof;
    std::vector<fe> trace_at_z1, trace_at_z2;        // DeepValues
    FriProof degree_proof;
    uint64_t pow_nonce = 0;
    ProofOptions options;
};

std::vector<uint8_t> write_proof(const StarkProof &P);
// false when the bytes are not exactly one StarkProof: short input, trailing bytes, or a Vec length the remaining bytes cannot hold
bool read_proof(const uint8_t *bytes, size_t len, StarkProof &P);
// one BatchMerkleProof {values, nodes, depth} alone (MerkleTree::prove_batch / verify_batch), with read_proof's rule
bool read_batch_proof(const uint8_t *bytes, size_t len, BatchMerkleProof &P);

// A proof the library returns (dg_proof_t): its bytes and the commitments the C-ABI exposes
struct Proof {
    std::vector<uint8_t> bytes;          // write_proof of the StarkProof
    uint8_t trace_root[32], constraint_root[32], pow_seed[32];
    unsigned long long pow_nonce = 0;
};

}  // namespace dg
