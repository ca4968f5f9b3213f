"""distaff_b200 -- H100-native (sm_90a) STARK prover backend for the Distaff VM.

Python host-side mirror of the reference interface for the prove hot path:
    distaff_b200.prove(trace, options)            <->  stark::prove        (/root/reference/src/stark/prover.rs:17)
    distaff_b200.prove_batch(traces, options)     <->  stark::prove of every trace, same-shape traces proven together
    distaff_b200.prove_traces(traces, options)    <->  stark::prove of every trace, traces of any shapes in one call
    distaff_b200.execute(source, inputs, ...)     <->  distaff::execute    (/root/reference/src/lib.rs:30-65), VM = host stand-in
    distaff_b200.verify(hash, inputs, outputs, p) <->  distaff::verify     (/root/reference/src/lib.rs:68-75, stark/verifier.rs:11-75)
    distaff_b200.verify_batch(items)              <->  distaff::verify of every proof, all checked together on the GPU
    distaff_b200.check_trace(trace, hash)         <->  the named transition / boundary constraints a trace breaks, before proving it
    distaff_b200.set_memory_limit(bytes)          <->  the most device memory the library may hold (plan_prove, memory_usage)
    distaff_b200.execute_batch(program, inputs)   <->  distaff::execute for many ProgramInputs: the VM and the proofs on the GPU
    distaff_b200.trace_batch(program, inputs)     <->  processor::execute for many ProgramInputs on the GPU (trace_shapes: shapes only)
    distaff_b200.execute_programs(jobs)           <->  execute_batch for jobs of many programs in one call (trace_programs: the traces)
    distaff_b200.execute_one(program, inputs)     <->  distaff::execute of one long execution, split across GPU threads (trace_one)
    distaff_b200.execute_many(jobs)               <->  execute_programs with every execution split as execute_one splits one (trace_many)
    distaff_b200.HasherTree(leaves)               <->  a Merkle tree of utils::hasher::digest, built on the GPU, with its smpath / pmpath inputs
    distaff_b200.prove_membership(tree, indexes)  <->  execute_batch of the smpath or pmpath program for leaves of a HasherTree
    distaff_b200.MerkleTree(leaves, hash)         <->  crypto::MerkleTree kept in device memory: paths of many leaves per call, leaf updates
    tree.prove_batch(indexes)                     <->  MerkleTree::prove_batch: a BatchMerkleProof gathered on the GPU
    distaff_b200.merkle_verify_paths / _batch     <->  MerkleTree::verify / verify_batch of many paths or batch proofs in one call
The compute path is hand-written CUDA behind the C-ABI of include/distaff_gpu.h; there is no CPU fallback.
"""
from .api import (ProofOptions, StarkProof, prove, prove_device, prove_batch, prove_batch_device, prove_traces, prove_traces_device, verify, verify_batch, execute, ntt, intt, lde,  # noqa: F401
                  merkle_build, hash_rows, hash64, find_pow_nonce, field_op, field_dot, eval_transitions, TraceReport, check_trace, check_traces,
                  check_traces_device, constraint_name, set_memory_limit, memory_usage, plan_prove, ProgramInputs, trace_batch, trace_shapes,
                  execute_batch, trace_programs, execute_programs, group_traces, trace_one, execute_one,
                  trace_many, execute_many, HasherTree, smpath_program, pmpath_program, prove_membership, MerkleTree,
                  BatchMerkleProof, merkle_verify_paths, merkle_verify_batch)
