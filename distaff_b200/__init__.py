"""distaff_b200 -- H100-native (sm_90a) STARK prover backend for the Distaff VM.

Python host-side mirror of the reference interface for the prove hot path:
    distaff_b200.prove(trace, options)            <->  stark::prove        (/root/reference/src/stark/prover.rs:17)
    distaff_b200.prove_batch(traces, options)     <->  stark::prove of every trace, same-shape traces proven together
    distaff_b200.execute(source, inputs, ...)     <->  distaff::execute    (/root/reference/src/lib.rs:30-65), VM = host stand-in
    distaff_b200.verify(hash, inputs, outputs, p) <->  distaff::verify     (/root/reference/src/lib.rs:68-75, stark/verifier.rs:11-75)
    distaff_b200.verify_batch(items)              <->  distaff::verify of every proof, all checked together on the GPU
The compute path is hand-written CUDA behind the C-ABI of include/distaff_gpu.h; there is no CPU fallback.
"""
from .api import (ProofOptions, StarkProof, prove, prove_device, prove_batch, prove_batch_device, verify, verify_batch, execute, ntt, intt, lde,  # noqa: F401
                  merkle_build, hash_rows, hash64, find_pow_nonce, field_op)
