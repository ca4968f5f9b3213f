"""ORACLE -- TEST INFRASTRUCTURE ONLY.  ctypes face of oracle/liboracle.so (the CPU restatement of the reference).

Importable only from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
The product package (distaff_b200/) never imports this module.
"""
import ctypes
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
u8p = ctypes.c_void_p


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(path):
            raise RuntimeError(f"{path} missing: run make -C oracle")
        L = ctypes.CDLL(path)
        L.or_prove.restype = ctypes.c_void_p
        L.or_prove.argtypes = [u8p, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, u8p, ctypes.c_uint32, u8p,
                               ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_int]
        L.or_prove_forged.restype = ctypes.c_void_p
        L.or_prove_forged.argtypes = L.or_prove.argtypes + [ctypes.c_int, ctypes.c_int64, ctypes.c_int64]
        L.or_result_error.restype = ctypes.c_char_p
        L.or_result_error.argtypes = [ctypes.c_void_p]
        L.or_result_proof_len.restype = ctypes.c_uint64
        L.or_result_proof_len.argtypes = [ctypes.c_void_p]
        L.or_result_proof.argtypes = [ctypes.c_void_p, u8p]
        L.or_result_stage_ms.argtypes = [ctypes.c_void_p, u8p]
        L.or_result_vector.restype = ctypes.c_uint64
        L.or_result_vector.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint32, u8p]
        L.or_result_free.argtypes = [ctypes.c_void_p]
        L.or_verify.restype = ctypes.c_int
        L.or_verify.argtypes = [u8p, u8p, ctypes.c_uint32, u8p, ctypes.c_uint32, u8p, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint32]
        L.or_set_threads.restype = ctypes.c_int
        L.or_set_threads.argtypes = [ctypes.c_int]
        L.or_field_op.argtypes = [ctypes.c_int, u8p, u8p, u8p]
        L.or_root_of_unity.argtypes = [ctypes.c_uint64, u8p]
        L.or_inv_many.argtypes = [u8p, u8p, ctypes.c_uint64]
        L.or_fft.argtypes = [u8p, ctypes.c_uint64, ctypes.c_int]
        L.or_fft_in_place.argtypes = [u8p, ctypes.c_uint64, u8p, ctypes.c_int]
        L.or_get_twiddles.argtypes = [u8p, ctypes.c_uint64, ctypes.c_int, u8p]
        L.or_poly_eval.argtypes = [u8p, ctypes.c_uint64, u8p, u8p]
        L.or_syn_div.argtypes = [u8p, ctypes.c_uint64, u8p]
        L.or_syn_div_expanded.argtypes = [u8p, ctypes.c_uint64, ctypes.c_uint64, u8p, ctypes.c_uint64]
        L.or_poly_div.restype = ctypes.c_uint64
        L.or_poly_div.argtypes = [u8p, ctypes.c_uint64, u8p, ctypes.c_uint64, u8p]
        L.or_lagrange.argtypes = [u8p, u8p, ctypes.c_uint64, u8p]
        L.or_quartic_interpolate_batch.argtypes = [u8p, u8p, ctypes.c_uint64, u8p]
        L.or_quartic_transpose.argtypes = [u8p, ctypes.c_uint64, ctypes.c_uint64, u8p]
        L.or_quartic_evaluate_batch.argtypes = [u8p, ctypes.c_uint64, u8p, u8p]
        L.or_power_series.argtypes = [u8p, ctypes.c_uint64, u8p]
        L.or_hash.restype = ctypes.c_int
        L.or_hash.argtypes = [ctypes.c_int, u8p, ctypes.c_uint64, u8p]
        L.or_hash_rows.argtypes = [u8p, ctypes.c_uint64, ctypes.c_uint64, u8p]
        L.or_merkle_nodes.restype = ctypes.c_int
        L.or_merkle_nodes.argtypes = [ctypes.c_int, u8p, ctypes.c_uint64, u8p]
        L.or_merkle_prove_batch.restype = ctypes.c_int64
        L.or_merkle_prove_batch.argtypes = [ctypes.c_int, u8p, ctypes.c_uint64, u8p, ctypes.c_uint64, u8p, ctypes.c_uint64]
        L.or_merkle_verify_batch.restype = ctypes.c_int
        L.or_merkle_verify_batch.argtypes = [ctypes.c_int, u8p, u8p, ctypes.c_uint64, u8p, ctypes.c_uint64]
        L.or_prng_vector.argtypes = [u8p, ctypes.c_uint64, u8p]
        L.or_chacha_words.argtypes = [u8p, ctypes.c_uint64, u8p]
        L.or_query_positions.restype = ctypes.c_int
        L.or_query_positions.argtypes = [u8p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64, u8p]
        L.or_find_pow_nonce.restype = ctypes.c_uint64
        L.or_find_pow_nonce.argtypes = [u8p, ctypes.c_uint32, u8p]
        L.or_constraint_coefficients.restype = ctypes.c_uint64
        L.or_constraint_coefficients.argtypes = [u8p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, u8p]
        L.or_hasher_digest.argtypes = [u8p, ctypes.c_uint32, u8p]
        L.or_eval_transition_raw.restype = ctypes.c_uint32
        L.or_eval_transition_raw.argtypes = [u8p, u8p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_uint64, u8p]
        L.or_op_flags.argtypes = [u8p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, u8p]
        L.or_eval_transitions.restype = ctypes.c_int
        L.or_eval_transitions.argtypes = [u8p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_uint32, u8p, ctypes.c_int,
                                          u8p, ctypes.c_char_p, ctypes.c_uint32]
        L.or_decoder_run_raw.restype = ctypes.c_uint32
        L.or_decoder_run_raw.argtypes = [u8p, u8p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, u8p, u8p, u8p]
        L.or_enforce_left_shift.restype = None
        L.or_enforce_left_shift.argtypes = [u8p, u8p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64, u8p, u8p]
        L.or_trace_state_fields.restype = ctypes.c_uint32
        L.or_trace_state_fields.argtypes = [u8p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, u8p]
        L.or_fri_roundtrip.restype = ctypes.c_int
        L.or_fri_roundtrip.argtypes = [u8p, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_uint64]
        L.or_sponge_round.restype = None
        L.or_sponge_round.argtypes = [u8p, u8p, u8p, ctypes.c_uint64]
        _LIB = L
    return _LIB


HASH_IDS = {"blake3": 0, "rescue": 1, "poseidon": 2, "gmimc": 3}
_MASK = 2**64 - 1


def set_threads(t):
    """Host threads of the oracle prover (1 = single thread, what the reference does: every FFT / batch call gets num_threads = 1)."""
    return lib().or_set_threads(int(t))


def _f(v):
    return np.array([v & _MASK, v >> 64], dtype=np.uint64)


def _fi(a):
    a = np.asarray(a, dtype=np.uint64).reshape(-1)
    return int(a[0]) | (int(a[1]) << 64)


def fvec(values):
    a = np.empty((len(values), 2), dtype=np.uint64)
    for i, v in enumerate(values):
        a[i, 0] = v & _MASK
        a[i, 1] = v >> 64
    return a


def ints(a):
    a = np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 2)
    return [int(lo) | (int(hi) << 64) for lo, hi in a]


def field_op(op, a, b=0):
    code = {"add": 0, "sub": 1, "mul": 2, "inv": 3, "exp": 4, "neg": 5}[op]
    out = np.zeros(2, dtype=np.uint64)
    fa, fb = _f(a), _f(b)
    lib().or_field_op(code, fa.ctypes.data, fb.ctypes.data, out.ctypes.data)
    return _fi(out)


def root_of_unity(order):
    out = np.zeros(2, dtype=np.uint64)
    lib().or_root_of_unity(order, out.ctypes.data)
    return _fi(out)


def fft(values, inverse=False):
    """natural-order DFT / inverse DFT of an (n,2) uint64 array; returns a new array"""
    a = np.ascontiguousarray(values, dtype=np.uint64).copy()
    lib().or_fft(a.ctypes.data, a.shape[0], 1 if inverse else 0)
    return a


def hash(name, data):
    out = ctypes.create_string_buffer(32)
    data = bytes(data)
    rc = lib().or_hash(HASH_IDS[name], data, len(data), out)
    if rc != 0:
        raise ValueError("hash failed")
    return out.raw


def merkle_nodes(name, leaves):
    """leaves: bytes of n*32 ; returns bytes n*32 (heap layout)"""
    n = len(leaves) // 32
    out = ctypes.create_string_buffer(n * 32)
    rc = lib().or_merkle_nodes(HASH_IDS[name], bytes(leaves), n, out)
    if rc != 0:
        raise ValueError("merkle failed")
    return out.raw


def merkle_prove_batch(name, leaves, indexes):
    n = len(leaves) // 32
    idx = np.array(indexes, dtype=np.uint64)
    cap = 32 * (len(indexes) + 2) * 70 + 1024
    out = ctypes.create_string_buffer(cap)
    r = lib().or_merkle_prove_batch(HASH_IDS[name], bytes(leaves), n, idx.ctypes.data, len(idx), out, cap)
    if r < 0:
        raise ValueError("prove_batch failed")
    return out.raw[:r]


def merkle_verify_batch(name, root, indexes, proof):
    idx = np.array(indexes, dtype=np.uint64)
    return lib().or_merkle_verify_batch(HASH_IDS[name], bytes(root), idx.ctypes.data, len(idx), bytes(proof), len(proof))


def prng_vector(seed, n):
    out = np.zeros((n, 2), dtype=np.uint64)
    lib().or_prng_vector(bytes(seed), n, out.ctypes.data)
    return ints(out)


def query_positions(seed, domain, ext, nq):
    out = np.zeros(nq, dtype=np.uint64)
    r = lib().or_query_positions(bytes(seed), domain, ext, nq, out.ctypes.data)
    if r < 0:
        raise ValueError("not enough positions")
    return [int(x) for x in out[:r]]


class ProveResult:
    def __init__(self, handle):
        self._h = handle
        L = lib()
        err = L.or_result_error(handle)
        self.error = err.decode() if err else None
        n = L.or_result_proof_len(handle)
        buf = ctypes.create_string_buffer(max(n, 1))
        if n:
            L.or_result_proof(handle, buf)
        self.proof = buf.raw[:n]
        ms = np.zeros(9, dtype=np.float64)
        L.or_result_stage_ms(handle, ms.ctypes.data)
        self.stage_ms = [float(x) for x in ms]

    def vector(self, name, index=0):
        L = lib()
        n = L.or_result_vector(self._h, name.encode(), index, None)
        out = np.zeros((max(n, 1), 2), dtype=np.uint64)
        L.or_result_vector(self._h, name.encode(), index, out.ctypes.data)
        return out[:n]

    def digest(self, name):
        return self.vector(name).tobytes()[:32]

    def digests(self, name):
        raw = self.vector(name).tobytes()
        return [raw[i:i + 32] for i in range(0, len(raw), 32)]

    def u64s(self, name):
        L = lib()
        n = L.or_result_vector(self._h, name.encode(), 0, None)
        out = np.zeros(max(n, 1), dtype=np.uint64)
        L.or_result_vector(self._h, name.encode(), 0, out.ctypes.data)
        return [int(x) for x in out[:n]]

    def __del__(self):
        try:
            lib().or_result_free(self._h)
        except Exception:
            pass


# stark.h Forgery::Kind: what or_prove_forged changes before it is committed
FORGERIES = {"transition": 1, "op_count": 2, "constraint_offset": 3, "deep_value": 4, "fri_offset": 5, "fri_alpha": 6,
             "remainder_point": 7, "layers": 8, "remainder_cut": 9}


def prove(registers, ctx_depth, loop_depth, inputs, outputs, ext=32, num_queries=50, grinding=20, keep_large=False, forge=None):
    """registers: (w, n, 2) uint64 column-major.  Returns ProveResult (check .error).  forge: None for an honest proof, or
    (kind, a[, b]) with kind a key of FORGERIES: a proof of a false statement whose commitments are all consistent (stark.h Forgery)."""
    regs = np.ascontiguousarray(registers, dtype=np.uint64)
    w, n = regs.shape[0], regs.shape[1]
    fi, fo = fvec(list(inputs)), fvec(list(outputs))
    args = (regs.ctypes.data, w, n, ctx_depth, loop_depth, fi.ctypes.data, len(fi), fo.ctypes.data, len(fo), ext, num_queries, grinding,
            1 if keep_large else 0)
    if forge is None:
        return ProveResult(lib().or_prove(*args))
    kind, a, b = (tuple(forge) + (0, 0))[:3]
    return ProveResult(lib().or_prove_forged(*args, FORGERIES[kind], a, b))


def extend(registers, blowup):
    """TraceTable::extend (trace_table.rs:143-169): (w, n, 2) register traces -> (w, n * blowup, 2) evaluations in LDE order"""
    regs = np.ascontiguousarray(registers, dtype=np.uint64)
    w, n = regs.shape[0], regs.shape[1]
    out = np.zeros((w, n * blowup, 2), dtype=np.uint64)
    for j in range(w):
        out[j, :n] = fft(regs[j], inverse=True)
        out[j] = fft(out[j])
    return out


def eval_transitions(ext, ctx_depth, loop_depth, stack_depth, blowup, seed, check):
    """The prover's transition loop over an extended trace: ext (w, n * blowup, 2) uint64 in LDE order, coefficients drawn from the
    32-byte seed.  Returns (values, error): values (8n, 2) in step order; error None, or with check the prover's message for the lowest
    failing step (values then None)."""
    a = np.ascontiguousarray(ext, dtype=np.uint64)
    n = a.shape[1] // blowup
    out = np.zeros((8 * n, 2), dtype=np.uint64)
    err = ctypes.create_string_buffer(512)
    rc = lib().or_eval_transitions(a.ctypes.data, ctx_depth, loop_depth, stack_depth, n, blowup, bytes(seed), 1 if check else 0,
                                   out.ctypes.data, err, 512)
    return (None, err.value.decode()) if rc else (out, None)


def verify(program_hash, inputs, outputs, proof):
    """returns None when the proof verifies, else the error string"""
    fi, fo = fvec(list(inputs)), fvec(list(outputs))
    err = ctypes.create_string_buffer(512)
    rc = lib().or_verify(bytes(program_hash), fi.ctypes.data, len(fi), fo.ctypes.data, len(fo), bytes(proof), len(proof), err, 512)
    return None if rc == 0 else err.value.decode()
