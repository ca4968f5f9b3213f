"""Host-side mirror of the reference's public interface for the prove path (names and argument meaning follow
/root/reference/src/lib.rs:30-75, /root/reference/src/stark/options.rs:16-91, /root/reference/src/stark/proof.rs:10-77)."""
import ctypes

import numpy as np

from . import backend, felt, hostvm


class ProofOptions:
    """stark::ProofOptions (options.rs:29-50): same argument checks, same defaults (options.rs:82-91)."""

    def __init__(self, extension_factor=32, num_queries=50, grinding_factor=20):
        assert extension_factor & (extension_factor - 1) == 0, "extension_factor must be a power of 2"
        assert extension_factor >= 16, "extension_factor cannot be smaller than 16"
        assert extension_factor <= 256, "extension_factor cannot be greater than 256"
        assert num_queries > 0, "num_queries must be greater than 0"
        assert num_queries <= 128, "num_queries cannot be greater than 128"
        assert grinding_factor <= 32, "grinding factor cannot be greater than 32"
        self.extension_factor = extension_factor
        self.num_queries = num_queries
        self.grinding_factor = grinding_factor

    def _c(self):
        return backend.DgOptions(self.extension_factor, self.num_queries, self.grinding_factor, 0)


class StarkProof:
    """Result of prove(): the bincode bytes of the reference's StarkProof plus a few commitments for differential tests."""

    def __init__(self, data, trace_root, constraint_root, pow_seed, pow_nonce, stats):
        self.bytes = data
        self.trace_root = trace_root
        self.constraint_root = constraint_root
        self.pow_seed = pow_seed
        self.pow_nonce = pow_nonce
        self.stats = stats

    def __len__(self):
        return len(self.bytes)


def _collect(handle, stats):
    L = backend.lib()
    try:
        n = ctypes.c_size_t(0)
        backend.check(L.dg_proof_serialized_len(handle, ctypes.byref(n)))
        buf = ctypes.create_string_buffer(n.value)
        backend.check(L.dg_proof_serialize(handle, buf, n.value))
        digs = []
        for which in range(3):
            d = ctypes.create_string_buffer(32)
            backend.check(L.dg_proof_digest(handle, which, d))
            digs.append(d.raw)
        nonce = backend.u64(0)
        backend.check(L.dg_proof_pow_nonce(handle, ctypes.byref(nonce)))
    finally:
        L.dg_proof_free(handle)
    st = {"stage_ms": [float(x) for x in stats.stage_ms], "h2d_ms": float(stats.h2d_ms), "total_ms": float(stats.total_ms),
          "kernel_launches": int(stats.kernel_launches)}
    return StarkProof(buf.raw, digs[0], digs[1], digs[2], nonce.value, st)


def prove(trace, options=None):
    """stark::prove(&mut trace, inputs, outputs, options) for a hostvm.ExecutionTrace (host memory in, proof bytes out)."""
    options = options or ProofOptions()
    regs = np.ascontiguousarray(trace.registers, dtype=np.uint64)
    w, n = regs.shape[0], regs.shape[1]
    cols = (backend.vp * w)(*[regs[j].ctypes.data for j in range(w)])
    t = backend.DgTrace(cols, w, n, trace.ctx_depth, trace.loop_depth)
    fi, fo = felt.from_ints(trace.public_inputs), felt.from_ints(trace.outputs)
    opt = options._c()
    handle = backend.vp()
    stats = backend.DgStats()
    backend.check(backend.lib().dg_prove(ctypes.byref(t), fi.ctypes.data, len(fi), fo.ctypes.data, len(fo), ctypes.byref(opt),
                                        ctypes.byref(handle), ctypes.byref(stats)))
    return _collect(handle, stats)


def prove_device(d_registers, width, length, ctx_depth, loop_depth, public_inputs, outputs, options=None):
    """Same, for register traces already resident in device memory (backend.DeviceBuffer or raw pointer)."""
    options = options or ProofOptions()
    ptr = d_registers.ptr if isinstance(d_registers, backend.DeviceBuffer) else int(d_registers)
    fi, fo = felt.from_ints(public_inputs), felt.from_ints(outputs)
    opt = options._c()
    handle = backend.vp()
    stats = backend.DgStats()
    backend.check(backend.lib().dg_prove_device(ptr, width, length, ctx_depth, loop_depth, fi.ctypes.data, len(fi), fo.ctypes.data, len(fo),
                                               ctypes.byref(opt), ctypes.byref(handle), ctypes.byref(stats)))
    return _collect(handle, stats)


def _batch_io(public_inputs_list, outputs_list):
    """per-trace public inputs / outputs as the pointer and count arrays of dg_prove_batch (the arrays are kept alive by the caller)"""
    ins = [felt.from_ints(x) for x in public_inputs_list]
    outs = [felt.from_ints(x) for x in outputs_list]
    k = len(ins)
    arrays = ((backend.vp * k)(*[a.ctypes.data for a in ins]), (backend.u32 * k)(*[len(a) for a in ins]),
              (backend.vp * k)(*[a.ctypes.data for a in outs]), (backend.u32 * k)(*[len(a) for a in outs]))
    return ins + outs, arrays


def _collect_batch(handles, status, stats):
    """one entry per trace: a StarkProof, or the DgError of a trace that failed with the library's message for it (stats: the
    whole batch)"""
    out = []
    msg = ctypes.create_string_buffer(512)
    for i, (h, rc) in enumerate(zip(handles, status)):
        if rc == 0:
            out.append(_collect(h, stats))
        else:
            backend.check(backend.lib().dg_batch_message(i, msg, len(msg)))
            out.append(backend.DgError(rc, msg.value.decode(errors="replace")))
    return out


def prove_batch(traces, options=None):
    """Proves many hostvm.ExecutionTraces.  Traces of one shape (width, length, ctx_depth, loop_depth) are proven together by one
    dg_prove_batch call, each stage launched once for all of them.  Returns a list in input order: a StarkProof (byte-identical to
    prove() of the same trace) or, for a trace that failed, a backend.DgError instance (returned, not raised).  Errors of a whole call
    (bad options, no device) raise as in prove()."""
    options = options or ProofOptions()
    opt = options._c()
    traces = list(traces)
    groups = {}
    for i, tr in enumerate(traces):
        groups.setdefault((tr.registers.shape[0], tr.registers.shape[1], tr.ctx_depth, tr.loop_depth), []).append(i)
    result = [None] * len(traces)
    for (w, n, ctx_depth, loop_depth), idx in groups.items():
        k = len(idx)
        regs = [np.ascontiguousarray(traces[i].registers, dtype=np.uint64) for i in idx]
        cols = [(backend.vp * w)(*[r[j].ctypes.data for j in range(w)]) for r in regs]
        ts = (backend.DgTrace * k)(*[backend.DgTrace(cols[m], w, n, ctx_depth, loop_depth) for m in range(k)])
        keep, (pin, nin, pout, nout) = _batch_io([traces[i].public_inputs for i in idx], [traces[i].outputs for i in idx])
        handles = (backend.vp * k)()
        status = (ctypes.c_int * k)()
        stats = backend.DgStats()
        backend.check(backend.lib().dg_prove_batch(ts, k, pin, nin, pout, nout, ctypes.byref(opt), handles, status, ctypes.byref(stats)))
        for i, entry in zip(idx, _collect_batch(list(handles), list(status), stats)):
            result[i] = entry
        del keep, regs, cols
    return result


def prove_batch_device(d_registers, count, width, length, ctx_depth, loop_depth, public_inputs_list, outputs_list, options=None):
    """prove_batch for `count` traces of one shape already in device memory: one allocation, proof-major [count][width][length]
    elements (backend.DeviceBuffer or raw pointer).  public_inputs_list / outputs_list hold one list per trace."""
    options = options or ProofOptions()
    assert len(public_inputs_list) == count and len(outputs_list) == count, "one list of public inputs and outputs per trace"
    ptr = d_registers.ptr if isinstance(d_registers, backend.DeviceBuffer) else int(d_registers)
    opt = options._c()
    keep, (pin, nin, pout, nout) = _batch_io(public_inputs_list, outputs_list)
    handles = (backend.vp * max(count, 1))()
    status = (ctypes.c_int * max(count, 1))()
    stats = backend.DgStats()
    backend.check(backend.lib().dg_prove_batch_device(ptr, count, width, length, ctx_depth, loop_depth, pin, nin, pout, nout, ctypes.byref(opt),
                                                     handles, status, ctypes.byref(stats)))
    del keep
    return _collect_batch(list(handles)[:count], list(status)[:count], stats)


def verify(program_hash, public_inputs, outputs, proof):
    """distaff::verify (lib.rs:68-75 -> stark/verifier.rs:11-75) on the GPU.  Returns None when the proof is accepted, otherwise the
    reference's error string (what `Err(msg)` carries); raises DgError for bytes that are not a serialized StarkProof."""
    data = proof.bytes if isinstance(proof, StarkProof) else bytes(proof)
    fi, fo = felt.from_ints(public_inputs), felt.from_ints(outputs)
    msg = ctypes.create_string_buffer(256)
    rc = backend.lib().dg_verify(bytes(program_hash), fi.ctypes.data, len(fi), fo.ctypes.data, len(fo), data, len(data), msg, 256)
    if rc == 0:
        return None
    if rc == -6:
        return msg.value.decode()
    backend.check(rc)


def verify_batch(items, stats=None):
    """verify() of many proofs in one dg_verify_batch call, each verifier stage launched once per group of proofs.  items: iterable of
    (program_hash, public_inputs, outputs, proof), proof a StarkProof or bytes; the proofs may differ in shape, length and options.
    Returns a list in input order: None (accepted), the reference's error string (rejected), or a backend.DgError instance for bytes
    that are not a serialized StarkProof -- returned, not raised, as prove_batch does.  Errors of the whole call raise.  A dict passed as
    `stats` receives total_ms, kernel_launches and groups."""
    items = list(items)
    if not items:
        return []
    k = len(items)
    hashes = [bytes(h) for h, _, _, _ in items]
    data = [p.bytes if isinstance(p, StarkProof) else bytes(p) for _, _, _, p in items]
    keep, (pin, nin, pout, nout) = _batch_io([i for _, i, _, _ in items], [o for _, _, o, _ in items])
    status = (ctypes.c_int * k)()
    st = backend.DgVerifyStats()
    backend.check(backend.lib().dg_verify_batch(k, (backend.vp * k)(*[ctypes.cast(ctypes.c_char_p(h), backend.vp) for h in hashes]), pin, nin, pout,
                                                nout, (backend.vp * k)(*[ctypes.cast(ctypes.c_char_p(d), backend.vp) for d in data]),
                                                (ctypes.c_size_t * k)(*[len(d) for d in data]), status, ctypes.byref(st)))
    del keep
    out = []
    msg = ctypes.create_string_buffer(512)
    for i, rc in enumerate(status):
        if rc == 0:
            out.append(None)
            continue
        backend.check(backend.lib().dg_batch_message(i, msg, len(msg)))
        text = msg.value.decode(errors="replace")
        out.append(text if rc == -6 else backend.DgError(rc, text))
    if stats is not None:
        stats.update(total_ms=float(st.total_ms), kernel_launches=int(st.kernel_launches), groups=int(st.groups))
    return out


def execute(source, public_inputs=(), secret_a=(), secret_b=(), num_outputs=1, options=None):
    """distaff::execute (lib.rs:30-65): run the program on the host VM, then prove on the GPU. Returns (outputs, proof)."""
    trace = hostvm.execute(source, public_inputs, secret_a, secret_b, num_outputs)
    return trace.outputs, prove(trace, options)


# ---- building blocks ------------------------------------------------------------------------------------------------------
def ntt(values, inverse=False):
    """polynom::eval_fft / interpolate_fft on (batch, n, 2) or (n, 2) uint64 arrays; returns a new array"""
    a = np.ascontiguousarray(values, dtype=np.uint64).copy()
    shape = a.shape
    n = shape[-2]
    batch = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
    assert n & (n - 1) == 0 and n >= 2
    backend.check(backend.lib().dg_ntt(a.ctypes.data, n.bit_length() - 1, batch, 1 if inverse else 0))
    return a


def intt(values):
    return ntt(values, inverse=True)


def lde(values, blowup=32):
    """TraceTable::extend for a (batch, n, 2) array of register traces: returns (batch, n*blowup, 2) evaluations in LDE order"""
    a = np.ascontiguousarray(values, dtype=np.uint64)
    if a.ndim == 2:
        a = a[None]
    batch, n = a.shape[0], a.shape[1]
    out = np.empty((batch, n * blowup, 2), dtype=np.uint64)
    backend.check(backend.lib().dg_lde(a.ctypes.data, out.ctypes.data, n.bit_length() - 1, blowup.bit_length() - 1, batch))
    return out


HASH_IDS = {"blake3": 0, "rescue": 1, "poseidon": 2}


def merkle_build(leaves, hash="blake3"):
    """crypto::build_merkle_nodes (merkle.rs:269-294): bytes (n*32) -> bytes (n*32), heap layout; hash in blake3 | rescue | poseidon"""
    leaves = bytes(leaves)
    n = len(leaves) // 32
    out = ctypes.create_string_buffer(n * 32)
    if hash == "blake3":
        backend.check(backend.lib().dg_merkle_build(leaves, n, out))
    else:
        backend.check(backend.lib().dg_merkle_build_with(HASH_IDS[hash], leaves, n, out))
    return out.raw


def hash64(messages, hash="rescue"):
    """crypto::hash::{blake3, rescue, poseidon} of n independent 64-byte messages: bytes (n*64) -> bytes (n*32)"""
    messages = bytes(messages)
    assert len(messages) % 64 == 0
    n = len(messages) // 64
    out = ctypes.create_string_buffer(max(1, n * 32))
    backend.check(backend.lib().dg_hash64(HASH_IDS[hash], messages, n, out))
    return out.raw[:n * 32]


def hash_rows(columns):
    """blake3 of every row of a column-major (w, rows, 2) uint64 matrix -> bytes rows*32"""
    a = np.ascontiguousarray(columns, dtype=np.uint64)
    w, rows = a.shape[0], a.shape[1]
    out = ctypes.create_string_buffer(rows * 32)
    backend.check(backend.lib().dg_hash_rows(a.ctypes.data, w, rows, out))
    return out.raw


def find_pow_nonce(seed, grinding_factor=20):
    nonce = backend.u64(0)
    out = ctypes.create_string_buffer(32)
    backend.check(backend.lib().dg_find_pow_nonce(bytes(seed), grinding_factor, ctypes.byref(nonce), out))
    return out.raw, nonce.value


def field_op(op, a, b=None, impl=0):
    code = {"add": 0, "sub": 1, "mul": 2, "inv": 3, "exp": 4, "dot6": 5}[op]
    fa = np.ascontiguousarray(a, dtype=np.uint64)
    fb = np.ascontiguousarray(b, dtype=np.uint64) if b is not None else None
    out = np.empty_like(fa)
    backend.check(backend.lib().dg_field_op(code, impl, fa.ctypes.data, fb.ctypes.data if fb is not None else None, out.ctypes.data, fa.shape[0]))
    return out[:fa.shape[0] // 6] if op == "dot6" else out


def field_dot(a, b, length):
    """sum of `length` products per group, accumulated unreduced as the kernels do: (groups * length, 2) arrays -> (groups, 2)"""
    fa = np.ascontiguousarray(a, dtype=np.uint64)
    fb = np.ascontiguousarray(b, dtype=np.uint64)
    assert fa.shape == fb.shape and fa.shape[0] % length == 0
    out = np.empty((fa.shape[0] // length, 2), dtype=np.uint64)
    backend.check(backend.lib().dg_field_dot(fa.ctypes.data, fb.ctypes.data, out.ctypes.data, out.shape[0], length))
    return out


def eval_transitions(ext, ctx_depth, loop_depth, stack_depth, blowup, seeds=None, coefs=None, check=False):
    """The prover's constraint kernel on extended traces: ext (count, w, n * blowup, 2) uint64 in LDE order.  Entry i combines its
    transition constraints with the coefficients drawn from seeds[i] (32 bytes) or, if given, coefs[i] ((2T, 2): coefA then coefB in
    evaluation order).  Returns (values (count, 8n, 2) in step order, first_violation: per entry 0 or 1 + the lowest violating trace
    step; only with check, which is the prover's trace-domain check)."""
    a = np.ascontiguousarray(ext, dtype=np.uint64)
    count, w, N = a.shape[0], a.shape[1], a.shape[2]
    assert w == 15 + ctx_depth + loop_depth + stack_depth and N % blowup == 0
    n = N // blowup
    assert n & (n - 1) == 0 and blowup & (blowup - 1) == 0, "trace length and extension factor must be powers of 2"
    T = 20 + max(ctx_depth, 1) + max(loop_depth, 1) + 2 + stack_depth
    sd = b"".join(bytes(s) for s in seeds) if seeds is not None else None
    cf = np.ascontiguousarray(coefs, dtype=np.uint64) if coefs is not None else None
    assert (sd is not None and len(sd) == 32 * count) or (cf is not None and cf.shape == (count, 2 * T, 2))
    out = np.empty((count, 8 * n, 2), dtype=np.uint64)
    first = (backend.u32 * count)()
    backend.check(backend.lib().dg_eval_transitions(a.ctypes.data, count, ctx_depth, loop_depth, stack_depth, n.bit_length() - 1,
                                                   blowup.bit_length() - 1, sd, cf.ctypes.data if cf is not None else None,
                                                   1 if check else 0, out.ctypes.data, first))
    return out, list(first)
