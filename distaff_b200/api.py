"""Host-side mirror of the reference's public interface for the prove path (names and argument meaning follow
/root/reference/src/lib.rs:30-75, /root/reference/src/stark/options.rs:16-91, /root/reference/src/stark/proof.rs:10-77)."""
import ctypes
import functools

import numpy as np

from . import backend, felt, hostvm


MAX_CONSTRAINT_DEGREE = 8       # stark/mod.rs: the constraint evaluation domain is 8 times the trace domain


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

    def security_level(self, optimistic=True):
        """ProofOptions::security_level (options.rs:68-79): log2(extension_factor / MAX_CONSTRAINT_DEGREE) bits per query, over all
        queries (optimistic) or half of them; the grinding factor is added once that reaches 80 bits."""
        security_factor = (self.extension_factor // MAX_CONSTRAINT_DEGREE).bit_length() - 1
        queries = self.num_queries if optimistic else self.num_queries // 2
        level = security_factor * queries
        return level + self.grinding_factor if level >= 80 else level

    def _key(self):
        return (self.extension_factor, self.num_queries, self.grinding_factor)

    def __eq__(self, other):
        return isinstance(other, ProofOptions) and self._key() == other._key()

    def __hash__(self):
        return hash(self._key())

    def __repr__(self):
        return "ProofOptions(extension_factor=%d, num_queries=%d, grinding_factor=%d)" % self._key()


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

    @property
    def options(self):
        """The ProofOptions the proof was made with: the last four bytes of its bincode (proof.rs:21, options.rs:15-23), log2 of the
        extension factor, num_queries, grinding_factor and the hash id (0, blake3)."""
        if len(self.bytes) < 4:
            raise ValueError("proof bytes too short to hold proof options")
        log_b, queries, grinding, hash_id = self.bytes[-4:]
        if hash_id != 0:
            raise ValueError("proof options name hash function %d; only blake3 (0) is serialisable" % hash_id)
        return ProofOptions(1 << log_b, queries, grinding)


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


def _dev_ptr(x):
    """the address of device memory given as a backend.DeviceBuffer or a raw pointer"""
    return x.ptr if isinstance(x, backend.DeviceBuffer) else int(x)


def _c_traces(traces):
    """the dg_trace_t array of hostvm.ExecutionTraces, and what keeps their columns alive"""
    regs = [np.ascontiguousarray(tr.registers, dtype=np.uint64) for tr in traces]
    cols = [(backend.vp * r.shape[0])(*[r[j].ctypes.data for j in range(r.shape[0])]) for r in regs]
    ts = (backend.DgTrace * max(len(traces), 1))(*[backend.DgTrace(c, r.shape[0], r.shape[1], tr.ctx_depth, tr.loop_depth)
                                                   for c, r, tr in zip(cols, regs, traces)])
    return ts, (regs, cols)


def _by_shape(traces):
    """{(width, length, ctx_depth, loop_depth): indices of the traces of that shape}, shapes in order of first appearance"""
    groups = {}
    for i, tr in enumerate(traces):
        groups.setdefault((tr.registers.shape[0], tr.registers.shape[1], tr.ctx_depth, tr.loop_depth), []).append(i)
    return groups


def _prove_one(entry, head, public_inputs, outputs, options):
    """entry(*head, inputs, outputs, options, proof, stats) for one trace (dg_prove, dg_prove_device): its StarkProof"""
    fi, fo = felt.from_ints(public_inputs), felt.from_ints(outputs)
    opt = (options or ProofOptions())._c()
    handle = backend.vp()
    stats = backend.DgStats()
    backend.check(entry(*head, fi.ctypes.data, len(fi), fo.ctypes.data, len(fo), ctypes.byref(opt), ctypes.byref(handle), ctypes.byref(stats)))
    return _collect(handle, stats)


def prove(trace, options=None):
    """stark::prove(&mut trace, inputs, outputs, options) for a hostvm.ExecutionTrace (host memory in, proof bytes out)."""
    ts, keep = _c_traces([trace])
    return _prove_one(backend.lib().dg_prove, (ts,), trace.public_inputs, trace.outputs, options)


def prove_device(d_registers, width, length, ctx_depth, loop_depth, public_inputs, outputs, options=None):
    """Same, for register traces already resident in device memory (backend.DeviceBuffer or raw pointer)."""
    return _prove_one(backend.lib().dg_prove_device, (_dev_ptr(d_registers), width, length, ctx_depth, loop_depth), public_inputs, outputs,
                      options)


def set_memory_limit(nbytes):
    """dg_set_memory_limit: the most device memory (bytes) the library may hold on the current device; 0 or None removes the limit.
    Shapes whose trace extension does not fit under it are proven in the evaluation-coset layout, with the same proof bytes."""
    nbytes = 0 if nbytes is None else int(nbytes)
    if nbytes < 0:
        raise ValueError("memory limit must be a non-negative number of bytes")
    backend.check(backend.lib().dg_set_memory_limit(nbytes))


def memory_usage():
    """dg_memory_usage: {"held": bytes the library holds now, "peak": the most it has held since the limit was last set}."""
    held, peak = ctypes.c_size_t(0), ctypes.c_size_t(0)
    backend.check(backend.lib().dg_memory_usage(ctypes.byref(held), ctypes.byref(peak)))
    return {"held": held.value, "peak": peak.value}


def plan_prove(width, length, count=1, options=None):
    """dg_plan_prove: what proving `count` traces of width x length would do, without running it: the layout ("full" or "eval_cosets"),
    the group size, the cosets extended per chunk and kept, bytes per proof and the fixed bytes beside them."""
    options = options or ProofOptions()
    width, length, count = int(width), int(length), int(count)
    if not 1 <= width < 128:
        raise ValueError("width must be in 1..127")
    if length < 16 or length & (length - 1):
        raise ValueError("length must be a power of 2 and at least 16")
    if count < 1:
        raise ValueError("count must be at least 1")
    opt = options._c()
    plan = backend.DgProvePlan()
    backend.check(backend.lib().dg_plan_prove(width, length, count, ctypes.byref(opt), ctypes.byref(plan)))
    return {"layout": "full" if plan.layout == 0 else "eval_cosets", "group": plan.group, "coset_chunk": plan.coset_chunk,
            "retained_cosets": plan.retained_cosets, "bytes_per_proof": plan.bytes_per_proof, "fixed_bytes": plan.fixed_bytes,
            "available_bytes": plan.available_bytes}


def _batch_io(public_inputs_list, outputs_list):
    """per-trace public inputs / outputs as the pointer and count arrays of dg_prove_batch (the arrays are kept alive by the caller)"""
    ins = [felt.from_ints(x) for x in public_inputs_list]
    outs = [felt.from_ints(x) for x in outputs_list]
    k = len(ins)
    arrays = ((backend.vp * k)(*[a.ctypes.data for a in ins]), (backend.u32 * k)(*[len(a) for a in ins]),
              (backend.vp * k)(*[a.ctypes.data for a in outs]), (backend.u32 * k)(*[len(a) for a in outs]))
    return ins + outs, arrays


def _messages(status, error=backend.DgError):
    """per entry of the thread's last batched call: None when it succeeded, else error(code, the library's message for it)"""
    msg = ctypes.create_string_buffer(512)
    out = []
    for i, rc in enumerate(status):
        if rc != 0:
            backend.check(backend.lib().dg_batch_message(i, msg, len(msg)))
        out.append(None if rc == 0 else error(rc, msg.value.decode(errors="replace")))
    return out


def _collect_batch(handles, status, stats):
    """one entry per trace: a StarkProof, or the DgError of a trace that failed with the library's message for it (stats: the
    whole batch)"""
    return [_collect(h, stats) if e is None else e for h, e in zip(handles, _messages(status))]


def _prove_batched(entry, head, public_inputs_list, outputs_list, opt):
    """entry(*head, public inputs / outputs, opt, proofs, status, stats) for a batched prove call, one trace per list of public inputs:
    _collect_batch of its results"""
    k = len(public_inputs_list)
    keep, io = _batch_io(public_inputs_list, outputs_list)
    handles = (backend.vp * max(k, 1))()
    status = (ctypes.c_int * max(k, 1))()
    stats = backend.DgStats()
    backend.check(entry(*head, *io, opt, handles, status, ctypes.byref(stats)))
    return _collect_batch(list(handles)[:k], list(status)[:k], stats)


def prove_batch(traces, options=None):
    """Proves many hostvm.ExecutionTraces.  Traces of one shape (width, length, ctx_depth, loop_depth) are proven together by one
    dg_prove_batch call, each stage launched once for all of them.  Returns a list in input order: a StarkProof (byte-identical to
    prove() of the same trace) or, for a trace that failed, a backend.DgError instance (returned, not raised).  Errors of a whole call
    (bad options, no device) raise as in prove()."""
    options = options or ProofOptions()
    opt = options._c()
    traces = list(traces)
    result = [None] * len(traces)
    for idx in _by_shape(traces).values():
        ts, keep = _c_traces([traces[i] for i in idx])
        proofs = _prove_batched(backend.lib().dg_prove_batch, (ts, len(idx)), [traces[i].public_inputs for i in idx],
                                [traces[i].outputs for i in idx], ctypes.byref(opt))
        for i, entry in zip(idx, proofs):
            result[i] = entry
    return result


def prove_batch_device(d_registers, count, width, length, ctx_depth, loop_depth, public_inputs_list, outputs_list, options=None):
    """prove_batch for `count` traces of one shape already in device memory: one allocation, proof-major [count][width][length]
    elements (backend.DeviceBuffer or raw pointer).  public_inputs_list / outputs_list hold one list per trace."""
    options = options or ProofOptions()
    assert len(public_inputs_list) == count and len(outputs_list) == count, "one list of public inputs and outputs per trace"
    opt = options._c()
    return _prove_batched(backend.lib().dg_prove_batch_device, (_dev_ptr(d_registers), count, width, length, ctx_depth, loop_depth),
                          public_inputs_list, outputs_list, ctypes.byref(opt))


def _options_arg(options, k, what):
    """(the C options argument, whether it holds one entry per trace / job): one ProofOptions (None: the defaults) for all k, or a
    list of k ProofOptions"""
    if options is None or isinstance(options, ProofOptions):
        return ctypes.byref((options or ProofOptions())._c()), False
    options = list(options)
    if len(options) != k:
        raise ValueError("options: one ProofOptions per %s, %d for %d %ss" % (what, len(options), k, what))
    for o in options:
        if not isinstance(o, ProofOptions):
            raise TypeError("options: each entry must be a ProofOptions, not %s" % type(o).__name__)
    return (backend.DgOptions * max(k, 1))(*[o._c() for o in options]), True


def prove_traces(traces, options=None):
    """Proves many hostvm.ExecutionTraces of any register shapes and lengths in one dg_prove_traces call: every stage is launched once
    per group of traces of one length, whatever their shapes (the constraint evaluation once per shape).  Returns what prove_batch
    returns, in input order: a StarkProof byte-identical to prove() of the same trace (its stats: the whole call's), or the
    backend.DgError of a trace that failed.  options: one ProofOptions for every trace, or a list with one per trace
    (dg_prove_traces_with_options): each proof is then prove() of its trace with its options, and the call runs in groups of one length
    and extension factor."""
    traces = list(traces)
    k = len(traces)
    opt, per_trace = _options_arg(options, k, "trace")
    ts, keep = _c_traces(traces)
    fn = backend.lib().dg_prove_traces_with_options if per_trace else backend.lib().dg_prove_traces
    return _prove_batched(fn, (ts, k), [tr.public_inputs for tr in traces], [tr.outputs for tr in traces], opt)


def prove_traces_device(d_registers, widths, lengths, ctx_depths, loop_depths, public_inputs_list, outputs_list, options=None):
    """prove_traces for traces already in device memory: trace i's widths[i] x lengths[i] registers (column-major) at d_registers[i]
    (backend.DeviceBuffer or raw pointer); the other arguments hold one entry per trace.  options as in prove_traces."""
    k = len(d_registers)
    assert all(len(a) == k for a in (widths, lengths, ctx_depths, loop_depths, public_inputs_list, outputs_list)), "one entry per trace"
    opt, per_trace = _options_arg(options, k, "trace")
    ptrs = (backend.vp * max(k, 1))(*[_dev_ptr(d) for d in d_registers])
    arr = lambda t, xs: (t * max(k, 1))(*[int(x) for x in xs])
    fn = backend.lib().dg_prove_traces_device_with_options if per_trace else backend.lib().dg_prove_traces_device
    head = (ptrs, arr(backend.u32, widths), arr(backend.u64, lengths), arr(backend.u32, ctx_depths), arr(backend.u32, loop_depths), k)
    return _prove_batched(fn, head, public_inputs_list, outputs_list, opt)


def group_traces(lengths, widths, ctx_depths, loop_depths, footprints, budget, cap, extension_factors=None):
    """dg_host_group_traces (no device): the groups prove_traces runs, as lists of trace indices in device order.  With
    extension_factors (one per trace; dg_host_group_traces_with_options) the partitions are those of per-trace options: one per
    (length, extension factor)."""
    k = len(lengths)
    arr = lambda t, xs: (t * max(k, 1))(*[int(x) for x in xs])
    order = (backend.u32 * max(k, 1))()
    sizes = (backend.u32 * max(k, 1))()
    n = backend.u32(0)
    rest = (arr(backend.u32, widths), arr(backend.u32, ctx_depths), arr(backend.u32, loop_depths), arr(backend.u64, footprints), int(budget),
            int(cap), order, sizes, ctypes.byref(n))
    if extension_factors is None:
        backend.check(backend.lib().dg_host_group_traces(k, arr(backend.u64, lengths), *rest))
    else:
        if len(extension_factors) != k:
            raise ValueError("extension_factors: one per trace, %d for %d traces" % (len(extension_factors), k))
        backend.check(backend.lib().dg_host_group_traces_with_options(k, arr(backend.u64, lengths), arr(backend.u32, extension_factors), *rest))
    out, at = [], 0
    for s in list(sizes)[:n.value]:
        out.append(list(order)[at:at + s])
        at += s
    return out


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
    out = _messages(status, lambda rc, text: text if rc == -6 else backend.DgError(rc, text))
    if stats is not None:
        stats.update(total_ms=float(st.total_ms), kernel_launches=int(st.kernel_launches), groups=int(st.groups))
    return out


# ---- checking a trace before proving it ---------------------------------------------------------------------------------------------
_NO_STEP = 2**64 - 1
MIN_OP_COUNT = 16           # lib.rs:48-52 (MIN_TRACE_LENGTH)


def constraint_name(ctx_depth, loop_depth, stack_depth, index):
    """name of transition constraint `index` (evaluation order) of a register shape: "op bit 3 binary", "sponge 1", "stack slot 5", ..."""
    buf = ctypes.create_string_buffer(64)
    backend.check(backend.lib().dg_host_constraint_name(ctx_depth, loop_depth, stack_depth, index, buf, len(buf)))
    return buf.value.decode()


def register_name(r, ctx_depth, loop_depth):
    """name of register r of the trace layout (trace_state.rs:115-118)"""
    if r == 0:
        return "op counter"
    for base, count, name in ((1, 4, "sponge"), (5, 3, "cf op bit"), (8, 5, "ld op bit"), (13, 2, "hd op bit"), (15, ctx_depth, "ctx stack"),
                              (15 + ctx_depth, loop_depth, "loop stack")):
        if r < base + count:
            return "%s %d" % (name, r - base)
    return "user stack %d" % (r - 15 - ctx_depth - loop_depth)


class TraceReport:
    """What check_trace finds in one trace, before any proving.
      ok                    no transition or boundary constraint fails, the op count is >= 16 and the program hash (if given) matches
      first_step            lowest trace step at which a transition constraint fails, or None (the last step, n - 1 -> 0, is exempt)
      violating_steps       number of such steps
      transitions           {constraint name: (steps at which it fails, its lowest such step)}, only the constraints that fail
      boundary              readable strings, one per register of the first or last row that breaks a boundary assertion
      first_row_registers / last_row_registers   those registers' indexes
      op_count              op counter of the last row; program_hash_matches 1, 0, or -1 when no hash was given
      masks                 (n, 3) uint32: bit j of word j // 32 at step k = constraint j fails at k (None unless asked for)"""

    def __init__(self, raw, shape, length, value_of, inputs, outputs, masks=None):
        ctx_depth, loop_depth, stack_depth = shape
        self.length = length
        self.n_constraints = int(raw.n_constraints)
        self.violating_steps = int(raw.violating_steps)
        self.first_step = None if raw.first_step == _NO_STEP else int(raw.first_step)
        self.transitions = {}
        for j in (range(self.n_constraints) if self.first_step is not None else ()):
            if raw.constraint_steps[j]:
                self.transitions[constraint_name(ctx_depth, loop_depth, stack_depth, j)] = (int(raw.constraint_steps[j]), int(raw.constraint_first[j]))
        stk = 15 + ctx_depth + loop_depth
        def registers(words):
            bits = int(words[0]) | (int(words[1]) << 64)
            return [r for r in range(128) if (bits >> r) & 1] if bits else []
        self.first_row_registers = registers(raw.first_row_registers)
        self.last_row_registers = registers(raw.last_row_registers)
        self.boundary = []
        for row, regs, claimed, what in (("first row", self.first_row_registers, inputs, "input"), ("last row", self.last_row_registers, outputs, "output")):
            for r in regs:
                if r >= stk:
                    expected = "%s %d" % (what, claimed[r - stk])
                else:
                    expected = "1" if row == "last row" and 5 <= r < 15 else "0"
                self.boundary.append("%s: %s (register %d) is %d, expected %s" % (
                    row, register_name(r, ctx_depth, loop_depth), r, value_of(row == "last row", r), expected))
        self.op_count = int(raw.op_count)
        self.op_count_ok = bool(raw.op_count_ok)
        self.program_hash_matches = int(raw.program_hash_matches)
        self.masks = masks

    @property
    def ok(self):
        return self.first_step is None and not self.boundary and self.op_count_ok and self.program_hash_matches != 0

    def __str__(self):
        if self.ok:
            return "trace ok: %d steps, %d operations" % (self.length, self.op_count)
        lines = []
        if self.first_step is not None:
            lines.append("transition constraints fail at %d of %d steps, first at step %d:" % (self.violating_steps, self.length - 1, self.first_step))
            lines += ["  %s: %d steps, first at step %d" % (name, s, f) for name, (s, f) in sorted(self.transitions.items(), key=lambda e: e[1][1])]
        if self.boundary:
            lines.append("boundary constraints fail:")
            lines += ["  " + b for b in self.boundary]
        if not self.op_count_ok:
            lines.append("the trace executes %d operations; a proof needs at least %d" % (self.op_count, MIN_OP_COUNT))
        if self.program_hash_matches == 0:
            lines.append("the program hash in the last row's sponge does not match the expected hash")
        return "\n".join(lines)

    __repr__ = __str__


def _hashes(program_hashes, count):
    if program_hashes is None:
        return None
    hs = [bytes(h) for h in program_hashes]
    assert len(hs) == count and all(len(h) == 32 for h in hs), "one 32-byte program hash per trace"
    return b"".join(hs)


def check_traces(traces, program_hashes=None, masks=False):
    """Checks hostvm.ExecutionTraces without proving them: one GPU pass per group of same-shape traces (dg_check_traces) evaluates every
    transition constraint at every step, and the first and last rows are compared with the boundary assertions for the trace's public
    inputs and outputs.  program_hashes: None, or one 32-byte hash per trace.  Returns a TraceReport per trace, in input order."""
    traces = list(traces)
    if program_hashes is not None:
        program_hashes = list(program_hashes)
    result = [None] * len(traces)
    for (w, n, ctx_depth, loop_depth), idx in _by_shape(traces).items():
        k = len(idx)
        ts, (regs, cols) = _c_traces([traces[i] for i in idx])
        keep, (pin, nin, pout, nout) = _batch_io([traces[i].public_inputs for i in idx], [traces[i].outputs for i in idx])
        hashes = _hashes([program_hashes[i] for i in idx], k) if program_hashes is not None else None
        reports = (backend.DgTraceReport * k)()
        step_masks = np.zeros((k, n, 3), dtype=np.uint32) if masks else None
        backend.check(backend.lib().dg_check_traces(ts, k, pin, nin, pout, nout, hashes, reports,
                                                    step_masks.ctypes.data if masks else None))
        shape = (ctx_depth, loop_depth, w - 15 - ctx_depth - loop_depth)
        for m, i in enumerate(idx):
            tr = traces[i]
            value_of = (lambda last, r, a=regs[m]: felt.to_ints(a[r, n - 1 if last else 0])[0])
            result[i] = TraceReport(reports[m], shape, n, value_of, list(tr.public_inputs), list(tr.outputs),
                                    step_masks[m] if masks else None)
        del keep, cols
    return result


def check_trace(trace, program_hash=None, masks=False):
    """check_traces of one trace: a TraceReport.  program_hash (32 bytes) is compared with the last row's sponge; masks=True also returns
    the per-step masks of failing constraints (report.masks, (n, 3) uint32)."""
    return check_traces([trace], None if program_hash is None else [program_hash], masks=masks)[0]


def check_traces_device(d_registers, count, width, length, ctx_depth, loop_depth, public_inputs_list, outputs_list, program_hashes=None,
                        d_masks=None):
    """check_traces for `count` traces of one shape already in device memory, proof-major [count][width][length] elements
    (backend.DeviceBuffer or raw pointer), used in place.  d_masks: None, or device memory of count * length * 3 uint32 that receives
    the per-step masks.  Returns a TraceReport per trace."""
    assert len(public_inputs_list) == count and len(outputs_list) == count, "one list of public inputs and outputs per trace"
    ptr = _dev_ptr(d_registers)
    mptr = None if d_masks is None else _dev_ptr(d_masks)
    keep, (pin, nin, pout, nout) = _batch_io(public_inputs_list, outputs_list)
    reports = (backend.DgTraceReport * max(count, 1))()
    backend.check(backend.lib().dg_check_traces_device(ptr, count, width, length, ctx_depth, loop_depth, pin, nin, pout, nout,
                                                       _hashes(program_hashes, count), reports, mptr))
    del keep

    def value_of(q, last, r):
        v = np.zeros(2, dtype=np.uint64)
        offset = ((q * width + r) * length + (length - 1 if last else 0)) * 16
        backend.check(backend.lib().dg_dev_download(v.ctypes.data, ptr + offset, 16))
        return felt.to_ints(v)[0]
    shape = (ctx_depth, loop_depth, width - 15 - ctx_depth - loop_depth)
    return [TraceReport(reports[q], shape, length, functools.partial(value_of, q), list(public_inputs_list[q]), list(outputs_list[q]))
            for q in range(count)]


def execute(source, public_inputs=(), secret_a=(), secret_b=(), num_outputs=1, options=None):
    """distaff::execute (lib.rs:30-65): run the program on the host VM, then prove on the GPU. Returns (outputs, proof)."""
    trace = hostvm.execute(source, public_inputs, secret_a, secret_b, num_outputs)
    return trace.outputs, prove(trace, options)


# ---- one program, many inputs, executed on the GPU ---------------------------------------------------------------------------------
MAX_STEPS = 2**22           # the longest trace the project plans for


class ProgramInputs:
    """ProgramInputs::new (programs/inputs.rs:12): public inputs (at most 8, else that execution fails) and the secret tapes A and B."""

    def __init__(self, public=(), secret_a=(), secret_b=()):
        self.public = [int(x) for x in public]
        self.secret_a = [int(x) for x in secret_a]
        self.secret_b = [int(x) for x in secret_b]


def _programs_args(jobs):
    """the dg_program_t table, program_of, dg_program_inputs_t array and num_outputs of a call (plus what they point into)"""
    programs, program_of, inputs, num_outputs = pack_jobs(jobs)
    k = len(inputs)
    cprogs = (backend.DgProgram * len(programs))(*[p.c_struct() for p in programs])
    arr = (backend.DgProgramInputs * k)()
    keep = [programs, cprogs]
    for i, x in enumerate(inputs):
        vals = [felt.from_ints(v) for v in (x.public, x.secret_a, x.secret_b)]
        keep += vals
        arr[i] = backend.DgProgramInputs(vals[0].ctypes.data, len(vals[0]), vals[1].ctypes.data, len(vals[1]), vals[2].ctypes.data, len(vals[2]))
    return programs, cprogs, (backend.u32 * k)(*program_of), arr, num_outputs, keep


def _execution_args(program, inputs):
    """the one-program case of _programs_args: the hostvm.Program, its dg_program_t, the dg_program_inputs_t array (plus what they point
    into, to keep alive)"""
    (prog,), cprogs, _, arr, _, keep = _programs_args([(program, x) for x in inputs])
    return prog, cprogs[0], arr, keep


def _fields(st, into=None):
    """a ctypes structure as a dict, also written into `into` when given: *_ms fields as floats, other numbers as ints, a nested
    structure as a dict"""
    d = {}
    for f, _ in st._fields_:
        v = getattr(st, f)
        d[f] = _fields(v) if isinstance(v, ctypes.Structure) else (float if f.endswith("_ms") else int)(v)
    if into is not None:
        into.update(d)
    return d


def _traces(call, jobs, programs, program_of, num_outputs):
    """The trace calls: call(info, registers_out, status) once without registers to size the buffers, then with one buffer per execution
    that call let through.  Returns a list in job order: a hostvm.ExecutionTrace with num_outputs[i] outputs, or the DgError of an
    execution that failed."""
    k = len(jobs)
    info = (backend.DgExecutionInfo * k)()
    status = (ctypes.c_int * k)()
    backend.check(call(info, None, status))
    regs = [np.empty((info[i].width, info[i].length, 2), dtype=np.uint64) if status[i] == 0 else None for i in range(k)]
    backend.check(call(info, (backend.vp * k)(*[r.ctypes.data if r is not None else None for r in regs]), status))
    result = _messages(status)
    for i, job in enumerate(jobs):
        if result[i] is None:
            sd, start, n = info[i].stack_depth, 15 + info[i].ctx_depth + info[i].loop_depth, info[i].length
            last = [felt.to_ints(regs[i][start + j, n - 1])[0] if j < sd else 0 for j in range(8)]
            result[i] = hostvm.ExecutionTrace(regs[i], info[i].ctx_depth, info[i].loop_depth, sd, programs[program_of[i]].hash,
                                              list(job[1].public), last[:num_outputs[i]])
    return result


def _proofs(call, num_outputs, per=8):
    """The execute calls: call(proofs_out, outputs16, status, prove_stats) with room for `per` output elements per execution.  Returns a
    list in execution order: (outputs, StarkProof), or the DgError of an execution that failed."""
    k = len(num_outputs)
    handles = (backend.vp * k)()
    outputs = np.zeros((k, per, 2), dtype=np.uint64)
    status = (ctypes.c_int * k)()
    pst = backend.DgStats()
    backend.check(call(handles, outputs.ctypes.data, status, ctypes.byref(pst)))
    return [e if e is not None else (felt.to_ints(outputs[i, :num_outputs[i]]) if num_outputs[i] else [], _collect(handles[i], pst))
            for i, e in enumerate(_messages(status))]


def trace_shapes(program, inputs, max_steps=MAX_STEPS):
    """The shape pass of dg_trace_batch alone: per input, a dict (width, length, steps, ctx_depth, loop_depth, stack_depth) or the
    DgError of an execution that failed."""
    inputs = list(inputs)
    if not inputs:
        return []
    _, cprog, arr, keep = _execution_args(program, inputs)
    k = len(inputs)
    info = (backend.DgExecutionInfo * k)()
    status = (ctypes.c_int * k)()
    backend.check(backend.lib().dg_trace_batch(ctypes.byref(cprog), k, arr, int(max_steps), info, None, status))
    return [e if e is not None else _fields(info[i]) for i, e in enumerate(_messages(status))]


def trace_batch(program, inputs, max_steps=MAX_STEPS, num_outputs=1):
    """processor::execute of one program (a hostvm.Program or assembly source) for every ProgramInputs, on the GPU, one thread per
    execution.  Returns a list in input order: a hostvm.ExecutionTrace (what hostvm.execute gives for the same inputs, byte for byte)
    or the DgError of an execution that failed, with the host VM's message ("execution exceeds N steps" past max_steps).  The buffers
    are sized by a shapes-only call first, so the shape pass runs twice."""
    jobs = [(program, x) for x in inputs]
    if not jobs:
        return []
    prog, cprog, arr, keep = _execution_args(program, [x for _, x in jobs])
    k = len(jobs)
    return _traces(lambda info, outs, status: backend.lib().dg_trace_batch(ctypes.byref(cprog), k, arr, int(max_steps), info, outs, status),
                   jobs, [prog], [0] * k, [num_outputs] * k)


def execute_batch(program, inputs, num_outputs=1, options=None, max_steps=MAX_STEPS):
    """distaff::execute (lib.rs:30-65) for every ProgramInputs: the program runs on the GPU, one thread per execution, and every trace is
    proven from the device memory it was generated in.  Returns a list in input order: (outputs, StarkProof) -- what execute() returns
    for the same inputs, byte for byte -- or the DgError of an execution that failed (in the VM or in the prover)."""
    options = options or ProofOptions()
    assert 0 <= num_outputs <= 8, "cannot have more than 8 outputs"
    jobs = [(program, x) for x in inputs]
    if not jobs:
        return []
    _, cprog, arr, keep = _execution_args(program, [x for _, x in jobs])
    k, opt = len(jobs), options._c()
    return _proofs(lambda handles, outputs16, status, pst: backend.lib().dg_execute_batch(
        ctypes.byref(cprog), k, arr, num_outputs, int(max_steps), ctypes.byref(opt), handles, outputs16, status, pst),
        [num_outputs] * k, max(num_outputs, 1))


# ---- one long execution, split across GPU threads ------------------------------------------------------------------------------------
def trace_one(program, inputs=None, max_steps=MAX_STEPS, num_outputs=1, segment_steps=0, stats=None):
    """processor::execute of one program (a hostvm.Program or assembly source) for one ProgramInputs on the GPU, split across threads
    (dg_trace_one): the sponge from a per-program table, one sequential pass that records checkpoints, and one thread per segment writing
    the rows.  Returns a hostvm.ExecutionTrace (what hostvm.execute gives, byte for byte); raises DgError when the execution fails, with
    the host VM's message.  segment_steps: 0 (the library chooses) or a power of two >= 16.  The buffer is sized by a call without
    registers first, so the table and the sequential pass run twice.  A dict passed as `stats` receives the full call's figures."""
    assert 0 <= num_outputs <= 8, "cannot have more than 8 outputs"
    jobs = [(program, inputs or ProgramInputs())]
    prog, cprog, arr, keep = _execution_args(program, [jobs[0][1]])
    st = backend.DgTraceOneStats()

    def call(info, outs, status):
        rc = backend.lib().dg_trace_one(ctypes.byref(cprog), arr, int(max_steps), int(segment_steps), info, None if outs is None else outs[0],
                                        ctypes.byref(st))
        _fields(st, stats)
        return rc
    return _traces(call, jobs, [prog], [0], [num_outputs])[0]


def execute_one(program, inputs=None, num_outputs=1, options=None, max_steps=MAX_STEPS, segment_steps=0, stats=None):
    """distaff::execute (lib.rs:30-65) of one program for one ProgramInputs, the execution split across GPU threads as in trace_one and
    the trace proven where it was written (dg_execute_one).  Returns (outputs, StarkProof) -- what execute() returns, byte for byte --
    and raises DgError when the execution or the proof fails.  `stats` as in trace_one."""
    options = options or ProofOptions()
    assert 0 <= num_outputs <= 8, "cannot have more than 8 outputs"
    _, cprog, arr, keep = _execution_args(program, [inputs or ProgramInputs()])
    opt, st = options._c(), backend.DgTraceOneStats()

    def call(handles, outputs16, status, pst):
        rc = backend.lib().dg_execute_one(ctypes.byref(cprog), arr, num_outputs, int(max_steps), int(segment_steps), ctypes.byref(opt), handles,
                                          outputs16, None, pst, ctypes.byref(st))
        _fields(st, stats)
        return rc
    return _proofs(call, [num_outputs])[0]


# ---- many programs, many inputs, executed on the GPU in one call ----------------------------------------------------------------------
def pack_jobs(jobs, compile=None):
    """The program table of a dg_trace_programs / dg_execute_programs call.  jobs: (program, ProgramInputs) or (program, ProgramInputs,
    num_outputs), the program an assembly source or a hostvm.Program.  Each distinct source is compiled once (by `compile`, default
    hostvm.compile_program) and each distinct program -- the same source, or the same Program object -- goes into the table once.
    Returns (programs, program_of, inputs, num_outputs), the last three in job order."""
    compile = compile or hostvm.compile_program
    programs, program_of, inputs, num_outputs = [], [], [], []
    index = {}
    for job in jobs:
        if len(job) not in (2, 3):
            raise ValueError("a job is (program, ProgramInputs) or (program, ProgramInputs, num_outputs)")
        program, x = job[0], job[1]
        no = int(job[2]) if len(job) == 3 else 1
        if not 0 <= no <= 8:
            raise ValueError("cannot have more than 8 outputs")
        key = ("source", program) if isinstance(program, str) else ("program", id(program))
        if key not in index:
            index[key] = len(programs)
            programs.append(compile(program) if isinstance(program, str) else program)
        program_of.append(index[key])
        inputs.append(x)
        num_outputs.append(no)
    return programs, program_of, inputs, num_outputs


def _trace_jobs(entry, jobs, st, stats, *args):
    """trace_programs / trace_many: the C entry named `entry` (programs, n_programs, count, program_of, inputs, *args, info, registers_out,
    status, st) through _traces, its stats structure st into the dict `stats`"""
    jobs = list(jobs)
    if not jobs:
        return []
    programs, cprogs, program_of, arr, num_outputs, keep = _programs_args(jobs)
    fn = getattr(backend.lib(), entry)
    result = _traces(lambda info, outs, status: fn(cprogs, len(programs), len(jobs), program_of, arr, *args, info, outs, status, ctypes.byref(st)),
                     jobs, programs, program_of, num_outputs)
    _fields(st, stats)
    return result


def _execute_jobs(entry, jobs, options, st, stats, *args):
    """execute_programs / execute_many: the C entry named `entry` (programs, n_programs, count, program_of, inputs, num_outputs, *args,
    options, proofs_out, outputs16, status, prove_stats, st) through _proofs, its stats structure st into the dict `stats`.  options: one
    ProofOptions, or a list with one per job (the entry's _with_options form)"""
    jobs = list(jobs)
    opt, per_job = _options_arg(options, len(jobs), "job")
    if not jobs:
        return []
    programs, cprogs, program_of, arr, num_outputs, keep = _programs_args(jobs)
    k, fn = len(jobs), getattr(backend.lib(), entry + "_with_options" if per_job else entry)
    result = _proofs(lambda handles, outputs16, status, pst: fn(cprogs, len(programs), k, program_of, arr, (backend.u32 * k)(*num_outputs), *args,
                                                                opt, handles, outputs16, status, pst, ctypes.byref(st)), num_outputs)
    _fields(st, stats)
    return result


def trace_programs(jobs, max_steps=MAX_STEPS, stats=None):
    """trace_batch for executions of different programs in one call (dg_trace_programs): each program's executions run in warps of
    their own, and one write launch per wave covers every trace shape.  Returns a list in job order: a hostvm.ExecutionTrace (with the
    job's num_outputs outputs, default 1) or the DgError of an execution that failed.  A dict passed as `stats` receives the VM passes'
    figures (shape_launches, write_launches, waves, prove_groups, lanes, shape_ms, write_ms) of the call that writes the traces; a
    shapes-only call sizes the buffers first."""
    return _trace_jobs("dg_trace_programs", jobs, backend.DgExecutionStats(), stats, int(max_steps))


def execute_programs(jobs, options=None, max_steps=MAX_STEPS, stats=None):
    """execute_batch for executions of different programs in one call (dg_execute_programs): the VM runs every job on the GPU, and each
    trace shape's traces are proven together, whichever programs they came from, in the device memory they were written to.  Returns a
    list in job order: (outputs, StarkProof) -- what execute_batch of that program alone returns, byte for byte -- or the DgError of an
    execution that failed.  `stats` as in trace_programs, prove_groups included.  options: one ProofOptions for every job, or a list with
    one per job (dg_execute_programs_with_options)."""
    return _execute_jobs("dg_execute_programs", jobs, options, backend.DgExecutionStats(), stats, int(max_steps))


# ---- many long executions, each split across GPU threads, in one call ------------------------------------------------------------------
def _segment_steps(segment_steps):
    s = int(segment_steps)
    if s != 0 and (s < 16 or s & (s - 1)):
        raise ValueError("segment_steps must be 0 or a power of two of at least 16")
    return s


def trace_many(jobs, max_steps=MAX_STEPS, segment_steps=0, stats=None):
    """trace_programs with every execution run as trace_one runs one (dg_trace_many): the programs' sponge tables, one sequential pass
    for every execution and the rows written by one thread per checkpoint.  jobs as in trace_programs (pack_jobs).  Returns a list in job
    order: a hostvm.ExecutionTrace (what trace_programs returns, byte for byte) or the DgError of an execution that failed.
    segment_steps: 0 (the library chooses) or a power of two >= 16.  The buffers are sized by a call without registers first, so the
    tables and the sequential pass run twice.  A dict passed as `stats` receives the full call's figures, the batch path's for the
    fallback executions under "fallback"."""
    return _trace_jobs("dg_trace_many", jobs, backend.DgManyStats(), stats, int(max_steps), _segment_steps(segment_steps))


def execute_many(jobs, options=None, max_steps=MAX_STEPS, segment_steps=0, stats=None):
    """execute_programs with every execution run as execute_one runs one (dg_execute_many): every trace is proven where it was written.
    Returns a list in job order: (outputs, StarkProof) -- what execute_programs returns, byte for byte -- or the DgError of an execution
    that failed.  segment_steps and `stats` as in trace_many; options as in execute_programs."""
    return _execute_jobs("dg_execute_many", jobs, options, backend.DgManyStats(), stats, int(max_steps), _segment_steps(segment_steps))


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


HASH_IDS = {"blake3": 0, "rescue": 1, "poseidon": 2, "hasher": 3}


def merkle_build(leaves, hash="blake3"):
    """crypto::build_merkle_nodes (merkle.rs:269-294): bytes (n*32) -> bytes (n*32), heap layout; hash in blake3 | rescue | poseidon |
    hasher (utils::hasher::digest, the VM's hash: a leaf is 2 field elements, and a tree of 2^d leaves is one smpath.n / pmpath.n verify,
    n = d + 1)"""
    leaves = bytes(leaves)
    n = len(leaves) // 32
    out = ctypes.create_string_buffer(n * 32)
    if hash == "blake3":
        backend.check(backend.lib().dg_merkle_build(leaves, n, out))
    else:
        backend.check(backend.lib().dg_merkle_build_with(HASH_IDS[hash], leaves, n, out))
    return out.raw


def hash64(messages, hash="rescue"):
    """crypto::hash::{blake3, rescue, poseidon} or utils::hasher::digest ("hasher") of n independent 64-byte messages: bytes (n*64) ->
    bytes (n*32)"""
    messages = bytes(messages)
    assert len(messages) % 64 == 0
    n = len(messages) // 64
    out = ctypes.create_string_buffer(max(1, n * 32))
    backend.check(backend.lib().dg_hash64(HASH_IDS[hash], messages, n, out))
    return out.raw[:n * 32]


# ---- Merkle trees of the VM's hash, and programs that prove membership of their leaves -----------------------------------------------
def _le_pairs(pairs):
    return b"".join(int(v).to_bytes(16, "little") for p in pairs for v in p)


def _int_pairs(raw):
    v = [int.from_bytes(raw[16 * k:16 * k + 16], "little") for k in range(len(raw) // 16)]
    return [(v[2 * k], v[2 * k + 1]) for k in range(len(v) // 2)]


def smpath_program(n):
    """Membership in a tree of 2^(n-1) leaves with the index private: the leaf and the path on the tapes, the index bits beside the path
    (HasherTree.smpath_inputs).  Outputs the root in stack order, [root[1], root[0]]."""
    _check_path_length(n)
    return f"begin read.ab smpath.{n} end"


def pmpath_program(n):
    """Membership in a tree of 2^(n-1) leaves with the index public: the index is the public input, the leaf and the path are on the tapes
    (HasherTree.pmpath_inputs).  Outputs the root in stack order, [root[1], root[0]]."""
    _check_path_length(n)
    return f"begin read.ab pmpath.{n} end"


def _check_path_length(n):
    if not 2 <= n <= 256:
        raise ValueError(f"a Merkle path has 2 to 256 entries (smpath.n / pmpath.n), not {n}")


class HasherTree:
    """A Merkle tree of utils::hasher::digest over L = 2^d leaves, each a pair of field elements, in the heap layout of
    merkle_build(..., "hasher"): nodes[L/2 + i] = digest(leaf[2i] | leaf[2i+1]), nodes[1] the root, nodes[0] zero.  Built on the GPU;
    `nodes` (L pairs) gives the heap instead, so that the path and tape logic runs on any heap.  Its paths are those of smpath.n /
    pmpath.n with n = depth = d + 1."""

    def __init__(self, leaves, nodes=None):
        self.leaves = [(int(a), int(b)) for a, b in leaves]
        L = len(self.leaves)
        if L < 2 or L & (L - 1) or L > 2**255:
            raise ValueError(f"a tree has 2^d leaves, 1 <= d <= 255, not {L}")
        if nodes is None:
            nodes = _int_pairs(merkle_build(_le_pairs(self.leaves), "hasher"))
        self.nodes = [(int(a), int(b)) for a, b in nodes]
        if len(self.nodes) != L:
            raise ValueError(f"the heap of {L} leaves has {L} nodes, not {len(self.nodes)}")

    @property
    def root(self):
        return list(self.nodes[1])

    @property
    def depth(self):
        """n of smpath.n / pmpath.n: the number of entries of a path"""
        return len(self.leaves).bit_length()

    def _index(self, i):
        i = int(i)
        if not 0 <= i < len(self.leaves):
            raise IndexError(f"leaf {i} of a tree of {len(self.leaves)} leaves")
        return i

    def path(self, i):
        """the path of examples/merkle.rs: [leaf i, leaf i^1, then the sibling of every node from leaf i's parent up to the root's child]"""
        i = self._index(i)
        p, k = [self.leaves[i], self.leaves[i ^ 1]], (len(self.leaves) + i) >> 1
        while k > 1:
            p.append(self.nodes[k ^ 1])
            k >>= 1
        return p

    def _smpath_tapes(self, i):
        """tapes A and B of smpath: the leaf, then per later entry (0, index bit) and the entry (merkle.rs:63-85)"""
        path, bits = self.path(i), i
        a, b = [path[0][0]], [path[0][1]]
        for node in path[1:]:
            a += [0, node[0]]
            b += [bits & 1, node[1]]
            bits >>= 1
        return a, b

    def tapes(self, i):
        """(tape A, tape B) of the program of examples/merkle.rs (hostvm.merkle_program(depth, i)), as generate_program_inputs
        (merkle.rs:63-94) lays them out: the smpath tapes, then every entry after the leaf again for pmpath"""
        a, b = self._smpath_tapes(self._index(i))
        path = self.path(i)
        return a + [e[0] for e in path[1:]], b + [e[1] for e in path[1:]]

    def smpath_inputs(self, i):
        """the ProgramInputs of smpath_program(depth) for leaf i"""
        a, b = self._smpath_tapes(self._index(i))
        return ProgramInputs([], a, b)

    def pmpath_inputs(self, i):
        """the ProgramInputs of pmpath_program(depth) for leaf i: the index public, the leaf and the path on the tapes"""
        path = self.path(i)
        return ProgramInputs([int(i)], [e[0] for e in path], [e[1] for e in path])


def prove_membership(tree, indexes, program="smpath", options=None):
    """Proves that leaves of a HasherTree, or of a MerkleTree of hash "hasher" (its paths from one dg_tree_paths call, laid out as
    HasherTree.smpath_inputs / pmpath_inputs lay them out), belong to it: one execute_batch call runs smpath_program(tree.depth) (index private) or
    pmpath_program(tree.depth) (index public) for every index.  Returns a list in index order: (program_hash, public_inputs, outputs,
    proof), an item of verify_batch whose outputs are the root in stack order, or a DgError for an entry whose execution failed or did not
    output the root."""
    if program not in ("smpath", "pmpath"):
        raise ValueError(f"program is smpath or pmpath, not {program!r}")
    if isinstance(tree, MerkleTree):
        indexes, inputs, root = tree._membership_inputs(indexes, program)
    else:
        indexes = [tree._index(i) for i in indexes]
        inputs = [tree.smpath_inputs(i) if program == "smpath" else tree.pmpath_inputs(i) for i in indexes]
        root = tree.root
    prog = hostvm.compile_program(smpath_program(tree.depth) if program == "smpath" else pmpath_program(tree.depth))
    want = root[::-1]
    out = []
    for i, x, r in zip(indexes, inputs, execute_batch(prog, inputs, num_outputs=2, options=options)):
        if isinstance(r, backend.DgError):
            out.append(r)
        elif r[0] != want:
            out.append(backend.DgError(-7, f"leaf {i}: the {program} program output {r[0]}, not the root"))
        else:
            out.append((prog.hash, x.public, r[0], r[1]))
    return out


class MerkleTree:
    """crypto::MerkleTree (merkle.rs:22-62) kept in device memory (dg_tree_*): L = 2^d leaves of 32 bytes and the heap of
    merkle_build(leaves, hash), built once on the GPU.  paths() gathers the authentication paths of many leaves in one call and copies
    only those; update() replaces leaves and rehashes only the nodes on their paths.  `leaves` is L x 32 bytes, a contiguous CUDA uint8
    tensor of L x 32 bytes on the library's device (copied into the tree's own buffer), or, for hash="hasher" only, a sequence of (a, b)
    field-element pairs as HasherTree takes them.  The tree holds 64 L bytes of the library's device memory until close()."""

    def __init__(self, leaves, hash="blake3"):
        if hash not in HASH_IDS:
            raise ValueError(f"hash is one of {', '.join(HASH_IDS)}, not {hash!r}")
        self.hash = hash
        self._h = None
        handle = backend.vp()
        if getattr(leaves, "is_cuda", False):
            import torch
            if leaves.dtype != torch.uint8 or not leaves.is_contiguous() or leaves.numel() % 32:
                raise ValueError("device leaves are a contiguous uint8 tensor of L x 32 bytes")
            torch.cuda.synchronize(leaves.device)                # the copy runs on the library's stream
            backend.check(backend.lib().dg_tree_new_device(HASH_IDS[hash], leaves.data_ptr(), leaves.numel() // 32, ctypes.byref(handle)))
        else:
            raw = self._leaf_bytes(leaves)
            backend.check(backend.lib().dg_tree_new(HASH_IDS[hash], raw, len(raw) // 32, ctypes.byref(handle)))
        self._h = handle.value
        n = backend.u64(0)
        backend.check(backend.lib().dg_tree_info(self._h, None, ctypes.byref(n), None))
        self._n = n.value

    def _leaf_bytes(self, leaves):
        if isinstance(leaves, (bytes, bytearray, memoryview, np.ndarray)):
            raw = leaves.tobytes() if isinstance(leaves, np.ndarray) else bytes(leaves)
        elif self.hash == "hasher":
            pairs = [(int(a), int(b)) for a, b in leaves]
            if any(not 0 <= v < 2**128 for p in pairs for v in p):
                raise ValueError("a leaf element is an integer in [0, 2^128)")
            raw = _le_pairs(pairs)
        else:
            raise TypeError(f"leaves of a {self.hash} tree are bytes of L x 32")
        if len(raw) % 32:
            raise ValueError(f"leaves are 32 bytes each, not {len(raw)} bytes in all")
        return raw

    def _handle(self):
        if not self._h:
            raise ValueError("the tree is closed")
        return self._h

    @staticmethod
    def _indexes(indexes):
        idx = np.asarray(indexes if isinstance(indexes, np.ndarray) else list(indexes), dtype=np.int64).reshape(-1)
        if (idx < 0).any():
            raise ValueError("leaf indexes are non-negative")
        return idx.astype(np.uint64)

    def __len__(self):
        return self._n

    @property
    def depth(self):
        """d + 1 for L = 2^d: the number of entries of a path, n of smpath.n / pmpath.n (HasherTree.depth)"""
        return self._n.bit_length()

    @property
    def root(self):
        """nodes[1], 32 bytes"""
        out = ctypes.create_string_buffer(32)
        backend.check(backend.lib().dg_tree_info(self._handle(), None, None, out))
        return out.raw

    def paths(self, indexes):
        """one dg_tree_paths call: per index, its depth entries of 32 bytes in MerkleTree::prove order (leaf i, leaf i ^ 1, then the
        sibling of every node from leaf i's parent up to the root's child).  An index >= len(tree) raises DgError naming it."""
        idx, e = self._indexes(indexes), self.depth
        if len(idx) == 0:
            return []
        out = ctypes.create_string_buffer(32 * e * len(idx))
        backend.check(backend.lib().dg_tree_paths(self._handle(), idx.ctypes.data, len(idx), out))
        raw = out.raw
        return [[raw[32 * (k * e + j):32 * (k * e + j + 1)] for j in range(e)] for k in range(len(idx))]

    def update(self, indexes, leaves):
        """the leaf at indexes[k] becomes leaves[k] (a repeated index: its last occurrence); rehashes only the changed paths and returns
        the new root.  A rejected call (an index out of range, a non-canonical hasher leaf) leaves the tree as it was."""
        idx, raw = self._indexes(indexes), self._leaf_bytes(leaves)
        if len(raw) != 32 * len(idx):
            raise ValueError(f"{len(idx)} indexes and {len(raw) // 32} leaves")
        root = ctypes.create_string_buffer(32)
        backend.check(backend.lib().dg_tree_update(self._handle(), idx.ctypes.data if len(idx) else None, raw, len(idx), root))
        return root.raw

    def prove_batch(self, indexes):
        """MerkleTree::prove_batch (merkle.rs:64-124): the compressed opening of many leaves as one BatchMerkleProof, values in request
        order.  An index >= len(tree) or a repeated index raises DgError with the crate's message."""
        idx = self._indexes(indexes)
        ptr = idx.ctypes.data if len(idx) else None
        n = ctypes.c_size_t(0)
        backend.check(backend.lib().dg_tree_prove_batch(self._handle(), ptr, len(idx), None, 0, ctypes.byref(n)))
        out = ctypes.create_string_buffer(n.value)
        backend.check(backend.lib().dg_tree_prove_batch(self._handle(), ptr, len(idx), out, n.value, ctypes.byref(n)))
        return BatchMerkleProof.from_bytes(out.raw)

    @staticmethod
    def verify(root, index, path, hash="blake3"):
        """MerkleTree::verify (merkle.rs:127-151): whether `path` (2 to 64 entries of 32 bytes) leads leaf `index` to `root`.  Only the low
        len(path) - 1 bits of the index are read, as in the reference."""
        (r,) = merkle_verify_paths(root, [index], [path], hash)
        if isinstance(r, backend.DgError):
            raise r
        return r

    @staticmethod
    def verify_batch(root, indexes, proof, hash="blake3"):
        """MerkleTree::verify_batch (merkle.rs:154-263) of a BatchMerkleProof (or its bytes); where the crate panics this raises DgError
        with the crate's message."""
        (r,) = merkle_verify_batch([(root, indexes, proof)], hash)
        if isinstance(r, backend.DgError):
            raise r
        return r

    def leaves(self):
        out = ctypes.create_string_buffer(32 * self._n)
        backend.check(backend.lib().dg_tree_read(self._handle(), out, None))
        return out.raw

    def nodes(self):
        """the heap of merkle_build: nodes[1] the root, nodes[0] zero"""
        out = ctypes.create_string_buffer(32 * self._n)
        backend.check(backend.lib().dg_tree_read(self._handle(), None, out))
        return out.raw

    def _index(self, i):
        i = int(i)
        if not 0 <= i < self._n:
            raise IndexError(f"leaf {i} of a tree of {self._n} leaves")
        return i

    def _membership_inputs(self, indexes, program):
        """prove_membership's indexes, ProgramInputs and root (field elements) from one paths() call"""
        if self.hash != "hasher":
            raise ValueError(f"membership proofs verify paths of the VM's hash: a MerkleTree of hash 'hasher', not {self.hash!r}")
        indexes = [self._index(i) for i in indexes]
        inputs = []
        for i, entries in zip(indexes, self.paths(indexes)):
            path = _int_pairs(b"".join(entries))
            if program == "smpath":                  # HasherTree.smpath_inputs: the leaf, then per entry (0, index bit) and the entry
                a, b, bits = [path[0][0]], [path[0][1]], i
                for node in path[1:]:
                    a += [0, node[0]]
                    b += [bits & 1, node[1]]
                    bits >>= 1
                inputs.append(ProgramInputs([], a, b))
            else:                                    # HasherTree.pmpath_inputs: the index public, the path on the tapes
                inputs.append(ProgramInputs([i], [e[0] for e in path], [e[1] for e in path]))
        return indexes, inputs, list(_int_pairs(self.root)[0])

    def close(self):
        if self._h:
            backend.lib().dg_tree_free(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BatchMerkleProof:
    """crypto::BatchMerkleProof (merkle.rs:14-18): values (32-byte bytes, one per requested index in request order), nodes (one list of
    32-byte bytes per normalised index) and depth.  to_bytes() / from_bytes() are its bincode: u64 count + 32 B per value; u64 count,
    then per slot u64 count + 32 B per node; u8 depth."""

    def __init__(self, values, nodes, depth):
        self.values = [bytes(v) for v in values]
        self.nodes = [[bytes(v) for v in slot] for slot in nodes]
        self.depth = int(depth)

    def to_bytes(self):
        u64 = lambda n: int(n).to_bytes(8, "little")
        return (u64(len(self.values)) + b"".join(self.values) + u64(len(self.nodes)) +
                b"".join(u64(len(slot)) + b"".join(slot) for slot in self.nodes) + bytes([self.depth]))

    @classmethod
    def from_bytes(cls, data):
        data, at = bytes(data), 0

        def take(n):
            nonlocal at
            if len(data) - at < n:
                raise ValueError("not a BatchMerkleProof: the bytes end early")
            at += n
            return data[at - n:at]

        def digests():
            n = int.from_bytes(take(8), "little")
            if n > (len(data) - at) // 32:
                raise ValueError("not a BatchMerkleProof: a length the bytes cannot hold")
            return [take(32) for _ in range(n)]
        values = digests()
        n = int.from_bytes(take(8), "little")
        if n > (len(data) - at) // 8:
            raise ValueError("not a BatchMerkleProof: a length the bytes cannot hold")
        nodes = [digests() for _ in range(n)]
        depth = take(1)[0]
        if at != len(data):
            raise ValueError("not a BatchMerkleProof: trailing bytes")
        return cls(values, nodes, depth)

    def __eq__(self, other):
        return isinstance(other, BatchMerkleProof) and (self.values, self.nodes, self.depth) == (other.values, other.nodes, other.depth)

    def __repr__(self):
        return f"BatchMerkleProof({len(self.values)} values, {sum(map(len, self.nodes))} nodes in {len(self.nodes)} slots, depth {self.depth})"


def _hash_id(hash):
    if hash not in HASH_IDS:
        raise ValueError(f"hash is one of {', '.join(HASH_IDS)}, not {hash!r}")
    return HASH_IDS[hash]


def _verdicts(status):
    """True (accepted), False (rejected) or the DgError of a malformed entry / a panic of the reference, per entry of the last call"""
    return [True if e is None else False if e.code == -6 else e for e in _messages(status)]


def merkle_verify_paths(roots, indexes, paths, hash="blake3"):
    """MerkleTree::verify (merkle.rs:127-151) of many paths in one dg_merkle_verify_paths call.  `roots` is one 32-byte root or one per path;
    `paths` is what MerkleTree.paths returns (lists of 32-byte entries, all of one length) or a uint8 array of shape (K, entries, 32).
    Returns a list per path: True, False, or a DgError for a path with an element >= M (hashes other than blake3)."""
    if isinstance(paths, np.ndarray):
        if paths.dtype != np.uint8 or paths.ndim != 3 or paths.shape[2] != 32:
            raise ValueError("a path array is uint8 of shape (K, entries, 32)")
        raw = np.ascontiguousarray(paths)
        k, entries = paths.shape[0], paths.shape[1]
    else:
        paths = [[bytes(e) for e in p] for p in paths]
        k, entries = len(paths), len(paths[0]) if paths else 2
        if any(len(p) != entries for p in paths) or any(len(e) != 32 for p in paths for e in p):
            raise ValueError("paths have one number of entries, each of 32 bytes")
        raw = np.frombuffer(b"".join(e for p in paths for e in p), dtype=np.uint8)
    idx = MerkleTree._indexes(indexes)
    if len(idx) != k:
        raise ValueError(f"{len(idx)} indexes and {k} paths")
    roots = bytes(roots) if isinstance(roots, (bytes, bytearray, memoryview)) else b"".join(bytes(r) for r in roots)
    if len(roots) % 32:
        raise ValueError("roots are 32 bytes each")
    if k == 0:
        return []
    status = (ctypes.c_int * k)()
    backend.check(backend.lib().dg_merkle_verify_paths(_hash_id(hash), roots, len(roots) // 32, idx.ctypes.data, raw.ctypes.data, entries, k,
                                                       status))
    return _verdicts(status)


def merkle_verify_batch(items, hash="blake3"):
    """MerkleTree::verify_batch (merkle.rs:154-263) of many batch proofs in one dg_merkle_verify_batch call.  items: (root, indexes, proof),
    proof a BatchMerkleProof or its bytes.  Returns a list per item: True, False, or a DgError where the reference panics or the input is
    malformed (bytes that are not one BatchMerkleProof, an element >= M for hashes other than blake3)."""
    items = list(items)
    k = len(items)
    if k == 0:
        return []
    roots = b"".join(bytes(r) for r, _, _ in items)
    if len(roots) != 32 * k:
        raise ValueError("roots are 32 bytes each")
    idx = [MerkleTree._indexes(i) for _, i, _ in items]
    data = [p.to_bytes() if isinstance(p, BatchMerkleProof) else bytes(p) for _, _, p in items]
    status = (ctypes.c_int * k)()
    backend.check(backend.lib().dg_merkle_verify_batch(_hash_id(hash), k, roots, (backend.vp * k)(*[a.ctypes.data if len(a) else None for a in idx]),
                                                       (backend.u32 * k)(*[len(a) for a in idx]),
                                                       (backend.vp * k)(*[ctypes.cast(ctypes.c_char_p(d), backend.vp) for d in data]),
                                                       (ctypes.c_size_t * k)(*[len(d) for d in data]), status))
    return _verdicts(status)


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
    code = {"add": 0, "sub": 1, "mul": 2, "inv": 3, "exp": 4, "dot6": 5, "mul_tw": 6}[op]
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
