"""Host-side mirror of the reference's public interface for the prove path (names and argument meaning follow
/root/reference/src/lib.rs:30-75, /root/reference/src/stark/options.rs:16-91, /root/reference/src/stark/proof.rs:10-77)."""
import ctypes
import functools

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


def prove_traces(traces, options=None):
    """Proves many hostvm.ExecutionTraces of any register shapes and lengths in one dg_prove_traces call: every stage is launched once
    per group of traces of one length, whatever their shapes (the constraint evaluation once per shape).  Returns what prove_batch
    returns, in input order: a StarkProof byte-identical to prove() of the same trace (its stats: the whole call's), or the
    backend.DgError of a trace that failed."""
    options = options or ProofOptions()
    opt = options._c()
    traces = list(traces)
    k = len(traces)
    regs = [np.ascontiguousarray(tr.registers, dtype=np.uint64) for tr in traces]
    cols = [(backend.vp * r.shape[0])(*[r[j].ctypes.data for j in range(r.shape[0])]) for r in regs]
    ts = (backend.DgTrace * max(k, 1))(*[backend.DgTrace(cols[i], r.shape[0], r.shape[1], tr.ctx_depth, tr.loop_depth)
                                        for i, (r, tr) in enumerate(zip(regs, traces))])
    keep, (pin, nin, pout, nout) = _batch_io([tr.public_inputs for tr in traces], [tr.outputs for tr in traces])
    handles = (backend.vp * max(k, 1))()
    status = (ctypes.c_int * max(k, 1))()
    st = backend.DgStats()
    backend.check(backend.lib().dg_prove_traces(ts, k, pin, nin, pout, nout, ctypes.byref(opt), handles, status, ctypes.byref(st)))
    del keep, regs, cols
    return _collect_batch(list(handles)[:k], list(status)[:k], st)


def prove_traces_device(d_registers, widths, lengths, ctx_depths, loop_depths, public_inputs_list, outputs_list, options=None):
    """prove_traces for traces already in device memory: trace i's widths[i] x lengths[i] registers (column-major) at d_registers[i]
    (backend.DeviceBuffer or raw pointer); the other arguments hold one entry per trace."""
    options = options or ProofOptions()
    k = len(d_registers)
    assert all(len(a) == k for a in (widths, lengths, ctx_depths, loop_depths, public_inputs_list, outputs_list)), "one entry per trace"
    ptrs = (backend.vp * max(k, 1))(*[d.ptr if isinstance(d, backend.DeviceBuffer) else int(d) for d in d_registers])
    arr = lambda t, xs: (t * max(k, 1))(*[int(x) for x in xs])
    opt = options._c()
    keep, (pin, nin, pout, nout) = _batch_io(public_inputs_list, outputs_list)
    handles = (backend.vp * max(k, 1))()
    status = (ctypes.c_int * max(k, 1))()
    st = backend.DgStats()
    backend.check(backend.lib().dg_prove_traces_device(ptrs, arr(backend.u32, widths), arr(backend.u64, lengths), arr(backend.u32, ctx_depths),
                                                      arr(backend.u32, loop_depths), k, pin, nin, pout, nout, ctypes.byref(opt), handles, status,
                                                      ctypes.byref(st)))
    del keep
    return _collect_batch(list(handles)[:k], list(status)[:k], st)


def group_traces(lengths, widths, ctx_depths, loop_depths, footprints, budget, cap):
    """dg_host_group_traces (no device): the groups prove_traces runs, as lists of trace indices in device order."""
    k = len(lengths)
    arr = lambda t, xs: (t * max(k, 1))(*[int(x) for x in xs])
    order = (backend.u32 * max(k, 1))()
    sizes = (backend.u32 * max(k, 1))()
    n = backend.u32(0)
    backend.check(backend.lib().dg_host_group_traces(k, arr(backend.u64, lengths), arr(backend.u32, widths), arr(backend.u32, ctx_depths),
                                                    arr(backend.u32, loop_depths), arr(backend.u64, footprints), int(budget), int(cap), order,
                                                    sizes, ctypes.byref(n)))
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
    ptr = d_registers.ptr if isinstance(d_registers, backend.DeviceBuffer) else int(d_registers)
    mptr = None if d_masks is None else (d_masks.ptr if isinstance(d_masks, backend.DeviceBuffer) else int(d_masks))
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


def _encoded(program):
    return hostvm.compile_program(program) if isinstance(program, str) else program


def _execution_args(program, inputs):
    """the dg_program_t and dg_program_inputs_t array of a call (plus the arrays they point into, to keep alive)"""
    prog = _encoded(program)
    cprog = prog.c_struct()
    keep = [prog, cprog]
    arr = (backend.DgProgramInputs * max(len(inputs), 1))()
    for i, x in enumerate(inputs):
        vals = [felt.from_ints(v) for v in (x.public, x.secret_a, x.secret_b)]
        keep += vals
        arr[i] = backend.DgProgramInputs(vals[0].ctypes.data, len(vals[0]), vals[1].ctypes.data, len(vals[1]), vals[2].ctypes.data, len(vals[2]))
    return prog, cprog, arr, keep


def _messages(status):
    msg = ctypes.create_string_buffer(512)
    out = []
    for i, rc in enumerate(status):
        if rc == 0:
            out.append(None)
            continue
        backend.check(backend.lib().dg_batch_message(i, msg, len(msg)))
        out.append(backend.DgError(rc, msg.value.decode(errors="replace")))
    return out


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
    errors = _messages(list(status))
    del keep
    return [e if e is not None else {f: int(getattr(info[i], f)) for f, _ in backend.DgExecutionInfo._fields_} for i, e in enumerate(errors)]


def trace_batch(program, inputs, max_steps=MAX_STEPS, num_outputs=1):
    """processor::execute of one program (a hostvm.Program or assembly source) for every ProgramInputs, on the GPU, one thread per
    execution.  Returns a list in input order: a hostvm.ExecutionTrace (what hostvm.execute gives for the same inputs, byte for byte)
    or the DgError of an execution that failed, with the host VM's message ("execution exceeds N steps" past max_steps).  The buffers
    are sized by a shapes-only call first, so the shape pass runs twice."""
    inputs = list(inputs)
    if not inputs:
        return []
    prog, cprog, arr, keep = _execution_args(program, inputs)
    k = len(inputs)
    shapes = trace_shapes(prog, inputs, max_steps)
    regs = [None if isinstance(s, backend.DgError) else np.empty((s["width"], s["length"], 2), dtype=np.uint64) for s in shapes]
    outs = (backend.vp * k)(*[r.ctypes.data if r is not None else None for r in regs])
    info = (backend.DgExecutionInfo * k)()
    status = (ctypes.c_int * k)()
    backend.check(backend.lib().dg_trace_batch(ctypes.byref(cprog), k, arr, int(max_steps), info, outs, status))
    errors = _messages(list(status))
    del keep
    result = []
    for i, (x, e) in enumerate(zip(inputs, errors)):
        if e is not None:
            result.append(e)
            continue
        sd, start, n = info[i].stack_depth, 15 + info[i].ctx_depth + info[i].loop_depth, info[i].length
        last = [felt.to_ints(regs[i][start + j, n - 1])[0] if j < sd else 0 for j in range(8)]
        result.append(hostvm.ExecutionTrace(regs[i], info[i].ctx_depth, info[i].loop_depth, sd, prog.hash, list(x.public), last[:num_outputs]))
    return result


def execute_batch(program, inputs, num_outputs=1, options=None, max_steps=MAX_STEPS):
    """distaff::execute (lib.rs:30-65) for every ProgramInputs: the program runs on the GPU, one thread per execution, and every trace is
    proven from the device memory it was generated in.  Returns a list in input order: (outputs, StarkProof) -- what execute() returns
    for the same inputs, byte for byte -- or the DgError of an execution that failed (in the VM or in the prover)."""
    options = options or ProofOptions()
    assert 0 <= num_outputs <= 8, "cannot have more than 8 outputs"
    inputs = list(inputs)
    if not inputs:
        return []
    _, cprog, arr, keep = _execution_args(program, inputs)
    k = len(inputs)
    opt = options._c()
    handles = (backend.vp * k)()
    outputs = np.zeros((k, max(num_outputs, 1), 2), dtype=np.uint64)
    status = (ctypes.c_int * k)()
    stats = backend.DgStats()
    backend.check(backend.lib().dg_execute_batch(ctypes.byref(cprog), k, arr, num_outputs, int(max_steps), ctypes.byref(opt), handles,
                                                outputs.ctypes.data, status, ctypes.byref(stats)))
    errors = _messages(list(status))
    del keep
    return [e if e is not None else (felt.to_ints(outputs[i, :num_outputs]) if num_outputs else [], _collect(handles[i], stats))
            for i, e in enumerate(errors)]


# ---- one long execution, split across GPU threads ------------------------------------------------------------------------------------
def _one_stats(stats, st):
    if stats is not None:
        stats.update({f: (float if f.endswith("_ms") else int)(getattr(st, f)) for f, _ in backend.DgTraceOneStats._fields_})


def trace_one(program, inputs=None, max_steps=MAX_STEPS, num_outputs=1, segment_steps=0, stats=None):
    """processor::execute of one program (a hostvm.Program or assembly source) for one ProgramInputs on the GPU, split across threads
    (dg_trace_one): the sponge from a per-program table, one sequential pass that records checkpoints, and one thread per segment writing
    the rows.  Returns a hostvm.ExecutionTrace (what hostvm.execute gives, byte for byte); raises DgError when the execution fails, with
    the host VM's message.  segment_steps: 0 (the library chooses) or a power of two >= 16.  The buffer is sized by a call without
    registers first, so the table and the sequential pass run twice.  A dict passed as `stats` receives the full call's figures."""
    assert 0 <= num_outputs <= 8, "cannot have more than 8 outputs"
    x = inputs or ProgramInputs()
    prog, cprog, arr, keep = _execution_args(program, [x])
    L, info, st = backend.lib(), backend.DgExecutionInfo(), backend.DgTraceOneStats()

    def call(out):
        rc = L.dg_trace_one(ctypes.byref(cprog), arr, int(max_steps), int(segment_steps), ctypes.byref(info), out, ctypes.byref(st))
        _one_stats(stats, st)
        backend.check(rc)

    call(None)
    regs = np.empty((info.width, info.length, 2), dtype=np.uint64)
    call(regs.ctypes.data)
    del keep
    sd, start, n = info.stack_depth, 15 + info.ctx_depth + info.loop_depth, info.length
    last = [felt.to_ints(regs[start + j, n - 1])[0] if j < sd else 0 for j in range(8)]
    return hostvm.ExecutionTrace(regs, info.ctx_depth, info.loop_depth, sd, prog.hash, list(x.public), last[:num_outputs])


def execute_one(program, inputs=None, num_outputs=1, options=None, max_steps=MAX_STEPS, segment_steps=0, stats=None):
    """distaff::execute (lib.rs:30-65) of one program for one ProgramInputs, the execution split across GPU threads as in trace_one and
    the trace proven where it was written (dg_execute_one).  Returns (outputs, StarkProof) -- what execute() returns, byte for byte --
    and raises DgError when the execution or the proof fails.  `stats` as in trace_one."""
    options = options or ProofOptions()
    assert 0 <= num_outputs <= 8, "cannot have more than 8 outputs"
    _, cprog, arr, keep = _execution_args(program, [inputs or ProgramInputs()])
    opt = options._c()
    handle = backend.vp()
    outputs = np.zeros((max(num_outputs, 1), 2), dtype=np.uint64)
    pst, st = backend.DgStats(), backend.DgTraceOneStats()
    rc = backend.lib().dg_execute_one(ctypes.byref(cprog), arr, num_outputs, int(max_steps), int(segment_steps), ctypes.byref(opt),
                                      ctypes.byref(handle), outputs.ctypes.data, None, ctypes.byref(pst), ctypes.byref(st))
    del keep
    _one_stats(stats, st)
    backend.check(rc)
    return (felt.to_ints(outputs[:num_outputs]) if num_outputs else []), _collect(handle.value, pst)


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


def _vm_stats(stats, st):
    if stats is not None:
        stats.update({f: (float if f.endswith("_ms") else int)(getattr(st, f)) for f, _ in backend.DgExecutionStats._fields_})


def trace_programs(jobs, max_steps=MAX_STEPS, stats=None):
    """trace_batch for executions of different programs in one call (dg_trace_programs): each program's executions run in warps of
    their own, and one write launch per wave covers every trace shape.  Returns a list in job order: a hostvm.ExecutionTrace (with the
    job's num_outputs outputs, default 1) or the DgError of an execution that failed.  A dict passed as `stats` receives the VM passes'
    figures (shape_launches, write_launches, waves, prove_groups, lanes, shape_ms, write_ms) of the call that writes the traces; a
    shapes-only call sizes the buffers first."""
    jobs = list(jobs)
    if not jobs:
        return []
    programs, cprogs, program_of, arr, num_outputs, keep = _programs_args(jobs)
    k, L = len(jobs), backend.lib()
    info = (backend.DgExecutionInfo * k)()
    status = (ctypes.c_int * k)()
    st = backend.DgExecutionStats()
    backend.check(L.dg_trace_programs(cprogs, len(programs), k, program_of, arr, int(max_steps), info, None, status, ctypes.byref(st)))
    regs = [np.empty((info[i].width, info[i].length, 2), dtype=np.uint64) if status[i] == 0 else None for i in range(k)]
    outs = (backend.vp * k)(*[r.ctypes.data if r is not None else None for r in regs])
    backend.check(L.dg_trace_programs(cprogs, len(programs), k, program_of, arr, int(max_steps), info, outs, status, ctypes.byref(st)))
    errors = _messages(list(status))
    _vm_stats(stats, st)
    result = []
    for i, (job, e) in enumerate(zip(jobs, errors)):
        if e is not None:
            result.append(e)
            continue
        sd, start, n = info[i].stack_depth, 15 + info[i].ctx_depth + info[i].loop_depth, info[i].length
        last = [felt.to_ints(regs[i][start + j, n - 1])[0] if j < sd else 0 for j in range(8)]
        result.append(hostvm.ExecutionTrace(regs[i], info[i].ctx_depth, info[i].loop_depth, sd, programs[program_of[i]].hash,
                                            list(job[1].public), last[:num_outputs[i]]))
    del keep
    return result


def execute_programs(jobs, options=None, max_steps=MAX_STEPS, stats=None):
    """execute_batch for executions of different programs in one call (dg_execute_programs): the VM runs every job on the GPU, and each
    trace shape's traces are proven together, whichever programs they came from, in the device memory they were written to.  Returns a
    list in job order: (outputs, StarkProof) -- what execute_batch of that program alone returns, byte for byte -- or the DgError of an
    execution that failed.  `stats` as in trace_programs, prove_groups included."""
    options = options or ProofOptions()
    jobs = list(jobs)
    if not jobs:
        return []
    programs, cprogs, program_of, arr, num_outputs, keep = _programs_args(jobs)
    k = len(jobs)
    opt = options._c()
    handles = (backend.vp * k)()
    outputs = np.zeros((k, 8, 2), dtype=np.uint64)
    status = (ctypes.c_int * k)()
    pst, st = backend.DgStats(), backend.DgExecutionStats()
    backend.check(backend.lib().dg_execute_programs(cprogs, len(programs), k, program_of, arr, (backend.u32 * k)(*num_outputs), int(max_steps),
                                                   ctypes.byref(opt), handles, outputs.ctypes.data, status, ctypes.byref(pst), ctypes.byref(st)))
    errors = _messages(list(status))
    _vm_stats(stats, st)
    del keep
    return [e if e is not None else (felt.to_ints(outputs[i, :num_outputs[i]]) if num_outputs[i] else [], _collect(handles[i], pst))
            for i, e in enumerate(errors)]


# ---- many long executions, each split across GPU threads, in one call ------------------------------------------------------------------
def _many_stats(stats, st):
    if stats is not None:
        stats.update({f: (float if f.endswith("_ms") else int)(getattr(st, f)) for f, _ in backend.DgManyStats._fields_ if f != "fallback"})
        fb = {}
        _vm_stats(fb, st.fallback)
        stats["fallback"] = fb


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
    jobs = list(jobs)
    s = _segment_steps(segment_steps)
    if not jobs:
        return []
    programs, cprogs, program_of, arr, num_outputs, keep = _programs_args(jobs)
    k, L = len(jobs), backend.lib()
    info = (backend.DgExecutionInfo * k)()
    status = (ctypes.c_int * k)()
    st = backend.DgManyStats()
    backend.check(L.dg_trace_many(cprogs, len(programs), k, program_of, arr, int(max_steps), s, info, None, status, ctypes.byref(st)))
    regs = [np.empty((info[i].width, info[i].length, 2), dtype=np.uint64) if status[i] == 0 else None for i in range(k)]
    outs = (backend.vp * k)(*[r.ctypes.data if r is not None else None for r in regs])
    backend.check(L.dg_trace_many(cprogs, len(programs), k, program_of, arr, int(max_steps), s, info, outs, status, ctypes.byref(st)))
    errors = _messages(list(status))
    _many_stats(stats, st)
    result = []
    for i, (job, e) in enumerate(zip(jobs, errors)):
        if e is not None:
            result.append(e)
            continue
        sd, start, n = info[i].stack_depth, 15 + info[i].ctx_depth + info[i].loop_depth, info[i].length
        last = [felt.to_ints(regs[i][start + j, n - 1])[0] if j < sd else 0 for j in range(8)]
        result.append(hostvm.ExecutionTrace(regs[i], info[i].ctx_depth, info[i].loop_depth, sd, programs[program_of[i]].hash,
                                            list(job[1].public), last[:num_outputs[i]]))
    del keep
    return result


def execute_many(jobs, options=None, max_steps=MAX_STEPS, segment_steps=0, stats=None):
    """execute_programs with every execution run as execute_one runs one (dg_execute_many): every trace is proven where it was written.
    Returns a list in job order: (outputs, StarkProof) -- what execute_programs returns, byte for byte -- or the DgError of an execution
    that failed.  segment_steps and `stats` as in trace_many."""
    options = options or ProofOptions()
    jobs = list(jobs)
    s = _segment_steps(segment_steps)
    if not jobs:
        return []
    programs, cprogs, program_of, arr, num_outputs, keep = _programs_args(jobs)
    k = len(jobs)
    opt = options._c()
    handles = (backend.vp * k)()
    outputs = np.zeros((k, 8, 2), dtype=np.uint64)
    status = (ctypes.c_int * k)()
    pst, st = backend.DgStats(), backend.DgManyStats()
    backend.check(backend.lib().dg_execute_many(cprogs, len(programs), k, program_of, arr, (backend.u32 * k)(*num_outputs), int(max_steps), s,
                                               ctypes.byref(opt), handles, outputs.ctypes.data, status, ctypes.byref(pst), ctypes.byref(st)))
    errors = _messages(list(status))
    _many_stats(stats, st)
    del keep
    return [e if e is not None else (felt.to_ints(outputs[i, :num_outputs[i]]) if num_outputs[i] else [], _collect(handles[i], pst))
            for i, e in enumerate(errors)]


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
