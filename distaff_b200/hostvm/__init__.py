"""Python face of the host-side VM stand-in (`distaff_b200/hostvm/vm.cpp`).

Mirrors the host half of `distaff::execute` (/root/reference/src/lib.rs:30-59): compile assembly, run the VM, return the
column-major register traces plus what `stark::prove` needs (ctx/loop depth, public inputs, outputs, program hash).
This is an input generator for tests / smoke / bench; the prove hot path never calls it.
"""
import ctypes
import os
import numpy as np

from .. import felt

_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "libdistaff_vm.so")
        if not os.path.exists(path):
            raise RuntimeError(f"{path} missing: run `python -c 'import __graft_entry__ as g; g.build()'` (or make -C distaff_b200/hostvm)")
        lib = ctypes.CDLL(path)
        lib.vm_execute.restype = ctypes.c_void_p
        lib.vm_execute.argtypes = [ctypes.c_char_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint32]
        lib.vm_error.restype = ctypes.c_char_p
        lib.vm_error.argtypes = [ctypes.c_void_p]
        for name in ("vm_width", "vm_ctx_depth", "vm_loop_depth", "vm_stack_depth"):
            getattr(lib, name).restype = ctypes.c_uint32
            getattr(lib, name).argtypes = [ctypes.c_void_p]
        lib.vm_length.restype = ctypes.c_uint64
        lib.vm_length.argtypes = [ctypes.c_void_p]
        lib.vm_program_hash.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        lib.vm_copy_trace.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        lib.vm_free.argtypes = [ctypes.c_void_p]
        lib.vm_compile.restype = ctypes.c_void_p
        lib.vm_compile.argtypes = [ctypes.c_char_p]
        lib.vm_compile_error.restype = ctypes.c_char_p
        lib.vm_compile_error.argtypes = [ctypes.c_void_p]
        lib.vm_compile_sizes.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        lib.vm_compile_copy.argtypes = [ctypes.c_void_p] * 6
        lib.vm_compile_free.argtypes = [ctypes.c_void_p]
        lib.vm_execute_program.restype = ctypes.c_void_p
        lib.vm_execute_program.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p,
                                           ctypes.c_uint32]
        _LIB = lib
    return _LIB


class ExecutionTrace:
    """What crosses the `stark::prove` seam (/root/reference/src/lib.rs:62)."""

    def __init__(self, registers, ctx_depth, loop_depth, stack_depth, program_hash, public_inputs, outputs):
        self.registers = registers          # (w, n, 2) uint64, column-major register traces
        self.ctx_depth = ctx_depth
        self.loop_depth = loop_depth
        self.stack_depth = stack_depth
        self.program_hash = program_hash    # 32 bytes
        self.public_inputs = public_inputs  # list[int]
        self.outputs = outputs              # list[int]

    @property
    def width(self):
        return self.registers.shape[0]

    @property
    def length(self):
        return self.registers.shape[1]


class Program:
    """A compiled program in the flat encoding of include/distaff_gpu.h (dg_program_t): the op codes with one hint per op, the blocks,
    the child lists, the root body and Program::hash() -- what the GPU interpreter (dg_trace_batch / dg_execute_batch) runs.  The
    arrays are ctypes arrays, so tests can alter an encoding before passing it on."""

    def __init__(self, ops, hints, blocks, children, root_first, root_count, hash32):
        from .. import backend
        self.ops = (ctypes.c_uint8 * max(len(ops), 1))(*ops)
        self.hints = (backend.DgOpHint * max(len(hints), 1))(*hints)
        self.n_ops = len(ops)
        self.blocks = (backend.DgBlock * max(len(blocks), 1))(*blocks)
        self.n_blocks = len(blocks)
        self.children = (ctypes.c_uint32 * max(len(children), 1))(*children)
        self.n_children = len(children)
        self.root_first, self.root_count = root_first, root_count
        self.hash = bytes(hash32)

    def c_struct(self):
        """the dg_program_t of this encoding (it points into this object's arrays)"""
        from .. import backend
        return backend.DgProgram(ctypes.cast(self.ops, ctypes.c_void_p), self.hints, self.n_ops, self.blocks, self.n_blocks, self.children,
                                 self.n_children, self.root_first, self.root_count, (ctypes.c_uint8 * 32)(*self.hash))


def compile_program(source):
    """Compiles assembly (programs::assembly::compile) into the program encoding: a Program, whose .hash is Program::hash()."""
    from .. import backend
    lib = _lib()
    h = lib.vm_compile(source.encode())
    try:
        err = lib.vm_compile_error(h)
        if err:
            raise RuntimeError("vm: " + err.decode())
        sizes = (ctypes.c_uint64 * 5)()
        lib.vm_compile_sizes(h, sizes)
        n_ops, n_blocks, n_children, root_first, root_count = (int(x) for x in sizes)
        ops = (ctypes.c_uint8 * max(n_ops, 1))()
        hints = (backend.DgOpHint * max(n_ops, 1))()
        blocks = (backend.DgBlock * n_blocks)()
        children = (ctypes.c_uint32 * n_children)()
        hash32 = ctypes.create_string_buffer(32)
        lib.vm_compile_copy(h, ops, hints, blocks, children, hash32)
    finally:
        lib.vm_compile_free(h)
    return Program(list(ops)[:n_ops], list(hints)[:n_ops], list(blocks), list(children), root_first, root_count, hash32.raw)


def execute_program(program, public_inputs=(), secret_a=(), secret_b=(), num_outputs=1):
    """execute() of a compiled Program: the encoding is decoded back into its block tree and run by the same VM, with the hashes the
    encoding carries.  Same result and errors as execute() of the source."""
    lib = _lib()
    prog = program.c_struct()
    return _run(lambda pub, sa, sb: lib.vm_execute_program(ctypes.byref(prog), pub.ctypes.data, len(pub), sa.ctypes.data, len(sa),
                                                          sb.ctypes.data, len(sb)), public_inputs, secret_a, secret_b, num_outputs)


def execute(source, public_inputs=(), secret_a=(), secret_b=(), num_outputs=1):
    lib = _lib()
    return _run(lambda pub, sa, sb: lib.vm_execute(source.encode(), pub.ctypes.data, len(pub), sa.ctypes.data, len(sa), sb.ctypes.data, len(sb)),
                public_inputs, secret_a, secret_b, num_outputs)


def _run(start, public_inputs, secret_a, secret_b, num_outputs):
    lib = _lib()
    pub = felt.from_ints(public_inputs)
    sa = felt.from_ints(secret_a)
    sb = felt.from_ints(secret_b)
    h = start(pub, sa, sb)
    try:
        err = lib.vm_error(h)
        if err:
            raise RuntimeError("vm: " + err.decode())
        w, n = lib.vm_width(h), lib.vm_length(h)
        regs = np.empty((w, n, 2), dtype=np.uint64)
        lib.vm_copy_trace(h, regs.ctypes.data)
        ph = ctypes.create_string_buffer(32)
        lib.vm_program_hash(h, ph)
        cd, ld, sd = lib.vm_ctx_depth(h), lib.vm_loop_depth(h), lib.vm_stack_depth(h)
    finally:
        lib.vm_free(h)
    assert num_outputs <= 8
    stack_start = 15 + cd + ld
    # outputs = top of the user stack at the last step, padded with zeros to the state's min depth 8 (lib.rs:45-46)
    last = [0] * 8
    for i in range(min(sd, 8)):
        last[i] = felt.to_ints(regs[stack_start + i, n - 1])[0]
    outputs = last[:num_outputs]
    return ExecutionTrace(regs, cd, ld, sd, ph.raw, list(public_inputs), outputs)


# ---- example programs (inputs of BASELINE.json's configs; /root/reference/src/examples/*.rs) --------------------------
def fibonacci_program(n):
    """examples/fibonacci.rs:33-42 ; inputs [1, 0], 1 output"""
    return f"begin repeat.{n - 1} swap dup.2 drop add end end"


def fibonacci(n):
    return execute(fibonacci_program(n), public_inputs=[1, 0], num_outputs=1)


COLLATZ_SOURCE = """
begin
    pad read dup push.1 ne
    while.true
        swap push.1 add swap dup isodd.128
        if.true
            push.3 mul push.1 add
        else
            push.2 div
        end
        dup push.1 ne
    end
    swap
end"""


def collatz(start):
    """examples/collatz.rs:10-23 ; secret tape A = [start], 1 output (number of steps)"""
    return execute(COLLATZ_SOURCE, secret_a=[start], num_outputs=1)


def merkle_program(depth, index):
    """examples/merkle.rs:41-57"""
    return f"begin read.ab dup.2 smpath.{depth} swap.2 push.{index} roll.4 swap swap.2 pmpath.{depth} end"


def merkle_paths(depth, count, seed=0):
    """`count` Merkle authentication paths of length `depth` verified back to back with the program of examples/merkle.rs:41-57 (paths
    drawn from field::prng_vector with the example's seeds, path number in byte 3, `seed` in bytes 4-5: different seeds give different
    traces of one shape).  The example itself is capped at depth 64 = 2^12
    steps by its own index arithmetic (examples/merkle.rs:75,106); four paths give BASELINE's 2^14-step Rescue-dominated trace."""
    import ctypes
    from .. import backend
    L = backend.lib()

    def prng_vector(seed, n):
        out = np.zeros((n, 2), dtype=np.uint64)
        backend.check(L.dg_host_prng_vector(bytes(seed), n, out.ctypes.data))
        return felt.to_ints(out)

    a_all, b_all, blocks = [], [], []
    for c in range(count):
        p0 = prng_vector(bytes([1, 2, 3, c, seed & 255, seed >> 8] + [0] * 26), depth)
        p1 = prng_vector(bytes([4, 5, 6, c, seed & 255, seed >> 8] + [0] * 26), depth)
        leaf_index = p0[0] % (2 ** (depth - 1))
        a, b = [p0[0]], [p1[0]]
        index = leaf_index + 2 ** (depth - 1)
        for i in range(1, depth):
            a += [0, p0[i]]
            b += [index & 1, p1[i]]
            index >>= 1
        for i in range(1, depth):
            a.append(p0[i])
            b.append(p1[i])
        a_all += a
        b_all += b
        blocks.append(f"read.ab dup.2 smpath.{depth} swap.2 push.{leaf_index} roll.4 swap swap.2 pmpath.{depth}")
    return execute("begin " + " drop.4 ".join(blocks) + " end", secret_a=a_all, secret_b=b_all, num_outputs=4)
