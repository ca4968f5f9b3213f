"""Sources and inputs of the programs the execution tests run, restated from tests/programs.py (which builds traces, not sources):
(name, source, public inputs, secret tape A, secret tape B, number of outputs)."""
import numpy as np

from distaff_b200 import hostvm

LOOP3 = ("push.2 push.1 while.true push.2 push.1 while.true push.2 push.1 while.true push.1 neg add dup push.0 ne end drop "
         "push.1 neg add dup push.0 ne end drop push.1 neg add dup push.0 ne end drop")
WIDE_SOURCE = "begin " + " ".join(f"push.{i + 1}" for i in range(26)) + " " + "block push.1 add " * 15 + "end " * 15 + " " + LOOP3 + " end"
IF_ELSE = "begin push.3 push.5 read if.true add else mul end end"

# the 17 programs of small_programs() (and tests/golden/oracle_proofs.json), in its order
SMALL = [
    ("fib13", hostvm.fibonacci_program(13), [1, 0], [], [], 1),
    ("fib_span", "begin swap dup.2 drop add swap dup.2 drop add swap dup.2 drop add end", [1, 0], [], [], 1),
    ("stack_ops", "begin swap swap.2 swap.4 roll.4 roll.8 pad.2 drop.2 dup dup.2 dup.4 drop.8 end", [1, 2, 3, 4, 5, 6, 7, 8], [], [], 8),
    ("logic", "begin not and or end", [1, 1, 0, 1], [], [], 2),
    ("arith", "begin add mul inv neg push.3 sub push.9 div end", [2, 3, 4], [], [], 1),
    ("eq", "begin eq swap.2 ne and end", [5, 5, 9, 6, 7], [], [], 1),
    ("cmp", "begin push.5 push.11 gt.8 push.7 push.3 lt.8 and end", [], [], [], 1),
    ("rc", "begin push.200 rc.8 push.300 rc.8 end", [], [], [], 2),
    ("choose", "begin choose swap.2 choose.2 end", [3, 4, 1, 5, 6, 7, 0, 8], [], [], 3),
    ("hash", "begin pad.2 hash.2 end", [5, 6], [], [], 2),
    ("if_else", IF_ELSE, [], [1], [], 1),
    ("if_else0", IF_ELSE, [], [0], [], 1),
    ("nested", "begin push.2 block push.3 block push.4 add end mul end add end", [1], [], [], 1),
    ("collatz3", hostvm.COLLATZ_SOURCE, [], [3], [], 1),
    ("deep_stack", "begin " + " ".join(f"push.{i + 1}" for i in range(22)) + " add mul swap.4 roll.8 dup.4 drop.8 end", [9, 8, 7], [], [], 4),
    ("deep_ctx", "begin push.1 block push.2 block push.3 block push.4 add end add end add end end", [], [], [], 1),
    ("nested_loops", "begin push.2 push.1 while.true push.3 push.1 while.true push.1 neg add dup push.0 ne end drop push.1 neg add dup "
                     "push.0 ne end end", [], [], [], 1),
]

# gt.n / lt.n / rc.n / eq on public inputs: with pmpath (merkle) every hint kind
COMPARE_SOURCE = "begin dup.2 gt.32 drop dup.2 lt.32 drop dup.2 eq drop dup.2 ne drop dup rc.32 drop end"


def merkle_case(depth, count, seed=0, index_of=None):
    """source, tape A, tape B of hostvm.merkle_paths(depth, count, seed); index_of(c) replaces the leaf index of path c"""
    from distaff_b200 import backend, felt
    L = backend.lib()

    def prng_vector(s, n):
        out = np.zeros((n, 2), dtype=np.uint64)
        backend.check(L.dg_host_prng_vector(bytes(s), n, out.ctypes.data))
        return felt.to_ints(out)

    a_all, b_all, blocks = [], [], []
    for c in range(count):
        p0 = prng_vector(bytes([1, 2, 3, c, seed & 255, seed >> 8] + [0] * 26), depth)
        p1 = prng_vector(bytes([4, 5, 6, c, seed & 255, seed >> 8] + [0] * 26), depth)
        leaf_index = p0[0] % (2 ** (depth - 1)) if index_of is None else index_of(c)
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
    return "begin " + " drop.4 ".join(blocks) + " end", a_all, b_all


def tape_growing_program():
    """rc.128 whose 2nd and 3rd BINACC also carry RcStart(128): the hints leave 381 bits on tape A before the macro has popped them,
    more than the 256 elements of scratch the shape pass starts with (a hand-made encoding; the assembler never emits it)"""
    prog = hostvm.compile_program("begin push.5 rc.128 end")
    binacc = [i for i in range(prog.n_ops) if prog.ops[i] == 0x7d]
    for i in binacc[1:3]:
        prog.hints[i].kind, prog.hints[i].n = 3, 128          # DG_HINT_RC_START
    return prog


def shared_block_program(levels=14, fanout=10):
    """a valid encoding whose every group body refers to the group below it `fanout` times: fanout ** levels paths through a DAG of
    levels + 3 blocks, nested 15 lists deep"""
    from distaff_b200 import backend
    ops = [0x00] + [0x7f] * 14 + [0x7f] * 15                  # span 0: BEGIN + 14 NOOP (the root's first), span 1: 15 NOOP
    hints = [backend.DgOpHint() for _ in ops]
    blocks = [backend.DgBlock(0, 0, 15, 0, 0), backend.DgBlock(0, 15, 15, 0, 0)]
    children = [1]                                          # the body of group 0: one span
    blocks.append(backend.DgBlock(1, 0, 1, 0, 0))
    for _ in range(levels - 1):
        first = len(children)
        for _ in range(fanout):
            children += [1, len(blocks) - 1]
        blocks.append(backend.DgBlock(1, first, 2 * fanout, 0, 0))
    root_first = len(children)
    children += [0, len(blocks) - 1]
    return hostvm.Program(ops, hints, blocks, children, root_first, 2, bytes(32))
