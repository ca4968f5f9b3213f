"""Inputs for testing the GPU VM against the host VM (distaff_b200/hostvm/vm.cpp), which runs the same program encoding on the CPU.

Three sets, each a list of Case (name, program, inputs, num_outputs), the program an assembly source or a hand-made hostvm.Program:
  edge_cases()        one family per op over operands at the field's and the 128-bit word's edges (bits 0, 63, 64, 127, M - 1, ...)
  failure_catalogue() one entry per code of distaff_b200/csrc/vm.h: a case that stops with exactly that message, or why no
                      execution can reach it (with an encoding the GPU rejects, where a validation rule is what rules it out)
  generated_cases()   structured random programs over the whole assembly language, most of which run to completion

Everything is deterministic: the same seed gives the same programs and inputs.  Nothing here needs a GPU.
"""
import collections
import ctypes
import random

import distaff_b200 as dg
from distaff_b200 import felt, hostvm

M = felt.M
C = 45 * 2**40 - 1                      # 2^128 mod M
X = dg.ProgramInputs
Case = collections.namedtuple("Case", "name program inputs num_outputs")

EDGE = [0, 1, 2, M - 1, M - 2, (M - 1) // 2, (M + 1) // 2, 2**63, 2**64 - 1, 2**64, 2**64 + 1, 2**127 - 1, 2**127, 2**127 + 1, C,
        2**128 - 2**88]
CMP_BITS = (4, 5, 31, 63, 64, 65, 127, 128)
PATH_DEPTHS = (2, 3, 64, 65, 128, 129, 130, 256)

# op codes (processor/opcodes.rs) and hint kinds (include/distaff_gpu.h)
OPCODES = {"begin": 0x00, "push": 0x1f, "cmp": 0x3f, "rescr": 0x5f, "assert": 0x60, "asserteq": 0x61, "eq": 0x62, "drop": 0x63,
           "drop4": 0x64, "choose": 0x65, "choose2": 0x66, "cswap2": 0x67, "add": 0x68, "mul": 0x69, "and": 0x6a, "or": 0x6b, "inv": 0x6c,
           "neg": 0x6d, "not": 0x6e, "read": 0x70, "read2": 0x71, "dup": 0x72, "dup2": 0x73, "dup4": 0x74, "pad2": 0x75, "swap": 0x78,
           "swap2": 0x79, "swap4": 0x7a, "roll4": 0x7b, "roll8": 0x7c, "binacc": 0x7d, "noop": 0x7f}
H_NONE, H_PUSH, H_EQ, H_RC, H_CMP, H_PMPATH = range(6)
# the op each hint kind belongs to (any other op with that hint fails; NONE belongs to every op but PUSH)
HINT_OP = {H_PUSH: 0x1f, H_EQ: 0x70, H_RC: 0x7d, H_CMP: 0x3f, H_PMPATH: 0x71}


def field_elements(rnd, n):
    return [rnd.randrange(M) for _ in range(n)]


# ---- a. edge operands, one family per op ---------------------------------------------------------------------------------------------
def edge_values(seed=0):
    return EDGE + field_elements(random.Random(seed), 3)


def _path_case(name, depth, index, rnd):
    """examples/merkle.rs for one path of `depth` with leaf `index` (tapes built as hostvm.merkle_paths builds them, values from rnd)"""
    p0, p1 = field_elements(rnd, depth), field_elements(rnd, depth)
    a, b = [p0[0]], [p1[0]]
    node = index + 2 ** (depth - 1)
    for i in range(1, depth):
        a += [0, p0[i]]
        b += [node & 1, p1[i]]
        node >>= 1
    a += p0[1:]
    b += p1[1:]
    src = f"begin read.ab dup.2 smpath.{depth} swap.2 push.{index} roll.4 swap swap.2 pmpath.{depth} end"
    return Case(name, src, X([], a, b), 4)


def edge_cases(seed=0):
    rnd = random.Random(seed)
    vals = edge_values(seed)
    out = []
    for op in ("add", "sub", "mul", "div", "eq", "ne", "assert.eq"):
        out += [Case(op, f"begin {op} end", X([x, y, 7]), 2) for x in vals for y in vals]
    for op in ("neg", "inv", "not", "assert"):
        out += [Case(op, f"begin {op} end", X([x, 7]), 2) for x in vals]
    for op in ("and", "or"):
        out += [Case(op, f"begin {op} end", X(p), 1) for x in vals for y in (0, 1) for p in ([x, y], [y, x])]
    for c in vals:
        out.append(Case("choose.1", "begin choose.1 end", X([vals[3], vals[9], c]), 1))
        out.append(Case("choose.2", "begin choose.2 end", X([vals[3], vals[9], vals[12], vals[14], c, 5]), 2))
    for k in (1, 2, 3, 4):
        out += [Case(f"hash.{k}", f"begin hash.{k} end", X([vals[(i + 5 * j) % len(vals)] for j in range(k)]), 4) for i in range(len(vals))]
    for n in CMP_BITS:
        top = min(2**n, M)
        base = rnd.randrange(top)
        pairs = [(base, base)]
        for bit in (0, 63, 64, 127):
            other = base ^ (1 << bit)
            if other < M:
                pairs += [(base, other), (other, base)]
        if 2**n < M:
            pairs += [(2**n - 1, 2**n), (rnd.randrange(2**n), 2**n + rnd.randrange(M - 2**n))]
        else:
            pairs += [(2**127 - 1, 2**127), (M - 1, M - 2), (2**128 - 2**88, 2**127 + 1)]
        for op in ("gt", "lt"):
            out += [Case(f"{op}.{n}", f"begin {op}.{n} end", X(p), 4) for x, y in pairs for p in ([x, y],)]
        vs = [v for v in (2**n - 1, 2**n, rnd.randrange(top)) if v < M]
        if n == 128:
            vs += [2**127, 2**127 + 1, M - 1, 2**128 - 2**88]
        for op in ("rc", "isodd"):
            out += [Case(f"{op}.{n}", f"begin {op}.{n} end", X([v, 3]), 2) for v in vs]
    for depth in PATH_DEPTHS:
        indices = {0, 1, 2**63, 2**64, 2**127, 2**127 | 2**64 | 2**63 | 1, rnd.randrange(2 ** min(depth - 1, 127))}
        for index in sorted(i for i in indices if i < 2 ** (depth - 1)):
            out.append(_path_case(f"path.{depth}", depth, index, rnd))
    return out


# ---- hand-made encodings ---------------------------------------------------------------------------------------------------------------
def encoding(source, ops=None, hints=None, hash32=None, block_hashes=None):
    """the encoding of `source` with ops {index: op}, hints {index: (kind, n, value)}, Program::hash() and block hashes
    {block: (hash0, hash1, hash2)} replaced.  Hints other than PushValue are not part of the program hash."""
    p = hostvm.compile_program(source)
    for i, op in (ops or {}).items():
        p.ops[i] = op
    for i, (kind, n, value) in (hints or {}).items():
        p.hints[i].kind, p.hints[i].n = kind, n
        ctypes.memmove(p.hints[i].value16, value.to_bytes(16, "little"), 16)
    for b, hs in (block_hashes or {}).items():
        for f, h in zip(("hash0", "hash1", "hash2"), hs):
            ctypes.memmove(getattr(p.blocks[b], f), h.to_bytes(16, "little"), 16)
    if hash32 is not None:
        p.hash = bytes(hash32)
    return p


def op_index(p, op, k=0):
    """index of the k-th `op` (a name of OPCODES) in the encoding"""
    return [i for i in range(p.n_ops) if p.ops[i] == OPCODES[op]][k]


def block_index(p, kind):
    return next(i for i in range(p.n_blocks) if p.blocks[i].kind == kind)


def _hinted(source, op, kind, n=0, value=0, k=0):
    p = hostvm.compile_program(source)
    return encoding(source, hints={op_index(p, op, k): (kind, n, value)})


def _with_op(source, at_op, new_op, k=0):
    p = hostvm.compile_program(source)
    return encoding(source, ops={op_index(p, at_op, k): new_op})


def _wrong_hash(source):
    h = bytearray(hostvm.compile_program(source).hash)
    h[0] ^= 1
    return encoding(source, hash32=bytes(h))


def _wrong_loop_image(source):
    p = hostvm.compile_program(source)
    b = block_index(p, 3)
    image = int.from_bytes(bytes(p.blocks[b].hash0), "little")
    rest = [int.from_bytes(bytes(getattr(p.blocks[b], f)), "little") for f in ("hash1", "hash2")]
    return encoding(source, block_hashes={b: ((image + 1) % M, *rest)})


def _short_span():
    p = hostvm.compile_program("begin noop end")
    p.blocks[0].count = 14
    return p


def _empty_root():
    p = hostvm.compile_program("begin noop end")
    p.root_count = 0
    return p


# ---- b. the failure catalogue --------------------------------------------------------------------------------------------------------
Reached = collections.namedtuple("Reached", "message step case max_steps")
Unreachable = collections.namedtuple("Unreachable", "reason program")

LOOP_SOURCE = "begin push.3 push.1 while.true push.1 neg add dup push.0 ne end drop end"
NEVER_STOPS = "begin push.1 while.true push.1 end end"
COUNTED_CMP = "begin gt.4 end"


def _reached(message, step, program, inputs, no=1, max_steps=None):
    return Reached(message, step, Case(message, program, inputs, no), max_steps)


def failure_catalogue():
    """{code name of vm.h: Reached or Unreachable}.  `step` is the step the message names (None for the codes without one)."""
    gt4 = hostvm.compile_program(COUNTED_CMP)
    return {
        "VM_ASSERT": _reached("ASSERT failed", 2, "begin assert end", X([2])),
        "VM_ASSERTEQ": _reached("ASSERTEQ failed", 2, "begin assert.eq end", X([2**64, 0])),
        "VM_STACK_UNDERFLOW": _reached("stack underflow", 2, "begin add end", X([1])),
        "VM_STACK_OVERFLOW": _reached("stack overflow", 201, "begin " + "push.1 " * 25 + "end", X(list(range(8)))),
        "VM_PUSH_VALUE": Unreachable("validate() rejects a PUSH without a PushValue hint ('PUSH value missing')",
                                     _hinted("begin push.5 end", "push", H_NONE)),
        "VM_EMPTY_TAPE_A": _reached("attempt to read from empty tape A", 2, "begin read end", X()),
        "VM_HINT_READ": _reached("invalid hint for READ", 2, _hinted("begin read end", "read", H_RC, 4), X([], [1])),
        "VM_PMPATH_TAPES": _reached("too few items on tapes for pmpath macro", 2, "begin pmpath.4 end", X([1, 2, 3], [1, 2], [1, 2])),
        "VM_EMPTY_TAPE": _reached("attempt to read from empty tape", 2, "begin read.ab end", X([], [1])),
        "VM_HINT_READ2": _reached("invalid hint for READ2", 2, _hinted("begin read.ab end", "read2", H_EQ), X([], [1], [2])),
        "VM_CHOOSE": _reached("CHOOSE on a non-binary condition", 2, "begin choose.1 end", X([1, 2, 2**64])),
        "VM_CHOOSE2": _reached("CHOOSE2 on a non-binary condition", 2, "begin choose.2 end", X([1, 2, 3, 4, 2**64 + 1, 5])),
        "VM_CSWAP2": _reached("CSWAP2 on a non-binary condition", 2, _with_op("begin choose.2 end", "choose2", OPCODES["cswap2"]),
                              X([1, 2, 3, 4, M - 1, 5])),
        "VM_INV_ZERO": _reached("cannot compute INV of 0", 2, "begin inv end", X([0])),
        "VM_NOT": _reached("NOT of a non-binary value", 2, "begin not end", X([2**127])),
        "VM_AND": _reached("AND of a non-binary value", 2, "begin and end", X([1, 2**64])),
        "VM_OR": _reached("OR of a non-binary value", 2, "begin or end", X([0, M - 1])),
        # eq with its aux value read from tape A instead of computed by the EqStart hint
        "VM_EQ_AUX": _reached("invalid AUX value for EQ", 3, _hinted("begin eq end", "read", H_NONE), X([5, 2**64 + 5], [7])),
        "VM_HINT_CMP": _reached("invalid hint for CMP", 10, _hinted(COUNTED_CMP, "cmp", H_PMPATH, 4), X([3, 9])),
        "VM_BINARY": _reached("expected binary input", 10, _hinted(COUNTED_CMP, "cmp", H_NONE), X([3, 9], [2], [0])),
        "VM_CMP_POW2": _reached("expected top of the stack to be a power of 2", 10,
                                encoding(COUNTED_CMP, hints={op_index(gt4, "push"): (H_PUSH, 0, 3)}), X([3, 9])),
        "VM_HINT_BINACC": _reached("invalid hint for BINACC", 12, _hinted("begin rc.4 end", "binacc", H_CMP, 4), X([3])),
        # bit 128 of the index: BINACC's power of two has become 2^128 mod M
        "VM_BINACC_POW2": Reached("expected 3rd value from the top of the stack to be a power of 2", 6176,
                                  _path_case("path.130", 130, 2**127 + 1, random.Random(7)), None),
        "VM_UNKNOWN_OP": _reached("unknown opcode", 2, _with_op("begin noop end", "noop", 0x01), X()),
        "VM_OPVALUE": _reached("op_value is non-zero for a non-PUSH operation", 1, _hinted("begin noop end", "noop", H_PUSH, 0, 9), X()),
        "VM_PUSH_ALIGN": Unreachable("validate() puts every PUSH on a multiple of 8 inside its span ('PUSH must be on a step which is a "
                                     "multiple of 8'), spans start on multiples of 16, and a PushValue on another op fails first",
                                     _with_op("begin noop end", "noop", OPCODES["push"], 2)),
        "VM_CTX_OVERFLOW": Unreachable("validate() rejects blocks nested more than 15 deep (the host VM runs them and stops with "
                                       "'context stack overflow')", "begin " + "block " * 16 + "noop " + "end " * 16 + "end"),
        "VM_CTX_UNDERFLOW": Unreachable("every end of a block pops the context its start pushed, and the root's context is there from "
                                        "the first step: no encoding can pop more", None),
        "VM_LOOP_OVERFLOW": Unreachable("validate() rejects loops nested more than 8 deep (the host VM runs them and stops with 'loop "
                                        "stack overflow')", "begin " + "push.1 while.true " * 9 + "push.0 " + "end " * 9 + "end"),
        "VM_LOOP_UNDERFLOW": Unreachable("a loop is wrapped or broken only at the end of its own body, after its start pushed the "
                                         "image: no encoding can pop more", None),
        "VM_START_ALIGN": Unreachable("validate() makes every span 16k + 15 ops long, so every block starts, ends, wraps and breaks on "
                                      "the step the decoder needs", _short_span()),
        "VM_END_ALIGN": Unreachable("as VM_START_ALIGN", _short_span()),
        "VM_LOOP_ALIGN": Unreachable("as VM_START_ALIGN", _short_span()),
        "VM_WRAP_ALIGN": Unreachable("as VM_START_ALIGN", _short_span()),
        "VM_BREAK_ALIGN": Unreachable("as VM_START_ALIGN", _short_span()),
        "VM_LOOP_IMAGE": _reached("hash of the last iteration doesn't match loop image", 64, _wrong_loop_image(LOOP_SOURCE), X()),
        "VM_SWITCH_COND": _reached("cannot select a branch based on a non-binary condition", 16,
                                   "begin noop if.true push.1 else push.2 end end", X([2**64])),
        "VM_LOOP_EXIT_COND": _reached("cannot exit loop based on a non-binary condition", 31,
                                      "begin push.1 while.true push.2 end end", X()),
        "VM_LOOP_ENTER_COND": _reached("cannot enter loop based on a non-binary condition", 15,
                                       "begin noop while.true push.1 push.0 end end", X([M - 1])),
        "VM_CAP": _reached("execution exceeds 1024 steps", None, NEVER_STOPS, X(), max_steps=1024),
        "VM_MIN_OPS": Unreachable("a root body starts with a span of at least 15 ops and closes with 15 NOOPs, so every execution "
                                  "runs at least 30; validate() rejects an empty root body", _empty_root()),
        "VM_HASH": _reached("program hash does not match trace hash", None, _wrong_hash(LOOP_SOURCE), X()),
        "VM_TAPE_SCRATCH": Unreachable("internal: the shape pass runs again with 16 times more tape scratch (see tape_scratch_case)",
                                       None),
        "VM_DIVERGED": Unreachable("a guard: control flow never reads the sponge, so the write pass retraces the shape pass", None),
    }


def input_failures():
    """executions that fail before they run, on their inputs: [(case, message)]"""
    src = "begin add end"
    return [
        (Case("tape B longer", src, X([1, 2], [1], [1, 2]), 1), "tape A cannot be shorter than tape B"),
        (Case("9 public inputs", src, X(list(range(9))), 1), "expected no more than 8 public inputs"),
        (Case("public input M", src, X([1, 2, M]), 1), "public input 2 is not a field element"),
        (Case("public input 2^128 - 1", src, X([2**128 - 1, 2]), 1), "public input 0 is not a field element"),
        (Case("tape A value M + 1", "begin read add end", X([1], [3, 4, M + 1]), 1), "tape A value 2 is not a field element"),
        (Case("tape B value 2^128 - 2^40", "begin read.ab add end", X([1], [3, 4], [2**128 - 2**40]), 1), "tape B value 0 is not a field element"),
        (Case("public before tapes", src, X([M, 1], [M]), 1), "public input 0 is not a field element"),
    ]


def tape_scratch_case():
    """rc.128 whose 2nd and 3rd BINACC also carry RcStart(128): more bits on tape A than the shape pass's first tape scratch holds"""
    p = hostvm.compile_program("begin push.5 rc.128 end")
    binacc = [i for i in range(p.n_ops) if p.ops[i] == OPCODES["binacc"]]
    for i in binacc[1:3]:
        p.hints[i].kind, p.hints[i].n = H_RC, 128
    return Case("tape scratch regrowth", p, X(), 2)


def short_hint_cases():
    """RcStart / CmpStart with n in 1..3: validation allows them, the assembler never emits them"""
    out = []
    for n in (1, 2, 3):
        out.append(Case(f"rc hint {n}", _hinted("begin rc.4 end", "binacc", H_RC, n), X([5], [1, 0, 1, 1, 0, 1]), 2))
        out.append(Case(f"cmp hint {n}", _hinted(COUNTED_CMP, "cmp", H_CMP, n), X([5, 3], [1, 0, 1, 1], [0, 1, 1, 0]), 4))
    return out


def catalogue_cases():
    """every case of the catalogue and around it that runs (the step cap's aside: the host VM has no cap)"""
    out = [e.case for e in failure_catalogue().values() if isinstance(e, Reached) and e.max_steps is None]
    out += [c for c, _ in input_failures()]
    out += [tape_scratch_case()] + short_hint_cases()
    out.append(Case("eq aux from tape", _hinted("begin eq end", "read", H_NONE), X([5, 2**64 + 5], [inv(5 - 2**64 - 5)]), 1))
    out.append(Case("wrong switch hash", encoding(IF_SOURCE, block_hashes={block_index(hostvm.compile_program(IF_SOURCE), 2): (1, 2, 0)}),
                    X([], [1]), 1))
    return out


IF_SOURCE = "begin read if.true push.3 else push.4 end end"


def inv(x):
    return pow(x % M, M - 2, M)


# ---- c. generated programs -----------------------------------------------------------------------------------------------------------
PUSH_VALUES = EDGE[:-1] + [3, 5, 2**32, 2**62]   # push values must be below M: 2^128 - 2^88 is; every one of EDGE is


class _Gen:
    """One random program.  The stack is modelled as a list of kinds, top first: 'z' (zero), 'b' (binary) or 'a'; ops that need binary
    operands or a depth the model does not have are mostly avoided, so that most programs run to completion."""

    def __init__(self, rnd, n_pub):
        self.r = rnd
        self.n_pub = n_pub
        self.loops = 0
        self.nest = 0

    def value(self):
        return self.r.choice(PUSH_VALUES)

    def op(self, s, floor, out):
        r = self.r
        avail = len(s) - floor
        grow = len(s) < 22
        choices = []
        if grow:
            choices += ["push", "push", "read", "read.ab", "pad", "dup"]
        if avail >= 1:
            choices += ["neg", "inv", "not", "rc", "isodd", "drop", "hash"]
        if avail >= 2:
            choices += ["add", "sub", "mul", "div", "eq", "ne", "gt", "lt", "swap", "and", "or", "assert.eq", "pick"]
        if avail >= 3:
            choices += ["choose.1"]
        if avail >= 4:
            choices += ["swap.2", "roll.4", "pick"]
        if avail >= 6:
            choices += ["choose.2"]
        if avail >= 8:
            choices += ["swap.4", "roll.8"]
        if avail >= 1 and s[0] in "bz" and r.random() < 0.15:
            choices += ["assert"]
        if not choices:                        # a full stack with nothing above the floor
            out.append("noop")
            return
        name = r.choice(choices)
        binary_needs = {"not": [0], "and": [0, 1], "or": [0, 1], "choose.1": [2], "choose.2": [4]}
        if name in binary_needs and any(s[i] not in "bz" for i in binary_needs[name]) and r.random() < 0.97:
            return self.op(s, floor, out)
        if name in ("inv", "div") and s[0] in "bz" and r.random() < 0.9:      # a zero divisor is likely
            return self.op(s, floor, out)
        if name == "push":
            v = self.value()
            out.append(f"push.{v}")
            s.insert(0, "z" if v == 0 else "b" if v == 1 else "a")
        elif name == "read":
            out.append("read")
            s.insert(0, "a")
        elif name == "read.ab":
            out.append("read.ab")
            s[:0] = ["a", "a"]
        elif name == "pad":
            n = r.randint(1, min(8, 26 - len(s)))
            out.append(f"pad.{n}")
            s[:0] = ["z"] * n
        elif name == "dup":
            n = r.randint(1, min(4, avail)) if avail else 0
            if n == 0:
                return self.op(s, floor, out)
            out.append(f"dup.{n}")
            s[:0] = s[:n]
        elif name == "drop":
            n = r.randint(1, min(8, avail))
            out.append(f"drop.{n}")
            del s[:n]
        elif name in ("neg", "inv"):
            out.append(name)
            s[0] = "a"
        elif name == "not":
            out.append("not")
            s[0] = "b"
        elif name in ("rc", "isodd"):
            n = r.choice([128] * 8 + [64, 8]) if name == "isodd" else r.choice([128, 64, 32, 8])
            out.append(f"{name}.{n}")
            s[0] = "b"
        elif name == "hash":
            k = r.randint(1, min(4, avail))
            out.append(f"hash.{k}")
            s[:k] = ["a", "a"]
        elif name in ("add", "sub", "mul", "div"):
            out.append(name)
            s[:2] = ["a"]
        elif name in ("eq", "ne", "and", "or"):
            out.append(name)
            s[:2] = ["b"]
        elif name in ("gt", "lt"):
            n = r.choice([128] * 8 + [65, 5])
            out.append(f"{name}.{n}")
            s[:2] = ["b"]
        elif name == "assert.eq":
            if r.random() < 0.9:
                out.append("dup")
                s.insert(0, s[0])
            out.append("assert.eq")
            del s[:2]
        elif name == "assert":
            out.append("assert")
            del s[:1]
        elif name == "swap":
            out.append("swap")
            s[0], s[1] = s[1], s[0]
        elif name == "swap.2":
            out.append("swap.2")
            s[:4] = s[2:4] + s[0:2]
        elif name == "swap.4":
            out.append("swap.4")
            s[:8] = s[4:8] + s[0:4]
        elif name == "roll.4":
            out.append("roll.4")
            s[:4] = [s[3]] + s[0:3]
        elif name == "roll.8":
            out.append("roll.8")
            s[:8] = [s[7]] + s[0:7]
        elif name == "pick":
            n = r.choice([1] if avail < 4 else [1, 2, 3])
            out.append(f"pick.{n}")
            s.insert(0, s[n])
        elif name == "choose.1":
            out.append("choose.1")
            s[:3] = ["a"]
        elif name == "choose.2":
            out.append("choose.2")
            s[:6] = ["a", "a"]

    def balance(self, s, depth, out):
        """drop or pad to `depth` (kinds below it unchanged)"""
        while len(s) > depth:
            n = min(8, len(s) - depth)
            out.append(f"drop.{n}")
            del s[:n]
        while len(s) < depth:
            n = min(8, depth - len(s))
            out.append(f"pad.{n}")
            s[:0] = ["z"] * n

    def condition(self, s, out):
        if s and s[0] in "bz" and self.r.random() < 0.5:
            return
        if len(s) >= 2 and self.r.random() < 0.5:
            out += ["dup.2", self.r.choice(["gt.128", "lt.128", "eq", "ne"])]
            s.insert(0, "b")
        elif self.r.random() < 0.9:
            out.append(f"push.{self.r.randint(0, 1)}")
            s.insert(0, "b")

    def body(self, s, floor, size, out):
        for _ in range(size):
            k = self.r.random()
            if self.nest < 3 and k < 0.08:
                self.nest += 1
                out.append("block")
                self.body(s, floor, self.r.randint(1, 4), out)
                out.append("end")
                self.nest -= 1
            elif self.nest < 3 and k < 0.18:
                self.nest += 1
                self.condition(s, out)
                if not s or len(s) <= floor:
                    s.insert(0, "a")
                    out.append("push.1")
                s.pop(0)
                depth = len(s)
                t = list(s)
                out.append("if.true")
                self.body(t, floor, self.r.randint(1, 4), out)
                self.balance(t, depth, out)
                if self.r.random() < 0.7:
                    f = list(s)
                    out.append("else")
                    start = len(out)
                    self.body(f, floor, self.r.randint(1, 4), out)
                    self.balance(f, depth, out)
                    if len(out) == start:
                        out.append("noop")
                else:
                    f = list(s)
                if out[-1] in ("if.true", "else"):
                    out.append("noop")
                out.append("end")
                s[:] = [x if x == y else "b" if x in "bz" and y in "bz" else "a" for x, y in zip(t, f)]
                self.nest -= 1
            elif self.nest < 3 and self.loops < 2 and k < 0.25:
                self.nest += 1
                self.loops += 1
                out += [f"push.{self.r.randint(1, 3)}", "push.1", "while.true"]
                s.insert(0, "a")                       # the counter, below the body's floor
                inner = len(s)
                t = list(s)
                self.body(t, inner, self.r.randint(1, 4), out)
                self.balance(t, inner, out)
                out += ["push.1", "neg", "add", "dup", "push.0", "ne", "end", "drop"]
                s.pop(0)
                self.loops -= 1
                self.nest -= 1
            elif self.nest < 3 and k < 0.30:
                self.nest += 1
                depth = len(s)
                out.append(f"repeat.{self.r.randint(2, 3)}")
                self.body(s, floor, self.r.randint(1, 3), out)
                self.balance(s, depth, out)
                if out[-1].startswith("repeat."):
                    out.append("noop")
                out.append("end")
                self.nest -= 1
            else:
                self.op(s, floor, out)

    def program(self):
        s = ["a"] * self.n_pub
        out = []
        self.body(s, 0, self.r.randint(3, 14), out)
        if not out:
            out.append("noop")
        return "begin " + " ".join(out) + " end", len(s)


def generated_cases(seed=1, programs=300, inputs_per_program=3):
    rnd = random.Random(seed)
    out = []
    for p in range(programs):
        n_pub = rnd.randint(0, 8)
        src, depth = _Gen(rnd, n_pub).program()
        for i in range(inputs_per_program):
            pub = [rnd.choice(PUSH_VALUES[1:] + [1, rnd.randrange(M)]) for _ in range(n_pub)]
            a = [rnd.choice([1, rnd.randrange(M), rnd.randrange(M), rnd.choice(EDGE)]) for _ in range(48)]
            b = [rnd.choice([1, rnd.randrange(M), rnd.randrange(M), rnd.choice(EDGE)]) for _ in range(24)]
            out.append(Case(f"generated {p}.{i}", src, X(pub, a, b), min(8, max(depth, 1))))
    return out


# ---- trace-length boundaries ----------------------------------------------------------------------------------------------------------
def noop_program(last_step):
    """a program whose last step is `last_step` (16 t + 15, t >= 1): BEGIN and NOOPs, then the root's closing 16 steps"""
    assert last_step % 16 == 15 and last_step >= 31
    return "begin " + "noop " * (last_step - 31 + 14) + "end"


def boundary_cases(ks=(5, 6, 8, 10, 12)):
    """last steps around 2^k: the last step is always 16 t + 15, so 2^k - 17, 2^k - 1 (the last row of a 2^k trace) and 2^k + 15 (the
    first that needs 2^(k+1) rows)"""
    out = []
    for k in ks:
        for last in (2**k - 17, 2**k - 1, 2**k + 15):
            if last >= 31:
                out.append(Case(f"last step {last}", noop_program(last), X([k]), 1))
    return out


# ---- the oracle -----------------------------------------------------------------------------------------------------------------------
_COMPILED = {}


def compiled(program):
    if not isinstance(program, str):
        return program
    if program not in _COMPILED:
        _COMPILED[program] = hostvm.compile_program(program)
    return _COMPILED[program]


def host(case):
    """the host VM on the case's encoding: an ExecutionTrace, or the message of its failure"""
    x = case.inputs
    try:
        return hostvm.execute_program(compiled(case.program), x.public, x.secret_a, x.secret_b, case.num_outputs)
    except RuntimeError as e:
        return str(e)[len("vm: "):]
