"""The case sets of tests/vm_cases.py on the host VM alone: what they cover (every opcode in a successful trace, every hint kind on every
op it belongs to and on one it does not, every failure code of the GPU VM either reached with its message and step or ruled out with a
reason), that they are deterministic, and the host VM's rule for inputs that are not field elements."""
import functools
import os
import re

import numpy as np
import pytest

from distaff_b200 import hostvm
from tests import vm_cases as vc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@functools.lru_cache(maxsize=None)
def _runs():
    """(case, host result) of every case that runs on the host VM"""
    cases = vc.edge_cases() + vc.catalogue_cases() + vc.generated_cases() + vc.boundary_cases()
    return [(c, vc.host(c)) for c in cases]


def _vm_codes():
    text = open(os.path.join(ROOT, "distaff_b200", "csrc", "vm.h")).read()
    body = text[text.index("enum VmCode"):]
    body = body[:body.index("};")]
    body = re.sub(r"//[^\n]*", "", body)
    return [n for n in re.findall(r"\b(VM_[A-Z0-9_]+)\b", body) if n not in ("VM_OK", "VM_NO_STEP")]


def _user_ops(tr):
    """the user op of every HACC row (flow bits, columns 5-7, all zero): columns 8-14 are its 7 bits"""
    bits = tr.registers[5:15, :, 0].astype(np.int64)
    flow = bits[0] + 2 * bits[1] + 4 * bits[2]
    user = sum(bits[3 + i] << i for i in range(7))
    return set(int(u) for u in user[flow == 0])


def _last_step(tr):
    flow = tr.registers[5, :, 0] & tr.registers[6, :, 0] & tr.registers[7, :, 0]
    return int(np.argmax(flow == 1))          # rows from the last step on are padding: every op bit 1


def test_every_opcode_occurs_in_a_successful_trace():
    seen = set()
    for _, r in _runs():
        if not isinstance(r, str):
            seen |= _user_ops(r)
    assert seen == set(vc.OPCODES.values()), sorted(set(vc.OPCODES.values()) - seen)
    assert len(seen) == 32


def test_every_hint_kind_on_its_op_and_on_another():
    pairs = set()
    programs = [c.program for c, _ in _runs()]
    programs += [e.program for e in vc.failure_catalogue().values() if isinstance(e, vc.Unreachable) and e.program is not None]
    for prog in {id(p): p for p in map(vc.compiled, programs)}.values():
        pairs |= {(prog.hints[i].kind, prog.ops[i]) for i in range(prog.n_ops)}
    for kind, op in vc.HINT_OP.items():
        assert (kind, op) in pairs, kind
        assert any(k == kind and o != op for k, o in pairs), kind
    for op in vc.OPCODES.values():
        if op != vc.OPCODES["push"]:
            assert (vc.H_NONE, op) in pairs, hex(op)
    assert (vc.H_NONE, vc.OPCODES["push"]) in pairs            # the catalogue's PUSH without a value
    assert len({k for k, _ in pairs}) == 6


def test_the_catalogue_lists_every_code_of_the_vm():
    cat = vc.failure_catalogue()
    assert sorted(cat) == sorted(_vm_codes())
    messages = open(os.path.join(ROOT, "distaff_b200", "csrc", "vm.cu")).read()
    reached = [k for k, e in cat.items() if isinstance(e, vc.Reached)]
    assert len(reached) >= 28
    for name, e in cat.items():
        if isinstance(e, vc.Unreachable):
            assert e.reason, name
            continue
        assert '"' + e.message.removesuffix(" 1024 steps") in messages, name        # vm_message's text


@pytest.mark.parametrize("name", [k for k, e in vc.failure_catalogue().items() if isinstance(e, vc.Reached) and e.max_steps is None])
def test_each_reachable_failure_gives_its_message_and_step(name):
    e = vc.failure_catalogue()[name]
    want = e.message if e.step is None else f"{e.message} at step {e.step}"
    assert vc.host(e.case) == want


def test_the_host_vm_reaches_what_validation_rules_out():
    """nesting deeper than the context or loop stack holds: the host VM runs the encoding and stops; the GPU call rejects it"""
    cat = vc.failure_catalogue()
    for name, want in (("VM_CTX_OVERFLOW", "context stack overflow at step 256"), ("VM_LOOP_OVERFLOW", "loop stack overflow at step 144")):
        assert vc.host(vc.Case(name, cat[name].program, vc.X(), 1)) == want


def test_inputs_that_are_not_field_elements_fail_before_the_vm_runs():
    for case, want in vc.input_failures():
        assert vc.host(case) == want, case.name
        x = case.inputs
        with pytest.raises(RuntimeError, match="^vm: " + re.escape(want) + "$"):
            hostvm.execute(case.program, x.public, x.secret_a, x.secret_b)
    # M - 1 and every other canonical value is accepted
    tr = hostvm.execute("begin add end", [vc.M - 1, vc.M - 1], [vc.M - 1], [vc.M - 1])
    assert tr.outputs == [vc.M - 2]


def test_paths_past_bit_127_stop_at_the_power_of_two():
    """pmpath.n reads n - 1 index bits, lowest first: bit 128 meets BINACC's power of two at 2^128 mod M, which is none"""
    for c, r in _runs():
        if c.name.startswith("path."):
            depth = int(c.name.split(".")[1])
            if depth <= 129:
                assert not isinstance(r, str), (c.name, r)
            else:
                assert r.startswith("expected 3rd value from the top of the stack to be a power of 2 at step "), (c.name, r)


def test_generated_programs_mostly_complete_and_fail_in_varied_ways():
    runs = [(c, r) for c, r in _runs() if c.name.startswith("generated")]
    assert len({c.program for c, _ in runs}) == 300 and len(runs) == 900
    ok = [r for _, r in runs if not isinstance(r, str)]
    assert 0.6 <= len(ok) / len(runs) <= 0.95
    failures = {r.split(" at step")[0] for _, r in runs if isinstance(r, str)}
    assert len(failures) >= 6, failures
    assert max(r.length for r in ok) <= 2**13
    assert {r.loop_depth for r in ok} >= {0, 1} and max(r.ctx_depth for r in ok) >= 3


def test_generator_is_deterministic():
    def key(cases):
        return [(c.name, c.program if isinstance(c.program, str) else bytes(c.program.ops), c.inputs.public, c.inputs.secret_a,
                 c.inputs.secret_b, c.num_outputs) for c in cases]
    assert key(vc.generated_cases(seed=5, programs=20)) == key(vc.generated_cases(seed=5, programs=20))
    assert key(vc.generated_cases(seed=5, programs=20)) != key(vc.generated_cases(seed=6, programs=20))
    assert key(vc.edge_cases()) == key(vc.edge_cases())
    assert key(vc.catalogue_cases()) == key(vc.catalogue_cases())


def test_trace_length_boundaries_on_the_host():
    for c, r in _runs():
        if c.name.startswith("last step"):
            last = int(c.name.split()[-1])
            assert _last_step(r) == last
            length = 16
            while length <= last:
                length *= 2
            assert r.length == length, c.name
