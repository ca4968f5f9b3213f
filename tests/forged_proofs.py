"""Forged proofs for the verifier tests: proofs of false statements whose commitments are all consistent.

The oracle's prover (oracle/stark.h, `Forgery`) changes one value before it is committed and derives every root, Fiat-Shamir draw,
PoW nonce, query position and opening from the changed value.  Such a proof passes the Merkle and PoW checks, so only the verifier's
algebraic checks can reject it: C(z) against the committed constraint values, each FRI fold against the next layer, the remainder
against the last fold and against the degree bound.  Bit flips almost never get that far.

`cases()` lists every case with the verdict the restated reference verifier must give, derived from what was changed:
- a false statement (a broken transition, a wrong op count, an offset constraint polynomial, a wrong DEEP value) and an offset first FRI
  layer make the DEEP composition at the queries differ from FRI layer 0 ("depth 0"); an op count below 16 fails before that;
- FRI values offset at layer d fail at depth d, a layer folded at the wrong point fails at depth d + 1, and both fail at the remainder
  when the next values are the remainder;
- a changed remainder value that no query opens fails the degree check over all remainder points;
- a proof with a different number of folds is still honest: the reference accepts it when 4^folds divides the trace length, and
  otherwise its truncating division of the degree bound (fri/verifier.rs:86) rejects the remainder;
- a remainder cut below the degree bound, and one cut to no more values than the bound, reach the two branches of the bound check.
  With a whole remainder of R points the bound is floor(7R / blowup), below the R - R / blowup points the check uses for every
  blowup >= 16, so no proof with a whole remainder reaches them.
"""
import functools
import os

from tests import programs

LDP = "verification of low-degree proof failed: "
DEPTH = LDP + "evaluations did not match column value at depth %d"
INCONSISTENT = LDP + "remainder values are inconsistent with values of the last column"
NOT_LOW_DEGREE = LDP + "remainder is not a valid degree %d polynomial"
BOUND_TOO_LARGE = LDP + "remainder degree is greater than number of remainder values"
MIN_OP_COUNT = "Verification of minimum operation count failed"
# the reference panics (index out of bounds) where the degree bound exceeds the remainder points it does not skip; the oracle throws
OUT_OF_BOUNDS = "exception: index out of bounds: the len is %d but the index is %d"

# (ext, queries, grinding) per program; collatz3 and the 65-register program stay away from blowup 256, where fri/verifier.rs:86
# rejects their honest proofs
OPTIONS = {
    "fib13": [(16, 30, 8), (32, 50, 8), (64, 20, 8), (128, 10, 4), (256, 5, 4)],
    "collatz3": [(16, 30, 8), (64, 20, 8)],
    "wide": [(16, 30, 8)],
    "deep_ctx": [(32, 50, 8), (128, 10, 4)],
}
# few queries, so that a PoW nonce whose queries open only the first half of the remainder is quick to find
CUT_OPTIONS = (16, 4, 8)


@functools.lru_cache(maxsize=None)
def traces():
    small = programs.small_programs()
    return {"fib13": small["fib13"], "collatz3": small["collatz3"], "wide": programs.wide_program(), "deep_ctx": small["deep_ctx"]}


def fri_layers(n, ext):
    """number of FRI layers of an honest proof (fri/prover.rs:21: fold while the domain exceeds 256 points)"""
    domain, layers = n * ext, 0
    while domain > 256:
        domain //= 4
        layers += 1
    return layers


def remainder_bound(n, layers):
    """the verifier's degree bound plus one at the remainder: get_composition_degree(n) + 1, divided by 4 per layer"""
    bound = 7 * n
    for _ in range(layers):
        bound //= 4
    return bound


def folded_verdict(n, layers):
    """verdict on an honest proof with `layers` FRI layers: the composition has degree 7n - 1 and each fold divides the degree by 4
    (rounding down), so the remainder fits the verifier's bound exactly when 4^layers divides n"""
    if n % 4 ** layers == 0:
        return None
    return NOT_LOW_DEGREE % ((remainder_bound(n, layers) - 1) % 2**64)       # usize arithmetic: a bound of 0 wraps


def _registers(tr):
    """a decoder register (sponge[0]), the first context register, the first loop register if any, and the top of the user stack"""
    regs = [1, 15]
    if tr.loop_depth:
        regs.append(15 + tr.ctx_depth)
    regs.append(15 + tr.ctx_depth + tr.loop_depth)
    return regs


def cases():
    """[(case id, program, (ext, queries, grinding), forge, expected oracle verdict)]"""
    out = []
    for prog, option_sets in OPTIONS.items():
        tr = traces()[prog]
        n = tr.length
        for k, opt in enumerate(option_sets):
            L = fri_layers(n, opt[0])
            tag = "%s/%d" % (prog, opt[0])
            add = lambda forge, want: out.append(("%s/%s" % (tag, ":".join(map(str, forge))), prog, opt, forge, want))
            if k == 0:                                 # false statements, at the first option set of each program
                add(("transition", n // 3), DEPTH % 0)
                add(("op_count", 16), DEPTH % 0)
                add(("op_count", 15), MIN_OP_COUNT)
                add(("constraint_offset", 1), DEPTH % 0)
                for j in _registers(tr):
                    for at in (0, 1):
                        add(("deep_value", j, at), DEPTH % 0)
            for d in range(L + 1):                     # every layer, and the remainder
                add(("fri_offset", d), DEPTH % d if d < L else INCONSISTENT)
            for d in range(L):
                add(("fri_alpha", d), DEPTH % (d + 1) if d + 1 < L else INCONSISTENT)
            add(("remainder_point",), NOT_LOW_DEGREE % (remainder_bound(n, L) - 1))
            add(("layers", -1), folded_verdict(n, L - 1))
            # more folds while the remainder keeps two rows for its tree
            extra = [e for e in (1, 2, 3) if n * opt[0] // 4 ** (L + e) >= 8]
            for e in extra if prog == "fib13" else extra[:1]:
                add(("layers", e), folded_verdict(n, L + e))
    tr = traces()["fib13"]
    L = fri_layers(tr.length, CUT_OPTIONS[0])
    bound = remainder_bound(tr.length, L)
    kept = [i for i in range(bound) if i % CUT_OPTIONS[0]]
    for cut, want in ((-1, BOUND_TOO_LARGE), (0, OUT_OF_BOUNDS % (len(kept), len(kept)))):
        out.append(("fib13/%d/remainder_cut:%d" % (CUT_OPTIONS[0], cut), "fib13", CUT_OPTIONS, ("remainder_cut", cut), want))
    return out


def honest_cases():
    """[(case id, program, options)] -- one honest proof per program and option set"""
    return [("%s/%d/honest" % (prog, opt[0]), prog, opt) for prog, option_sets in OPTIONS.items() for opt in option_sets]


def prove(po, prog, opt, forge=None):
    tr = traces()[prog]
    r = po.prove(tr.registers, tr.ctx_depth, tr.loop_depth, tr.public_inputs, tr.outputs, *opt, forge=forge)
    assert r.error is None, (prog, opt, forge, r.error)
    return r.proof


@functools.lru_cache(maxsize=None)
def _proven(po):
    threads = po.set_threads(0)                     # more host threads change no byte of a proof (test_oracle_stark.py)
    po.set_threads(os.cpu_count() or 1)
    try:
        forged = [(cid, prog, opt, forge, want, prove(po, prog, opt, forge)) for cid, prog, opt, forge, want in cases()]
        honest = [(cid, prog, opt, prove(po, prog, opt)) for cid, prog, opt in honest_cases()]
    finally:
        po.set_threads(threads)
    return forged, honest


def proven(po):
    """(forged, honest): [(case id, program, options, forge, expected verdict, proof bytes)], [(case id, program, options, proof bytes)]"""
    return _proven(po)
