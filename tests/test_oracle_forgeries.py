"""The oracle's verifier on forged proofs (tests/forged_proofs.py): proofs of false statements whose commitments are all consistent,
one per algebraic check of the verifier and per FRI depth.  Each forged proof is well formed and passes the PoW and Merkle checks,
and the verifier rejects it at the check that the changed value reaches, with the reference's message; honest proofs with one fold
fewer are accepted."""
import pytest

from tests import forged_proofs as fp

# verdicts that a proof with consistent commitments never gets
NOT_CONSISTENT = ("Merkle", "proof-of-work", "query positions", "truncated", "trailing", "bad length", "too short", "wrong number",
                  "wrong width", "unsupported")


@pytest.fixture(scope="module")
def proven(po):
    return fp.proven(po)


def test_honest_proofs_are_accepted(po, proven):
    _, honest = proven
    for cid, prog, opt, proof in honest:
        tr = fp.traces()[prog]
        assert po.verify(tr.program_hash, tr.public_inputs, tr.outputs, proof) is None, cid


def test_every_forgery_gets_its_verdict(po, proven):
    forged, _ = proven
    for cid, prog, opt, forge, want, proof in forged:
        tr = fp.traces()[prog]
        got = po.verify(tr.program_hash, tr.public_inputs, tr.outputs, proof)
        assert got == want, (cid, got, want)
        assert got is None or not any(s in got for s in NOT_CONSISTENT), (cid, got)


def test_forgeries_keep_the_commitments_and_options(po, proven):
    """the same trace root, options and register shape as the honest proof, and different bytes.  That the PoW and the trace and
    constraint Merkle proofs hold follows from the verdicts: every one but the op-count minimum comes after those checks."""
    forged, honest = proven
    honest_by = {(prog, opt): proof for _, prog, opt, proof in honest}
    for cid, prog, opt, forge, want, proof in forged:
        ref = honest_by.get((prog, opt))
        if ref is None:
            continue
        assert proof != ref, cid
        assert proof[-4:] == ref[-4:] and proof[32:36] == ref[32:36], cid          # options; domain depth and register shape
        if forge[0] != "transition":
            assert proof[:32] == ref[:32], cid                                     # the trace root


def test_every_fri_depth_of_every_proof_is_reached(proven):
    forged, _ = proven
    for prog, option_sets in fp.OPTIONS.items():
        n = fp.traces()[prog].length
        for opt in option_sets:
            L = fp.fri_layers(n, opt[0])
            seen = {want for cid, p, o, forge, want, _ in forged if p == prog and o == opt}
            assert {fp.DEPTH % d for d in range(L)} <= seen, (prog, opt)
            assert fp.INCONSISTENT in seen and fp.NOT_LOW_DEGREE % (fp.remainder_bound(n, L) - 1) in seen, (prog, opt)


def test_coverage_of_the_verifier_messages(proven):
    forged, _ = proven
    seen = {want for *_, want, _ in forged}
    deepest = max(fp.fri_layers(fp.traces()[p].length, o[0]) for p, opts in fp.OPTIONS.items() for o in opts)
    assert deepest == 5
    for want in [fp.DEPTH % d for d in range(deepest)] + [fp.INCONSISTENT, fp.BOUND_TOO_LARGE, fp.MIN_OP_COUNT, None]:
        assert want in seen, want
    assert any(w and w.startswith(fp.LDP + "remainder is not a valid degree ") for w in seen)
    assert any(w and w.startswith("exception: index out of bounds") for w in seen)
    assert fp.NOT_LOW_DEGREE % (2**64 - 1) in seen                                  # a degree bound of 0, as usize arithmetic wraps it
    accepted = [cid for cid, *_, want, _ in forged if want is None]
    assert any("layers:-1" in c for c in accepted) and any("layers:1" in c for c in accepted)

