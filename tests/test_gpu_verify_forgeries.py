"""-m gpu: the GPU verifier (dg_verify / dg_verify_batch, distaff_b200/csrc/verifier.cu) on forged proofs (tests/forged_proofs.py):
proofs of false statements whose commitments are all consistent, so that only the algebraic checks can reject them -- C(z), every FRI
fold at every depth, the remainder against the last fold and against its degree bound.  Every verdict must be the restated reference
verifier's, string for string, alone and in batches that mix the forgeries with honest proofs of several shapes."""
import os
import pickle
import random
import subprocess
import sys

import pytest

from tests import forged_proofs as fp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    backend.device_info()
    return distaff_b200


@pytest.fixture(scope="module")
def items(po):
    """[(case id, (program hash, inputs, outputs, proof), oracle verdict)] over the forged and the honest proofs"""
    forged, honest = fp.proven(po)
    out = []
    for cid, prog, _, _, _, proof in forged + [(cid, prog, opt, None, None, proof) for cid, prog, opt, proof in honest]:
        tr = fp.traces()[prog]
        args = (tr.program_hash, tr.public_inputs, tr.outputs, proof)
        out.append((cid, args, po.verify(*args)))
    return out


def single(dg, args):
    from distaff_b200 import backend
    try:
        return dg.verify(*args)
    except backend.DgError as e:
        return e


def agrees(got, want):
    """the reference's verdict; where the oracle throws (the reference panics), any rejection"""
    if want is not None and want.startswith("exception: "):
        return got is not None
    return got == want


def test_dg_verify_gives_the_oracle_verdict(dg, po, items):
    forged, _ = fp.proven(po)
    expected = {cid: want for cid, *_, want, _ in forged}
    seen = set()
    for cid, args, want in items:
        assert want == expected.get(cid), (cid, want)                  # honest proofs: None
        got = single(dg, args)
        assert agrees(got, want), (cid, got, want)
        if want is not None and want.startswith("exception: "):
            assert got == fp.BOUND_TOO_LARGE, (cid, got)      # where the reference panics, the GPU verifier reports the bound
        seen.add(got)
    # the checks the forgeries reach on the GPU
    deepest = max(fp.fri_layers(fp.traces()[p].length, o[0]) for p, opts in fp.OPTIONS.items() for o in opts)
    for want in [fp.DEPTH % d for d in range(deepest)] + [fp.INCONSISTENT, fp.BOUND_TOO_LARGE, fp.MIN_OP_COUNT, fp.NOT_LOW_DEGREE % (2**64 - 1)]:
        assert want in seen, want
    assert any(isinstance(g, str) and g.startswith(fp.LDP + "remainder is not a valid degree ") for g in seen)
    accepted = [cid for cid, args, want in items if want is None and not cid.endswith("/honest")]
    assert any("layers:-1" in c for c in accepted) and any("layers:1" in c for c in accepted)


def test_one_shuffled_batch(dg, items):
    order = list(range(len(items)))
    random.Random(11).shuffle(order)
    batch = [items[k] for k in order]
    stats = {}
    got = dg.verify_batch([args for _, args, _ in batch], stats=stats)
    assert stats["groups"] == 1
    for (cid, args, want), v in zip(batch, got):
        alone = single(dg, args)
        assert (str(v), type(v)) == (str(alone), type(alone)), (cid, v, alone)
        assert agrees(v, want), (cid, v, want)
        if cid.endswith("/honest"):
            assert v is None, cid


def test_group_splitting_gives_the_same_verdicts(dg, items, tmp_path):
    """DG_BATCH_GROUP=3 splits the batch into groups of 3 (in a fresh process, as a user would set it)"""
    order = list(range(len(items)))
    random.Random(12).shuffle(order)
    batch = [items[k][1] for k in order]
    want = [repr(v) for v in dg.verify_batch(batch)]
    path = tmp_path / "items.pickle"
    path.write_bytes(pickle.dumps(batch))
    code = ("import sys, pickle; sys.path.insert(0, %r)\n"
            "import distaff_b200 as dg\n"
            "items = pickle.loads(open(%r, 'rb').read())\n"
            "stats = {}\n"
            "print(repr([repr(v) for v in dg.verify_batch(items, stats=stats)]))\n"
            "print(stats['groups'])\n" % (ROOT, str(path)))
    env = dict(os.environ, DG_BATCH_GROUP="3")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.strip().splitlines()
    assert lines[-2] == repr(want)
    decided = sum(1 for cid, _, w in items if w == fp.MIN_OP_COUNT)      # decided before the device phase: in no group
    assert int(lines[-1]) == -(-(len(items) - decided) // 3)
