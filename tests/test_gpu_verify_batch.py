"""-m gpu tests of batched verification (dg_verify_batch / verify_batch): every verdict of a batch -- return code and message -- must be
the one dg_verify gives for that proof alone, whatever else the batch holds, and both must reproduce the verdicts that the
single-proof verifier gave before it became the K = 1 case of the batched pipeline (tests/golden/verify_corpus.json)."""
import hashlib
import json
import os
import random
import subprocess
import sys

import pytest

from tests import programs
from tests.golden import make_verify_corpus as corpus

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    backend.device_info()
    return distaff_b200


@pytest.fixture(scope="module")
def corpus_cases(dg):
    golden = json.load(open(corpus.PATH))
    pm = corpus.proofs(dg)
    for name, (_, proof) in pm.items():
        assert hashlib.sha256(proof).hexdigest() == golden["proof_sha256"][name], name
    return corpus.cases(pm), golden["cases"]


def fib_traces(k):
    from distaff_b200 import hostvm
    return [hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[1 + i, i]) for i in range(k)]


def as_code(v):
    """verify_batch entry -> (return code, message) as dg_verify reports it"""
    from distaff_b200 import backend
    if v is None:
        return 0, ""
    if isinstance(v, str):
        return -6, v
    assert isinstance(v, backend.DgError)
    prefix = "distaff_gpu error %d: " % v.code
    assert str(v).startswith(prefix)
    return v.code, str(v)[len(prefix):]


def item(tr, proof, inputs=None, outputs=None, program_hash=None):
    return (program_hash or tr.program_hash, tr.public_inputs if inputs is None else inputs, tr.outputs if outputs is None else outputs, proof)


def test_honest_mixed_batch(dg, po):
    import bench
    small = programs.small_programs()
    entries = [(name, tr, dg.prove(tr).bytes) for name, tr in small.items()]
    wide = programs.wide_program()
    entries.append(("wide", wide, dg.prove(wide).bytes))
    for prog, ext, queries, grinding in (("collatz3", 16, 30, 8), ("collatz3", 64, 20, 12), ("hash", 128, 128, 1), ("fib13", 256, 5, 4),
                                         ("collatz3", 256, 5, 4)):
        entries.append((f"{prog}/{ext}", small[prog], dg.prove(small[prog], dg.ProofOptions(ext, queries, grinding)).bytes))
    big, _ = bench.build_trace(16)
    entries.append(("bench16", big, dg.prove(big).bytes))
    stats = {}
    got = dg.verify_batch([item(tr, proof) for _, tr, proof in entries], stats=stats)
    assert stats["groups"] == 1 and stats["kernel_launches"] > 0 and stats["total_ms"] > 0
    for (name, tr, proof), v in zip(entries, got):
        want = dg.verify(tr.program_hash, tr.public_inputs, tr.outputs, proof)
        assert v == want, name
        if name != "bench16":
            assert v == po.verify(tr.program_hash, tr.public_inputs, tr.outputs, proof), name
    # fri/verifier.rs:86 rejects the honest blowup-256 proof of a 2^11-step trace: the same quirk in the batch
    assert got[-2] is not None and "remainder" in got[-2]
    assert all(v is None for v in got[:-2] + got[-1:])


def test_corpus_through_dg_verify_and_one_batch(dg, po, corpus_cases):
    cases, golden = corpus_cases
    assert len(cases) > 400
    single = {cid: list(corpus.verify_one(*rest)) for cid, *rest in cases}
    batch = dg.verify_batch([tuple(rest) for _, *rest in cases])
    for (cid, h, i, o, proof), v in zip(cases, batch):
        assert single[cid] == golden[cid], (cid, single[cid], golden[cid])
        assert list(as_code(v)) == golden[cid], (cid, as_code(v), golden[cid])
    # the restated reference verifier agrees on the cases test_gpu_verify.py compares it on: the reference's tampering cases, and single
    # bit flips past the header of proofs with the default options (a flipped domain depth moves the query positions, and then the GPU
    # verifier's constraint-leaf lookup fails before the reference would compare the trace root)
    for (cid, h, i, o, proof), v in zip(cases, batch):
        name, kind, *rest = cid.split("/")
        L = len(proof)
        if kind == "flip" and not (name in ("fib13", "collatz3", "hash", "deep_stack")
                                   and (44 <= int(rest[0]) < L - 16 or int(rest[0]) in (L - 12, L - 5))):
            continue
        if kind in ("truncate", "append"):
            continue
        want = po.verify(h, i, o, proof)
        if want is not None and (want.startswith("exception") or "too short" in want):
            assert v is not None, cid
        elif not isinstance(v, Exception):
            assert v == want, (cid, v, want)


def test_verdicts_do_not_depend_on_the_rest_of_the_batch(dg, corpus_cases):
    cases, golden = corpus_cases
    items = [tuple(rest) for _, *rest in cases]
    want = [golden[cid] for cid, *_ in cases]
    assert [list(as_code(v)) for v in dg.verify_batch(items[::-1])] == want[::-1]
    order = list(range(len(items)))
    random.Random(3).shuffle(order)
    got = dg.verify_batch([items[k] for k in order])
    assert [list(as_code(v)) for v in got] == [want[k] for k in order]
    # a malformed proof between honest ones, and one honest proof 100 times
    honest = [k for k, (cid, *_) in enumerate(cases) if cid.endswith("/honest") and golden[cid][0] == 0]
    junk = [k for k, (cid, *_) in enumerate(cases) if golden[cid][0] == -1][0]
    got = dg.verify_batch([items[honest[0]], items[junk], items[honest[1]]])
    assert got[0] is None and got[2] is None and as_code(got[1])[0] == -1
    assert dg.verify_batch([items[honest[0]]] * 100) == [None] * 100


def test_rng_callbacks_see_the_per_proof_sequences(dg, po, corpus_cases):
    from distaff_b200 import backend, felt
    cases, golden = corpus_cases
    picked = [c for c in cases if c[0].startswith(("fib13/", "wide/", "collatz3_e16/"))][::3]
    log = []

    def draw_field(seed, count):
        log.append(("field", seed, count))
        return felt.from_ints(po.prng_vector(seed, count)).tobytes()

    def draw_positions(seed, domain, ext, nq):
        log.append(("positions", seed, domain, ext, nq))
        return po.query_positions(seed, domain, ext, nq)

    try:
        backend.set_rng_callbacks(draw_field, draw_positions)
        single = []
        for cid, *rest in picked:
            single.append(list(corpus.verify_one(*rest)))
        want_log, log[:] = list(log), []
        got = dg.verify_batch([tuple(rest) for _, *rest in picked])
    finally:
        backend.set_rng_callbacks()
    assert log == want_log and len(log) > len(picked)
    for (cid, *_), s, v in zip(picked, single, got):
        assert s == golden[cid] and list(as_code(v)) == golden[cid], cid


def test_group_splitting_gives_the_same_verdicts(dg):
    """DG_BATCH_GROUP=3 splits a batch of 7 into groups of 3, 3 and 1 (in a fresh process, as a user would set it)"""
    trs = fib_traces(7)
    items = [item(t, p.bytes) for t, p in zip(trs, dg.prove_batch(trs))]
    items[3] = item(trs[3], items[3][3], outputs=[5])
    stats = {}
    want = dg.verify_batch(items, stats=stats)
    assert stats["groups"] == 1 and want[3] is not None and want.count(None) == 6
    code = ("import sys; sys.path.insert(0, %r)\n"
            "import distaff_b200 as dg\n"
            "from distaff_b200 import hostvm\n"
            "trs = [hostvm.execute(hostvm.fibonacci_program(13), public_inputs=[1 + i, i]) for i in range(7)]\n"
            "items = [(t.program_hash, t.public_inputs, t.outputs, p.bytes) for t, p in zip(trs, dg.prove_batch(trs))]\n"
            "items[3] = items[3][:2] + ([5],) + items[3][3:]\n"
            "stats = {}\n"
            "print(repr(dg.verify_batch(items, stats=stats)))\n"
            "print(stats['groups'])\n" % ROOT)
    env = dict(os.environ, DG_BATCH_GROUP="3")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.strip().splitlines()
    assert lines[-2] == repr(want)
    assert int(lines[-1]) == 3


def test_batch_shares_launches(dg):
    trs = fib_traces(64)
    items = [item(t, p.bytes) for t, p in zip(trs, dg.prove_batch(trs))]
    dg.verify_batch(items[:1])                         # warm-up: twiddle tables of this domain
    one, many = {}, {}
    assert dg.verify_batch(items[:1], stats=one) == [None]
    assert dg.verify_batch(items, stats=many) == [None] * 64
    print("kernel launches: one proof %d, 64 proofs %d" % (one["kernel_launches"], many["kernel_launches"]))
    assert one["kernel_launches"] == many["kernel_launches"] <= 8
    # each further register shape adds its row hash and its constraint launch
    small = programs.small_programs()
    others = [small[n] for n in ("collatz3", "deep_stack", "deep_ctx")]
    extra = [item(t, dg.prove(t).bytes) for t in others]
    dg.verify_batch(extra)
    mixed = {}
    assert dg.verify_batch(items + extra, stats=mixed) == [None] * 67
    shapes = {(t.ctx_depth, t.loop_depth, t.stack_depth) for t in [trs[0]] + others}
    widths = {t.width for t in [trs[0]] + others}
    assert mixed["groups"] == 1
    assert mixed["kernel_launches"] == one["kernel_launches"] + (len(shapes) - 1) + (len(widths) - 1) <= one["kernel_launches"] + 2 * 3


def test_scale(dg):
    trs = fib_traces(100)
    proofs = [p.bytes for p in dg.prove_batch(trs)]
    distinct = [item(t, p) for t, p in zip(trs, proofs)]
    single = [dg.verify(*it) for it in distinct]
    assert single == [None] * 100
    got = dg.verify_batch([distinct[i % 100] for i in range(2000)])
    assert got == [None] * 2000
    # and with one wrong output in every tenth distinct proof
    bad = [it if k % 10 else it[:2] + ([it[2][0] + 1],) + it[3:] for k, it in enumerate(distinct)]
    want = [dg.verify(*it) for it in bad]
    assert dg.verify_batch([bad[i % 100] for i in range(2000)]) == [want[i % 100] for i in range(2000)]
