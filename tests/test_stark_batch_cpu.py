"""The batched provers' host logic without a GPU (StarkPlan.prove_batch, PlainStarkPlan.prove_batch and
sa_stark.sign_batch through tests/stark_batch_cases.py's test double): the fixture's two signatures proven as one
batch give the recorded bytes from the batch's draw stream; a batch of synthetic proofs equals sequential proofs fed
the matching slices of its stream; a batch holding a broken witness or a false boundary raises what proving the
proofs in order raises first, with that proof's index; an empty batch does no device work; and sign_batch gives
what sign gives."""
import hashlib
import random

import pytest

import stark_batch_cases as SB
import stark_cases as C
import stark_plain_cases as S
import sa_engine
import sa_stark

G = C.golden()
GP = S.golden()


@pytest.fixture(autouse=True)
def double_engine():
    prev = sa_engine._ENGINE
    sa_engine.set_engine(SB.BatchStarkEngine())
    yield
    sa_engine.set_engine(prev)


def signatures(g, fast):
    first, second = g["rpsss"], g["rpsss_second"]
    st = C.params(first) if fast else S.stark(first)
    return first, second, st


@pytest.mark.parametrize("fast", [True, False])
def test_fixture_signatures_as_one_batch(fast):
    first, second, st = signatures(G if fast else GP, fast)
    recs = (first, second)
    traces, boundaries = zip(*[C.inputs(r) for r in recs])
    draws = C.Urandom(SB.batch_draws([r["draws"] for r in recs], SB.ntrace(first)))
    streams = [C.stream(r) for r in recs]
    if fast:
        zpoly, zvals = C.zerofier(st)
        plan = sa_stark.StarkPlan(st, C.air(first), zpoly)
        proofs = SB.run_batch(plan, list(traces), list(boundaries), draws, streams, C.zerofier_codeword(zvals, True))
    else:
        plan = sa_stark.PlainStarkPlan(st, C.air(first))
        proofs = SB.run_batch(plan, list(traces), list(boundaries), draws, streams)
    assert isinstance(proofs, list), proofs
    assert draws.count == len(first["draws"]) + len(second["draws"])
    for rec, proof, ps in zip(recs, proofs, streams):
        assert hashlib.sha256(proof).hexdigest() == rec["proof_sha256"]
        assert ps.serialize() == proof


@pytest.mark.parametrize("fast", [True, False])
def test_synthetic_batch_equals_sequential(fast):
    st, cons, trace, boundary = C.synthetic(5, 10)
    # three statements of one AIR: the valid trace, and for FastStark two traces broken at a middle row (still
    # proofs); the plain prover refuses those, so there the valid trace three times, each with its own draws
    traces = [trace]
    for k in (1, 2):
        if not fast:
            traces.append(trace)
            continue
        t = [list(r) for r in trace]
        t[len(t) // 2][0] = C.T.fe((t[len(t) // 2][0].value + k) % C.P)
        traces.append(t)
    B = len(traces)
    zpoly, zvals = C.zerofier(st)
    zcw = C.zerofier_codeword(zvals, True)
    plan = sa_stark.StarkPlan(st, cons, zpoly) if fast else sa_stark.PlainStarkPlan(S.plain_stark(st), cons)
    nt = st.num_registers * st.num_randomizers
    rng = random.Random(9)
    per = [[rng.randrange(C.P) for _ in range(nt + plan.max_degree + 1)] for _ in range(B)]
    got = SB.run_batch(plan, traces, [boundary] * B, C.Urandom(SB.batch_draws(per, nt)), None,
                       zcw if fast else None)
    assert isinstance(got, list) and len(got) == B, got
    for b in range(B):
        if fast:
            want, _ = C.run(st, traces[b], None, boundary, zpoly, zcw, C.Urandom(per[b]), plan=plan)
        else:
            want = S.run(None, traces[b], None, boundary, C.Urandom(per[b]), plan=plan)
        assert got[b] == want, b


# the fixtures' failing cases (FastStark proves a broken witness: only its false boundary raises)
FAILING = [(fast, bad) for fast in (True, False) for bad in ("broken_witness", "false_boundary")
           if "raises" in (G if fast else GP)[bad]]


@pytest.mark.parametrize("fast,bad", FAILING)
@pytest.mark.parametrize("at", [0, 1, 2])
def test_failure_is_the_first_sequential_failure(fast, bad, at):
    g = G if fast else GP
    rec, good = g[bad], g["three_register"]
    st = C.params(rec) if fast else S.stark(rec)
    assert C.air(rec) == C.air(good) and rec["params"] == good["params"]
    recs = [good] * 3
    recs[at] = rec
    traces, boundaries = zip(*[C.inputs(r) for r in recs])
    zpoly, zvals = C.zerofier(C.params(rec))
    zcw = C.zerofier_codeword(zvals, True)
    plan = sa_stark.StarkPlan(st, C.air(rec), zpoly) if fast else sa_stark.PlainStarkPlan(st, C.air(rec))
    got = SB.run_batch(plan, list(traces), list(boundaries), C.Urandom([7] * 100000), None, zcw if fast else None)
    # sequentially, the proofs before `at` succeed and proof `at` raises the recorded message
    assert isinstance(got, AssertionError), got
    assert str(got).startswith(rec["raises"]) and got.proof_index == at


def test_refused_boundary_raises_at_its_proof():
    rec = GP["three_register"]
    st = S.stark(rec)
    trace, boundary = C.inputs(rec)
    plan = sa_stark.PlainStarkPlan(st, C.air(rec))
    refused = [b for b in boundary if b[1] != 1]  # register 1 without boundary points
    got = SB.run_batch(plan, [trace] * 3, [boundary, refused, boundary], C.Urandom([7] * 100000))
    assert isinstance(got, AssertionError) and got.proof_index == 1


def test_empty_batch_does_no_device_work():
    rec = GP["three_register"]
    plan = sa_stark.PlainStarkPlan(S.stark(rec), C.air(rec))
    eng = sa_engine.get_engine()
    before = len(eng.calls)
    assert plan.prove_batch([], []) == [] and len(eng.calls) == before


@pytest.mark.parametrize("fast", [True, False])
def test_sign_batch_is_sign(fast):
    g = G if fast else GP
    first, second = g["rpsss"], g["rpsss_second"]
    signer = SB.Signer(first, fast)
    docs = [bytes.fromhex(first["document"]), bytes.fromhex(second["document"])]
    # one document: the recorded signature
    real = sa_stark.os.urandom
    try:
        sa_stark.os.urandom = C.Urandom(first["draws"])
        one = sa_stark.sign_batch(signer, 1, docs[:1])
    finally:
        sa_stark.os.urandom = real
    assert [hashlib.sha256(s).hexdigest() for s in one] == [first["proof_sha256"]]
    # two documents with one key: the two sequential signatures from the matching slices of the draws
    nt = SB.ntrace(first)
    per = [[str(v) for v in range(11, 11 + len(first["draws"]))], [str(v) for v in range(5, 5 + len(first["draws"]))]]
    try:
        sa_stark.os.urandom = C.Urandom(SB.batch_draws(per, nt))
        two = sa_stark.sign_batch(signer, 1, docs)
        want = []
        for d, ds in zip(docs, per):
            sa_stark.os.urandom = C.Urandom(ds)
            want.append(signer.sign(1, d))
    finally:
        sa_stark.os.urandom = real
    assert two == want and two[0] != two[1]
