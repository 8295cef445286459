"""Seeded provers without a GPU (StarkPlan and PlainStarkPlan with seeds, and sign_batch with seeds, through the test
double of tests/stark_seeded_cases.py, whose sample_seeded runs the CPU emulation of csrc/sample.cuh): a seeded proof
is the unseeded proof with os.urandom = seeded_urandom(seed), for the fixtures' AIRs and synthetic AIRs; nothing calls
os.urandom; a batch is its proofs alone; failures keep the unseeded message and proof_index; seeded signatures are
sign's under seeded_urandom; bad seeds are refused before device work; and the test-side verifier accepts seeded
proofs."""
import pytest

import stark_batch_cases as SB
import stark_cases as C
import stark_plain_cases as S
import stark_seeded_cases as SS
import stark_verify as V
import sa_engine
import sa_stark

G = C.golden()
GP = S.golden()


@pytest.fixture(autouse=True)
def double_engine():
    prev = sa_engine._ENGINE
    sa_engine.set_engine(SS.SeededStarkEngine())
    yield
    sa_engine.set_engine(prev)


def fixture_plan(rec, fast):
    if fast:
        st = C.params(rec)
        zpoly, zvals = C.zerofier(st)
        return sa_stark.StarkPlan(st, C.air(rec), zpoly), C.zerofier_codeword(zvals, True)
    return sa_stark.PlainStarkPlan(S.stark(rec), C.air(rec)), None


CASES = [(True, k) for k in sorted(G)] + [(False, k) for k in sorted(GP)]


@pytest.mark.parametrize("fast,name", CASES)
def test_fixture_case_equals_the_host_route(fast, name):
    rec = (G if fast else GP)[name]
    try:
        plan, zcw = fixture_plan(rec, fast)
    except (AssertionError, ValueError) as e:  # a plan the unseeded path refuses too: nothing to draw
        pytest.skip("the plan is refused: %s" % e)
    trace, boundary = C.inputs(rec)
    s = [SS.seed(fast, name)]
    got = SS.seeded(plan, [trace], [boundary], s, zcw, [C.stream(rec)])
    want = SS.route(plan, [trace], [boundary], s, zcw, [C.stream(rec)])
    assert SS.same(got, want), (got, want)
    assert isinstance(got, list) == ("raises" not in rec)
    if isinstance(got, list):
        # the seed changes the proof
        other = SS.seeded(plan, [trace], [boundary], [SS.seed(fast, name, 1)], zcw, [C.stream(rec)])
        assert other != got


@pytest.mark.parametrize("fast", [True, False], ids=["faststark", "plain"])
@pytest.mark.parametrize("log_fri", [10, 12])
def test_synthetic_single_and_batch(fast, log_fri):
    st, cons, trace, boundary = C.synthetic(40 + log_fri, log_fri)
    zpoly, zvals = C.zerofier(st)
    zcw = C.zerofier_codeword(zvals, True) if fast else None
    plan = sa_stark.StarkPlan(st, cons, zpoly) if fast else sa_stark.PlainStarkPlan(S.plain_stark(st), cons)
    seeds = [SS.seed(log_fri, b) for b in range(3)]
    batch = SS.seeded(plan, [trace] * 3, [boundary] * 3, seeds, zcw)
    assert isinstance(batch, list) and len(set(batch)) == 3, batch
    assert batch == SS.route(plan, [trace] * 3, [boundary] * 3, seeds, zcw)
    # each proof alone, and in another batch position, is the same bytes
    for b in range(3):
        assert SS.seeded(plan, [trace], [boundary], [seeds[b]], zcw) == [batch[b]]
    assert SS.seeded(plan, [trace] * 2, [boundary] * 2, seeds[2:0:-1], zcw) == [batch[2], batch[1]]
    if fast:
        root = C.O.merkle_root_np(C.O.to_np(zvals))
        for proof in batch:
            assert V.verify(st, proof, cons, boundary, root)


@pytest.mark.parametrize("fast", [True, False], ids=["faststark", "plain"])
def test_no_randomizer_upload(fast):
    """with seeds the uploads are the callers' rows and the seeds: no randomizer crosses to the device"""
    st, cons, trace, boundary = C.synthetic(7, 10)
    zpoly, zvals = C.zerofier(st)
    zcw = C.zerofier_codeword(zvals, True) if fast else None
    plan = sa_stark.StarkPlan(st, cons, zpoly) if fast else sa_stark.PlainStarkPlan(S.plain_stark(st), cons)
    eng = sa_engine.get_engine()
    before = len(eng.calls)
    assert isinstance(SS.seeded(plan, [trace] * 2, [boundary] * 2, [SS.seed(1), SS.seed(2)], zcw), list)
    calls = eng.calls[before:]
    uploads = [c[1] for c in calls if c[0] == "upload"]
    assert uploads[0] == 2 * st.num_registers * st.original_trace_length
    assert (st.num_registers * (st.original_trace_length + st.num_randomizers) not in uploads and
            plan.max_degree + 1 not in uploads and 2 * (plan.max_degree + 1) not in uploads)
    assert [c for c in calls if c[0] in ("upload_seeds", "sample_seeded")] == [
        ("upload_seeds", 2), ("sample_seeded", 2, 0, st.num_registers * st.num_randomizers, st.num_registers),
        ("sample_seeded", 2, st.num_registers * st.num_randomizers, plan.max_degree + 1, 1)]


# failing fixture cases whose AIR and parameters are three_register's, so that they batch with it
FAILING = [(fast, bad) for fast in (True, False) for bad in ("broken_witness", "false_boundary")
           if "raises" in (G if fast else GP)[bad]]


@pytest.mark.parametrize("fast,bad", FAILING)
@pytest.mark.parametrize("at", [0, 1, 2])
def test_failure_at_each_position(fast, bad, at):
    g = G if fast else GP
    rec, good = g[bad], g["three_register"]
    plan, zcw = fixture_plan(rec, fast)
    recs = [good] * 3
    recs[at] = rec
    traces, boundaries = zip(*[C.inputs(r) for r in recs])
    seeds = [SS.seed(bad, b) for b in range(3)]
    got = SS.seeded(plan, list(traces), list(boundaries), seeds, zcw)
    want = SS.route(plan, list(traces), list(boundaries), seeds, zcw)
    assert isinstance(got, AssertionError) and str(got).startswith(rec["raises"]) and got.proof_index == at
    assert SS.same(got, want)


@pytest.mark.parametrize("fast,name", [(False, "cancelled_top"), (True, "below_zerofier"), (False, "tiny_broken")])
def test_other_failures_in_a_batch(fast, name):
    """the degree mismatch and the other refusals of an AIR of their own, twice in one batch: the first proof's"""
    rec = (G if fast else GP)[name]
    plan, zcw = fixture_plan(rec, fast)
    trace, boundary = C.inputs(rec)
    seeds = [SS.seed(name, b) for b in range(2)]
    got = SS.seeded(plan, [trace] * 2, [boundary] * 2, seeds, zcw)
    assert isinstance(got, AssertionError) and str(got).startswith(rec["raises"]) and got.proof_index == 0
    assert SS.same(got, SS.route(plan, [trace] * 2, [boundary] * 2, seeds, zcw))


def test_refused_boundary_with_seeds():
    rec = GP["three_register"]
    plan, _ = fixture_plan(rec, False)
    trace, boundary = C.inputs(rec)
    refused = [b for b in boundary if b[1] != 1]
    seeds = [SS.seed("refused", b) for b in range(3)]
    got = SS.seeded(plan, [trace] * 3, [boundary, refused, boundary], seeds)
    assert isinstance(got, AssertionError) and got.proof_index == 1
    assert SS.same(got, SS.route(plan, [trace] * 3, [boundary, refused, boundary], seeds))


@pytest.mark.parametrize("fast", [True, False])
def test_sign_batch_with_seeds(fast):
    g = G if fast else GP
    first, second = g["rpsss"], g["rpsss_second"]
    signer = SB.Signer(first, fast)
    docs = [bytes.fromhex(first["document"]), bytes.fromhex(second["document"]), b"third"]
    seeds = [SS.seed("sign", d) for d in docs]
    real = sa_stark.os.urandom
    try:
        sa_stark.os.urandom = SS.refuse_urandom
        got = sa_stark.sign_batch(signer, 1, docs, seeds)
        want = []
        for d, s in zip(docs, seeds):
            sa_stark.os.urandom = sa_stark.seeded_urandom(s)
            want.append(sa_stark.sign_batch(signer, 1, [d])[0])
    finally:
        sa_stark.os.urandom = real
    assert got == want and len(set(got)) == 3


BAD_SEEDS = [[b"short"], [bytes(33)], [bytearray(32)], ["x" * 32], [None], [bytes(32)] * 2, [], bytes(32), 5]


@pytest.mark.parametrize("bad", BAD_SEEDS, ids=range(len(BAD_SEEDS)))
def test_bad_seeds_refused_before_device_work(bad):
    rec = GP["three_register"]
    plan, _ = fixture_plan(rec, False)
    fplan, zcw = fixture_plan(G["three_register"], True)
    trace, boundary = C.inputs(rec)
    eng = sa_engine.get_engine()
    before = len(eng.calls)
    with pytest.raises(AssertionError, match="seeds"):
        plan.prove_batch([trace], [boundary], seeds=bad)
    with pytest.raises(AssertionError, match="seeds"):
        fplan.prove_batch([trace], [boundary], zcw, seeds=bad)
    with pytest.raises(AssertionError, match="seeds"):
        sa_stark.sign_batch(SB.Signer(GP["rpsss"], False), 1, [b"doc"], bad)
    if isinstance(bad, list) and len(bad) == 1 and bad[0] is not None:  # seed=None is the unseeded proof
        with pytest.raises(AssertionError, match="seeds"):
            plan.prove(trace, boundary, seed=bad[0])
    assert len(eng.calls) == before
