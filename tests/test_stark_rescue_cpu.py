"""Device Rescue and SignerPlan without a GPU (sa_rescue.hash_batch / trace_batch and sa_stark.SignerPlan through the
test double of tests/stark_rescue_cases.py, whose rescue runs the CPU emulation of csrc/rescue.cuh): the batches equal
the fixture's hashes and traces from one upload and one launch; the two recorded keys and documents signed as one
batch give the recorded RPSSS and FastRPSSS signatures; seeded signatures equal the seeded_urandom route; a plan
serves many calls and equals sign_batch per key; refusals come before any device work; and no trace element is
uploaded."""
import hashlib
import os

import pytest

import rescue_cases as R
import stark_batch_cases as SB
import stark_cases as C
import stark_plain_cases as S
import stark_rescue_cases as SR
import stark_seeded_cases as SS
import sa_engine
import sa_rescue
import sa_stark

G = C.golden()
GP = S.golden()
T = C.T


@pytest.fixture(autouse=True)
def double_engine():
    prev = sa_engine._ENGINE
    sa_engine.set_engine(SR.RescueStarkEngine())
    yield
    sa_engine.set_engine(prev)


def test_hash_and_trace_batch_equal_the_fixture():
    g = R.golden()
    rp = SR.RescuePrime()
    xs = [T.fe(int(c["input"])) for c in g["cases"]]
    eng = sa_engine.get_engine()
    before = len(eng.calls)
    hashes = sa_rescue.hash_batch(rp, xs)
    calls = [c[0] for c in eng.calls[before:]]
    assert calls.count("upload") == 1 and calls.count("rescue") == 1
    assert [str(h.value) for h in hashes] == [c["hash"] for c in g["cases"]]
    assert all(type(h) is type(xs[0]) and h.field is rp.field for h in hashes)
    before = len(eng.calls)
    traces = sa_rescue.trace_batch(rp, xs)
    calls = [c[0] for c in eng.calls[before:]]
    assert calls.count("upload") == 1 and calls.count("rescue") == 1
    assert [[[str(v.value) for v in row] for row in t] for t in traces] == [c["trace"] for c in g["cases"]]
    assert sa_rescue.hash_batch(rp, []) == [] and sa_rescue.trace_batch(rp, []) == []
    # plain ints are elements too
    assert sa_rescue.hash_batch(rp, [1]) == [T.fe(int(g["cases"][9]["hash"]))]


def test_batch_refusals_before_device_work():
    rp = SR.RescuePrime()
    eng = sa_engine.get_engine()
    before = len(eng.calls)
    for bad in ([R.P], [-1], [1.0], ["1"], [T.fe(1), R.P + 5]):
        for fn in (sa_rescue.hash_batch, sa_rescue.trace_batch):
            with pytest.raises(AssertionError):
                fn(rp, bad)
    wide = SR.RescuePrime()
    wide.m = 3
    with pytest.raises(AssertionError):
        sa_rescue.hash_batch(wide, [1])
    with pytest.raises(AssertionError):
        sa_rescue.trace_batch(wide, [])
    assert len(eng.calls) == before


def signers(fast):
    g = G if fast else GP
    first, second = g["rpsss"], g["rpsss_second"]
    return first, second, SR.Signer(first, fast)


def with_draws(values, fn):
    real = os.urandom
    os.urandom = values
    try:
        return fn()
    finally:
        os.urandom = real


@pytest.mark.parametrize("fast", [True, False], ids=["fastrpsss", "rpsss"])
def test_recorded_two_key_batch(fast):
    first, second, signer = signers(fast)
    plan = sa_stark.SignerPlan(signer)
    recs = (first, second)
    draws = C.Urandom(SB.batch_draws([r["draws"] for r in recs], SB.ntrace(first)))
    sks = [T.fe(int(r["sk"])) for r in recs]
    docs = [bytes.fromhex(r["document"]) for r in recs]
    sigs = with_draws(draws, lambda: plan.sign(sks, docs))
    assert draws.count == len(first["draws"]) + len(second["draws"])
    assert [hashlib.sha256(s).hexdigest() for s in sigs] == [r["proof_sha256"] for r in recs]


@pytest.mark.parametrize("fast", [True, False], ids=["fastrpsss", "rpsss"])
def test_seeded_signatures_equal_the_route_and_plan_serves_many_calls(fast):
    first, second, signer = signers(fast)
    plan = sa_stark.SignerPlan(signer)
    sks = [T.fe(int(first["sk"])), T.fe(int(second["sk"])), T.fe(5)]
    docs = [b"one", b"two", b"three"]
    seeds = [SS.seed("rescue", fast, b) for b in range(3)]
    got = SR.seeded_sign(plan, sks, docs, seeds)
    assert len(set(got)) == 3
    assert got == SR.route(signer, sks, docs, seeds)
    # a second call on the same plan, in another order and batch size: each signature is its own
    assert SR.seeded_sign(plan, sks[2:0:-1], docs[2:0:-1], seeds[2:0:-1]) == [got[2], got[1]]
    assert SR.seeded_sign(plan, sks[:1], docs[:1], seeds[:1]) == got[:1]


@pytest.mark.parametrize("fast", [True, False], ids=["fastrpsss", "rpsss"])
def test_one_key_equals_sign_batch(fast):
    first, _, signer = signers(fast)
    plan = sa_stark.SignerPlan(signer)
    sk = T.fe(int(first["sk"]))
    docs = [b"alpha", b"beta", b"gamma"]
    n = len(first["draws"])
    per = [[str(v) for v in range(11 + 7 * b, 11 + 7 * b + n)] for b in range(3)]
    stream = SB.batch_draws(per, SB.ntrace(first))
    got = with_draws(C.Urandom(stream), lambda: plan.sign([sk] * 3, docs))
    want = with_draws(C.Urandom(stream), lambda: sa_stark.sign_batch(signer, sk, docs))
    assert got == want and len(set(got)) == 3


def test_refusals_before_device_work():
    first, _, signer = signers(True)
    plan = sa_stark.SignerPlan(signer)
    eng = sa_engine.get_engine()
    before = len(eng.calls)
    sk = T.fe(int(first["sk"]))
    with pytest.raises(AssertionError):
        plan.sign([sk, sk], [b"x"])
    for bad in (R.P, -1, 2.5, "7", None):
        with pytest.raises(AssertionError):
            plan.sign([sk, bad], [b"x", b"y"])
    with pytest.raises(AssertionError):
        plan.sign([sk], [b"x"], seeds=[b"short"])
    with pytest.raises(AssertionError):
        plan.sign([sk], [b"x"], seeds=[SS.seed(1), SS.seed(2)])
    assert plan.sign([], []) == [] and plan.sign([], [], seeds=[]) == []
    assert len(eng.calls) == before
    # a Stark of the wrong shape is refused when the plan is built
    bad = SR.Signer(first, True)
    bad.rp.N = 26
    with pytest.raises(AssertionError):
        sa_stark.SignerPlan(bad)


@pytest.mark.parametrize("fast", [True, False], ids=["fastrpsss", "rpsss"])
def test_no_trace_element_is_uploaded(fast):
    first, second, signer = signers(fast)
    plan = sa_stark.SignerPlan(signer)
    eng = sa_engine.get_engine()
    sks = [T.fe(int(first["sk"])), T.fe(int(second["sk"]))]
    docs = [b"a", b"b"]
    before = len(eng.calls)
    SR.seeded_sign(plan, sks, docs, [SS.seed(0), SS.seed(1)])
    assert SR.uploads(eng, before) == [2]  # the keys
    nrand = signer.stark.num_randomizers
    before = len(eng.calls)
    with_draws(C.Urandom([str(v) for v in range(1, 5000)]), lambda: plan.sign(sks, docs))
    # the keys, the trace randomizer rows, the randomizer polynomials
    assert SR.uploads(eng, before) == [2, 2 * 2 * nrand, 2 * (plan.plan.max_degree + 1)]
