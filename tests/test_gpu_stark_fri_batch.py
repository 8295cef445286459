"""The provers with fri_batch=True on the H100 (StarkPlan.prove_batch, PlainStarkPlan.prove_batch, sign_batch and
SignerPlan.sign): the recorded two-signature fixtures byte for byte; synthetic batches at 2^12 x 16, 2^16 x 4 and
2^20 x 2 equal to the default route and accepted by VerifierPlan; 16 seeded SignerPlan.sign keys equal to the default
route and accepted; and the FRI stage reads the roots once per round plus a fixed number of openings, whatever B."""
import random

import pytest

import oracle as O
import stark_cases as C
import stark_plain_cases as S
import stark_rescue_cases as SR
import verify_cases as V
import test_fri_batch_cpu as CPU
from test_gpu_air import release

import sa_engine  # noqa: E402
import sa_stark  # noqa: E402

pytestmark = pytest.mark.gpu
P = C.P


@pytest.fixture(scope="module")
def eng():
    sa_engine.set_engine(None)
    e = sa_engine.get_engine()
    assert e.name == "cuda"
    return e


@pytest.fixture(autouse=True)
def _cuda_engine(eng):
    sa_engine.set_engine(eng)
    yield
    release(eng)


@pytest.mark.parametrize("fast", [True, False])
def test_fixture_signatures_with_batched_fri(eng, fast):
    CPU.test_fixture_signatures_with_batched_fri(None, fast)


@pytest.mark.parametrize("fast", [True, False])
def test_sign_batch_with_batched_fri(eng, fast):
    CPU.test_sign_batch_with_batched_fri(None, fast)


def batch_case(log_fri, B, seed):
    st, cons, trace, boundary = C.synthetic(seed, log_fri)
    zpoly, zvals = C.zerofier(st)
    plan = sa_stark.StarkPlan(st, cons, zpoly)
    seeds = [bytes([log_fri, b]) * 16 for b in range(B)]
    return st, cons, trace, boundary, zvals, plan, seeds


@pytest.mark.parametrize("log_fri,B", [(12, 16), (16, 4), (20, 2)])
def test_synthetic_batch_equals_default_route_and_verifies(eng, log_fri, B):
    st, cons, trace, boundary, zvals, plan, seeds = batch_case(log_fri, B, log_fri)
    zcw = C.zerofier_codeword(zvals, True)
    default = plan.prove_batch([trace] * B, [boundary] * B, zcw, seeds=seeds)
    got = plan.prove_batch([trace] * B, [boundary] * B, zcw, seeds=seeds, fri_batch=True)
    assert got == default and len(set(got)) == B
    root = O.merkle_root_np(O.to_np(zvals))
    assert sa_stark.VerifierPlan(st, cons, root).verify_batch(got, [boundary] * B) == [True] * B


def test_plain_synthetic_batch_equals_default_route(eng):
    st, cons, trace, boundary = C.synthetic(8, 12)
    plan = sa_stark.PlainStarkPlan(S.plain_stark(st), cons)
    seeds = [bytes([8, b]) * 16 for b in range(4)]
    default = plan.prove_batch([trace] * 4, [boundary] * 4, seeds=seeds)
    assert plan.prove_batch([trace] * 4, [boundary] * 4, seeds=seeds, fri_batch=True) == default


@pytest.mark.parametrize("fast", [True, False], ids=["fastrpsss", "rpsss"])
def test_seeded_16_keys_equal_the_default_route_and_verify(eng, fast):
    g = C.golden() if fast else S.golden()
    first = g["rpsss"]
    signer = SR.Signer(first, fast)
    if fast:
        signer.transition_zerofier_root = bytes.fromhex(first["zerofier_root"])
    plan = sa_stark.SignerPlan(signer)
    plan.stream = V.SignatureProofStream
    rng = random.Random(16 + fast)
    sks = [C.T.fe(rng.randrange(P)) for _ in range(16)]
    docs = [b"document %d" % d for d in range(16)]
    seeds = [bytes([fast, d]) * 16 for d in range(16)]
    default = plan.sign(sks, docs, seeds)
    got = plan.sign(sks, docs, seeds, fri_batch=True)
    assert got == default and len(set(got)) == 16
    assert plan.verify([signer.rp.hash(sk) for sk in sks], docs, got) == [True] * 16


def test_fri_stage_transfers(eng):
    """at 2^12, B = 2 and B = 8: the FRI stage's reads are the roots of each round, the last codewords, one gather
    per layer but the last and one path read per layer"""
    counts = []
    for B in (2, 8):
        st, cons, trace, boundary, zvals, plan, seeds = batch_case(12, B, 3)
        log = []
        inner = plan.fri.prove_batch
        count = eng._count

        def record(kind, nbytes):
            log.append(kind)
            count(kind, nbytes)

        def counted(*args, **kw):
            eng._count = record
            try:
                return inner(*args, **kw)
            finally:
                eng._count = count
        plan.fri.prove_batch = counted
        try:
            got = plan.prove_batch([trace] * B, [boundary] * B, C.zerofier_codeword(zvals, True), seeds=seeds,
                                   fri_batch=True)
        finally:
            del plan.fri.prove_batch
        assert len(got) == B
        counts.append(log.count("d2h"))
    rounds = plan.fri.num_rounds()
    assert counts == [rounds + 1 + (rounds - 1) + rounds] * 2
