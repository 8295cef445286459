"""Batched verification without a GPU: sa_stark.VerifierPlan and SignerPlan.verify through the test double of
tests/verify_cases.py, whose verify_chunk restates every device check in Python ints.  Proofs of the fixture cases
(regenerated from their recorded draws) get the reference's recorded verdict, tampered copies are rejected at the
check the reference fails first, mixed batches equal per-proof verdicts, malformed streams are False on the plan and
go to the original method under enable_verify, and refusals come before device work."""
import pickle

import pytest

import stark_cases as C
import stark_plain_cases as S
import stark_rescue_cases as SR
import verify_cases as V
import sa_engine
import sa_stark

G = C.golden()
GP = S.golden()


@pytest.fixture(autouse=True)
def double_engine():
    prev = sa_engine._ENGINE
    sa_engine.set_engine(V.VerifyEngine())
    yield
    sa_engine.set_engine(prev)
    sa_stark.disable()


def fast_case(name):
    rec = G[name]
    stark = C.params(rec)
    proof, ps, _ = C.run_case(rec, stark=stark)
    return rec, stark, proof, C.inputs(rec)[1], bytes.fromhex(rec["zerofier_root"])


def plain_case(name):
    rec = GP[name]
    stark = S.stark(rec)
    proof, _, _ = S.run_case(rec, st=stark)
    return rec, stark, proof, C.inputs(rec)[1]


def stream_of(rec):
    return C.stream(rec)


@pytest.mark.parametrize("name", V.FAST)
def test_fast_verdicts_and_messages_recorded_from_the_reference(name):
    assert V.check_recorded(name, True) == 1 + len(V.kinds(True))


@pytest.mark.parametrize("name", V.PLAIN)
def test_plain_verdicts_and_messages_recorded_from_the_reference(name):
    assert V.check_recorded(name, False) == 1 + len(V.kinds(False))


def test_mixed_batch_equals_per_proof():
    rec, stark, proof, boundary, root = fast_case("tiny")
    plan = sa_stark.VerifierPlan(stark, C.air(rec), root)
    k, rounds = stark.fri.num_colinearity_tests, stark.fri.num_rounds()
    proofs = [proof] + [V.tamper(proof, stark.num_registers, rounds, k, t) for t in V.kinds(True)]
    single = [plan.verify_batch([p], [boundary], reasons=True)[0] for p in proofs]
    assert plan.verify_batch(proofs, [boundary] * len(proofs), reasons=True) == single
    order = list(reversed(range(len(proofs))))
    got = plan.verify_batch([proofs[i] for i in order], [boundary] * len(proofs), reasons=True)
    assert got == [single[i] for i in order]
    assert single[0] == (True, None)


def test_wrong_boundary_is_rejected():
    rec, stark, proof, boundary, root = fast_case("tiny")
    plan = sa_stark.VerifierPlan(stark, C.air(rec), root)
    c, r, v = boundary[-1]
    wrong = boundary[:-1] + [(c, r, type(v)(v.value + 1, v.field))]
    assert plan.verify_batch([proof, proof], [boundary, wrong]) == [True, False]


def test_malformed_goes_to_the_original_method_under_enable_verify():
    rec, stark, proof, boundary, root = fast_case("tiny")
    calls = []

    class Fast(type(stark)):
        def verify(self, proof, transition_constraints, boundary, transition_zerofier_root, proof_stream=None):
            calls.append(proof)
            return "original"
    stark.__class__ = Fast
    sa_stark.enable_verify(Fast)
    assert stark.verify(proof, C.air(rec), boundary, root) is True
    bad = pickle.dumps(pickle.loads(proof)[:-1])
    assert stark.verify(bad, C.air(rec), boundary, root) == "original" and calls == [bad]
    sa_stark.disable()
    assert stark.verify(proof, C.air(rec), boundary, root) == "original"


def test_enable_and_disable_in_any_order():
    class A:
        def verify(self, *a):
            return "a"

        def prove(self, *a):
            return "pa"

    class B(A):
        pass
    own = A.__dict__["verify"]
    sa_stark.enable_verify(A)
    sa_stark.enable(A)
    sa_stark.enable_verify_plain(B)
    sa_stark.enable_plain(B)
    assert A.__dict__["verify"] is not own and A.__dict__["prove"] is sa_stark.prove
    assert "verify" in B.__dict__ and "prove" in B.__dict__ and B.__dict__["prove"] is sa_stark.prove_plain
    sa_stark.disable()
    assert A().verify() == "a" and B().verify() == "a" and "verify" not in B.__dict__ and "prove" not in B.__dict__
    assert A().prove() == "pa"
    sa_stark.enable_plain(B)
    sa_stark.enable_verify(B)
    sa_stark.disable()
    assert "verify" not in B.__dict__ and "prove" not in B.__dict__


@pytest.mark.parametrize("fast", [True, False], ids=["fastrpsss", "rpsss"])
def test_signer_plan_verify(fast):
    g = G if fast else GP
    first, second = g["rpsss"], g["rpsss_second"]
    signer = SR.Signer(first, fast)
    if fast:
        signer.transition_zerofier_root = bytes.fromhex(first["zerofier_root"])
    plan = sa_stark.SignerPlan(signer)
    plan.stream = V.SignatureProofStream
    sks = [C.T.fe(int(first["sk"])), C.T.fe(int(second["sk"]))]
    docs = [b"one", b"two"]
    sigs = SR.seeded_sign(plan, sks, docs, [bytes([1]) * 32, bytes([2]) * 32])
    pks = [C.T.fe(int(first["pk"])), C.T.fe(int(second["pk"]))]
    assert plan.verify(pks, docs, sigs) == [True, True]
    assert plan.verify(pks, docs[::-1], sigs) == [False, False]
    assert plan.verify(pks[::-1], docs, sigs) == [False, False]


def test_refusals_before_device_work():
    rec, stark, proof, boundary, root = fast_case("tiny")
    plan = sa_stark.VerifierPlan(stark, C.air(rec), root)
    eng = sa_engine.get_engine()
    before = len(eng.calls)
    with pytest.raises(AssertionError):
        plan.verify_batch([proof], [])
    with pytest.raises(AssertionError):
        plan.verify_batch([proof], [[(0, 0, C.T.fe(1))]])  # register 1 has no point
    assert plan.verify_batch([b"not a pickle"], [boundary]) == [False]
    assert len(eng.calls) == before


def test_a_batch_across_chunks_equals_one_chunk(monkeypatch):
    stark, cons, boundary, root, proof = V.case("tiny", True)
    plan = sa_stark.VerifierPlan(stark, cons, root)
    k, rounds = stark.fri.num_colinearity_tests, stark.fri.num_rounds()
    proofs = [proof] + [V.tamper(proof, stark.num_registers, rounds, k, t) for t in V.kinds(True)] + [proof]
    whole = plan.verify_batch(proofs, [boundary] * len(proofs), reasons=True)
    eng = sa_engine.get_engine()
    before = len(eng.calls)
    monkeypatch.setattr(sa_stark, "CHUNK_BYTES", 2 * plan._bytes(plan._parse(proof, boundary, None)) + 1)
    assert plan.verify_batch(proofs, [boundary] * len(proofs), reasons=True) == whole
    chunks = [c[1] for c in eng.calls[before:] if c[0] == "verify_chunk"]
    assert len(chunks) > 1 and max(chunks) == 2 and sum(chunks) == len(proofs) - 1  # the truncated one is malformed
