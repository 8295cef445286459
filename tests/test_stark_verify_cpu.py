"""The test-side verifier (tests/stark_verify.py) is neither vacuous nor too strict, on proofs the test double of
tests/stark_cases.py builds (the reference's bytes): it gives the fixture's recorded verdicts, accepts synthetic proofs,
rejects a proof with any one committed object changed, and its per-index equation fails exactly where the prover's
committed codewords, weights or shifts were perturbed."""
import pickle
import random

import pytest

import oracle as O
import stark_cases as C
import stark_verify as V
import sa_engine

G = C.golden()
VERDICTS = {"faststark": True, "three_register": True, "tiny": True, "broken_witness": False}


@pytest.fixture(autouse=True)
def double_engine():
    prev = sa_engine._ENGINE
    sa_engine.set_engine(C.StarkEngine())
    yield
    sa_engine.set_engine(prev)


def prove_synthetic(seed, log_fri, **recorder):
    """(stark, constraints, boundary, proof, zerofier codeword as ints, Recorder) of a synthetic case"""
    stark, cons, trace, boundary = C.synthetic(seed, log_fri)
    zpoly, zvals = C.zerofier(stark)
    rng = random.Random(seed)
    draws = C.Urandom([rng.randrange(C.P) for _ in range(stark.num_registers * stark.num_randomizers
                                                         + stark.fri_domain_length)])
    with V.Recorder(sa_engine.get_engine(), **recorder) as rec:
        proof, _ = C.run(stark, trace, cons, boundary, zpoly, C.zerofier_codeword(zvals, True), draws)
    assert isinstance(proof, bytes), proof
    return stark, cons, boundary, proof, zvals, rec


def root(values):
    return O.merkle_root_np(O.to_np(values))


def test_recorded_verdicts_cover_the_plain_stream_cases():
    assert {k for k, r in G.items() if r.get("verify") is not None and r["stream"] == "plain"} == set(VERDICTS)
    assert all(G[k]["verify"] is v for k, v in VERDICTS.items())


@pytest.mark.parametrize("name", sorted(VERDICTS))
def test_fixture_verdict(name):
    rec = G[name]
    proof, ps, draws = C.run_case(rec)
    C.check(rec, proof, ps, draws)
    _, boundary = C.inputs(rec)
    got = V.verify(C.params(rec), proof, C.air(rec), boundary, bytes.fromhex(rec["zerofier_root"]))
    assert got is VERDICTS[name]


@pytest.mark.parametrize("log_fri", [10, 12])
def test_synthetic_accepted(log_fri):
    stark, cons, boundary, proof, zvals, _ = prove_synthetic(log_fri, log_fri)
    assert V.verify(stark, proof, cons, boundary, root(zvals))


# ---- tampering: one object of one kind changed in an accepted proof ----
def _bump(fe):
    return C.T.fe((fe.value + 1) % C.P)


def _flip(b):
    return bytes([b[0] ^ 1]) + b[1:]


def _layout(stark, objects):
    """positions in the proof's object list (fast_stark.py:100-175 and fri.py's commit and query order)"""
    nregs, k = stark.num_registers, stark.num_colinearity_checks
    rounds = stark.fri.num_rounds()
    last = nregs + 1 + rounds
    block = 2 * 4 * k  # a leaf and a path per quadrupled index
    after_fri = len(objects) - (nregs + 2) * block
    assert after_fri == last + 1 + (rounds - 1) * 4 * k
    return {"fri_root": nregs + 1, "last": last, "fri_leaf": last + 1, "fri_path": last + 1 + k,
            "boundary": after_fri, "randomizer": after_fri + nregs * block,
            "zerofier": after_fri + (nregs + 1) * block}


def _tamper(kind, stark, objects):
    at = _layout(stark, objects)
    o = list(objects)
    if kind == "boundary_root":
        o[0] = _flip(o[0])
    elif kind == "randomizer_root":
        o[stark.num_registers] = _flip(o[stark.num_registers])
    elif kind == "fri_root":
        o[at["fri_root"]] = _flip(o[at["fri_root"]])
    elif kind == "fri_leaf":
        a, b, c = o[at["fri_leaf"]]
        o[at["fri_leaf"]] = (_bump(a), b, c)
    elif kind == "fri_path":
        o[at["fri_path"]] = [_flip(o[at["fri_path"]][0])] + o[at["fri_path"]][1:]
    elif kind == "last_codeword":
        o[at["last"]] = [_bump(o[at["last"]][0])] + o[at["last"]][1:]
    else:
        what, part = kind.rsplit("_", 1)
        i = at[what] + (part == "path")
        o[i] = _bump(o[i]) if part == "leaf" else [_flip(o[i][0])] + o[i][1:]
    assert o != list(objects)
    return pickle.dumps(o)


TAMPER = ["boundary_root", "randomizer_root", "fri_root", "fri_leaf", "fri_path", "last_codeword",
          "boundary_leaf", "boundary_path", "randomizer_leaf", "randomizer_path", "zerofier_leaf", "zerofier_path"]


@pytest.fixture(scope="module")
def accepted():
    prev = sa_engine._ENGINE
    sa_engine.set_engine(C.StarkEngine())
    try:
        stark, cons, boundary, proof, zvals, _ = prove_synthetic(21, 10)
    finally:
        sa_engine.set_engine(prev)
    return stark, cons, boundary, proof, root(zvals)


def test_repickled_proof_accepted(accepted):
    """the control of the tampering cases: loading and re-pickling the untouched objects changes nothing"""
    stark, cons, boundary, proof, zroot = accepted
    assert V.verify(stark, pickle.dumps(pickle.loads(proof)), cons, boundary, zroot)


@pytest.mark.parametrize("kind", TAMPER)
def test_tampered_proof_rejected(accepted, kind):
    stark, cons, boundary, proof, zroot = accepted
    assert V.verify(stark, _tamper(kind, stark, pickle.loads(proof)), cons, boundary, zroot) is False


# ---- checker sensitivity: the prover's outputs perturbed before the proof is built ----
def _sweep(stark, cons, boundary, proof, zvals, rec):
    """the indices of the whole FRI domain where combination_at fails, with the proof's Fiat-Shamir weights"""
    st = V.Statement(stark, cons, boundary)
    w = V.weights(stark, proof, len(cons))
    return V.failures(st, range(st.n), rec.committed, rec.combined, O.to_np(zvals), w), w


def test_unperturbed_sweep_holds_everywhere():
    stark, cons, boundary, proof, zvals, rec = prove_synthetic(22, 10)
    bad, w = _sweep(stark, cons, boundary, proof, zvals, rec)
    assert bad == [] and rec.weights == w


@pytest.mark.parametrize("at", [0, 3, 1021])
def test_perturbed_boundary_codeword_fails_at_its_index(at):
    """register 1's codeword + 1 at `at`: the equation fails there and where `at` is the next row's index"""
    def bump(vecs):
        vecs[1, at] = O.to_np([(V.element(vecs[1], at) + 1) % C.P])[0]
    stark, cons, boundary, proof, zvals, rec = prove_synthetic(23, 10, on_committed=bump)
    bad, _ = _sweep(stark, cons, boundary, proof, zvals, rec)
    n = stark.fri_domain_length
    assert bad == sorted({at, (at - stark.expansion_factor) % n})


def test_swapped_weights_fail_everywhere():
    def swap(terms):
        (a, sa, wa), (b, sb, wb) = terms[1], terms[2]
        return [terms[0], (a, sa, wb), (b, sb, wa)] + terms[3:]
    stark, cons, boundary, proof, zvals, rec = prove_synthetic(24, 10, on_terms=swap)
    bad, _ = _sweep(stark, cons, boundary, proof, zvals, rec)
    assert len(bad) == stark.fri_domain_length


@pytest.mark.parametrize("term", [2, -1])
def test_shifted_term_fails_everywhere(term):
    """a transition quotient's (term 2) or a boundary quotient's (the last term) shift one higher"""
    def shift(terms):
        vec, s, w = terms[term]
        terms[term] = (vec, s + 1, w)
        return terms
    stark, cons, boundary, proof, zvals, rec = prove_synthetic(25, 10, on_terms=shift)
    bad, _ = _sweep(stark, cons, boundary, proof, zvals, rec)
    assert len(bad) == stark.fri_domain_length
