"""The plain prover's host logic (sa_stark.PlainStarkPlan, the device route of stark.py's Stark.prove) without a
GPU: every case of tests/golden/stark_plain.json through the test double of tests/stark_plain_cases.py gives the
reference's proof bytes and stream prefixes, or its message, after the same os.urandom draws; the caller's trace is
not touched; one plan serves two signatures; enable_plain, enable and disable rebind and restore in every order; a
synthetic AIR's plain proof is its FastStark proof without the zerofier openings; and the inputs the schedule does
not fold are refused."""
import hashlib
import itertools
import os
import pickle
import random

import pytest

import stark_cases as C
import stark_plain_cases as S
import sa_engine
import sa_stark

G = S.golden()
CASES = sorted(G)


@pytest.fixture(autouse=True)
def double_engine():
    prev = sa_engine._ENGINE
    sa_engine.set_engine(S.PlainStarkEngine())
    yield
    sa_engine.set_engine(prev)


@pytest.mark.parametrize("name", CASES)
def test_case_reproduces_the_reference(name):
    """the proof bytes and every prefix digest, or the reference's message, with the reference's draw count"""
    rec = G[name]
    proof, ps, draws = S.run_case(rec)
    S.check(rec, proof, ps, draws)


@pytest.mark.parametrize("name", CASES)
def test_plan_restates_the_bounds(name):
    rec = G[name]
    plan = sa_stark.PlainStarkPlan(S.stark(rec), C.air(rec))
    assert plan.bounds == rec["params"]["transition_quotient_degree_bounds"]
    assert plan.max_degree == rec["params"]["max_degree"]


def test_fixture_covers_the_issue_cases():
    nregs = {k: G[k]["params"]["num_registers"] * G[k]["params"]["num_randomizers"] for k in G}
    assert G["three_register"]["repeated_indices"] and G["three_register"]["verify"] is True
    for name in ("broken_witness", "below_zerofier", "tiny_broken"):
        # the transition division raises, after the trace randomizers alone
        assert G[name]["raises"] == sa_stark.REMAINDER and len(G[name]["draws"]) == nregs[name], name
    assert G["false_boundary"]["raises"] == sa_stark.REMAINDER
    # the cancelled top terms: a degree mismatch after the randomizer polynomial's draws
    rec = G["cancelled_top"]
    assert rec["raises"] == sa_stark.DEGREE_MISMATCH
    assert len(rec["draws"]) == nregs["cancelled_top"] + rec["params"]["max_degree"] + 1
    assert min(G["below_zerofier"]["params"]["transition_quotient_degree_bounds"]) < -1


def test_caller_trace_unchanged():
    rec = G["three_register"]
    trace, boundary = C.inputs(rec)
    rows = [list(r) for r in trace]
    ids = [id(r) for r in trace]
    proof = S.run(S.stark(rec), trace, C.air(rec), boundary, C.Urandom(rec["draws"]))
    assert hashlib.sha256(proof).hexdigest() == rec["proof_sha256"]
    assert len(trace) == len(rows) and [id(r) for r in trace] == ids and [list(r) for r in trace] == rows


def test_one_plan_serves_two_signatures():
    first, second = G["rpsss"], G["rpsss_second"]
    st = S.stark(first)
    plan = sa_stark.PlainStarkPlan(st, C.air(first))
    for rec in (first, second):
        proof, ps, draws = S.run_case(rec, plan=plan, st=st)
        S.check(rec, proof, ps, draws)


def _stand_ins():
    class Fast:
        def prove(self, *a, **k):
            return "fast host"

    class Plain:
        def prove(self, *a, **k):
            return "plain host"
    return Fast, Plain


@pytest.mark.parametrize("order", list(itertools.permutations(["plain", "fast", "disable"])))
def test_enable_plain_enable_disable_in_every_order(order):
    Fast, Plain = _stand_ins()
    originals = {Fast: Fast.__dict__["prove"], Plain: Plain.__dict__["prove"]}
    on = set()
    for step in order + ("disable",):
        if step == "plain":
            sa_stark.enable_plain(Plain)
            sa_stark.enable_plain(Plain)  # idempotent
            on.add(Plain)
        elif step == "fast":
            sa_stark.enable(Fast)
            on.add(Fast)
        else:
            sa_stark.disable()
            on.clear()
        assert Plain.__dict__["prove"] is (sa_stark.prove_plain if Plain in on else originals[Plain])
        assert Fast.__dict__["prove"] is (sa_stark.prove if Fast in on else originals[Fast])
    assert (Fast().prove(), Plain().prove()) == ("fast host", "plain host")


def test_engine_calls_are_the_planned_ones():
    """one interpolation, one boundary apply, one exact apply per division order and no unchecked one, one
    commitment of nregs + 1 codewords, one combination, and the zerofier built once"""
    rec = G["three_register"]
    eng = sa_engine.get_engine()
    proof, ps, draws = S.run_case(rec)
    S.check(rec, proof, ps, draws)
    names = [c[0] for c in eng.calls]
    nregs = rec["params"]["num_registers"]
    assert names.count("interp_apply") == 1 and names.count("boundary_quotients") == 1
    assert names.count("air_quotients_exact") == 2 and "air_quotients" not in names
    assert [c for c in eng.calls if c[0] == "merkle_trees"] == [("merkle_trees", nregs + 1,
                                                                 rec["params"]["fri_domain_length"])]
    assert names.count("coset_combine_evaluate") == 1 and names.count("merkle_open_batch") == 1
    assert names.count("zerofier") == 1


@pytest.mark.parametrize("seed", [3, 4])
def test_synthetic_plain_proof_is_faststark_without_zerofier_openings(seed):
    params, cons, trace, boundary = C.synthetic(seed, 10)
    rng = random.Random(seed)
    values = [rng.randrange(C.P) for _ in range(3 * params.num_randomizers + params.fri_domain_length)]
    plain, fast = S.pair(params, cons, trace, boundary, values)
    assert isinstance(plain, bytes) and isinstance(fast, bytes)
    objects = S.without_zerofier_openings(fast, params.num_colinearity_checks)
    assert pickle.loads(plain) == objects and plain == pickle.dumps(objects)


def test_one_cycle_raises_the_reference_index_error():
    """Stark's transition_zerofier has no points for one cycle: IndexError at the division, after the trace
    randomizers and the boundary quotients"""
    st = S.plain_stark(sa_stark.Params(C.T.field, 4, 2, 4, 2, 1, 2))
    air = [{(0, 0, 0, 1, 0): 1, (0, 1, 0, 0, 0): C.P - 1}, {(0, 0, 0, 0, 1): 1, (0, 0, 1, 0, 0): C.P - 1}]
    trace = [C.T.elems([5, 7])]
    boundary = [(0, 0, C.T.fe(5)), (0, 1, C.T.fe(7))]
    draws = C.Urandom(list(range(100, 200)))
    real = os.urandom
    os.urandom = draws
    try:
        with pytest.raises(IndexError):
            sa_stark.prove_plain(st, trace, air, boundary)
    finally:
        os.urandom = real
    assert draws.count == 2 * st.num_randomizers


def test_refusals():
    """inputs the schedule does not fold raise AssertionError instead of proving other bytes"""
    rec = G["three_register"]
    st = S.stark(rec)
    air = C.air(rec)
    nvars = 1 + 2 * st.num_registers
    n = st.fri.domain_length
    # a division order above 2^30
    with pytest.raises(AssertionError, match="above 2"):
        sa_stark.PlainStarkPlan(st, air + [{(1 << 30,) + (0,) * (nvars - 1): 1}])
    # a combination longer than the FRI domain: a bound of n makes max_degree 2n - 1
    with pytest.raises(AssertionError, match="max_degree"):
        sa_stark.PlainStarkPlan(st, air + [{(n + st.original_trace_length - 1,) + (0,) * (nvars - 1): 1}])
    # a boundary the boundary plan refuses: register 1 without boundary points
    trace, boundary = C.inputs(rec)
    plan = sa_stark.PlainStarkPlan(st, air)
    proof = S.run(st, trace, None, [b for b in boundary if b[1] != 1], C.Urandom(rec["draws"]), plan=plan)
    assert isinstance(proof, AssertionError) and not isinstance(proof, bytes)
    # a trace of another length than the plan's
    proof = S.run(st, trace[:-1], None, boundary, C.Urandom(rec["draws"]), plan=plan)
    assert isinstance(proof, AssertionError) and "rows" in str(proof)
