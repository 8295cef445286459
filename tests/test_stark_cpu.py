"""The device prover's host logic (sa_stark) without a GPU: every case of tests/golden/stark.json through the test
double of tests/stark_cases.py gives the reference's proof bytes and stream prefixes, or its message, after the same
os.urandom draws; Params restates what FastStark derives; the caller's trace is not touched; enable/disable rebind
and restore; a plain-list zerofier codeword proves the same bytes as a device list; one plan serves two signatures;
and the inputs the schedule cannot decide exactly are refused."""
import hashlib
import json
import os

import pytest

import stark_cases as C
import sa_engine
import sa_stark

G = C.golden()
CASES = sorted(G)


@pytest.fixture(autouse=True)
def double_engine():
    prev = sa_engine._ENGINE
    sa_engine.set_engine(C.StarkEngine())
    yield
    sa_engine.set_engine(prev)


@pytest.mark.parametrize("name", CASES)
def test_params_restate_faststark(name):
    rec = G[name]
    p, st = rec["params"], C.params(rec)
    assert (st.num_randomizers, st.omicron_domain_length, st.fri_domain_length) == \
        (p["num_randomizers"], p["omicron_domain_length"], p["fri_domain_length"])
    assert [str(v.value) for v in (st.generator, st.omega, st.omicron)] == [p["generator"], p["omega"], p["omicron"]]
    air = C.air(rec)
    assert st.transition_quotient_degree_bounds(air) == p["transition_quotient_degree_bounds"]
    assert st.max_degree(air) == p["max_degree"]
    _, boundary = C.inputs(rec)
    T = len(rec["trace"]) + st.num_randomizers
    assert st.boundary_quotient_degree_bounds(T, boundary) == p["boundary_quotient_degree_bounds"]
    assert isinstance(st.fri, C.sa_stark._fri.Fri) and st.fri.domain_length == st.fri_domain_length


@pytest.mark.parametrize("name", CASES)
def test_case_reproduces_the_reference(name):
    """the proof bytes and every prefix digest, or the reference's message, with the reference's draw count"""
    rec = G[name]
    proof, ps, draws = C.run_case(rec)
    C.check(rec, proof, ps, draws)


def test_fixture_agrees_with_the_earlier_fixtures():
    """the seed-600 run is faststark_trace.json's and the first signature is rpsss.json's"""
    with open(os.path.join(C.HERE, "golden", "faststark_trace.json")) as f:
        assert G["faststark"]["proof_sha256"] == json.load(f)["proof_sha256"]
    with open(os.path.join(C.HERE, "golden", "rpsss.json")) as f:
        assert G["rpsss"]["proof_sha256"] == json.load(f)["signature_sha256"]
    assert G["three_register"]["repeated_indices"]
    assert G["broken_witness"].get("verify") is False or "raises" in G["broken_witness"]
    assert G["false_boundary"]["raises"].startswith(sa_stark.REMAINDER)
    assert G["below_zerofier"]["raises"] == sa_stark.LARGER_DEGREE
    assert G["tiny_broken"]["raises"] == sa_stark.REMAINDER


@pytest.mark.parametrize("name", ["three_register", "false_boundary", "tiny"])
def test_plain_list_zerofier_codeword(name):
    """a zerofier codeword given as a list of the caller's elements proves the same bytes"""
    rec = G[name]
    proof, ps, draws = C.run_case(rec, device_list=False)
    C.check(rec, proof, ps, draws)


def test_caller_trace_unchanged():
    rec = G["three_register"]
    stark = C.params(rec)
    zpoly, zvals = C.zerofier(stark)
    trace, boundary = C.inputs(rec)
    rows = [list(r) for r in trace]
    ids = [id(r) for r in trace]
    proof, _ = C.run(stark, trace, C.air(rec), boundary, zpoly, C.zerofier_codeword(zvals, True),
                     C.Urandom(rec["draws"]))
    assert hashlib.sha256(proof).hexdigest() == rec["proof_sha256"]
    assert len(trace) == len(rows) and [id(r) for r in trace] == ids and [list(r) for r in trace] == rows


def test_one_plan_serves_two_signatures():
    first, second = G["rpsss"], G["rpsss_second"]
    stark = C.params(first)
    zpoly, _ = C.zerofier(stark)
    plan = sa_stark.StarkPlan(stark, C.air(first), zpoly)
    for rec in (first, second):
        proof, ps, draws = C.run_case(rec, plan=plan, stark=stark)
        C.check(rec, proof, ps, draws)


def test_enable_disable_rebind_a_stand_in_class():
    class Stand:
        def prove(self, *a, **k):
            return "host"

    class Sub(Stand):
        pass
    original = Stand.__dict__["prove"]
    sa_stark.enable(Stand)
    sa_stark.enable(Stand)  # idempotent
    assert Stand.prove is sa_stark.prove
    sa_stark.enable(Sub)
    assert Sub.__dict__["prove"] is sa_stark.prove
    sa_stark.disable()
    assert Stand.__dict__["prove"] is original and "prove" not in Sub.__dict__
    assert Sub().prove() == "host"
    sa_stark.disable()  # idempotent
    assert Stand.__dict__["prove"] is original


def test_enabled_class_proves_through_the_device_schedule():
    """a stand-in FastStark whose prove is rebound: the unmodified call site gets the reference's bytes"""
    rec = G["tiny"]

    class Stark(sa_stark.Params):
        def prove(self, *a, **k):
            raise RuntimeError("the host prover")
    p = rec["params"]
    stark = Stark(C.T.field, p["expansion_factor"], p["num_colinearity_checks"], p["security_level"],
                  p["num_registers"], p["num_cycles"], p["transition_constraints_degree"])
    zpoly, zvals = C.zerofier(stark)
    trace, boundary = C.inputs(rec)
    sa_stark.enable(Stark)
    try:
        real = os.urandom
        os.urandom = C.Urandom(rec["draws"])
        try:
            proof = stark.prove(trace, C.air(rec), boundary, zpoly, C.zerofier_codeword(zvals, True))
        finally:
            os.urandom = real
    finally:
        sa_stark.disable()
    assert hashlib.sha256(proof).hexdigest() == rec["proof_sha256"]
    with pytest.raises(RuntimeError):
        stark.prove()


def test_engine_calls_are_the_planned_ones():
    """one interpolation, one boundary apply, one apply per division order, one commitment of nregs + 1 codewords,
    one combination"""
    rec = G["three_register"]
    eng = sa_engine.get_engine()
    proof, ps, draws = C.run_case(rec)
    C.check(rec, proof, ps, draws)
    names = [c[0] for c in eng.calls]
    nregs = rec["params"]["num_registers"]
    assert names.count("interp_apply") == 1 and names.count("boundary_quotients") == 1
    assert names.count("air_quotients") == 2  # the linear and the cubic constraints divide at different orders
    assert [c for c in eng.calls if c[0] == "merkle_trees"] == [("merkle_trees", nregs + 1,
                                                                 rec["params"]["fri_domain_length"])]
    assert names.count("coset_combine_evaluate") == 1 and names.count("merkle_open_batch") == 1
    assert "interpolate" not in names[names.index("interp_plan") + 1:names.index("boundary_plan")]


def test_refusals():
    """inputs the schedule cannot decide exactly raise instead of proving other bytes"""
    rec = G["three_register"]
    stark = C.params(rec)
    zpoly, zvals = C.zerofier(stark)
    air = C.air(rec)
    # a zerofier of another degree than num_cycles - 1
    with pytest.raises(AssertionError, match="zerofier has degree"):
        sa_stark.StarkPlan(stark, air, C.T.Polynomial(zpoly.coefficients + [C.T.fe(0)] + [C.T.fe(1)]))
    with pytest.raises(AssertionError, match="zero polynomial"):
        sa_stark.StarkPlan(stark, air, C.T.Polynomial([C.T.fe(0)]))
    # a constraint of degree at or above the omicron domain's length
    nvars = 1 + 2 * stark.num_registers
    big = {(stark.omicron_domain_length,) + (0,) * (nvars - 1): 1}
    with pytest.raises(AssertionError, match="omicron domain"):
        sa_stark.StarkPlan(stark, air + [big], zpoly)
    # a numerator below its degree bound: its top terms cancel on every trace
    plan = sa_stark.StarkPlan(stark, air + [{(0, 1, 0, 0, 0, 0, 0): 1, (0, 0, 0, 0, 0, 0, 0): 1,
                                             (0, 2, 0, 0, 0, 0, 0): 0}], zpoly)
    trace, boundary = C.inputs(rec)
    proof, _ = C.run(stark, trace, None, boundary, zpoly, C.zerofier_codeword(zvals, True), C.Urandom(rec["draws"]),
                     plan=plan)
    assert isinstance(proof, AssertionError) and "cannot be decided" in str(proof)
    # a trace of another length than the plan's
    proof, _ = C.run(stark, trace[:-1], None, boundary, zpoly, C.zerofier_codeword(zvals, True),
                     C.Urandom(rec["draws"]), plan=plan)
    assert isinstance(proof, AssertionError) and "rows" in str(proof)


def test_import_does_not_load_torch():
    import subprocess
    import sys
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import sa_stark; "
            "print('torch' in sys.modules)" % (os.path.join(os.path.dirname(C.HERE), "oracle"), C.sa_stark.__file__
                                               .rsplit(os.sep, 1)[0]))
    out = subprocess.check_output([sys.executable, "-c", code], text=True)
    assert out.strip() == "False"


def test_synthetic_case_is_deterministic():
    a = C.synthetic_prove(3, 10)
    b = C.synthetic_prove(3, 10)
    assert isinstance(a[0], bytes) and a == b
