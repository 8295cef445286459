"""The provers' geometric route without a GPU: with the test double's tree cap lowered below the randomized trace
length, StarkPlan and PlainStarkPlan interpolate the trace with one geometric plan of (omicron, T) (and the plain
prover takes its zerofier from geo_zerofier), through the CPU emulation of the library's schedules, and every proof,
single or batched, is the tree route's bytes from the same draws."""
import random

import pytest

import stark_batch_cases as SB
import stark_cases as C
import stark_geo_cases as SG
import stark_plain_cases as S
import sa_engine
import sa_stark


@pytest.fixture
def engines():
    prev = sa_engine._ENGINE
    yield
    sa_engine.set_engine(prev)


def prove(engine, fast, st, cons, traces, boundary, per):
    """(proofs, calls) of a batch through `engine`, each proof with its own draws `per[b]`"""
    sa_engine.set_engine(engine)
    nt = st.num_registers * st.num_randomizers
    if fast:
        zpoly, zvals = C.zerofier(st)
        plan = sa_stark.StarkPlan(st, cons, zpoly)
        got = SB.run_batch(plan, traces, [boundary] * len(traces), C.Urandom(SB.batch_draws(per, nt)), None,
                           C.zerofier_codeword(zvals, True))
    else:
        plan = sa_stark.PlainStarkPlan(S.plain_stark(st), cons)
        got = SB.run_batch(plan, traces, [boundary] * len(traces), C.Urandom(SB.batch_draws(per, nt)))
    assert isinstance(got, list), got
    return got, [c[0] for c in engine.calls]


@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("fast", [True, False], ids=["faststark", "plain"])
@pytest.mark.parametrize("log_fri", [10, 11])
def test_geometric_route_gives_the_tree_routes_bytes(engines, fast, batch, log_fri):
    st, cons, trace, boundary = C.synthetic(3 + log_fri, log_fri)
    rng = random.Random(log_fri)
    nt = st.num_registers * st.num_randomizers
    T = st.original_trace_length + st.num_randomizers
    per = [[rng.randrange(C.P) for _ in range(nt + (1 << log_fri))] for _ in range(batch)]
    tree, tree_calls = prove(SB.BatchStarkEngine(), fast, st, cons, [trace] * batch, boundary, per)
    geo, geo_calls = prove(SG.GeoStarkEngine(16), fast, st, cons, [trace] * batch, boundary, per)
    assert geo == tree
    assert "interp_plan" in tree_calls and "geo_interp_plan" not in tree_calls
    assert "geo_interp_plan" in geo_calls and "interp_plan" not in geo_calls
    assert geo_calls.count("geo_interp_apply") == 1 and T > 16
    # the plain prover's zerofier over ncycles - 1 points: by the tree at the parent's cap, geometric below it
    assert ("geo_zerofier" in geo_calls) == (not fast) and "geo_zerofier" not in tree_calls
    # every call but the route's own is the tree route's
    route = {"interp_plan", "geo_interp_plan", "zerofier", "geo_zerofier", "upload", "interp_apply",
             "geo_interp_apply"}
    assert [c for c in geo_calls if c not in route] == [c for c in tree_calls if c not in route]


def test_at_or_below_the_cap_the_calls_are_the_tree_routes(engines):
    """a cap at the trace length: the double with the geometric calls makes exactly the parent's calls"""
    st, cons, trace, boundary = C.synthetic(4, 10)
    T = st.original_trace_length + st.num_randomizers
    per = [[5 + i for i in range(st.num_registers * st.num_randomizers + 1024)]]
    for fast in (True, False):
        tree, tree_calls = prove(SB.BatchStarkEngine(), fast, st, cons, [trace], boundary, per)
        geo, geo_calls = prove(SG.GeoStarkEngine(T), fast, st, cons, [trace], boundary, per)
        assert geo == tree and geo_calls == tree_calls
