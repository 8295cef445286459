"""The provers' geometric route on the device.  With the engine's tree cap lowered, FastStark, plain and batched proofs
at 2^12, 2^16 and 2^20 FRI domains are the tree route's bytes from the same draws.  Above the real cap, a trace of
2^20 - 7 cycles (a randomized trace of 2^20 + 1 rows, a 2^24 FRI domain): the trace polynomials give the trace rows and
the randomizers back at sampled points, the test-side verifier accepts the FastStark proof with its zerofier from
geo_zerofier, and the plain proof is that proof without its zerofier openings."""
import os
import random
import sys

import numpy as np
import pytest

import oracle as O
import stark_batch_cases as SB
import stark_cases as C
import stark_plain_cases as S
import stark_verify as V

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "stark-anatomy_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)
import sa_devlist  # noqa: E402
import sa_engine  # noqa: E402
import sa_stark  # noqa: E402

pytestmark = pytest.mark.gpu
P = O.P
GIB = 1 << 30


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
    import torch
    torch.cuda.synchronize()


def proofs(eng, fast, st, cons, traces, boundary, per):
    """a batch's proofs through the current route, each proof with its own draws, and the plan"""
    nt = st.num_registers * st.num_randomizers
    draws = C.Urandom(SB.batch_draws(per, nt))
    if fast:
        zpoly, zvals = C.zerofier(st)
        plan = sa_stark.StarkPlan(st, cons, zpoly)
        got = SB.run_batch(plan, traces, [boundary] * len(traces), draws, None, C.zerofier_codeword(zvals, True))
    else:
        plan = sa_stark.PlainStarkPlan(S.plain_stark(st), cons)
        got = SB.run_batch(plan, traces, [boundary] * len(traces), draws)
    assert isinstance(got, list), got
    return got, plan


@pytest.mark.parametrize("batch", [1, 2])
@pytest.mark.parametrize("fast", [True, False], ids=["faststark", "plain"])
@pytest.mark.parametrize("log_fri", [12, 16, pytest.param(20, marks=pytest.mark.slow)])
def test_lowered_cap_gives_the_tree_routes_bytes(eng, monkeypatch, log_fri, fast, batch):
    st, cons, trace, boundary = C.synthetic(40 + log_fri, log_fri)
    rng = random.Random(log_fri)
    per = [[rng.randrange(P) for _ in range(st.num_registers * st.num_randomizers + (1 << log_fri))]
           for _ in range(batch)]
    traces = [trace] * batch
    tree, plan = proofs(eng, fast, st, cons, traces, boundary, per)
    assert isinstance(plan.interp, sa_engine.InterpPlan)
    monkeypatch.setattr(eng, "tree_fits", lambda k: k <= 16)
    geo, plan = proofs(eng, fast, st, cons, traces, boundary, per)
    assert isinstance(plan.interp, sa_engine.GeoInterpPlan)
    assert geo == tree


NCYCLES = (1 << 20) - 7  # with 2 colinearity checks a randomized trace of 2^20 + 1 rows


@pytest.fixture(scope="module")
def case24(eng):
    return air24()


def air24():
    """(Params, constraints, trace rows as ints, boundary as ints) of a two-register AIR over NCYCLES cycles:
    r0' = r0 r1 + a, r1' = b r1 + x; transition degree 2, so the omicron domain has 2^22 points and FRI 2^24"""
    rng = random.Random(24)
    st = sa_stark.Params(C.T.field, 4, 2, 4, 2, NCYCLES, transition_constraints_degree=2)
    assert st.randomized_trace_length == (1 << 20) + 1 and st.fri_domain_length == 1 << 24
    a, b = rng.randrange(1, P), rng.randrange(2, P)
    cons = [{(0, 0, 0, 1, 0): 1, (0, 1, 1, 0, 0): P - 1, (0, 0, 0, 0, 0): P - a},
            {(0, 0, 0, 0, 1): 1, (0, 0, 1, 0, 0): P - b, (1, 0, 0, 0, 0): P - 1}]
    w = st.omicron.value
    r0, r1, x = rng.randrange(P), rng.randrange(P), 1
    rows = []
    for _ in range(NCYCLES):
        rows.append([r0, r1])
        r0, r1, x = (r0 * r1 + a) % P, (b * r1 + x) % P, x * w % P
    boundary = [(0, 0, rows[0][0]), (0, 1, rows[0][1]), (NCYCLES - 1, 0, rows[-1][0])]
    return st, cons, rows, boundary


def fe_trace(rows):
    return [C.T.elems(r) for r in rows]


def fe_boundary(boundary):
    return [(c, r, C.T.fe(v)) for c, r, v in boundary]


@pytest.mark.slow
def test_trace_polynomials_above_the_tree(eng, case24):
    st, cons, rows, boundary = case24
    zpoly = O.from_np(eng.download(eng.geo_zerofier(st.omicron.value, NCYCLES - 1)).view(np.uint64))
    plan = sa_stark.StarkPlan(st, cons, zpoly)
    assert isinstance(plan.interp, sa_engine.GeoInterpPlan)
    T, nregs = plan.trace_length, plan.nregs
    rng = random.Random(5)
    rand = [rng.randrange(P) for _ in range(nregs * st.num_randomizers)]
    real = sa_stark.os.urandom
    sa_stark.os.urandom = C.Urandom(rand)
    try:
        polys = plan._trace_polynomials(eng, [fe_trace(rows)])
    finally:
        sa_stark.os.urandom = real
    idx = sorted(set(rng.sample(range(NCYCLES), 56)) | set(range(NCYCLES, T)))
    w = st.omicron.value
    pts = eng.upload(O.to_np([pow(w, i, P) for i in idx]).view(np.int64))
    for s in range(nregs):
        got = O.from_np(eng.download(eng.poly_eval(polys[s].contiguous(), pts, mode=1)).view(np.uint64))
        want = [rows[i][s] if i < NCYCLES else rand[(i - NCYCLES) * nregs + s] for i in idx]
        assert got == want, s


@pytest.mark.slow
def test_proofs_above_the_tree(eng, case24):
    """the FastStark proof verifies; the plain proof from the same draws is it without the zerofier openings"""
    import torch
    st, cons, rows, boundary = case24
    n = st.fri_domain_length
    torch.cuda.empty_cache()
    assert eng.lib.sa_release_workspaces() == 0
    if torch.cuda.mem_get_info(eng.device)[0] < 16 * GIB:
        pytest.skip("the 2^24 proofs need 16 GiB free on the device")
    z = eng.geo_zerofier(st.omicron.value, NCYCLES - 1)
    zpoly = O.from_np(eng.download(z).view(np.uint64))
    cw = eng.coset_evaluate(z, n.bit_length() - 1, st.omega.value, st.generator.value)
    zcw = sa_devlist.DeviceCodeword(cw, None, C.T.field, n)
    plan = sa_stark.StarkPlan(st, cons, zpoly)
    rng = random.Random(6)
    values = [rng.randrange(P) for _ in range(st.num_registers * st.num_randomizers + plan.max_degree + 1)]
    fast, _ = C.run(st, fe_trace(rows), None, fe_boundary(boundary), zpoly, zcw, C.Urandom(values), plan=plan)
    assert isinstance(fast, bytes), fast
    assert V.verify(st, fast, cons, fe_boundary(boundary), zcw.root())
    del plan
    plain = S.run(None, fe_trace(rows), None, fe_boundary(boundary), C.Urandom(values),
                  plan=sa_stark.PlainStarkPlan(S.plain_stark(st), cons))
    assert isinstance(plain, bytes), plain
    import pickle
    assert pickle.loads(plain) == S.without_zerofier_openings(fast, st.num_colinearity_checks)
