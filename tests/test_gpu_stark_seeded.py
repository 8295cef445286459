"""Seeded proofs on the H100 (StarkPlan, PlainStarkPlan and sign_batch with seeds through CudaEngine): every fixture
case equals the host route under seeded_urandom; at 2^12, 2^16 and 2^20 FRI domains single and batched seeded proofs
equal that route and the test-side verifier accepts them; no randomizer crosses the link; the plain seeded proof is
its FastStark twin minus the zerofier openings; and, marked slow, a 2^20 + 1-row randomized trace (2^24 FRI domain)
whose seeded proof verifies and equals the host route."""
import pickle

import numpy as np
import pytest

import oracle as O
import stark_cases as C
import stark_plain_cases as S
import stark_seeded_cases as SS
import stark_verify as V
import test_stark_seeded_cpu as CPU
from test_gpu_air import release
from test_gpu_stark_geo import NCYCLES, air24, fe_boundary, fe_trace

import sa_devlist  # noqa: E402  (on sys.path through test_gpu_air)
import sa_engine  # noqa: E402
import sa_stark  # noqa: E402

pytestmark = pytest.mark.gpu
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
    release(eng)


@pytest.mark.parametrize("fast,name", CPU.CASES)
def test_fixture_case_equals_the_host_route(eng, fast, name):
    CPU.test_fixture_case_equals_the_host_route(fast, name)


@pytest.mark.parametrize("fast", [True, False])
def test_sign_batch_with_seeds(eng, fast):
    CPU.test_sign_batch_with_seeds(fast)


def synthetic_plan(log_fri, fast, seed=40):
    st, cons, trace, boundary = C.synthetic(seed + log_fri, log_fri)
    zpoly, zvals = C.zerofier(st)
    zcw = C.zerofier_codeword(zvals, True) if fast else None
    plan = sa_stark.StarkPlan(st, cons, zpoly) if fast else sa_stark.PlainStarkPlan(S.plain_stark(st), cons)
    return st, cons, trace, boundary, zvals, zcw, plan


@pytest.mark.parametrize("fast", [True, False], ids=["faststark", "plain"])
@pytest.mark.parametrize("log_fri", [12, 16, 20])
def test_synthetic_single_and_batch(eng, fast, log_fri):
    st, cons, trace, boundary, zvals, zcw, plan = synthetic_plan(log_fri, fast)
    B = 3 if log_fri < 20 else 2
    seeds = [SS.seed(log_fri, b) for b in range(B)]
    batch = SS.seeded(plan, [trace] * B, [boundary] * B, seeds, zcw)
    assert isinstance(batch, list) and len(set(batch)) == B, batch
    assert batch == SS.route(plan, [trace] * B, [boundary] * B, seeds, zcw)
    assert SS.seeded(plan, [trace], [boundary], seeds[-1:], zcw) == batch[-1:]
    if fast:
        root = O.merkle_root_np(O.to_np(zvals))
        assert all(V.verify(st, proof, cons, boundary, root) is True for proof in batch)


def test_plain_is_the_faststark_twin(eng):
    """one seed, one AIR: the plain proof's objects are the FastStark proof's without its zerofier openings"""
    st, cons, trace, boundary, _, zcw, fplan = synthetic_plan(16, True, seed=60)
    pplan = sa_stark.PlainStarkPlan(S.plain_stark(st), cons)
    s = [SS.seed("twin")]
    fast = SS.seeded(fplan, [trace], [boundary], s, zcw)[0]
    plain = SS.seeded(pplan, [trace], [boundary], s)[0]
    assert pickle.loads(plain) == S.without_zerofier_openings(fast, st.num_colinearity_checks)


@pytest.mark.parametrize("fast", [True, False], ids=["faststark", "plain"])
def test_transfers(eng, fast):
    """at a FRI domain of 2^16, B = 2: the uploads are the callers' rows, the seeds and index lists; nothing of a
    randomized trace's or a randomizer polynomial's size crosses to the device"""
    st, cons, trace, boundary, _, zcw, plan = synthetic_plan(16, fast)
    nregs, T = st.num_registers, st.original_trace_length + st.num_randomizers
    log = []
    count = eng._count

    def record(kind, nbytes):
        log.append((kind, int(nbytes)))
        count(kind, nbytes)
    eng._count = record
    try:
        got = SS.seeded(plan, [trace] * 2, [boundary] * 2, [SS.seed(1), SS.seed(2)], zcw)
    finally:
        eng._count = count
    assert isinstance(got, list), got
    h2d = [n for kind, n in log if kind == "h2d"]
    assert h2d[:2] == [2 * 32, 16 * 2 * nregs * st.original_trace_length]
    randomized = {16 * 2 * nregs * T, 16 * nregs * T, 16 * (plan.max_degree + 1), 32 * (plan.max_degree + 1)}
    assert not randomized & set(h2d), h2d


@pytest.mark.slow
def test_seeded_proof_above_the_tree(eng):
    """a 2^20 + 1-row randomized trace (2^24 FRI domain): the seeded FastStark proof verifies and equals the host
    route under seeded_urandom"""
    import torch
    st, cons, rows, boundary = air24()
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
    trace, bnd = fe_trace(rows), fe_boundary(boundary)
    s = [SS.seed("2^24")]
    got = SS.seeded(plan, [trace], [bnd], s, zcw)
    assert isinstance(got, list), got
    assert V.verify(st, got[0], cons, bnd, zcw.root())
    assert got == SS.route(plan, [trace], [bnd], s, zcw)
