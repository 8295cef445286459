"""The plain prover on the H100 (sa_stark.PlainStarkPlan through CudaEngine): every case of
tests/golden/stark_plain.json gives the reference's proof bytes, or its message, the two RPSSS signatures included
(replayed from the fixture's recorded trace, AIR and draws); one plan serves both signatures; at FRI domains 2^16 to
2^22 the plain proof of test_gpu_stark_scale's synthetic AIRs is the FastStark proof with the same draws minus its
zerofier openings, and the test-side verifier accepts that FastStark twin; and at 2^20 a witness broken at one
middle row raises the remainder message after exactly the trace randomizers, with no whole-row download."""
import pickle
import random

import numpy as np
import pytest

import oracle as O
import stark_cases as C
import stark_plain_cases as S
import stark_verify as V
import sa_engine
import sa_stark
from test_gpu_stark_scale import fe, fe_boundary, need_device, synthetic, zerofier

pytestmark = pytest.mark.gpu
G = S.golden()
P = O.P


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


@pytest.mark.parametrize("name", sorted(G))
def test_case_byte_identical(eng, name):
    rec = G[name]
    proof, ps, draws = S.run_case(rec)
    S.check(rec, proof, ps, draws)


def test_one_plan_two_signatures(eng):
    first, second = G["rpsss"], G["rpsss_second"]
    st = S.stark(first)
    plan = sa_stark.PlainStarkPlan(st, C.air(first))
    for rec in (first, second):
        proof, ps, draws = S.run_case(rec, plan=plan, st=st)
        S.check(rec, proof, ps, draws)


MATRIX = [  # (log_fri, nregs, expansion_factor, colinearity_checks)
    (16, 1, 4, 2),
    (16, 3, 16, 8),
    (18, 3, 4, 2),
    (20, 3, 4, 2),
    pytest.param(22, 9, 4, 2, marks=pytest.mark.slow),
]


@pytest.mark.parametrize("log_fri,nregs,ef,checks", MATRIX)
def test_plain_is_faststark_without_zerofier_openings(eng, log_fri, nregs, ef, checks):
    need_device(eng, log_fri, 9 * (nregs + 1) + 48)
    stark, cons, rows, boundary = synthetic(log_fri, log_fri, nregs, ef, checks)
    zpoly, zcw = zerofier(eng, stark)
    rng = random.Random(log_fri)
    values = [rng.randrange(P) for _ in range(nregs * stark.num_randomizers + stark.fri_domain_length)]
    plain, fast = S.pair(stark, cons, fe(rows), fe_boundary(boundary), values, zcw, zpoly)
    assert isinstance(plain, bytes) and isinstance(fast, bytes), (plain, fast)
    objects = S.without_zerofier_openings(fast, checks)
    assert pickle.loads(plain) == objects
    assert plain == pickle.dumps(objects)
    zroot = O.merkle_root_np(eng.download(zcw.device_vector()).view(np.uint64))
    assert V.verify(stark, fast, cons, fe_boundary(boundary), zroot)


def test_broken_witness_at_2_20_raises_without_row_downloads(eng):
    """register 0 off by one at a middle row: the remainder message after the trace randomizers alone, and nothing
    near a row's size read back"""
    log_fri = 20
    need_device(eng, log_fri, 9 * 4 + 48)
    stark, cons, rows, boundary = synthetic(20, log_fri, 3, 4, 2)
    c = len(rows) // 2
    assert all(bc != c for bc, _, _ in boundary)
    broken = [list(r) for r in rows]
    broken[c][0] = (broken[c][0] + 1) % P
    st = S.plain_stark(stark)
    plan = sa_stark.PlainStarkPlan(st, cons)
    log = []
    count = eng._count

    def record(kind, nbytes):
        log.append((kind, int(nbytes)))
        count(kind, nbytes)
    draws = C.Urandom([7] * (1 << 21))
    eng._count = record
    try:
        proof = S.run(st, fe(broken), None, fe_boundary(boundary), draws, plan=plan)
    finally:
        eng._count = count
    assert isinstance(proof, AssertionError) and str(proof).startswith(sa_stark.REMAINDER), proof
    assert draws.count == 3 * stark.num_randomizers
    d2h = [b for k, b in log if k == "d2h"]
    assert max(d2h, default=0) < 16 * 1024, d2h  # flags and single elements; a trace row is 16 * 2^16 bytes
