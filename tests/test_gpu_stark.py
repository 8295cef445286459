"""The device prover on the H100 (sa_stark through CudaEngine): every case of tests/golden/stark.json gives the
reference's proof bytes, or its message, the RPSSS signature and the seed-600 proof included; one StarkPlan serves
both signatures and its buffers are unchanged afterwards; synthetic AIRs at FRI domains 2^10 ... 2^16 prove the bytes
the test double proves; the prover's host<->device traffic is the trace, the randomizer, the indices and small reads;
and the out= forms of coset_evaluate and boundary_quotients write where they are told."""
import hashlib
import json
import os

import numpy as np
import pytest

import stark_cases as C
import oracle as O
import sa_engine
import sa_stark

pytestmark = pytest.mark.gpu
G = C.golden()


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
    proof, ps, draws = C.run_case(rec)
    C.check(rec, proof, ps, draws)


def test_recorded_runs_of_the_earlier_fixtures(eng):
    """the seed-600 proof is faststark_trace.json's, the signature rpsss.json's"""
    with open(os.path.join(C.HERE, "golden", "faststark_trace.json")) as f:
        want = json.load(f)["proof_sha256"]
    proof, _, _ = C.run_case(G["faststark"])
    assert hashlib.sha256(proof).hexdigest() == want
    with open(os.path.join(C.HERE, "golden", "rpsss.json")) as f:
        want = json.load(f)["signature_sha256"]
    proof, _, _ = C.run_case(G["rpsss"])
    assert hashlib.sha256(proof).hexdigest() == want


def test_plain_list_zerofier_codeword(eng):
    rec = G["rpsss"]
    proof, ps, draws = C.run_case(rec, device_list=False)
    C.check(rec, proof, ps, draws)


def test_one_plan_two_signatures_plan_unchanged(eng):
    first, second = G["rpsss"], G["rpsss_second"]
    stark = C.params(first)
    zpoly, _ = C.zerofier(stark)
    plan = sa_stark.StarkPlan(stark, C.air(first), zpoly)
    buffers = [plan.interp.plan, plan.zerofier] + [p.plan for _, p, _, _ in plan.groups]
    before = [b.clone() for b in buffers]
    for rec in (first, second):
        proof, ps, draws = C.run_case(rec, plan=plan, stark=stark)
        C.check(rec, proof, ps, draws)
    assert all(bool((a == b).all()) for a, b in zip(before, buffers))


@pytest.mark.parametrize("log_fri", [10, 12, 14, 16])
def test_synthetic_matches_the_double(eng, log_fri):
    got = C.synthetic_prove(log_fri, log_fri)
    assert isinstance(got[0], bytes), got[0]
    sa_engine.set_engine(C.StarkEngine())
    want = C.synthetic_prove(log_fri, log_fri)
    sa_engine.set_engine(eng)
    assert got == want


def test_transfers(eng):
    """at a FRI domain of 2^16 the prove uploads the trace, the randomizer and index lists, and outside FRI reads
    nothing near a codeword's or a quotient's size"""
    log_fri = 16
    n = 1 << log_fri
    stark, cons, trace, boundary = C.synthetic(5, log_fri)
    zpoly, zvals = C.zerofier(stark)
    zcw = C.zerofier_codeword(zvals, True)
    plan = sa_stark.StarkPlan(stark, cons, zpoly)
    log, inside = [], [False]
    count = eng._count

    def record(kind, nbytes):
        log.append((kind, int(nbytes), inside[0]))
        count(kind, nbytes)
    fri_prove = plan.fri.prove

    def prove_marked(codeword, ps):
        inside[0] = True
        try:
            return fri_prove(codeword, ps)
        finally:
            inside[0] = False
    eng._count = record
    plan.fri.prove = prove_marked
    try:
        proof, _ = C.run(stark, trace, None, boundary, zpoly, zcw, C.Urandom([7] * (1 << 20)), plan=plan)
    finally:
        eng._count = count
        del plan.fri.prove
    assert isinstance(proof, bytes), proof
    T = plan.trace_length
    nregs = stark.num_registers
    h2d = [b for k, b, f in log if k == "h2d" and not f]
    for b in (16 * nregs * T, 16 * (plan.max_degree + 1)):  # the trace columns, the randomizer
        h2d.remove(b)
    assert max(h2d) <= 1024, h2d  # index lists, and the boundary's points and values for its plan
    d2h = [b for k, b, f in log if k == "d2h" and not f]
    assert max(d2h) < 16 * (n // 16), d2h


def test_out_forms(eng):
    """coset_evaluate and boundary_quotients write into a caller's rows, refuse a wrong one, and default as before"""
    import torch
    from boundary_cases import make_case
    log_n = 8
    n = 1 << log_n
    boundary, omicron, trace, _, _, root, offset = make_case(3, log_n, 2, [2, 1])
    t = eng.upload(O.to_np([v for row in trace for v in row]).view(np.int64)).reshape(2, len(trace[0]), 2)
    plan = eng.boundary_plan(boundary, 2, omicron, log_n, root, offset)
    buf = torch.full((3, n, 2), 7, dtype=torch.int64, device=eng.device)
    q0, cw0, f0 = eng.boundary_quotients(plan, t)
    q1, cw1, f1 = eng.boundary_quotients(plan, t, out=buf[:2])
    assert cw1.data_ptr() == buf.data_ptr() and bool((buf[:2] == cw0).all()) and bool((buf[2] == 7).all())
    coeffs = t[0]
    want = eng.coset_evaluate(coeffs, log_n, root, offset)
    got = eng.coset_evaluate(coeffs, log_n, root, offset, out=buf[2])
    assert got.data_ptr() == buf[2].data_ptr() and bool((buf[2] == want).all())
    for bad in (buf[:1], buf[:, :n // 2], buf.transpose(0, 1)[:2], buf[:2].to(torch.int32)):
        with pytest.raises(sa_engine.SaError):
            eng.boundary_quotients(plan, t, out=bad)
    with pytest.raises(sa_engine.SaError):
        eng.coset_evaluate(coeffs, log_n, root, offset, out=buf[:2])
