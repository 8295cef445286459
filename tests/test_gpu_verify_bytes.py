"""Verification from the proof bytes on the device (DESIGN section 3.17): the fixture cases and every tamper kind get
the reference's recorded verdicts through the device route (observed by wrapping VerifierPlan._parse, which only
the host route calls); a mixed batch of canonical proofs, re-encodings, a truncated stream and a boundary whose
interpolation raises gives the host route's output, exceptions and proof_index; a proof whose zerofier values are
zero raises "divide by zero" from the device route at its index, after a later boundary's exception; 64
seeded FastRPSSS and RPSSS signatures verify with no _parse call; adversarial bytes are refused without a CUDA error;
a fixed launch count per chunk; and no spills in the new kernels."""
import os
import re
import subprocess
import tempfile

import pytest

import stark_cases as C
import stark_plain_cases as S
import stark_rescue_cases as SR
import transcript_emu as TE
import verify_cases as V
from test_gpu_air import release
from test_transcript_emu_cpu import mutations, reencodings

import sa_engine  # noqa: E402
import sa_stark  # noqa: E402

pytestmark = pytest.mark.gpu
G = C.golden()
GP = S.golden()
PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "stark-anatomy_b200")


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


@pytest.fixture
def host_parses(monkeypatch):
    calls = []
    parse = sa_stark.VerifierPlan._parse

    def wrapped(self, proof, *args):
        calls.append(proof)
        return parse(self, proof, *args)
    monkeypatch.setattr(sa_stark.VerifierPlan, "_parse", wrapped)
    return calls


def on_host(fn):
    prev = sa_engine._ENGINE
    sa_engine.set_engine(V.VerifyEngine())
    try:
        return fn()
    finally:
        sa_engine.set_engine(prev)


def outcome(fn):
    try:
        return fn()
    except AssertionError as exc:
        return ("raised", str(exc), getattr(exc, "proof_index", None))


@pytest.mark.parametrize("name,fast", [(n, True) for n in V.FAST] + [(n, False) for n in V.PLAIN])
def test_recorded_verdicts_on_the_device_route(name, fast, monkeypatch):
    assert V.check_recorded(name, fast) == 1 + len(V.kinds(fast))
    stark, cons, boundary, root, proof = V.case(name, fast)
    k, rounds = stark.fri.num_colinearity_tests, stark.fri.num_rounds()
    proofs = [proof if r["kind"] == "none" else V.tamper(proof, stark.num_registers, rounds, k, r["kind"])
              for r in V.recorded(name, fast)]
    calls = []
    parse = sa_stark.VerifierPlan._parse
    monkeypatch.setattr(sa_stark.VerifierPlan, "_parse", lambda self, p, *a: calls.append(p) or parse(self, p, *a))
    run = lambda: sa_stark.VerifierPlan(stark, cons, root).verify_batch(proofs, [boundary] * len(proofs),  # noqa
                                                                       reasons=True)
    got = run()
    truncated = V.tamper(proof, stark.num_registers, rounds, k, "truncated")
    assert calls == [truncated]  # only the truncated stream is read on the host
    monkeypatch.setattr(sa_stark.VerifierPlan, "_parse", parse)
    assert got == on_host(run)


def test_mixed_batch_equals_host_route():
    stark, cons, boundary, root, proof = V.case("three_register", True)
    k, rounds = stark.fri.num_colinearity_tests, stark.fri.num_rounds()
    proofs = [proof] + list(reencodings(proof).values()) + \
        [V.tamper(proof, stark.num_registers, rounds, k, t) for t in ("truncated", "fri_leaf_b", "boundary_leaf")]
    bounds = [boundary] * len(proofs)
    run = lambda p, b: outcome(lambda: sa_stark.VerifierPlan(stark, cons, root).verify_batch(p, b, reasons=True))  # noqa
    assert run(proofs, bounds) == on_host(lambda: run(proofs, bounds))
    # a boundary whose interpolation raises, after a proof the device reads
    empty_reg = [(c, r, v) for c, r, v in boundary if r != 0]
    bad = bounds[:3] + [empty_reg] + bounds[4:]
    got = run(proofs, bad)
    assert got == on_host(lambda: run(proofs, bad)) and got[0] == "raised" and got[2] == 3
    # a plain batch with a host-route proof between two device-route ones
    sp, consp, bp, _, pp = V.case("tiny", False)
    plain = lambda ps: outcome(lambda: sa_stark.VerifierPlan(sp, consp).verify_batch(ps, [bp] * len(ps),  # noqa
                                                                                  reasons=True))
    batch = [pp] * 3 + [V.tamper(pp, sp.num_registers, sp.fri.num_rounds(), sp.fri.num_colinearity_tests,
                                 "truncated")] + [pp] * 3
    assert plain(batch) == on_host(lambda: plain(batch))


def test_divide_by_zero_on_the_device_route(host_parses):
    """a proof whose opened zerofier values are zero raises "divide by zero" with its index from the device route,
    after the checks of every chunk; a boundary that raises at a later index comes first, as _parse raises it before
    any check; both as the host route gives them"""
    stark, cons, boundary, root, proof = V.case("three_register", True)
    zroot, dz = TE.zero_zerofier_proof(stark, cons, boundary, root, proof)
    k, rounds = stark.fri.num_colinearity_tests, stark.fri.num_rounds()
    proofs = [proof, proof] + list(reencodings(proof).values()) + [dz] + \
        [V.tamper(proof, stark.num_registers, rounds, k, t) for t in ("fri_leaf_b", "boundary_leaf", "truncated")] + \
        [dz, proof, proof]
    at = proofs.index(dz)
    bounds = [boundary] * len(proofs)
    run = lambda b: outcome(lambda: sa_stark.VerifierPlan(stark, cons, zroot).verify_batch(proofs, b))  # noqa: E731
    got = run(bounds)
    assert got == ("raised", "divide by zero", at) and dz not in host_parses
    assert got == on_host(lambda: run(bounds))
    later = list(bounds)
    later[at + 4] = [(c, r, v) for c, r, v in boundary if r != 0]
    got = run(later)
    assert got[0] == "raised" and got[2] == at + 4 and got != ("raised", "divide by zero", at)
    assert got == on_host(lambda: run(later))


@pytest.mark.parametrize("fast", [True, False], ids=["fastrpsss", "rpsss"])
def test_64_signatures_read_on_the_device(eng, fast, host_parses):
    g = G if fast else GP
    first = g["rpsss"]
    signer = SR.Signer(first, fast)
    if fast:
        signer.transition_zerofier_root = bytes.fromhex(first["zerofier_root"])
    plan = sa_stark.SignerPlan(signer)
    plan.stream = V.SignatureProofStream
    sks = [C.T.fe(11 + 5 * d) for d in range(64)]
    docs = [b"signed %d" % d for d in range(64)]
    sigs = plan.sign(sks, docs, [bytes([d, 7]) * 16 for d in range(64)])
    pks = [signer.rp.hash(sk) for sk in sks]
    nregs, rounds = plan.stark.num_registers, plan.stark.fri.num_rounds()
    sigs[17] = V.tamper(sigs[17], nregs, rounds, plan.stark.fri.num_colinearity_tests, "fri_leaf_c")
    want = [True] * 64
    want[17] = False
    assert plan.verify(pks, docs, sigs) == want
    assert host_parses == []
    counts = []
    for _ in range(2):
        before = eng.launch_count()
        assert plan.verify(pks, docs, sigs) == want
        counts.append(eng.launch_count() - before)
    assert counts[0] == counts[1]


def test_adversarial_bytes_refused(eng, host_parses):
    import random
    stark, cons, boundary, root, proof = V.case("tiny", True)
    rng = random.Random(5)
    muts = list(mutations(proof, rng, 6)) + [b"", b"\x80", proof[:2], proof + proof]
    plan = sa_stark.VerifierPlan(stark, cons, root)
    got = plan.verify_batch(muts, [boundary] * len(muts), reasons=True)
    assert all(m in host_parses for m in muts[-4:])  # refused, so read on the host
    assert got == on_host(lambda: sa_stark.VerifierPlan(stark, cons, root).verify_batch(
        muts, [boundary] * len(muts), reasons=True))
    eng.torch.cuda.synchronize()


def test_launches_per_chunk(eng, monkeypatch, host_parses):
    stark, cons, boundary, root, proof = V.case("three_register", True)
    plan = sa_stark.VerifierPlan(stark, cons, root)
    k, rounds = stark.fri.num_colinearity_tests, stark.fri.num_rounds()
    n = sa_stark.DEVICE_ROUTE_MIN_PROOFS
    proofs = [proof, V.tamper(proof, stark.num_registers, rounds, k, "boundary_leaf")] * n
    whole = plan.verify_batch(proofs, [boundary] * len(proofs), reasons=True)
    monkeypatch.setattr(sa_stark, "CHUNK_BYTES", 1)  # one chunk per proof
    counts = []
    for count in (n, 2 * n):
        before = eng.launch_count()
        assert plan.verify_batch(proofs[:count], [boundary] * count, reasons=True) == whole[:count]
        counts.append(eng.launch_count() - before)
    assert counts[1] == 2 * counts[0] and host_parses == []


def test_new_kernels_have_no_spills():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress",
                              "550", "-c", "-Xptxas", "-v", "-o", os.path.join(tmp, "transcript.o"),
                              os.path.join(PKG, "csrc", "transcript.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    reports = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", res.stderr)
    assert len(reports) >= 6 and all(r == ("0", "0") for r in reports), res.stderr[-3000:]
