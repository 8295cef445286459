"""SignerPlan on the device: the two recorded keys and documents signed as one batch give the recorded RPSSS and
FastRPSSS signatures byte for byte; seeded 16-key batches equal the host route (oracle trace, each signature alone
under seeded_urandom), and the test-side verifier accepts every FastRPSSS signature under its own public key and
document; with seeds, no trace element and no randomizer crosses the link.  The stand-in signer takes its constants
from tests/golden/rescue.json and its AIR from the recorded signature case."""
import hashlib
import os
import pickle
import random
from hashlib import blake2s, shake_256

import pytest

import stark_batch_cases as SB
import stark_cases as C
import stark_plain_cases as S
import stark_rescue_cases as SR
import stark_seeded_cases as SS
import stark_verify as V
from test_gpu_air import release

import sa_engine  # noqa: E402
import sa_stark  # noqa: E402

pytestmark = pytest.mark.gpu
G = C.golden()
GP = S.golden()
T = C.T


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


def signers(fast):
    g = G if fast else GP
    first, second = g["rpsss"], g["rpsss_second"]
    return first, second, SR.Signer(first, fast)


@pytest.mark.parametrize("fast", [True, False], ids=["fastrpsss", "rpsss"])
def test_recorded_two_key_batch(eng, fast):
    first, second, signer = signers(fast)
    plan = sa_stark.SignerPlan(signer)
    recs = (first, second)
    draws = C.Urandom(SB.batch_draws([r["draws"] for r in recs], SB.ntrace(first)))
    real = os.urandom
    os.urandom = draws
    try:
        sigs = plan.sign([T.fe(int(r["sk"])) for r in recs], [bytes.fromhex(r["document"]) for r in recs])
    finally:
        os.urandom = real
    assert [hashlib.sha256(s).hexdigest() for s in sigs] == [r["proof_sha256"] for r in recs]
    assert [len(s) for s in sigs] == [r["proof_len"] for r in recs]


def signature_stream(document):
    """a ProofStream class whose verifier Fiat-Shamir carries the document's prefix, as rpsss.py's does"""
    prefix = blake2s(bytes(document)).digest()
    base = sa_stark.sa_host.ip.ProofStream

    class Stream(base):
        def verifier_fiat_shamir(self, num_bytes=32):
            return shake_256(prefix + pickle.dumps(self.objects[:self.read_index])).digest(num_bytes)
    return base, Stream


def verify_signature(signer, pk, document, signature, monkeypatch):
    ip = sa_stark.sa_host.ip
    base, stream = signature_stream(document)
    monkeypatch.setattr(ip, "ProofStream", stream)
    try:
        root = C.O.merkle_root_np(C.O.to_np(signer.zerofier_values))
        return V.verify(signer.stark, signature, signer.rp.air, signer.rp.boundary_constraints(pk), root)
    finally:
        monkeypatch.setattr(ip, "ProofStream", base)


@pytest.mark.parametrize("fast", [True, False], ids=["fastrpsss", "rpsss"])
def test_seeded_16_keys_equal_the_host_route(eng, fast, monkeypatch):
    first, _, signer = signers(fast)
    plan = sa_stark.SignerPlan(signer)
    rng = random.Random(16 + fast)
    sks = [T.fe(rng.randrange(C.P)) for _ in range(16)]
    docs = [("document %d" % d).encode() for d in range(16)]
    seeds = [SS.seed("gpu-rescue", fast, d) for d in range(16)]
    got = SR.seeded_sign(plan, sks, docs, seeds)
    assert len(set(got)) == 16
    assert got == SR.route(signer, sks, docs, seeds)
    if fast:
        for sk, d, sig in zip(sks, docs, got):
            assert verify_signature(signer, signer.rp.hash(sk), d, sig, monkeypatch) is True
        # and not under another key's public key
        assert verify_signature(signer, signer.rp.hash(sks[1]), docs[0], got[0], monkeypatch) is False


@pytest.mark.parametrize("fast", [True, False], ids=["fastrpsss", "rpsss"])
def test_seeded_sign_moves_no_trace_and_no_randomizer(eng, fast, monkeypatch):
    """B = 4: the only upload of more than one element is the keys; what else crosses to the device is single
    elements, the seeds and index lists"""
    _, _, signer = signers(fast)
    plan = sa_stark.SignerPlan(signer)
    B = 4
    sizes, log = [], []
    upload, count = eng.upload, eng._count

    def counting_upload(buf):
        out = upload(buf)
        sizes.append(out.shape[0])
        return out

    def record(kind, nbytes):
        log.append((kind, int(nbytes)))
        count(kind, nbytes)
    monkeypatch.setattr(eng, "upload", counting_upload)
    monkeypatch.setattr(eng, "_count", record)
    got = SR.seeded_sign(plan, [T.fe(v) for v in (3, 5, 7, 11)], [b"a", b"b", b"c", b"d"],
                         [SS.seed("link", b) for b in range(B)])
    monkeypatch.undo()
    assert len(set(got)) == B
    # the keys, then single elements (FRI's scalars): no trace row and no randomizer
    assert sizes[0] == B and max(sizes[1:], default=0) <= 1, sizes
    h2d = [n for kind, n in log if kind == "h2d"]
    assert h2d[0] == 16 * B and 32 * B in h2d, h2d  # the keys, and the seeds
