"""The transcript reader (csrc/transcript.cuh) on the CPU through tests/emu/emu_transcript.cpp: SHAKE-256, blake2b
over seed || zero bytes and the reductions mod p against hashlib and Python ints; the fixture proofs and every
tampered copy read from their bytes with the digests of the stream's verifier_fiat_shamir, _parse's draws and
_pack's sections byte for byte; re-encodings pickle.loads still reads refused; and a seeded byte-level fuzz in which
every mutation is refused or read exactly as the host route reads it."""
import ctypes
import hashlib
import pickle
import pickletools
import random

import pytest

import stark_cases as C  # noqa: F401  puts the drop-in on sys.path
import verify_cases as V
import sa_engine
import sa_host
import sa_stark
import transcript_emu as TE

P = V.P


@pytest.fixture(autouse=True)
def double_engine():
    prev = sa_engine._ENGINE
    sa_engine.set_engine(V.VerifyEngine())
    yield
    sa_engine.set_engine(prev)


@pytest.fixture(scope="module")
def lib():
    return TE.lib()


def test_shake256(lib):
    rng = random.Random(3)
    out = ctypes.create_string_buffer(32)
    lengths = list(range(601)) + [136 * m + d for m in range(1, 12) for d in (-2, -1, 0, 1, 2)]
    for n in lengths:
        msg = rng.randbytes(n)
        lib.emu_shake256(out, msg, ctypes.c_size_t(n))
        assert out.raw == hashlib.shake_256(msg).digest(32), n


def test_blake2b_of_seed_and_zeros(lib):
    rng = random.Random(4)
    out = ctypes.create_string_buffer(64)
    for zeros in list(range(0, 300)) + [479, 480, 481, 1000]:
        seed = rng.randbytes(32)
        lib.emu_blake2b_zeros(out, seed, ctypes.c_uint64(zeros))
        assert out.raw == hashlib.blake2b(seed + bytes(zeros)).digest(), zeros


def test_reductions(lib):
    out = ctypes.create_string_buffer(16)
    values = [0, 1, 2 ** 256 - 1, 2 ** 512 - 1, 2 ** 128 - 1, 2 ** 128] + \
        [m * P + d for m in (1, 2, 3, 2 ** 100, 2 ** 127) for d in (-1, 0, 1)] + \
        [m * P + d for m in (2 ** 128, 2 ** 383) for d in (-1, 0, 1)]
    for v in values:
        for nbytes in (32, 64):
            if v < 1 << (8 * nbytes):
                lib.emu_reduce_be(out, v.to_bytes(nbytes, "big"), nbytes)
                assert int.from_bytes(out.raw, "little") == v % P, (v, nbytes)


def cases():
    return [(n, True) for n in V.FAST] + [(n, False) for n in V.PLAIN]


def host_fs(proof, plan, stream=None):
    """the stream's own verifier_fiat_shamir at each of the plan's Fiat-Shamir points"""
    ps = (stream if stream is not None else sa_host.ip.ProofStream()).deserialize(proof)
    js = [plan.nregs + 1 + m for m in range(plan.rounds + 1)] + [plan.nregs + plan.rounds + 2]
    out = []
    for j in js:
        ps.read_index = j
        out.append(ps.verifier_fiat_shamir())
    return out


def check_same(lib, plan, proofs, boundary, stream=None):
    """each proof is refused, or read exactly as _parse and _pack read it: its Fiat-Shamir digests, draws and last
    root, and its sections alone byte for byte _pack's of its _parse; the whole batch's sections too when every
    proof is accepted.  Returns the accepted flags"""
    prefix = sa_stark.VerifierPlan._fs_prefix(stream)
    assert prefix is not None
    parsed = [plan._parse(p, boundary, stream) for p in proofs]
    st = plan._statement(boundary)
    sec, out, ws, L = TE.run(lib, plan, [(p, prefix, st) for p in proofs])
    flags = [TE.accepted(out, j) for j in range(len(proofs))]
    for j, pr in enumerate(parsed):
        if flags[j]:
            assert pr is not None, j
            fsd, weights, alphas, top = TE.draws(lib, plan, ws, j)
            assert fsd == host_fs(proofs[j], plan, stream)
            assert (weights, alphas, top) == (pr.weights, pr.alphas, pr.top_indices)
            assert out[80 * j + 16:80 * j + 80] == pr.fri_roots[-1]
            alone, out1, _, _ = TE.run(lib, plan, [(proofs[j], prefix, st)])
            assert TE.accepted(out1, 0) and alone == plan._pack([pr])[0], j
    if all(flags):
        raw, L2 = plan._pack(parsed)
        assert sec == raw
    return flags


@pytest.mark.parametrize("name,fast", cases())
def test_fixtures_and_tampered_copies(lib, name, fast):
    stark, cons, boundary, root, proof = V.case(name, fast)
    plan = sa_stark.VerifierPlan(stark, cons, root)
    k, rounds = stark.fri.num_colinearity_tests, stark.fri.num_rounds()
    kinds = [t for t in V.kinds(fast) if t != "truncated"]
    proofs = [proof] + [V.tamper(proof, stark.num_registers, rounds, k, t) for t in kinds]
    assert check_same(lib, plan, proofs, boundary) == [True] * len(proofs)
    truncated = V.tamper(proof, stark.num_registers, rounds, k, "truncated")
    assert check_same(lib, plan, [truncated], boundary) == [False]


def reencodings(proof):
    """copies pickle.loads reads as the same objects that are not what the pickler writes at the running protocol"""
    objs = pickle.loads(proof)
    other = 5 if pickle.DEFAULT_PROTOCOL != 5 else 4
    out = {"protocol 2": pickle.dumps(objs, protocol=2), "protocol %d" % other: pickle.dumps(objs, protocol=other),
           "optimized": pickletools.optimize(proof)}
    ops = list(pickletools.genops(proof))
    for op, arg, pos in ops:
        if op.name == "LONG1":
            n = proof[pos + 1]
            out["long1 padded"] = proof[:pos + 1] + bytes([n + 1]) + proof[pos + 2:pos + 2 + n] + b"\0" + \
                proof[pos + 2 + n:]
            break
    out["foreign module"] = proof.replace(b"\x8c\x07algebra", b"\x8c\x07algebrb", 1)
    return out


def test_reencodings_refused(lib):
    stark, cons, boundary, root, proof = V.case("tiny", True)
    plan = sa_stark.VerifierPlan(stark, cons, root)
    for what, p in reencodings(proof).items():
        assert check_same(lib, plan, [p], boundary) == [False], what
    # a small value written as BININT: an element of the last codeword set to 5, then its encoding widened
    objs = pickle.loads(proof)
    objs[plan.nregs + 1 + plan.rounds][1].value = 5
    p = pickle.dumps(objs)
    at = p.index(b"\x4b\x05")
    widened = p[:at] + b"\x4a\x05\x00\x00\x00" + p[at + 2:]
    assert check_same(lib, plan, [p], boundary) == [True]
    assert check_same(lib, plan, [widened], boundary) == [False]


def mutations(proof, rng, count):
    ops = list(pickletools.genops(proof))
    frames = [pos for op, _, pos in ops if op.name == "FRAME"]
    gets = [pos for op, _, pos in ops if op.name in ("BINGET", "LONG_BINGET")]
    for i in range(count):
        kind = i % 6
        b = bytearray(proof)
        if kind == 0:
            at = rng.randrange(len(b))
            b[at] ^= 1 << rng.randrange(8)
        elif kind == 1:
            del b[rng.randrange(len(b)):]
        elif kind == 2:
            at = rng.choice(frames)
            n = int.from_bytes(b[at + 1:at + 9], "little") + rng.choice((-1, 1))
            b[at + 1:at + 9] = n.to_bytes(8, "little")
        elif kind == 3:
            at = rng.choice(gets)
            b[at + 1] = (b[at + 1] + rng.choice((-2, -1, 1, 2))) % 256
        elif kind == 4:
            b += rng.randbytes(rng.randrange(1, 5))
        else:
            at = rng.randrange(len(b))
            b[at] = rng.randrange(256)
        yield bytes(b)


@pytest.mark.parametrize("name,fast", [("tiny", True), ("tiny", False)])
def test_fuzz_refused_or_exact(lib, name, fast):
    stark, cons, boundary, root, proof = V.case(name, fast)
    plan = sa_stark.VerifierPlan(stark, cons, root)
    rng = random.Random(11 + fast)
    muts = list(mutations(proof, rng, 1500))
    accepted = 0
    for at in range(0, len(muts), 100):
        flags = check_same(lib, plan, muts[at:at + 100], boundary)
        accepted += sum(flags)
    assert 0 < accepted < len(muts)


@pytest.mark.parametrize("fast", [True, False], ids=["fastrpsss", "rpsss"])
def test_recorded_signatures_with_their_document_prefix(lib, fast):
    recs, signer, sigs = TE.recorded_signatures(fast)
    rp = signer.rp
    plan = sa_stark.VerifierPlan(signer.stark, rp.transition_constraints(signer.stark.omicron),
                                 bytes.fromhex(recs[0]["zerofier_root"]) if fast else None)
    for rec, sig in zip(recs, sigs):
        doc = bytes.fromhex(rec["document"])
        stream = V.SignatureProofStream(doc)
        assert sa_stark.VerifierPlan._fs_prefix(stream) == hashlib.blake2s(doc).digest()
        assert len([op for op, _, _ in pickletools.genops(sig) if op.name == "FRAME"]) > 1
        boundary = rp.boundary_constraints(rp.hash(C.T.fe(int(rec["sk"]))))
        assert check_same(lib, plan, [sig], boundary, stream) == [True]
        # under another document's prefix the digests differ, and stay the stream's own
        other = V.SignatureProofStream(doc + b"!")
        assert check_same(lib, plan, [sig], boundary, other) == [True]


def test_zero_zerofier_proof_is_read_and_divides_by_zero(lib):
    stark, cons, boundary, root, proof = V.case("tiny", True)
    zroot, dz = TE.zero_zerofier_proof(stark, cons, boundary, root, proof)
    plan = sa_stark.VerifierPlan(stark, cons, zroot)
    assert check_same(lib, plan, [dz, proof], boundary) == [True, True]
    with pytest.raises(AssertionError, match="divide by zero") as exc:
        plan.verify_batch([proof, dz, dz], [boundary] * 3)
    assert exc.value.proof_index == 1
