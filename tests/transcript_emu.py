"""The device route's chunk (sa_stark.VerifierPlan._transcript_chunk) run through tests/emu/emu_transcript.cpp, the
CPU emulation of sa_transcript_sections, shared by the transcript tests."""
import ctypes

import __graft_entry__ as G
import sa_host
import sa_stark

_vp = ctypes.c_void_p


def lib():
    lib = ctypes.CDLL(G.build_emu_transcript())
    lib.emu_transcript_bytes.restype = ctypes.c_size_t
    lib.emu_transcript_sections.restype = ctypes.c_int
    return lib


def _u64(xs):
    return (ctypes.c_uint64 * len(xs))(*xs)


class Aligned:
    """a zeroed host buffer whose address is 16-byte aligned, as the device's allocations are (fe is alignas(16))"""

    def __init__(self, n, data=b""):
        self.buf = ctypes.create_string_buffer(n + 16)
        self.addr = (ctypes.addressof(self.buf) + 15) & ~15
        self.n = n
        ctypes.memmove(self.addr, data, len(data))

    @property
    def raw(self):
        return ctypes.string_at(self.addr, self.n)


def run(lib, plan, items):
    """(sections, out, workspace, L) of one chunk of (proof, prefix, statement or None) items"""
    raw, parts, L, nstat = plan._transcript_chunk(items)
    shape = _u64(plan._transcript_shape())
    B = len(items)
    wsb = lib.emu_transcript_bytes(shape)
    assert wsb > 0
    sec = Aligned(max(L["bytes"], 16))
    out = Aligned(sa_stark.TRANSCRIPT_OUT * B)
    ws = Aligned(wsb * B)
    buf = Aligned(len(raw), raw)
    base = buf.addr
    zroot = base + parts["zroot"] if plan.zerofier_root is not None else None
    assert lib.emu_transcript_sections(_vp(sec.addr), _u64([L[n] for n in sa_stark.SECTIONS]), _vp(out.addr),
                                       _vp(ws.addr), _vp(base + parts["proofs"]),
                                       _vp(base + parts["proof_at"]), _vp(base + parts["prefixes"]),
                                       _vp(base + parts["statement"]), ctypes.c_size_t(nstat), _vp(zroot),
                                       ctypes.c_size_t(B), shape) == 0
    return sec.raw[:L["bytes"]], out.raw, ws, L


def accepted(out, j):
    return out[sa_stark.TRANSCRIPT_OUT * j] == 1


def draws(lib, plan, ws, j):
    """(Fiat-Shamir digests, weights, alphas, indices) the emulation drew for proof j"""
    shape = _u64(plan._transcript_shape())
    nfs, W = plan.rounds + 2, plan._transcript_shape()[6]
    fsd, w, a = (ctypes.create_string_buffer(n) for n in (32 * nfs, 16 * W, 16 * plan.rounds))
    top = (ctypes.c_uint64 * plan.k)()
    lib.emu_transcript_draws(fsd, w, a, top, _vp(ws.addr), ctypes.c_size_t(j), shape)
    fe = lambda raw: [int.from_bytes(raw[16 * i:16 * (i + 1)], "little") for i in range(len(raw) // 16)]  # noqa
    return [fsd.raw[32 * m:32 * (m + 1)] for m in range(nfs)], fe(w.raw), fe(a.raw), list(top)


def zero_zerofier_proof(stark, cons, boundary, root, proof):
    """(a zerofier root, a copy of the FastStark proof whose opened zerofier leaves are zero): the root of the all-zero
    codeword, whose leaves and paths replace the proof's zerofier openings.  Fiat-Shamir does not see the openings, so
    every other check passes, and a plan with that root meets a zero zerofier value at the first combination index"""
    import pickle
    plan = sa_stark.VerifierPlan(stark, cons, root)
    pr = plan._parse(proof, boundary, None)
    objs = pickle.loads(proof)
    zero = sa_host.algebra.FieldElement(0, objs[plan.nregs + 1 + plan.rounds][0].field)  # the stream's one Field
    codeword = [zero] * plan.n
    merkle = sa_host.merkle.Merkle
    at = plan.nregs + 1 + plan.rounds + 1 + (plan.rounds - 1) * 4 * plan.k + (plan.nregs + 1) * 8 * plan.k
    for q, (i, _, _) in enumerate(pr.opened[plan.nregs + 1][1]):
        objs[at + 2 * q] = zero
        objs[at + 2 * q + 1] = merkle.open(i, codeword)
    return merkle.commit(codeword), pickle.dumps(objs)


def recorded_signatures(fast):
    """(the two recorded signature records, their Signer, the signatures regenerated from the recorded draws)"""
    import os
    import stark_batch_cases as SB
    import stark_cases as C
    import stark_plain_cases as S
    import stark_rescue_cases as SR
    g = C.golden() if fast else S.golden()
    recs = (g["rpsss"], g["rpsss_second"])
    signer = SR.Signer(recs[0], fast)
    plan = sa_stark.SignerPlan(signer)
    draws = C.Urandom(SB.batch_draws([r["draws"] for r in recs], SB.ntrace(recs[0])))
    real = os.urandom
    os.urandom = draws
    try:
        sigs = plan.sign([C.T.fe(int(r["sk"])) for r in recs], [bytes.fromhex(r["document"]) for r in recs])
    finally:
        os.urandom = real
    import hashlib
    assert [hashlib.sha256(s).hexdigest() for s in sigs] == [r["proof_sha256"] for r in recs]
    return recs, signer, sigs
