"""Cases of the device Rescue and SignerPlan tests, shared by the CPU suite (tests/test_stark_rescue_cpu.py) and the
GPU suite (tests/test_gpu_stark_rescue.py): the seeded test double of tests/stark_seeded_cases.py plus ``rescue`` on
the CPU emulation of csrc/rescue.cuh, a stand-in RescuePrime whose constants come from tests/golden/rescue.json and
whose hash and trace come from the independent oracle, and a stand-in signer over a recorded signature case."""
import numpy as np

import rescue_cases as R
import stark_cases as C
import stark_plain_cases as S
import stark_seeded_cases as SS
import sa_stark
from sa_engine import SA_ERRORS, SaError

T = C.T


class RescueStarkEngine(SS.SeededStarkEngine):
    name = "oracle-test-double-stark-rescue"
    RESCUE_MAX_ROUNDS = R.MAX_ROUNDS

    def rescue(self, inputs, constants, rounds, alpha, alphainv, hashes=None, trace=None, inst_stride=None,
               lane_stride=None):
        """CudaEngine.rescue's checks, then the emulated kernel over a grid of 37 threads"""
        lane_stride = rounds + 1 if lane_stride is None else lane_stride
        inst_stride = 2 * lane_stride if inst_stride is None else inst_stride
        self._log("rescue", inputs.shape[0], rounds, hashes is not None, trace is not None)
        vecs = [v for v in (inputs, constants, hashes, trace) if v is not None]
        if (any(v.dtype != np.uint64 or v.shape[-1] != 2 or not v.flags.c_contiguous for v in vecs)
                or (hashes is None and trace is None) or not 1 <= rounds <= R.MAX_ROUNDS
                or not all(0 <= int(e) < 1 << 128 for e in (alpha, alphainv)) or min(inst_stride, lane_stride) < 0
                or constants.size // 2 < 4 + 4 * rounds):
            raise SaError(SA_ERRORS[-6])
        count = inputs.size // 2
        if hashes is not None and hashes.size // 2 < count:
            raise SaError(SA_ERRORS[-6])
        if trace is not None and count and (count - 1) * inst_stride + lane_stride + rounds >= trace.size // 2:
            raise SaError(SA_ERRORS[-6])
        if count == 0:
            return hashes, trace
        rc = R.emu(hashes, trace, inputs.reshape(-1, 2), constants, rounds, alpha, alphainv, inst_stride,
                   lane_stride, 37)
        if rc:
            raise SaError(SA_ERRORS[rc])
        return hashes, trace


def uploads(eng, since):
    """the element counts of the double's uploads after call `since`"""
    return [c[1] for c in eng.calls[since:] if c[0] == "upload"]


class RescuePrime:
    """a RescuePrime of the fixture's constants over the drop-in's field: hash and trace from the oracle"""
    m = 2

    def __init__(self, air=None):
        g = R.golden()
        self.field = T.field
        self.N = g["N"]
        self.alpha, self.alphainv = R.exponents(g)
        mds = [T.fe(int(v)) for v in g["mds"]]
        self.MDS = [mds[:2], mds[2:]]
        self.round_constants = [T.fe(int(v)) for v in g["round_constants"]]
        self.air = air

    def _run(self, x):
        h, t = R.oracle(R.to_np([x.value]), R.to_np(R.constants()), self.N, self.alpha, self.alphainv)
        return T.fe(R.from_np(h)[0]), [[T.fe(v) for v in row] for row in R.dense_trace(t)[0]]

    def hash(self, x):
        return self._run(x)[0]

    def trace(self, x):
        return self._run(x)[1]

    def boundary_constraints(self, output):
        return [(0, 1, self.field.zero()), (self.N, 0, output)]

    def transition_constraints(self, omicron):
        return self.air


class Signer:
    """a stand-in for RPSSS / FastRPSSS: the fixture case's Params (or its plain-Stark restatement) and AIR, and the
    RescuePrime above; sign(sk, d) is the unmodified signing route (host hash and trace, then prove or prove_plain).
    Its module is stark_cases, whose SignatureProofStream SignerPlan and sign_batch pick up."""
    __module__ = C.__name__

    def __init__(self, rec, fast):
        self.stark = C.params(rec) if fast else S.stark(rec)
        self.rp = RescuePrime(C.air(rec))
        if fast:
            zpoly, zvals = C.zerofier(self.stark)
            self.transition_zerofier = zpoly
            self.transition_zerofier_codeword = C.zerofier_codeword(zvals, True)
            self.zerofier_values = zvals

    def sign(self, sk, document):
        ps = C.SignatureProofStream(document)
        rp = self.rp
        trace, boundary = rp.trace(sk), rp.boundary_constraints(rp.hash(sk))
        air = rp.transition_constraints(self.stark.omicron)
        if hasattr(self, "transition_zerofier"):
            return sa_stark.prove(self.stark, trace, air, boundary, self.transition_zerofier,
                                  self.transition_zerofier_codeword, ps)
        return sa_stark.prove_plain(self.stark, trace, air, boundary, ps)


def route(signer, sks, documents, seeds):
    """the host route: each signature alone with os.urandom = seeded_urandom(its seed)"""
    real = SS.os.urandom
    try:
        out = []
        for sk, d, s in zip(sks, documents, seeds):
            SS.os.urandom = sa_stark.seeded_urandom(s)
            out.append(signer.sign(sk, d))
        return out
    finally:
        SS.os.urandom = real


def seeded_sign(plan, sks, documents, seeds):
    """plan.sign with seeds and os.urandom refused"""
    real = SS.os.urandom
    SS.os.urandom = SS.refuse_urandom
    try:
        return plan.sign(sks, documents, seeds)
    finally:
        SS.os.urandom = real
