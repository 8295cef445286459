"""Cases of the batched verifier tests, shared by the CPU suite (tests/test_verify_cpu.py) and the GPU suite
(tests/test_gpu_verify.py): a test double whose verify_chunk restates every device check of one chunk in Python ints
and hashlib from the packed buffer, a signature stream with the reference's verifier side, and tampered copies of a
proof."""
import hashlib
import json
import os
import pickle

import numpy as np

import oracle as O
import sa_stark
import stark_cases as C
import stark_plain_cases as S
import stark_rescue_cases as SR
import verify_tamper as T_

P = O.P
HERE = os.path.dirname(os.path.abspath(__file__))


def _fe(raw, at, count):
    a = np.frombuffer(raw, dtype="<u8", count=2 * count, offset=at).reshape(-1, 2)
    return [int(lo) | int(hi) << 64 for lo, hi in a]


def _ints(raw, at, count, dtype):
    return [int(v) for v in np.frombuffer(raw, dtype=dtype, count=count, offset=at)]


def colinear(x0, y0, x1, y1, x2, y2):
    """test_colinearity's Lagrange interpolant in ints, inverse(0) = 0: True when its degree is 1"""
    inv = lambda v: pow(v % P, P - 2, P)  # noqa: E731
    c0 = y0 * inv(x0 - x1) * inv(x0 - x2) % P
    c1 = y1 * inv(x1 - x0) * inv(x1 - x2) % P
    c2 = y2 * inv(x2 - x0) * inv(x2 - x1) % P
    quad = (c0 + c1 + c2) % P
    lin = (c0 * (x1 + x2) + c1 * (x0 + x2) + c2 * (x0 + x1)) % P
    return quad == 0 and lin != 0


def merkle_ok(root, index, path, value):
    h = hashlib.blake2b(str(value).encode()).digest()
    for sib in path:
        h = hashlib.blake2b(sib + h if index & 1 else h + sib).digest()
        index >>= 1
    return index == 0 and h == root


def air_value(terms, point):
    acc = 0
    for k, v in terms:
        t = v
        for x, e in zip(point, k):
            t = t * pow(x, e, P) % P
        acc += t
    return acc % P


def horner(coef, x):
    acc = 0
    for c in reversed(coef):
        acc = (acc * x + c) % P
    return acc


class VerifyEngine(SR.RescueStarkEngine):
    """the Rescue / seeded / batched double plus the verifier's calls, each restated from its definition"""
    name = "oracle-test-double-verify"

    def air_program(self, constraints, nregs):
        self._log("air_program", len(constraints), nregs)
        return [[(tuple(int(e) for e in k), int(getattr(v, "value", v)) % P)
                 for k, v in getattr(a, "dictionary", a).items()] for a in constraints]

    def upload_bytes(self, buf):
        self._log("upload_bytes", len(buf))
        return bytes(buf)

    def verify_chunk(self, raw, L):
        self._log("verify_chunk", L["proofs"])
        npath, ncol, B, k, m, nregs, ncons = (L[x] for x in ("paths", "colinear", "proofs", "k", "last_len", "nregs",
                                                              "ncons"))
        idx = _ints(raw, L["leaf_index"], npath, "<u8")
        depth = _ints(raw, L["depth"], npath, "<u4")
        poff = _ints(raw, L["path_offset"], npath, "<u8")
        leaves = _fe(raw, L["leaves"], npath)
        mflags = []
        for i in range(npath):
            root = raw[L["roots"] + 64 * i:L["roots"] + 64 * (i + 1)]
            path = [raw[L["digests"] + 64 * (poff[i] + l):L["digests"] + 64 * (poff[i] + l + 1)]
                    for l in range(depth[i])]
            mflags.append(0 if merkle_ok(root, idx[i], path, leaves[i]) else 1)
        ay, by, cy, alpha = (_fe(raw, L[x], ncol) for x in ("ay", "by", "cy", "alpha"))
        aidx, rnd = _ints(raw, L["a_index"], ncol, "<u8"), _ints(raw, L["round"], ncol, "<u4")
        cflags = []
        for i in range(ncol):
            e = 1 << rnd[i]
            ax = pow(L["fri_offset"], e, P) * pow(L["fri_omega"], e * aidx[i], P) % P
            cflags.append(0 if colinear(ax, ay[i], P - ax, by[i], alpha[i], cy[i]) else 1)
        R = 4 + 2 * nregs
        W = 1 + 2 * ncons + 2 * nregs
        Q = W + ncons + nregs + 2 * nregs * L["blen"]
        items = _fe(raw, L["items"], B * k * R)
        pdata = _fe(raw, L["proof_data"], B * Q)
        zcoef = None if L["zcoef"] is None else O.from_np(np.asarray(L["zcoef"]))
        n, blen = 1 << L["log_n"], L["blen"]
        kflags = []
        for j in range(B * k):
            it, pr = items[j * R:(j + 1) * R], pdata[(j // k) * Q:(j // k + 1) * Q]
            w, shifts, bc = pr[:W], pr[W:W + ncons + nregs], pr[W + ncons + nregs:]
            i = it[0]
            x = L["offset"] * pow(L["omega"], i % n, P) % P
            xn = L["offset"] * pow(L["omega"], (i + L["ef"]) % n, P) % P
            cur, nxt = [], []
            acc = w[0] * it[2 + 2 * nregs]
            for s in range(nregs):
                z, ip = bc[2 * s * blen:(2 * s + 1) * blen], bc[(2 * s + 1) * blen:(2 * s + 2) * blen]
                cur.append((it[2 + s] * horner(z, x) + horner(ip, x)) % P)
                nxt.append((it[2 + nregs + s] * horner(z, xn) + horner(ip, xn)) % P)
                acc += it[2 + s] * (w[W - 2 * nregs + 2 * s] + w[W - 2 * nregs + 2 * s + 1] *
                                    pow(x, shifts[ncons + s], P))
            zval = it[3 + 2 * nregs] if zcoef is None else horner(zcoef, x)
            if zval == 0:
                kflags.append(2)
                continue
            zinv = pow(zval, P - 2, P)
            for c, terms in enumerate(L["prog"]):
                q = air_value(terms, [x] + cur + nxt) * zinv % P
                acc += q * (w[1 + 2 * c] + w[2 + 2 * c] * pow(x, shifts[c], P))
            kflags.append(0 if acc % P == it[1] else 1)
        last = _fe(raw, L["last"], B * m)
        degrees, roots = [], b""
        for b in range(B):
            row = last[b * m:(b + 1) * m]
            coeffs = O.from_np(O.intt_np(L["last_omega"], O.to_np(row)))
            degrees.append(max([j for j, v in enumerate(coeffs) if v], default=-1))
            roots += O.merkle_tree_np(O.to_np(row))[1].tobytes()
        u32 = lambda v: np.array(v, dtype=np.uint32)  # noqa: E731
        return u32(mflags), u32(cflags), u32(kflags), np.array(degrees, dtype=np.int64), roots


class SignatureProofStream(C.SignatureProofStream):
    """the fixture's signature stream with the reference's verifier side too (rpsss.py:16-22): the document's blake2s
    prefix in verifier_fiat_shamir, and deserialize keeping the document"""

    def verifier_fiat_shamir(self, num_bytes=32):
        return hashlib.shake_256(self.prefix + pickle.dumps(self.objects[:self.read_index])).digest(num_bytes)

    def deserialize(self, bb):
        sps = SignatureProofStream(self.document)
        sps.objects = pickle.loads(bb)
        return sps


FAST = ["tiny", "faststark", "three_register", "broken_witness"]  # the cases verify.json records
PLAIN = ["tiny", "stark", "three_register"]


# ---- tampered copies of a proof (tests/verify_tamper.py) and the reference's verdicts on them ----
tamper = T_.tamper
kinds = T_.kinds


def golden():
    with open(os.path.join(HERE, "golden", "verify.json")) as f:
        return json.load(f)


def case(name, fast):
    """(stark, constraints, boundary, zerofier root or None, proof) of a stark.json / stark_plain.json case, the proof
    proven again through the current engine from the recorded draws"""
    if fast:
        rec = C.golden()[name]
        stark = C.params(rec)
        proof = C.run_case(rec, stark=stark)[0]
        root = bytes.fromhex(rec["zerofier_root"])
    else:
        rec = S.golden()[name]
        stark = S.stark(rec)
        proof = S.run_case(rec, st=stark)[0]
        root = None
    assert hashlib.sha256(proof).hexdigest() == rec["proof_sha256"]
    return stark, C.air(rec), C.inputs(rec)[1], root, proof


def recorded(name, fast):
    """the reference's records of one case, in verify.json's order (the proof itself first)"""
    return [r for r in golden()["records"] if r["case"] == name and r["verifier"] == ("fast" if fast else "plain")]


def check_recorded(name, fast):
    """every recorded proof of the case in one verify_batch call: the reference's verdict and printed message, or
    "malformed" where the reference raised on a stream outside the shape; then each one under enable_verify, whose
    printed text is the reference's and which hands the malformed stream to the original method"""
    import contextlib
    import io
    stark, cons, boundary, root, proof = case(name, fast)
    recs = recorded(name, fast)
    k, rounds = stark.fri.num_colinearity_tests, stark.fri.num_rounds()
    proofs = [proof if r["kind"] == "none" else tamper(proof, stark.num_registers, rounds, k, r["kind"])
              for r in recs]
    assert [hashlib.sha256(p).hexdigest() for p in proofs] == [r["sha256"] for r in recs]
    got = sa_stark.VerifierPlan(stark, cons, root).verify_batch(proofs, [boundary] * len(proofs), reasons=True)
    for r, (verdict, reason) in zip(recs, got):
        if r["raises"] is not None:
            assert (verdict, reason) == (False, sa_stark.MALFORMED), r["kind"]
        elif r["verdict"]:
            assert (verdict, reason) == (True, None), r["kind"]
        elif r["printed"]:
            assert (verdict, reason) == (False, r["printed"].rstrip("\n")), r["kind"]
        else:
            assert verdict is False and reason in ("leaf path", "combination"), (r["kind"], reason)

    class Original(type(stark)):
        def verify(self, *args):
            raise AssertionError("ProofStream: cannot pull object; queue empty.")
    stark.__class__ = Original
    (sa_stark.enable_verify if fast else sa_stark.enable_verify_plain)(Original)
    try:
        for r, p in zip(recs, proofs):
            out = io.StringIO()
            args = (p, cons, boundary, root) if fast else (p, cons, boundary)
            with contextlib.redirect_stdout(out):
                try:
                    result = stark.verify(*args)
                except AssertionError as e:
                    result = ["AssertionError", str(e)]
            assert out.getvalue() == r["printed"], r["kind"]
            assert result == (r["verdict"] if r["raises"] is None else r["raises"]), r["kind"]
    finally:
        sa_stark.disable()
        stark.__class__ = Original.__mro__[1]
    return len(recs)
