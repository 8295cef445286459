#!/usr/bin/env python3
"""Generate tests/golden/verify.json by running the UNMODIFIED Python reference's verifiers: FastStark.verify and
Stark.verify on the proofs of the small stark.json / stark_plain.json cases (proven again by the reference from their
recorded draws) and on one tampered copy of each kind (tests/verify_tamper.py), so that sa_stark.VerifierPlan
(tests/test_verify_cpu.py, tests/test_gpu_verify.py) can be held to the reference's verdicts and printed messages
without the reference present.

    STARK_REFERENCE=<reference>/code python tests/golden/make_golden_verify.py   # ~1 minute

Each record names the case, the verifier ("fast" or "plain") and the tamper kind ("none" for the proof itself), and
holds the SHA-256 of the verified bytes, the reference's verdict (true / false, or null when it raised), the text it
printed, and the exception's type and message when it raised.  The RPSSS / FastRPSSS signatures are not recorded: the
reference's verify takes several minutes per signature there.
"""
import contextlib
import hashlib
import io
import json
import os
import pickle
import sys

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden import P, dump, fe, field  # noqa: E402

import fast_stark as fs  # noqa: E402
import stark as st  # noqa: E402
from multivariate import MPolynomial  # noqa: E402
import verify_tamper  # noqa: E402

FAST = ["tiny", "faststark", "three_register", "broken_witness"]
PLAIN = ["tiny", "stark", "three_register"]


class Replay:
    def __init__(self, values):
        self.values, self.count = [int(v) for v in values], 0

    def __call__(self, n):
        assert n == 17
        v = self.values[self.count]
        self.count += 1
        return v.to_bytes(17, "big")


def case(rec, fast):
    p = rec["params"]
    cls = fs.FastStark if fast else st.Stark
    stark = cls(field, p["expansion_factor"], p["num_colinearity_checks"], p["security_level"], p["num_registers"],
                p["num_cycles"], transition_constraints_degree=p["transition_constraints_degree"])
    air = [MPolynomial({tuple(t["e"]): fe(int(t["c"])) for t in cons}) for cons in rec["air"]]
    trace = [[fe(int(v)) for v in row] for row in rec["trace"]]
    boundary = [(int(c), int(r), fe(int(v))) for c, r, v in rec["boundary"]]
    real = os.urandom
    os.urandom = Replay(rec["draws"])
    try:
        if fast:
            tz, tzc, tzr = stark.preprocess()
            assert tzr.hex() == rec["zerofier_root"]
            proof = stark.prove(trace, air, boundary, tz, tzc)
        else:
            tzr = None
            proof = stark.prove(trace, air, boundary)
    finally:
        os.urandom = real
    assert hashlib.sha256(proof).hexdigest() == rec["proof_sha256"], "the reference's proof is not the recorded one"
    return stark, air, boundary, proof, tzr


def verdict(stark, air, boundary, proof, tzr):
    out = io.StringIO()
    rec = {"verdict": None, "printed": "", "raises": None}
    try:
        with contextlib.redirect_stdout(out):
            v = stark.verify(proof, air, boundary, tzr) if tzr is not None else stark.verify(proof, air, boundary)
        rec["verdict"] = bool(v)
    except Exception as e:  # noqa: BLE001 -- the reference's exception is what is recorded
        rec["raises"] = [type(e).__name__, str(e)]
    rec["printed"] = out.getvalue()
    return rec


def main():
    records = []
    for fast, names, fixture in ((True, FAST, "stark.json"), (False, PLAIN, "stark_plain.json")):
        with open(os.path.join(HERE, fixture)) as f:
            g = json.load(f)
        for name in names:
            rec = g[name]
            stark, air, boundary, proof, tzr = case(rec, fast)
            k, rounds = stark.fri.num_colinearity_tests, stark.fri.num_rounds()
            for kind in ["none"] + verify_tamper.kinds(fast):
                data = proof if kind == "none" else verify_tamper.tamper(proof, stark.num_registers, rounds, k, kind)
                r = {"case": name, "verifier": "fast" if fast else "plain", "kind": kind,
                     "sha256": hashlib.sha256(data).hexdigest()}
                r.update(verdict(stark, air, boundary, data, tzr))
                records.append(r)
                print(name, r["verifier"], kind, r["verdict"], repr(r["printed"]), r["raises"])
    assert P == field.p
    dump("verify.json", {"records": records})


if __name__ == "__main__":
    main()
