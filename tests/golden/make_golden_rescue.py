#!/usr/bin/env python3
"""Generate tests/golden/rescue.json by running the UNMODIFIED Python reference's RescuePrime, so that the Rescue
kernel (csrc/rescue.cuh), its CPU emulation and the test-side oracle (tests/emu/rescue_oracle.cpp) can be held to the
reference's hashes and traces without the reference present.

    STARK_REFERENCE=<reference>/code python tests/golden/make_golden_rescue.py   # a few seconds

Contents: the instance's constants (m, N, alpha, alphainv, the MDS matrix row-major, the round constants in order)
and, for each input, its hash and its whole trace (rows 0 .. N of [register 0, register 1]).  The inputs are 0, 1, 2,
p - 2, p - 1, 2^64 - 1, 2^64, 2^119, 2^127; both inputs of the reference's known-answer test
(test_rescue_prime.py:8-9); the secret keys of the four recorded signatures of stark.json and stark_plain.json (each
trace is checked against the one recorded there); and 16 inputs of random.Random(1400).randrange(p).  Field elements
are decimal strings."""
import json
import os
import random
import sys

REF = os.environ["STARK_REFERENCE"]
sys.path.insert(0, REF)
HERE = os.path.dirname(os.path.abspath(__file__))

from algebra import FieldElement  # noqa: E402
from rescue_prime import RescuePrime  # noqa: E402


def main():
    rp = RescuePrime()
    p = rp.field.p
    fixed = [0, 1, 2, p - 2, p - 1, (1 << 64) - 1, 1 << 64, 1 << 119, 1 << 127]
    known = [1, 57322816861100832358702415967512842988]
    keys, recorded = [], {}
    for name in ("stark.json", "stark_plain.json"):
        with open(os.path.join(HERE, name)) as f:
            g = json.load(f)
        for case in ("rpsss", "rpsss_second"):
            sk = int(g[case]["sk"])
            keys.append(sk)
            recorded[sk] = g[case]["trace"]
    rng = random.Random(1400)
    randoms = [rng.randrange(p) for _ in range(16)]

    cases = []
    for kind, values in (("fixed", fixed), ("known_answer", known), ("signature_key", keys), ("random", randoms)):
        for x in values:
            e = FieldElement(x, rp.field)
            trace = [[str(s.value) for s in row] for row in rp.trace(e)]
            if x in recorded:
                assert trace == recorded[x], "the reference's trace differs from the recorded signature's"
            cases.append({"kind": kind, "input": str(x), "hash": str(rp.hash(e).value), "trace": trace})
    assert cases[9]["hash"] == "244180265933090377212304188905974087294"  # test_rescue_prime.py:8
    assert cases[10]["hash"] == "89633745865384635541695204788332415101"  # test_rescue_prime.py:9
    out = {"m": rp.m, "N": rp.N, "alpha": str(rp.alpha), "alphainv": str(rp.alphainv),
           "mds": [str(v.value) for row in rp.MDS for v in row],
           "round_constants": [str(v.value) for v in rp.round_constants], "random_seed": 1400, "cases": cases}
    with open(os.path.join(HERE, "rescue.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
