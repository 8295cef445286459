#!/usr/bin/env python3
"""Generate tests/golden/stark_plain.json by running the UNMODIFIED Python reference's plain prover: whole
Stark.prove runs (and RPSSS signatures) with os.urandom replaced by a seeded stream, so that sa_stark's plain prover
(tests/test_stark_plain_cpu.py, tests/test_gpu_stark_plain.py) can be held to the reference's proof bytes without the
reference present.

Needs a checkout of the reference, named as for make_golden.py (whose helpers it uses):

    STARK_REFERENCE=<reference>/code python tests/golden/make_golden_stark_plain.py   # ~6 minutes (two signatures)

The record format is make_golden_stark.py's, with the derived parameters Stark does not keep as attributes computed
from what it does keep, and prefix digests over the nregs + 1 committed codewords (the plain proof opens no
zerofier): after the boundary roots, after the randomizer root, after FRI and after each opening block.
"""
import hashlib
import os
import pickle
import random
import sys

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import P, Fri, dump, fe, field  # noqa: E402
from make_golden_stark import Draws, enc_air, three_register_air, three_register_trace  # noqa: E402

import stark as st  # noqa: E402
from multivariate import MPolynomial  # noqa: E402


def params(stark, ncycles, tcd, air, boundary, trace_len):
    return {"expansion_factor": stark.expansion_factor, "num_colinearity_checks": stark.num_colinearity_checks,
            "security_level": stark.security_level, "num_registers": stark.num_registers, "num_cycles": ncycles,
            "transition_constraints_degree": tcd, "num_randomizers": stark.num_randomizers,
            "omicron_domain_length": len(stark.omicron_domain), "fri_domain_length": stark.fri.domain_length,
            "generator": str(stark.generator.value), "omega": str(stark.omega.value),
            "omicron": str(stark.omicron.value),
            "transition_quotient_degree_bounds": stark.transition_quotient_degree_bounds(air),
            "max_degree": stark.max_degree(air),
            "boundary_quotient_degree_bounds": stark.boundary_quotient_degree_bounds(trace_len, boundary)}


def prefix_digests(objects, nregs, nquad):
    """SHA-256 of the pickled prefixes: after the boundary roots, the randomizer root, FRI and each opening block"""
    block = 2 * nquad
    after_fri = len(objects) - (nregs + 1) * block
    cuts = [nregs, nregs + 1, after_fri] + [after_fri + block * (j + 1) for j in range(nregs + 1)]
    return [hashlib.sha256(pickle.dumps(objects[:k])).hexdigest() for k in cuts]


def run(stark, ncycles, tcd, trace, air, boundary, draws, proof_stream=None, document=None, verify=True):
    """one Stark.prove, recorded"""
    print("prove: %d registers, %d cycles, FRI domain %d" % (stark.num_registers, ncycles, stark.fri.domain_length),
          flush=True)
    indices = []
    orig_prove = Fri.prove

    def prove_w(self, codeword, ps):
        res = orig_prove(self, codeword, ps)
        indices.append(list(res))
        return res
    rec = {"params": params(stark, ncycles, tcd, air, boundary, len(trace) + stark.num_randomizers),
           "trace": [[str(v.value) for v in row] for row in trace], "air": enc_air(air),
           "boundary": [[c, r, str(v.value)] for c, r, v in boundary],
           "stream": "plain" if document is None else "signature"}
    if document is not None:
        rec["document"] = document.hex()
    before = [list(row) for row in trace]
    draws.values = []
    Fri.prove = prove_w
    try:
        proof = stark.prove(trace, air, boundary, proof_stream)
    except AssertionError as e:
        rec["raises"] = str(e)
        rec["draws"] = list(draws.values)
        return rec, None
    finally:
        Fri.prove = orig_prove
    assert trace == before
    rec["draws"] = list(draws.values)
    objects = pickle.loads(proof)
    nquad = 4 * len(indices[0])
    n = stark.fri.domain_length
    quad = sorted([i for i in indices[0]] + [(i + stark.expansion_factor) % n for i in indices[0]])
    quad = sorted(quad + [(i + n // 2) % n for i in quad])
    rec.update({"proof_sha256": hashlib.sha256(proof).hexdigest(), "proof_len": len(proof),
                "prefix_sha256": prefix_digests(objects, stark.num_registers, nquad),
                "indices": indices[0], "repeated_indices": len(set(quad)) < len(quad), "verify": None})
    if verify:
        rec["verify"] = bool(stark.verify(proof, air, boundary))
    return rec, proof


def gen_stark(out):
    """test_stark.py's parameters (Rescue-Prime, expansion factor 4, 2 colinearity checks, security level 2, the
    declared degree 2), seed 1000"""
    from rescue_prime import RescuePrime
    rng = random.Random(1000)
    draws = Draws(rng)
    os.urandom = draws
    rp = RescuePrime()
    stark = st.Stark(field, 4, 2, 2, rp.m, rp.N + 1)
    input_element = fe(rng.randrange(P))
    trace = rp.trace(input_element)
    air = rp.transition_constraints(stark.omicron)
    boundary = rp.boundary_constraints(rp.hash(input_element))
    out["stark"], _ = run(stark, rp.N + 1, 2, trace, air, boundary, draws)


def gen_rpsss(out):
    """RPSSS keygen + sign, seed 1100, "Hello, World!", then a second key and document.  The draws of a signature are
    recorded as draw_stream [seed, skip, count]: the count values after the first skip of the seeded stream (a keygen
    draw precedes each signature); the second signature's AIR is the first's (air_of)"""
    import rpsss
    rng = random.Random(1100)
    draws = Draws(rng)
    os.urandom = draws
    r = rpsss.RPSSS()
    air = r.rp.transition_constraints(r.stark.omicron)
    skip = 0
    for name, doc in (("rpsss", b"Hello, World!"), ("rpsss_second", b"A second document, signed with another key")):
        sk, pk = r.keygen()
        trace = r.rp.trace(sk)
        boundary = r.rp.boundary_constraints(pk)
        sps = rpsss.SignatureProofStream(doc)
        rec, _ = run(r.stark, r.rp.N + 1, 3, trace, air, boundary, draws, sps, doc, verify=False)
        rec.update({"sk": str(sk.value), "pk": str(pk.value)})
        rec["draw_stream"] = [1100, skip + 1, len(rec.pop("draws"))]
        skip += 1 + rec["draw_stream"][2]
        if name == "rpsss_second":
            del rec["air"]
            rec["air_of"] = "rpsss"
        out[name] = rec


def gen_three_register(out):
    """make_golden_stark.py's three-register AIR on Stark: the first seed from 1200 whose quadrupled indices repeat.
    Then a broken witness (the remainder message at the transition division, after the trace randomizers), a false
    boundary value, a constraint of degree below the zerofier's (x^3 - 2x: degree 3 < deg Z = 15, a non-zero
    remainder), and a constraint whose maximal-degree terms cancel (a b c - c b a: a zero coefficient at degree
    3 (T - 1), so the declared bound is above the quotient's degree)"""
    ncycles = 16
    for seed in range(1200, 1400):
        rng = random.Random(seed)
        draws = Draws(rng)
        os.urandom = draws
        stark = st.Stark(field, 8, 8, 16, 3, ncycles, transition_constraints_degree=3)
        air = three_register_air(stark)
        trace = three_register_trace(rng, ncycles)
        last = ncycles - 1
        boundary = [(0, 0, trace[0][0]), (0, 1, trace[0][1]), (0, 2, trace[0][2]), (5, 0, trace[5][0]),
                    (last, 0, trace[last][0]), (last, 2, trace[last][2])]
        rec, proof = run(stark, ncycles, 3, trace, air, boundary, draws, verify=False)
        if rec.get("repeated_indices"):
            break
    rec["verify"] = bool(stark.verify(proof, air, boundary))
    rec["seed"] = seed
    out["three_register"] = rec

    broken = [list(row) for row in trace]
    broken[7][2] = broken[7][2] + fe(1)
    rec, _ = run(stark, ncycles, 3, broken, air, boundary, draws)
    rec["seed"] = seed
    out["broken_witness"] = rec

    false_boundary = list(boundary)
    false_boundary[3] = (5, 0, trace[5][0] + fe(1))
    rec, _ = run(stark, ncycles, 3, trace, air, false_boundary, draws)
    out["false_boundary"] = rec

    v = MPolynomial.variables(1 + 2 * 3, field)
    low = air + [v[0] * v[0] * v[0] - MPolynomial.constant(fe(2)) * v[0]]
    rec, _ = run(stark, ncycles, 3, trace, low, boundary, draws)
    out["below_zerofier"] = rec

    cur = v[1:4]
    cancel = air + [air[2] + cur[0] * cur[1] * cur[2] - cur[2] * cur[1] * cur[0]]
    rec, _ = run(stark, ncycles, 3, trace, cancel, boundary, draws)
    out["cancelled_top"] = rec


def gen_tiny(out):
    """make_golden_stark.py's four-cycle AIR (one colinearity check, two registers), seed 1300, then its broken
    witness"""
    ncycles = 4
    rng = random.Random(1300)
    draws = Draws(rng)
    os.urandom = draws
    stark = st.Stark(field, 4, 1, 2, 2, ncycles, transition_constraints_degree=2)
    v = MPolynomial.variables(1 + 2 * 2, field)
    cur, nxt = v[1:3], v[3:5]
    air = [nxt[0] - cur[0] - cur[1], nxt[1] - cur[0] * cur[1]]
    a, b = fe(rng.randrange(P)), fe(rng.randrange(P))
    trace = [[a, b]]
    for _ in range(ncycles - 1):
        a, b = a + b, a * b
        trace.append([a, b])
    boundary = [(0, 0, trace[0][0]), (0, 1, trace[0][1]), (ncycles - 1, 0, trace[-1][0])]
    out["tiny"], _ = run(stark, ncycles, 2, trace, air, boundary, draws)
    broken = [list(row) for row in trace]
    broken[2][1] = broken[2][1] + fe(3)
    out["tiny_broken"], _ = run(stark, ncycles, 2, broken, air, boundary, draws)


if __name__ == "__main__":
    real_urandom = os.urandom
    out = {}
    try:
        gen_stark(out)
        gen_three_register(out)
        gen_tiny(out)
        if "--no-rpsss" not in sys.argv:
            gen_rpsss(out)
    finally:
        os.urandom = real_urandom
    dump("stark_plain.json", out)
