#!/usr/bin/env python3
"""Generate tests/golden/stark.json by running the UNMODIFIED Python reference: whole FastStark.prove runs (and
FastRPSSS signatures) with os.urandom replaced by a seeded stream, so that sa_stark (tests/test_stark_cpu.py,
tests/test_gpu_stark.py) can be held to the reference's proof bytes without the reference present.

Needs a checkout of the reference, named as for make_golden.py (whose helpers it uses):

    STARK_REFERENCE=<reference>/code python tests/golden/make_golden_stark.py   # ~3 minutes (two signatures)

Each case records the parameters and what FastStark derives from them, the original trace rows, the AIR as
exponent dicts ({"e": exponents, "c": coefficient}), the boundary as [cycle, register, value], the field values the
prove drew from os.urandom in order (the stub's 17 bytes reduced mod p; a test can hand each one back as 17
big-endian bytes), the proof stream kind ("plain", or "signature" with the document), and then either the proof's
SHA-256, length and prefix digests (SHA-256 of the pickled stream prefix after the boundary roots, after the
randomizer root, after FRI and after each opening block) with the reference's verify result, or the message of the
AssertionError the prove raised.  Field elements are decimal strings.
"""
import hashlib
import os
import pickle
import random
import sys

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import P, Fri, dump, fe, field  # noqa: E402

import fast_stark as fs  # noqa: E402
from multivariate import MPolynomial  # noqa: E402


class Draws:
    """os.urandom from a seeded random.Random (as make_golden.py seeds it), recording each 17-byte draw's value"""

    def __init__(self, rng):
        self.rng, self.values = rng, []

    def __call__(self, n):
        b = bytes(self.rng.getrandbits(8) for _ in range(n))
        self.values.append(str(int.from_bytes(b, "big") % P))
        return b


def enc_air(air):
    return [[{"e": list(k), "c": str(v.value)} for k, v in a.dictionary.items()] for a in air]


def params(stark, ncycles, tcd, air, boundary, trace_len):
    return {"expansion_factor": stark.expansion_factor, "num_colinearity_checks": stark.num_colinearity_checks,
            "security_level": stark.security_level, "num_registers": stark.num_registers, "num_cycles": ncycles,
            "transition_constraints_degree": tcd, "num_randomizers": stark.num_randomizers,
            "omicron_domain_length": stark.omicron_domain_length, "fri_domain_length": stark.fri_domain_length,
            "generator": str(stark.generator.value), "omega": str(stark.omega.value),
            "omicron": str(stark.omicron.value),
            "transition_quotient_degree_bounds": stark.transition_quotient_degree_bounds(air),
            "max_degree": stark.max_degree(air),
            "boundary_quotient_degree_bounds": stark.boundary_quotient_degree_bounds(trace_len, boundary)}


def prefix_digests(objects, nregs, nquad):
    """SHA-256 of the pickled prefixes: after the boundary roots, the randomizer root, FRI and each opening block"""
    total = len(objects)
    block = 2 * nquad
    after_fri = total - (nregs + 2) * block
    cuts = [nregs, nregs + 1, after_fri] + [after_fri + block * (j + 1) for j in range(nregs + 2)]
    return [hashlib.sha256(pickle.dumps(objects[:k])).hexdigest() for k in cuts]


def run(stark, ncycles, tcd, trace, air, boundary, draws, zerofier, zerofier_codeword, zerofier_root,
        proof_stream=None, document=None, verify=True):
    """one prove, recorded"""
    print("prove: %d registers, %d cycles, FRI domain %d" % (stark.num_registers, ncycles, stark.fri_domain_length),
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
           "zerofier_root": zerofier_root.hex(),
           "stream": "plain" if document is None else "signature"}
    if document is not None:
        rec["document"] = document.hex()
    before = list(trace)
    draws.values = []
    Fri.prove = prove_w
    try:
        proof = stark.prove(trace, air, boundary, zerofier, zerofier_codeword, proof_stream)
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
    quad = sorted([i for i in indices[0]] + [(i + stark.expansion_factor) % stark.fri_domain_length
                                               for i in indices[0]])
    quad = sorted(quad + [(i + stark.fri_domain_length // 2) % stark.fri_domain_length for i in quad])
    rec.update({"proof_sha256": hashlib.sha256(proof).hexdigest(), "proof_len": len(proof),
                "prefix_sha256": prefix_digests(objects, stark.num_registers, nquad),
                "indices": indices[0], "repeated_indices": len(set(quad)) < len(quad), "verify": None})
    if verify:
        rec["verify"] = bool(stark.verify(proof, air, boundary, zerofier_root))
    return rec, proof


def gen_faststark(out):
    """test_fast_stark.py's parameters, seed 600: make_golden.py's faststark_trace.json run"""
    from rescue_prime import RescuePrime
    rng = random.Random(600)
    draws = Draws(rng)
    os.urandom = draws
    rp = RescuePrime()
    stark = fs.FastStark(field, 4, 2, 2, rp.m, rp.N + 1, transition_constraints_degree=3)
    tz, tzc, tzr = stark.preprocess()
    input_element = fe(rng.randrange(P))
    trace = rp.trace(input_element)
    air = rp.transition_constraints(stark.omicron)
    boundary = rp.boundary_constraints(rp.hash(input_element))
    out["faststark"], _ = run(stark, rp.N + 1, 3, trace, air, boundary, draws, tz, tzc, tzr)


def gen_rpsss(out):
    """FastRPSSS keygen + sign, seed 700, "Hello, World!" (rpsss.json's run), then a second key and document"""
    import fast_rpsss
    rng = random.Random(700)
    draws = Draws(rng)
    os.urandom = draws
    r = fast_rpsss.FastRPSSS()
    air = r.rp.transition_constraints(r.stark.omicron)
    for name, doc in (("rpsss", b"Hello, World!"), ("rpsss_second", b"A second document, signed with another key")):
        sk, pk = r.keygen()
        trace = r.rp.trace(sk)
        boundary = r.rp.boundary_constraints(pk)
        sps = fast_rpsss.SignatureProofStream(doc)
        rec, _ = run(r.stark, r.rp.N + 1, 3, trace, air, boundary, draws, r.transition_zerofier,
                       r.transition_zerofier_codeword, r.transition_zerofier_root, sps, doc, verify=False)
        rec.update({"sk": str(sk.value), "pk": str(pk.value)})
        out[name] = rec


def three_register_air(stark):
    """a' = b, b' = a b c + 5 (cubic), c' = c + a (linear)"""
    v = MPolynomial.variables(1 + 2 * 3, field)
    cur, nxt = v[1:4], v[4:7]
    return [nxt[0] - cur[1], nxt[1] - cur[0] * cur[1] * cur[2] - MPolynomial.constant(fe(5)),
            nxt[2] - cur[2] - cur[0]]


def three_register_trace(rng, ncycles):
    a, b, c = fe(rng.randrange(P)), fe(rng.randrange(P)), fe(rng.randrange(P))
    trace = [[a, b, c]]
    for _ in range(ncycles - 1):
        a, b, c = b, a * b * c + fe(5), c + a
        trace.append([a, b, c])
    return trace


def gen_three_register(out):
    """mixed constraint degrees (the linear and the cubic divide at different orders), expansion factor 8, several
    boundary points on register 0; the seed is the first from 800 whose quadrupled indices repeat.  Then the same AIR
    with a witness that breaks the linear constraint at one row, a false boundary value, and one more constraint of
    degree below the zerofier's"""
    ncycles = 16
    for seed in range(800, 1000):
        rng = random.Random(seed)
        draws = Draws(rng)
        os.urandom = draws
        stark = fs.FastStark(field, 8, 8, 16, 3, ncycles, transition_constraints_degree=3)
        tz, tzc, tzr = stark.preprocess()
        air = three_register_air(stark)
        trace = three_register_trace(rng, ncycles)
        last = ncycles - 1
        boundary = [(0, 0, trace[0][0]), (0, 1, trace[0][1]), (0, 2, trace[0][2]), (5, 0, trace[5][0]),
                    (last, 0, trace[last][0]), (last, 2, trace[last][2])]
        rec, proof = run(stark, ncycles, 3, trace, air, boundary, draws, tz, tzc, tzr, verify=False)
        if rec.get("repeated_indices"):
            break
    rec["verify"] = bool(stark.verify(proof, air, boundary, tzr))
    rec["seed"] = seed
    out["three_register"] = rec

    broken = [list(row) for row in trace]
    broken[7][2] = broken[7][2] + fe(1)  # c' = c + a fails from row 6 to 7 and from 7 to 8; b' uses c at row 7
    rec, _ = run(stark, ncycles, 3, broken, air, boundary, draws, tz, tzc, tzr)
    rec["seed"] = seed
    out["broken_witness"] = rec

    false_boundary = list(boundary)
    false_boundary[3] = (5, 0, trace[5][0] + fe(1))
    rec, _ = run(stark, ncycles, 3, trace, air, false_boundary, draws, tz, tzc, tzr)
    out["false_boundary"] = rec

    v = MPolynomial.variables(1 + 2 * 3, field)
    low = air + [v[0] * v[0] * v[0] - MPolynomial.constant(fe(2)) * v[0]]  # x^3 - 2x: degree 3 < deg Z = 15
    rec, _ = run(stark, ncycles, 3, trace, low, boundary, draws, tz, tzc, tzr)
    out["below_zerofier"] = rec


def gen_tiny(out):
    """four cycles and one colinearity check: the linear constraint's numerator has degree 7, so the reference
    divides it by long division; the quadratic one (degree 14) goes through the transform at order 16.  Then a
    witness that breaks the linear constraint, which that long division refuses"""
    ncycles = 4
    rng = random.Random(900)
    draws = Draws(rng)
    os.urandom = draws
    stark = fs.FastStark(field, 4, 1, 2, 2, ncycles, transition_constraints_degree=2)
    tz, tzc, tzr = stark.preprocess()
    v = MPolynomial.variables(1 + 2 * 2, field)
    cur, nxt = v[1:3], v[3:5]
    air = [nxt[0] - cur[0] - cur[1], nxt[1] - cur[0] * cur[1]]
    a, b = fe(rng.randrange(P)), fe(rng.randrange(P))
    trace = [[a, b]]
    for _ in range(ncycles - 1):
        a, b = a + b, a * b
        trace.append([a, b])
    boundary = [(0, 0, trace[0][0]), (0, 1, trace[0][1]), (ncycles - 1, 0, trace[-1][0])]
    out["tiny"], _ = run(stark, ncycles, 2, trace, air, boundary, draws, tz, tzc, tzr)
    broken = [list(row) for row in trace]
    broken[2][1] = broken[2][1] + fe(3)
    out["tiny_broken"], _ = run(stark, ncycles, 2, broken, air, boundary, draws, tz, tzc, tzr)


if __name__ == "__main__":
    real_urandom = os.urandom
    out = {}
    try:
        gen_faststark(out)
        gen_three_register(out)
        gen_tiny(out)
        if "--no-rpsss" not in sys.argv:
            gen_rpsss(out)
    finally:
        os.urandom = real_urandom
    dump("stark.json", out)
