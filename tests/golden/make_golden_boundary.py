#!/usr/bin/env python3
"""Generate tests/golden/boundary.json by running the UNMODIFIED Python reference: FastStark's boundary quotients
(T_s - I_s) / Z_s with the reference's boundary_zerofiers, boundary_interpolants and Polynomial division, and their
fast_coset_evaluate codewords on the FRI domain (fast_stark.py:92-106), which pin sa_boundary_plan /
sa_boundary_quotients (tests/test_boundary_cpu.py, tests/test_gpu_boundary.py) without the reference present.

Needs a checkout of the reference, named as for make_golden.py (whose helpers it uses), and the recorded
tests/golden/faststark_trace.json:

    STARK_REFERENCE=<reference>/code python tests/golden/make_golden_boundary.py   # a few seconds

Encoding: field elements are decimal strings; a boundary is a list of [cycle, register, value]; a codeword is kept as
its vector digest (blake2b over the 16-byte little-endian values, BASELINE.md section 3); a register whose division
raises has null for its quotient and codeword digest.
"""
import json
import os
import random
import sys

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, Polynomial, dump, enc, fe, field, rand_elems, refntt, vector_digest  # noqa: E402

REMAINDER = "cannot perform polynomial division because remainder is not zero"


def case(omicron, omega, order, boundary, trace_polys, nregs, ncoef):
    """the reference's per-register zerofier, interpolant, quotient and codeword; trace rows padded to ncoef"""
    import fast_stark as fs

    class Regs(fs.FastStark):  # the reference's boundary_zerofiers / boundary_interpolants over this omicron
        def __init__(self):
            self.num_registers, self.omicron = nregs, omicron
    st = Regs()
    zerofiers, interpolants = st.boundary_zerofiers(boundary), st.boundary_interpolants(boundary)
    g = field.generator()
    quotients, digests = [], []
    for s in range(nregs):
        try:
            q = (trace_polys[s] - interpolants[s]) / zerofiers[s]
        except AssertionError as e:
            assert str(e) == REMAINDER
            quotients.append(None)
            digests.append(None)
            continue
        quotients.append(enc(q.coefficients))
        digests.append(vector_digest(refntt.fast_coset_evaluate(q, g, omega, order)))
    rows = [list(tp.coefficients) + [field.zero()] * (ncoef - len(tp.coefficients)) for tp in trace_polys]
    assert all(len(r) == ncoef for r in rows)
    return {"log_n": order.bit_length() - 1, "root": str(omega.value), "offset": str(g.value),
            "omicron": str(omicron.value), "nregs": nregs,
            "boundary": [[c, r, str(v.value)] for c, r, v in boundary], "trace": [enc(r) for r in rows],
            "zerofiers": [enc(z.coefficients) for z in zerofiers],
            "interpolants": [enc(i.coefficients) for i in interpolants],
            "quotients": quotients, "codeword_digests": digests}


def clean_trace(omicron, boundary, nregs, rng, rlen, zeros=0):
    """I_s + Z_s R_s of rlen coefficients, R_s seeded: rlen - deg Z_s coefficients, the top `zeros` of them zero"""
    polys = []
    for s in range(nregs):
        pts = [(omicron ^ c, v) for c, r, v in boundary if r == s]
        z = Polynomial.zerofier_domain([p for p, _ in pts])
        i = Polynomial.interpolate_domain([p for p, _ in pts], [v for _, v in pts])
        k = rlen - z.degree()
        r = Polynomial(rand_elems(rng, k - zeros) + [field.zero()] * zeros)
        polys.append(i + z * r)
    return polys


def gen_boundary():
    """Five cases: the seeded FastStark run of faststark_trace.json (its boundary rebuilt from the seed; the recorded
    boundary quotients and codewords checked again here); the same run with the output value off by one (register 0's
    division raises); three registers with 1, 3 and 5 boundary points and trace polynomials I + Z R; two registers
    whose T - I has zero top coefficients, so the quotient is shorter than ncoef - deg Z; and the config-5 size
    (omicron of order 1024, trace polynomials of 284 coefficients, FRI domain 4096)."""
    from rescue_prime import RescuePrime
    with open(os.path.join(HERE, "faststark_trace.json")) as f:
        rec = json.load(f)
    calls, p = rec["calls"], rec["params"]
    rp = RescuePrime()
    poly = lambda c: Polynomial([fe(int(v)) for v in c])  # noqa: E731
    fz = [c for c in calls if c["fn"] == "fast_zerofier"][0]
    omicron = fe(int(fz["args"][1]["f"]))
    n = p["fri_domain_length"]
    omega = field.primitive_nth_root(n)
    trace_polys = [poly(c["out"]["poly"]) for c in calls if c["fn"] == "fast_interpolate"]
    ncoef = len(trace_polys[0].coefficients)
    # gen_faststark_trace's first draw from its seeded generator is the hash input
    output = rp.hash(fe(random.Random(rec["urandom_seed"]).randrange(field.p)))
    boundary = rp.boundary_constraints(output)
    out = {"faststark": case(omicron, omega, n, boundary, trace_polys, rp.m, ncoef)}
    evals = [c for c in calls if c["fn"] == "fast_coset_evaluate"]
    assert out["faststark"]["quotients"] == [evals[1]["args"][0]["poly"], evals[2]["args"][0]["poly"]]
    assert out["faststark"]["codeword_digests"] == [vector_digest([fe(int(v)) for v in e["out"]["l"]])
                                                    for e in evals[1:3]]
    false = rp.boundary_constraints(output + field.one())
    out["false_boundary"] = case(omicron, omega, n, false, trace_polys, rp.m, ncoef)
    assert out["false_boundary"]["quotients"][0] is None and out["false_boundary"]["quotients"][1] is not None

    rng = random.Random(900)
    multi = [(c, s, fe(rng.randrange(field.p))) for s, k in enumerate((1, 3, 5)) for c in rng.sample(range(28), k)]
    out["multi"] = case(omicron, omega, n, multi, clean_trace(omicron, multi, 3, rng, ncoef), 3, ncoef)
    assert all(q is not None for q in out["multi"]["quotients"])
    short = [(c, s, fe(rng.randrange(field.p))) for s, k in enumerate((2, 4)) for c in rng.sample(range(28), k)]
    out["short"] = case(omicron, omega, n, short, clean_trace(omicron, short, 2, rng, ncoef, zeros=3), 2, ncoef)
    assert all(len(q) < ncoef - (2, 4)[s] for s, q in enumerate(out["short"]["quotients"]))

    rng = random.Random(901)
    order = 1024
    omicron = field.primitive_nth_root(order)
    big = [(0, 1, field.zero()), (rp.N, 0, fe(rng.randrange(field.p))), (5, 0, fe(rng.randrange(field.p)))]
    out["config5"] = case(omicron, field.primitive_nth_root(4 * order), 4 * order, big,
                          clean_trace(omicron, big, 2, rng, 284), 2, 284)
    out["config5"]["seed"] = 901
    dump("boundary.json", out)


if __name__ == "__main__":
    gen_boundary()
