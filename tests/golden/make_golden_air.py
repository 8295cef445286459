#!/usr/bin/env python3
"""Generate tests/golden/air.json by running the UNMODIFIED Python reference: the Rescue-Prime AIR and the
reference's transition quotients (evaluate_symbolic + fast_coset_divide, fast_stark.py:108-113), which pin
sa_air_plan / sa_air_quotients (tests/test_air_cpu.py, tests/test_gpu_air.py) without the reference present.

Needs a checkout of the reference, named as for make_golden.py (whose helpers it uses), and the recorded
tests/golden/faststark_trace.json:

    STARK_REFERENCE=<reference>/code python tests/golden/make_golden_air.py   # ~1 minute

Encoding: field elements are decimal strings; exponent vectors are full length (1 + 2 registers).
"""
import json
import os
import random
import sys

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import HERE, Polynomial, dump, enc, fe, field, rand_elems, refntt  # noqa: E402


def gen_air():
    """The Rescue-Prime AIR with the reference's evaluate_symbolic + fast_coset_divide quotients (fast_stark.py:108-113):
    the seeded FastStark run of faststark_trace.json (its recorded trace polynomials and quotients, checked again
    here), the same trace polynomials with one coefficient changed (a false witness: the division is not clean and
    the reference truncates it), and the config-5 size (omicron of order 1024, seeded trace polynomials of 284
    coefficients).  ~1 minute of reference time."""
    from rescue_prime import RescuePrime
    from multivariate import MPolynomial  # noqa: F401  (the AIR's type)
    with open(os.path.join(HERE, "faststark_trace.json")) as f:
        rec = json.load(f)
    calls = rec["calls"]
    poly = lambda c: Polynomial([fe(int(v)) for v in c])  # noqa: E731
    rp = RescuePrime()
    nvars = 1 + 2 * rp.m
    g = field.generator()

    def enc_air(air):
        out = []
        for a in air:
            out.append([{"e": list(k) + [0] * (nvars - len(k)), "c": str(v.value)} for k, v in a.dictionary.items()])
        return out

    def case(omicron, order, zerofier, trace_polys):
        air = rp.transition_constraints(omicron)
        point = [Polynomial([field.zero(), field.one()])] + trace_polys + [tp.scale(omicron) for tp in trace_polys]
        quotients = [refntt.fast_coset_divide(a.evaluate_symbolic(point), zerofier, g, omicron, order) for a in air]
        qlen = len(quotients[0].coefficients)
        assert all(len(q.coefficients) == qlen for q in quotients)
        return {"log_n": order.bit_length() - 1, "root": str(omicron.value), "offset": str(g.value),
                "step": str(omicron.value), "qlen": qlen, "air": enc_air(air),
                "zerofier": enc(zerofier.coefficients), "trace": [enc(tp.coefficients) for tp in trace_polys],
                "quotients": [enc(q.coefficients) for q in quotients]}

    fz = [c for c in calls if c["fn"] == "fast_zerofier"][0]
    omicron, order = fe(int(fz["args"][1]["f"])), fz["args"][2]["i"]
    zerofier = poly(fz["out"]["poly"])
    trace_polys = [poly(c["out"]["poly"]) for c in calls if c["fn"] == "fast_interpolate"]
    recorded = [c["out"]["poly"] for c in calls if c["fn"] == "fast_coset_divide"]
    out = {"faststark": case(omicron, order, zerofier, trace_polys)}
    assert out["faststark"]["quotients"] == recorded
    bad = [Polynomial(list(tp.coefficients)) for tp in trace_polys]
    bad[0].coefficients[5] = bad[0].coefficients[5] + field.one()
    out["false_witness"] = case(omicron, order, zerofier, bad)
    assert out["false_witness"]["quotients"] != recorded
    rng = random.Random(800)
    order = 1024
    omicron = field.primitive_nth_root(order)
    zerofier = refntt.fast_zerofier([omicron ^ i for i in range(rp.N)], omicron, order)
    out["config5"] = case(omicron, order, zerofier, [Polynomial(rand_elems(rng, 284)) for _ in range(rp.m)])
    out["config5"]["seed"] = 800
    dump("air.json", out)


if __name__ == "__main__":
    gen_air()
