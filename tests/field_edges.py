"""Boundary operands for the field arithmetic of field.cuh (plain Python ints, no GPU).

Random operands reach the carry boundaries of the 128-bit product and of the modular add / sub only about
once in 2^32 tries, so a dropped carry there slips past any random campaign.  This module builds the
operands on purpose:

* product pairs whose low 128 bits t_lo = (a * b) mod 2^128 are chosen.  t_lo alone fixes every
  intermediate of the device reduction (x = e0 * P3 mod 2^32, the borrow w of e3 - x, m3 = e3 - x mod 2^32
  and the whole m * P3 chain); for an odd b, a = t_lo * b^-1 mod 2^128 gives that t_lo, and the pair is
  kept when a < p (about 80 % are).  The limbs e0, e1, e2 of t_lo run over {0, 1, 2^31, 2^32 - 2,
  2^32 - 1, random} and e3 over {x, x + 1, x - 1, 0, 2^32 - 1}.
* products of the special elements (0, 1, p - 2, p - 1, (p + 1) / 2, 2^128 mod p) with each other and
  with random elements, and pairs solved for the products 0, 1 and p - 1.
* add / sub pairs at a + b in {p - 1, p, p + 1, 2^128 - 1, 2^128, 2^128 + 1}, carries through every limb,
  a == b and a - b in {0, -1, -(p - 1)}.
* elements to invert.

Every expected value is computed on Python ints ((a * b) % p, (a +- b) % p, pow(a, p - 2, p)).
`device_reduction` restates the device's intermediates only to count which boundary classes the vectors
hit; `build()` asserts that every class is there at least MIN_PER_CLASS times, so a later edit cannot
quietly hollow the set out.
"""
import random
from collections import Counter

P = 1 + 407 * (1 << 119)
P3 = 0xCB800000  # top 32-bit limb of p; the low limbs are (1, 0, 0)
R = 1 << 128
M32 = (1 << 32) - 1
MIN_PER_CLASS = 8

SPECIAL = [0, 1, P - 2, P - 1, (P + 1) // 2, R % P]
LIMB_VALUES = ["0", "1", "2^31", "2^32-2", "2^32-1", "rand"]
TOP_RULES = ["x", "x+1", "x-1", "0", "2^32-1"]
SUM_TARGETS = {"p-1": P - 1, "p": P, "p+1": P + 1, "2^128-1": R - 1, "2^128": R, "2^128+1": R + 1}


def limbs(v):
    return [(v >> (32 * i)) & M32 for i in range(4)]


def device_reduction(a, b):
    """the intermediates of field.cuh's device fe_montmul for the product a * b: x = e0 * P3 mod 2^32,
    w = [e3 < x], m3 = (e3 - x) mod 2^32, and top = [t_hi < ((m * P3) >> 32) + w], the borrow that
    triggers the masked add-back of p.  Used for class counts only, never for expected values."""
    t = a * b
    e0, e1, e2, e3 = limbs(t % R)
    x = (e0 * P3) & M32
    w = int(e3 < x)
    m3 = (e3 - x) & M32
    m = e0 | (e1 << 32) | (e2 << 64) | (m3 << 96)
    u = ((m * P3) >> 32) + w
    r = (t >> 128) - u  # a * b * 2^-128 mod p, before the add-back, in (-p, p)
    return {"e": (e0, e1, e2, e3), "x": x, "w": w, "m3": m3, "top": int(r < 0), "r": r}


def _limb_value(name, rng):
    if name == "rand":
        return rng.randrange(1 << 32)
    return {"0": 0, "1": 1, "2^31": 1 << 31, "2^32-2": M32 - 1, "2^32-1": M32}[name]


def _top_value(rule, x):
    return {"x": x, "x+1": (x + 1) & M32, "x-1": (x - 1) & M32, "0": 0, "2^32-1": M32}[rule]


def _solve_low(t_lo, rng):
    """(a, b), both < p, with (a * b) mod 2^128 == t_lo"""
    while True:
        b = rng.randrange(1, P, 2)
        a = t_lo * pow(b, -1, R) % R
        if a < P:
            return a, b


def product_pairs(rng):
    """list of (a, b, tag) with a, b < p"""
    out = []
    for n0 in LIMB_VALUES:
        for n1 in LIMB_VALUES:
            for n2 in LIMB_VALUES:
                for rule in TOP_RULES:
                    for _ in range(2):  # two operand pairs (and two draws of the random limbs) per pattern
                        e0, e1, e2 = (_limb_value(n, rng) for n in (n0, n1, n2))
                        e3 = _top_value(rule, (e0 * P3) & M32)
                        a, b = _solve_low(e0 | (e1 << 32) | (e2 << 64) | (e3 << 96), rng)
                        out.append((a, b, "low:%s,%s,%s,%s" % (n0, n1, n2, rule)))
    for a in SPECIAL:
        for b in SPECIAL:
            out.append((a, b, "special"))
        for _ in range(4):
            r = rng.randrange(P)
            out.append((a, r, "special"))
            out.append((r, a, "special"))
    for target in (0, 1, P - 1):
        for _ in range(MIN_PER_CLASS):
            b = rng.randrange(1, P)
            a = target * pow(b, P - 2, P) % P
            out.append((a, b, "product=%d" % target if target < 2 else "product=p-1"))
    return out


def addsub_pairs(rng):
    """list of (a, b, tag) with a, b < p"""
    out = []
    for name, s in SUM_TARGETS.items():
        lo, hi = max(0, s - (P - 1)), min(P - 1, s)  # a in [lo, hi] keeps b = s - a in [0, p)
        for a in [lo, hi] + [rng.randint(lo, hi) for _ in range(MIN_PER_CLASS)]:
            out.append((a, s - a, "sum=" + name))
    for k in (1, 2, 3):
        c = (1 << (32 * k)) - 1
        out += [(c, 1, "carry%d" % k), (1, c, "carry%d" % k)]
        for _ in range(MIN_PER_CLASS // 2):
            r = rng.randrange(P - c)
            out += [(c + r, 1, "carry%d" % k), (c, 1 + r, "carry%d" % k)]  # (a carry chain that starts higher up)
    for a in SPECIAL + [rng.randrange(P) for _ in range(MIN_PER_CLASS)]:
        out.append((a, a, "a==b"))
        if a + 1 < P:
            out.append((a, a + 1, "diff=-1"))
    out.append((0, P - 1, "diff=-(p-1)"))
    out += [(a, b, "special") for a in SPECIAL for b in SPECIAL]
    return out


def inverse_operands(rng):
    vals = [v for v in SPECIAL if v] + [2, 3, P - 3, (P - 1) // 2, P3 << 96, (1 << 96) - 1, 1 << 96]
    vals += [1 << k for k in range(0, 128, 7)] + [(1 << k) - 1 for k in range(2, 128, 9)]
    vals += [rng.randrange(1, P) for _ in range(64)]
    return [v % P for v in vals if v % P]


def _check_coverage(muls, addsubs, invs):
    c = Counter()
    for a, b, tag in muls:
        assert 0 <= a < P and 0 <= b < P
        c[tag.split(":")[0] if tag.startswith("low") else tag] += 1
        d = device_reduction(a, b)
        e3 = d["e"][3]
        c["w=%d" % d["w"]] += 1
        c["top=%d" % d["top"]] += 1
        if d["m3"] == 0 and d["w"] == 0:
            c["e3==x"] += 1
        if d["m3"] == M32 and d["w"] == 1:
            c["e3==x-1"] += 1
        if e3 == ((d["x"] + 1) & M32):
            c["e3==x+1"] += 1
        if tag.startswith("low:"):
            for i, name in enumerate(tag[4:].split(",")[:3]):
                c["e%d=%s" % (i, name)] += 1
    for a, b, tag in addsubs:
        assert 0 <= a < P and 0 <= b < P
        c[tag] += 1
    for name in SUM_TARGETS:
        assert sum(1 for a, b, _ in addsubs if a + b == SUM_TARGETS[name]) >= MIN_PER_CLASS, name
    assert len(invs) >= MIN_PER_CLASS and all(0 < v < P for v in invs)
    need = ["low", "special", "product=0", "product=1", "product=p-1", "w=0", "w=1", "top=0", "top=1",
            "e3==x", "e3==x-1", "e3==x+1", "a==b", "diff=-1", "carry1", "carry2", "carry3"]
    need += ["e%d=%s" % (i, v) for i in range(3) for v in LIMB_VALUES]
    need += ["sum=" + s for s in SUM_TARGETS]
    for cls in need:
        assert c[cls] >= MIN_PER_CLASS, (cls, c[cls])
    assert c["diff=-(p-1)"] >= 1
    return c


def build(seed=2024):
    """(muls, addsubs, invs, class_counts): product pairs and add / sub pairs as lists of (a, b, tag),
    elements to invert as a list of ints; the same seed gives the same vectors"""
    rng = random.Random(seed)
    muls, addsubs, invs = product_pairs(rng), addsub_pairs(rng), inverse_operands(rng)
    return muls, addsubs, invs, _check_coverage(muls, addsubs, invs)
