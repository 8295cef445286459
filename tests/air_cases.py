"""Cases of the transition quotient tests, shared by the CPU emulation (tests/test_air_cpu.py) and the GPU suite
(tests/test_gpu_air.py): seeded AIRs in FastStark's variable layout and their quotients restated with Python ints --
the numerator in coefficients (MPolynomial.evaluate_symbolic's polynomial), divided on the coset at order n and not
truncated -- plus the fixture tests/golden/air.json.

An AIR of C constraints over nregs registers at n = 2^log_n mixes, constraint by constraint in turn: random terms; a
dense x-polynomial (consecutive x exponents) times one trace monomial; sparse high x powers; a constant; the zero
polynomial (no terms); terms with zero coefficients; several groups that share trace monomials.  Every term's degree
bound e_0 + (sum of the trace exponents) (max_ncoef - 1) stays below n."""
import json
import os
import random

import oracle as O

P = O.P
HERE = os.path.dirname(os.path.abspath(__file__))
KINDS = ("random", "dense", "sparse", "constant", "empty", "zeros", "groups")


# ---- polynomials as lists of Python ints, products by Kronecker substitution (exact, fast at these sizes) ----
def pmul(a, b):
    if not a or not b:
        return []
    width = 34  # bytes per slot: products < 2^254, sums of up to 2^17 of them
    pack = lambda v: int.from_bytes(b"".join(x.to_bytes(width, "little") for x in v), "little")  # noqa: E731
    raw = (pack(a) * pack(b)).to_bytes(width * (len(a) + len(b) - 1), "little")
    return [int.from_bytes(raw[k:k + width], "little") % P for k in range(0, len(raw), width)]


def padd(a, b):
    if len(a) < len(b):
        a, b = b, a
    return [(x + (b[i] if i < len(b) else 0)) % P for i, x in enumerate(a)]


def ppow(a, e, cache):
    key = (id(a), e)
    if key not in cache:
        if e == 0:
            cache[key] = [1]
        elif e == 1:
            cache[key] = a
        else:
            h = ppow(a, e // 2, cache)
            r = pmul(h, h)
            cache[key] = pmul(r, a) if e % 2 else r
    return cache[key]


def numerator(constraint, trace, step):
    """C(x, T(x), T(step x)) in coefficients, constraint a {exponent tuple: coefficient} dict: per trace monomial,
    its x-polynomial times the monomial"""
    nxt = [[v * pow(step, j, P) % P for j, v in enumerate(row)] for row in trace]
    point = trace + nxt
    groups = {}
    for k, v in constraint.items():
        xs = groups.setdefault(tuple(k[1:]), {})
        xs[k[0]] = (xs.get(k[0], 0) + v) % P
    cache, acc = {}, []
    for e, xs in groups.items():
        term = [0] * (max(xs) + 1)
        for x, v in xs.items():
            term[x] = v
        for row, ev in zip(point, e):
            if ev:
                term = pmul(term, ppow(row, ev, cache))
        acc = padd(acc, term)
    return acc


def evaluate(constraint, trace, step, x):
    """C(x, T(x), T(step x)) at one point, with Python ints"""
    def horner(row, at):
        r = 0
        for c in reversed(row):
            r = (r * at + c) % P
        return r
    vals = [horner(row, x) for row in trace] + [horner(row, step * x % P) for row in trace]
    acc = 0
    for k, v in constraint.items():
        t = v * pow(x, k[0], P)
        for val, ev in zip(vals, k[1:]):
            t = t * pow(val, ev, P) % P
        acc += t
    return acc % P


def coset_quotient(num, zerofier, n, root, offset):
    """U[j] * offset^-j, U = intt(ntt(num * offset^i) / ntt(Z * offset^i)) at order n, all n coefficients"""
    def ev(coeffs):
        return O.ntt(root, [c * pow(offset, i, P) % P for i, c in enumerate(coeffs)] + [0] * (n - len(coeffs)))
    u = O.intt(root, [a * O.inverse(b) % P for a, b in zip(ev(num), ev(zerofier))])
    inv = O.inverse(offset)
    return [c * pow(inv, j, P) % P for j, c in enumerate(u)]


def quotients(air, trace, zerofier, n, root, offset, step):
    return [coset_quotient(numerator(c, trace, step), zerofier, n, root, offset) for c in air]


# ---- seeded AIRs ----
def make_air(seed, log_n, nregs, ncons, max_ncoef):
    """ncons constraints over 1 + 2 nregs variables whose terms keep e_0 + tdeg (max_ncoef - 1) < n"""
    rng = random.Random(seed)
    n, nvars = 1 << log_n, 1 + 2 * nregs
    span = max_ncoef - 1

    def trace_exps(tdeg):
        e = [0] * (2 * nregs)
        for _ in range(tdeg):
            e[rng.randrange(2 * nregs)] += 1
        return e

    def room(e):  # the largest x exponent a term with trace exponents e may have
        return n - 1 - sum(e) * span

    def top_tdeg():  # the largest trace degree that leaves x^0
        return (n - 1) // span if span else 3

    air = []
    for c in range(ncons):
        kind = KINDS[(c + seed) % len(KINDS)]
        d = {}
        if kind == "random":
            for _ in range(rng.randrange(1, 7)):
                e = trace_exps(rng.randrange(0, min(3, top_tdeg()) + 1))
                d[tuple([rng.randrange(room(e) + 1)] + e)] = rng.randrange(P)
        elif kind == "dense":
            e = trace_exps(min(1, top_tdeg()))
            for x in range(min(room(e), 40) + 1):
                d[tuple([x] + e)] = rng.randrange(P)
        elif kind == "sparse":
            for tdeg in (0, min(1, top_tdeg())):
                e = trace_exps(tdeg)
                for x in sorted({room(e), room(e) // 2, room(e) // 3 + 1, 0}):
                    if 0 <= x <= room(e):
                        d[tuple([x] + e)] = rng.randrange(P)
        elif kind == "constant":
            d[(0,) * nvars] = rng.randrange(P)
        elif kind == "zeros":
            for _ in range(3):
                e = trace_exps(rng.randrange(0, min(2, top_tdeg()) + 1))
                d[tuple([rng.randrange(room(e) + 1)] + e)] = 0
            d[tuple([0] + trace_exps(min(1, top_tdeg())))] = rng.randrange(1, P)
        elif kind == "groups":
            for _ in range(3):
                e = trace_exps(rng.randrange(0, min(3, top_tdeg()) + 1))
                for x in rng.sample(range(room(e) + 1), min(4, room(e) + 1)):
                    d[tuple([x] + e)] = rng.choice([1, P - 1, rng.randrange(P)])
        air.append(d)
    return air


def make_case(seed, log_n, nregs, ncons, offset_kind="random", step_kind="root", short=False, qlen=None):
    """a full case: (air, trace rows, zerofier, max_ncoef, root, offset, step, qlen)"""
    rng = random.Random(seed)
    n = 1 << log_n
    max_ncoef = max(1, min(n, 1 + (n // 2) // 3 + rng.randrange(2)))
    ncoef = max(1, max_ncoef - 1 - rng.randrange(max(1, max_ncoef // 2))) if short else max_ncoef
    air = make_air(seed, log_n, nregs, ncons, max_ncoef)
    trace = [[rng.randrange(P) for _ in range(ncoef)] for _ in range(nregs)]
    zerofier = [rng.randrange(P) for _ in range(rng.randrange(1, n + 1))]
    zerofier[-1] = zerofier[-1] or 1
    root = O.primitive_nth_root(n)
    offset = {"random": rng.randrange(2, P), "zero": 0, "one": 1}[offset_kind]
    step = {"root": root, "power": pow(root, rng.randrange(n), P), "outside": O.GENERATOR}[step_kind]
    return air, trace, zerofier, max_ncoef, root, offset, step, n if qlen is None else qlen


def flatten(air, nregs):
    """the C ABI's arrays: coefficient limbs, exponents, term_start"""
    nvars = 1 + 2 * nregs
    coeffs, exps, starts = [], [], [0]
    for d in air:
        for k, v in d.items():
            k = tuple(k) + (0,) * (nvars - len(k))
            coeffs += [v & 0xFFFFFFFFFFFFFFFF, v >> 64]
            exps += list(k)
        starts.append(len(exps) // nvars)
    return coeffs, exps, starts


def plan_bytes_rule(log_n, max_ncoef, nregs, nterms):
    """DESIGN section 2: 3 S for the zerofier's coset division plan, S for (offset step)^j, S for x_i, then the
    program of 1 + nterms (2 + ceil(nregs / 2)) elements, every section rounded up to 16 elements; 0 when invalid"""
    n = 1 << log_n if 1 <= log_n <= 30 else 0
    if not n or nregs < 1 or not 1 <= max_ncoef <= n or nterms >= 1 << 32:
        return 0
    sec = lambda k: (k + 15) // 16 * 16  # noqa: E731
    return 16 * (5 * sec(n) + sec(1 + nterms * (2 + (nregs + 1) // 2)))


# ---- the fixture ----
def golden():
    with open(os.path.join(HERE, "golden", "air.json")) as f:
        g = json.load(f)
    return g


def golden_air(rec):
    """the fixture's constraints as {exponent tuple: int} dicts"""
    return [{tuple(t["e"]): int(t["c"]) for t in cons} for cons in rec["air"]]


def ints(xs):
    return [int(x) for x in xs]
