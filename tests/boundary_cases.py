"""Cases of the boundary quotient tests, shared by the CPU emulation (tests/test_boundary_cpu.py) and the GPU suite
(tests/test_gpu_boundary.py): seeded boundaries and trace polynomials, and the outputs restated with Python ints --
the reference's long division (T - I) / Z (univariate.py:80-97) and fast_coset_evaluate of the quotient for a clean
division; the coset values (T - I)(x_i) / Z(x_i), their inverse transform and its tail for any trace -- plus the
fixture tests/golden/boundary.json.

A case's register s has k_s boundary points omicron^c at distinct odd cycles c of an omicron of order 4n, so no point
lies on the coset offset * <root> for offset 1 or a random offset.  A clean register's trace polynomial is I + Z R
with R seeded; a false one's boundary value is changed by one afterwards, as a witness that breaks a boundary
constraint."""
import json
import os
import random

import oracle as O
from air_cases import padd, pmul

P = O.P
HERE = os.path.dirname(os.path.abspath(__file__))


# ---- the restatements ----
def divide(num, den):
    """univariate.py:80-97 on lists of ints: (quotient, remainder), the quotient deg num - deg Z + 1 coefficients
    long (or [] when deg num < deg Z), as Polynomial.divide builds it"""
    dn, dd = O.degree(num), O.degree(den)
    assert dd >= 0
    if dn < dd:
        return [], [c % P for c in num]
    rem = [c % P for c in num[:dn + 1]]
    inv = O.inverse(den[dd])
    quo = [0] * (dn - dd + 1)
    for shift in range(dn - dd, -1, -1):
        c = rem[shift + dd] * inv % P
        quo[shift] = c
        if c:
            for j in range(dd + 1):
                rem[shift + j] = (rem[shift + j] - c * den[j]) % P
    return quo, rem


def psub(a, b):
    return padd(a, [(P - v) % P for v in b])


def coset_values(coeffs, n, root, offset):
    """fast_coset_evaluate at order n (zero padded)"""
    return O.ntt(root, [c * pow(offset, i, P) % P for i, c in enumerate(coeffs)] + [0] * (n - len(coeffs)))


def expected(trace, zerofier, interpolant, n, root, offset):
    """one register's (quot row, codeword, flag) as the apply defines them, for any trace: V = (T - I)(x_i) / Z(x_i),
    U = intt(V), quot[j] = U[j] offset^-j for j < ncoef, flag = U non-zero at some j >= ncoef - deg Z"""
    ncoef = len(trace)
    num = coset_values(psub(trace, interpolant), n, root, offset)
    den = coset_values(zerofier, n, root, offset)
    cw = [a * O.inverse(b) % P for a, b in zip(num, den)]
    u = O.intt(root, cw)
    inv = O.inverse(offset)
    quot = [u[j] * pow(inv, j, P) % P for j in range(ncoef)]
    flag = any(u[j] for j in range(max(0, ncoef - (len(zerofier) - 1)), n))
    return quot, cw, flag


def reference(trace, zerofier, interpolant, n, root, offset):
    """the reference's (T - I) / Z: (quotient, codeword) for a clean division, None when it raises"""
    q, r = divide(psub(trace, interpolant), zerofier)
    if any(r):
        return None
    return q, O.fast_coset_evaluate(q, offset, root, n) if q else [0] * n


# ---- seeded cases ----
def boundary_rows(boundary, nregs, omicron):
    """per register: (points, values), and its zerofier and interpolant from the oracle"""
    out = []
    for s in range(nregs):
        pts = [(pow(omicron, c, P), v) for c, r, v in boundary if r == s]
        xs, vs = [x for x, _ in pts], [v for _, v in pts]
        z = O.from_np(O.zerofier_np(O.to_np(xs)))
        i = O.from_np(O.interpolate_np(O.to_np(xs), O.to_np(vs)))
        out.append((z, i))
    return out


def make_case(seed, log_n, nregs, npoints, offset_kind="random", ncoef=None, false_regs=(), const_values=False):
    """(boundary, omicron, trace rows, rows, R rows, root, offset): register s has npoints[s] boundary points (below n);
    trace polynomials of ncoef coefficients (default: about n / 4, at least deg Z), I + Z R for the registers not in
    false_regs.  With const_values every value of a register is the same, so I is a constant."""
    rng = random.Random(seed)
    n = 1 << log_n
    root = O.primitive_nth_root(n)
    omicron = O.primitive_nth_root(4 * n)
    offset = {"random": rng.randrange(2, P), "one": 1, "generator": O.GENERATOR}[offset_kind]
    if ncoef is None:
        ncoef = max(max(npoints), min(n, n // 4 + rng.randrange(3)))
    boundary = []
    for s in range(nregs):
        v0 = rng.randrange(P)
        for c in rng.sample(range(1, 4 * n, 2), npoints[s]):
            boundary.append((c, s, v0 if const_values else rng.randrange(P)))
    rng.shuffle(boundary)
    rows = boundary_rows(boundary, nregs, omicron)
    trace, rs = [], []
    for z, i in rows:
        r = [rng.randrange(P) for _ in range(max(0, ncoef - (len(z) - 1)))]
        t = padd(i, pmul(z, r)) if r else list(i)
        t = (t + [0] * ncoef)[:ncoef]
        trace.append(t)
        rs.append(r)
    if false_regs:
        for k, (c, s, v) in enumerate(boundary):
            if s in false_regs:
                boundary[k] = (c, s, (v + 1) % P)
                false_regs = tuple(x for x in false_regs if x != s)
        rows = boundary_rows(boundary, nregs, omicron)
    return boundary, omicron, trace, rows, rs, root, offset


def plan_bytes_rule(log_n, nregs):
    """DESIGN section 2: 2 S for offset^i and offset^-i, nregs S for 1/Z_s(x_i), nregs S for I_s(x_i), then
    sec16(nregs) for the degrees, S = sec16(n); 0 when invalid or past 2^64 bytes"""
    if not 1 <= log_n <= 30 or nregs < 1:
        return 0
    sec = lambda k: (k + 15) // 16 * 16  # noqa: E731
    b = 16 * ((2 + 2 * nregs) * sec(1 << log_n) + sec(nregs))
    return b if b < 1 << 64 else 0


# ---- the fixture ----
def golden():
    with open(os.path.join(HERE, "golden", "boundary.json")) as f:
        return json.load(f)


def ints(xs):
    return [int(x) for x in xs]


def digest(values):
    """the fixture's codeword digest: blake2b over the 16-byte little-endian values"""
    return O.vector_digest(O.to_np(values))


def golden_boundary(rec):
    return [(int(c), int(r), int(v)) for c, r, v in rec["boundary"]]
