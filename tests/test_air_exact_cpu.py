"""CPU emulation of the exact transition quotients (tests/emu/emu_air_exact.cpp over csrc/air.cuh's air_quotients_exact):
the rows bit for bit those of the unchecked apply, and each remainder flag exactly the reference's test of
Polynomial.__truediv__ (univariate.py:50-53), restated as long division with Python ints.

The AIRs mix tests/air_cases.py's seeded constraints (numerators in the trace, almost never divisible) with
constraints in x alone whose numerators are built: Q Z (exact), Q Z plus a remainder at a chosen degree below deg Z,
the zero polynomial (no terms, or zero coefficients only) and a non-zero numerator below the zerofier's degree.  The
engine's tail is n - deg Z."""
import ctypes
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O
from air_cases import P, make_case, numerator, pmul, padd, quotients
from test_air_cpu import apply, plan

SA_EROOTORDER, SA_ESIZE = -2, -6


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu_air_exact())
    sz, vp, ci = ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int
    lib.emu_air_plan_bytes.restype = sz
    lib.emu_air_plan_bytes.argtypes = [ci, sz, sz, sz]
    lib.emu_air_plan.restype = ci
    lib.emu_air_plan.argtypes = [vp, vp, vp, vp, sz, sz, sz, vp, sz, ci, vp, vp, vp]
    lib.emu_air_quotients.restype = ci
    lib.emu_air_quotients.argtypes = [vp, vp, vp, sz, sz, sz, sz, ci, vp]
    lib.emu_air_quotients_exact.restype = ci
    lib.emu_air_quotients_exact.argtypes = [vp, vp, vp, vp, sz, sz, sz, sz, sz, ci, vp]
    lib.emu_air_store_atomics.restype = ctypes.c_longlong
    return lib


def remainder(num, z):
    """num mod z with Python ints (z's top coefficient non-zero)"""
    r = list(num)
    dz = len(z) - 1
    inv = O.inverse(z[-1])
    for top in range(len(r) - 1, dz - 1, -1):
        c = r[top] * inv % P
        if c:
            for i, zc in enumerate(z):
                r[top - dz + i] = (r[top - dz + i] - c * zc) % P
    return r[:dz]


def divides(num, z):
    return not any(remainder(num, z))


def x_constraint(coeffs, nregs):
    """the constraint sum_i coeffs[i] x^i (a term per non-zero coefficient)"""
    return {(i,) + (0,) * (2 * nregs): c for i, c in enumerate(coeffs) if c}


def built(rng, kind, z, n, nregs):
    """a constraint in x alone of the given kind, for the zerofier z (deg Z = len(z) - 1)"""
    dz = len(z) - 1
    q = [rng.randrange(P) for _ in range(rng.randrange(1, n - dz + 1))]
    if kind == "exact":
        return x_constraint(pmul(q, z), nregs)
    if kind == "remainder":  # Q Z + r x^k, k < deg Z
        k = rng.randrange(dz)
        return x_constraint(padd(pmul(q, z), [0] * k + [rng.randrange(1, P)]), nregs)
    if kind == "zero":
        return {} if rng.randrange(2) else {(rng.randrange(n),) + (0,) * (2 * nregs): 0}
    if kind == "low":  # 0 < deg N < deg Z, or a non-zero constant
        d = rng.randrange(dz)
        return x_constraint([rng.randrange(P) for _ in range(d)] + [rng.randrange(1, P)], nregs)
    raise ValueError(kind)


BUILT = ("exact", "remainder", "zero", "low")


def exact_case(seed, log_n, nregs, ncons):
    """air_cases' case with every other constraint replaced by a built one (deg Z >= 1 where one is built)"""
    air, trace, z, max_ncoef, root, offset, step, qlen = make_case(seed, log_n, nregs, ncons)
    rng = random.Random(seed + 1)
    n = 1 << log_n
    if n > 1 and len(z) < 2:
        z = [rng.randrange(P), 1]
    for c in range(ncons):
        if (c + seed) % 2 == 0 and len(z) >= 2:
            air[c] = built(rng, BUILT[(c // 2 + seed) % len(BUILT)], z, n, nregs)
    return air, trace, z, max_ncoef, root, offset, step, qlen


def run_exact(E, air, trace, z, max_ncoef, root, offset, step, qlen, log_n, tail):
    """(rc, unchecked rows, exact rows, flags) from one plan"""
    nregs, ncons = len(trace), len(air)
    rc, buf = plan(E, air, nregs, max_ncoef, z, log_n, root, offset, step)
    assert rc == 0
    plain = np.zeros((ncons * qlen, 2), np.uint64)
    assert apply(E, plain, buf, trace, nregs, qlen, ncons, log_n, root) == 0
    out = np.zeros_like(plain)
    flags = np.zeros(ncons, np.uint32)
    t = O.to_np([v for row in trace for v in row])
    rc = E.emu_air_quotients_exact(O._ptr(out), O._ptr(flags), O._ptr(buf), O._ptr(t), nregs, len(trace[0]), qlen,
                                   ncons, tail, log_n, O._ptr(O._fe(root)))
    return rc, plain, out, flags


def expected_atomics(rows, tail, n):
    """one atomicOr per (warp, row) with a non-zero coefficient at j >= tail: warps of 32 consecutive indices c n + j"""
    return len({((c * n + j) // 32, c) for c, row in enumerate(rows) for j in range(tail, n) if row[j]})


def check(E, seed, log_n, nregs, ncons):
    n = 1 << log_n
    air, trace, z, max_ncoef, root, offset, step, qlen = exact_case(seed, log_n, nregs, ncons)
    tail = n - (len(z) - 1)
    rc, plain, out, flags = run_exact(E, air, trace, z, max_ncoef, root, offset, step, qlen, log_n, tail)
    assert rc == 0
    assert np.array_equal(out, plain)
    # the reference's test, restated twice: long division of the numerator, and the coset row's tail
    want = [0 if divides(numerator(a, trace, step), z) else 1 for a in air]
    rows = quotients(air, trace, z, n, root, offset, step)
    assert want == [int(any(r[tail:])) for r in rows]
    assert flags.tolist() == want
    assert E.emu_air_store_atomics() == expected_atomics(rows, tail, n)
    return want


@pytest.mark.parametrize("ncons", [1, 2, 7])
@pytest.mark.parametrize("nregs", [1, 2, 3])
@pytest.mark.parametrize("log_n", list(range(1, 11)))
def test_flags_are_the_remainder_test(E, log_n, nregs, ncons):
    check(E, 1000 * log_n + 10 * nregs + ncons, log_n, nregs, ncons)


@pytest.mark.parametrize("log_n", [4, 6])
def test_remainder_at_every_degree_below_the_zerofier(E, log_n):
    """Q Z + x^k for every k < deg Z: each flagged, and Q Z alone clean"""
    n, nregs = 1 << log_n, 1
    rng = random.Random(log_n)
    z = [rng.randrange(P) for _ in range(n // 2)] + [1]
    q = [rng.randrange(P) for _ in range(n - len(z) + 1)]
    base = pmul(q, z)
    air = [x_constraint(base, nregs)] + [x_constraint(padd(base, [0] * k + [rng.randrange(1, P)]), nregs)
                                         for k in range(len(z) - 1)]
    root = O.primitive_nth_root(n)
    trace = [[rng.randrange(P) for _ in range(3)]]
    rc, plain, out, flags = run_exact(E, air, trace, z, 3, root, 7, root, n, log_n, n - (len(z) - 1))
    assert rc == 0 and np.array_equal(out, plain)
    assert flags.tolist() == [0] + [1] * (len(z) - 1)


def test_errors_leave_outputs_untouched(E):
    log_n = 4
    n = 1 << log_n
    air, trace, z, max_ncoef, root, offset, step, qlen = exact_case(3, log_n, 2, 2)
    rc, buf = plan(E, air, 2, max_ncoef, z, log_n, root, offset, step)
    assert rc == 0
    t = O.to_np([v for row in trace for v in row])
    good = dict(nregs=2, ncoef=len(trace[0]), qlen=qlen, ncons=2, tail=n - (len(z) - 1), log_n=log_n, root=root)
    bad = [(dict(tail=n + 1), SA_ESIZE), (dict(qlen=0), SA_ESIZE), (dict(qlen=n + 1), SA_ESIZE),
           (dict(ncons=0), SA_ESIZE), (dict(nregs=0), SA_ESIZE), (dict(ncoef=0), SA_ESIZE),
           (dict(ncoef=n + 1), SA_ESIZE), (dict(log_n=31), SA_ESIZE),
           (dict(root=O.primitive_nth_root(n * 2)), SA_EROOTORDER)]
    for change, code in bad:
        a = dict(good, **change)
        out = np.full((max(1, a["ncons"]) * max(1, a["qlen"]), 2), 0x1234, np.uint64)
        flags = np.full(2, 0x77, np.uint32)
        rc = E.emu_air_quotients_exact(O._ptr(out), O._ptr(flags), O._ptr(buf), O._ptr(t), a["nregs"], a["ncoef"],
                                       a["qlen"], a["ncons"], a["tail"], a["log_n"], O._ptr(O._fe(a["root"])))
        assert rc == code, change
        assert (out == 0x1234).all() and (flags == 0x77).all(), change
