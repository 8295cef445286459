"""The verifier's element functions (csrc/verify.cuh) on the CPU through tests/emu/emu_verify.cpp: Merkle paths at
depths 1 to 20 and every index parity against hashlib and merkle.py's recursion restated; the colinearity test
against Polynomial.interpolate_domain restated in Python ints on random triples, constant lines, collinear triples
and alpha in {ax, bx}; the AIR at a point against stark_verify's term-by-term evaluation on air.json and random AIRs
of 1, 2, 3 and 5 registers; the combination against stark_verify.combination_at."""
import ctypes
import hashlib
import random

import numpy as np
import pytest

import __graft_entry__ as G
import air_cases as A
import stark_cases as C
import stark_verify as SV
from sa_engine import _air_arrays

P = C.P
_vp, _u64p = ctypes.c_void_p, ctypes.POINTER(ctypes.c_uint64)


@pytest.fixture(scope="module")
def lib():
    lib = ctypes.CDLL(G.build_emu_verify())
    lib.emu_air_point.restype = lib.emu_verify_combination.restype = ctypes.c_int
    return lib


def fe_bytes(values):
    return b"".join((int(v) % P).to_bytes(16, "little") for v in values)


def ptr(buf):
    return ctypes.cast(ctypes.c_char_p(buf), _vp) if isinstance(buf, bytes) else buf.ctypes.data_as(_vp)


def limbs(x):
    return (ctypes.c_uint64 * 2)(x & (2 ** 64 - 1), x >> 64)


def verify_(root, index, path, leaf):
    """merkle.py:28-40 restated: the recursion over the path"""
    assert 0 <= index < 1 << len(path)
    h = hashlib.blake2b
    if len(path) == 1:
        return root == (h(leaf + path[0]).digest() if index == 0 else h(path[0] + leaf).digest())
    nxt = h(leaf + path[0]).digest() if index % 2 == 0 else h(path[0] + leaf).digest()
    return verify_(root, index >> 1, path[1:], nxt)


def root_of(index, path, value):
    h = hashlib.blake2b(str(value).encode()).digest()
    for sib in path:
        h = hashlib.blake2b(sib + h if index & 1 else h + sib).digest()
        index >>= 1
    return h


def test_merkle_paths(lib):
    rng = random.Random(1)
    roots, leaves, idx, depth, digests, poff, want = [], [], [], [], [], [], []
    for d in range(1, 21):
        for index in sorted({0, 1, (1 << d) - 1, (1 << d) - 2, rng.randrange(1 << d), 0x5555555 % (1 << d)}):
            value = rng.randrange(P)
            path = [rng.randbytes(64) for _ in range(d)]
            root = root_of(index, path, value)
            for case in range(4):  # right, a wrong sibling, a wrong root, an index at 2^d (refused as failed)
                p, r, i = list(path), root, index
                if case == 1:
                    p[rng.randrange(d)] = bytes(64)
                elif case == 2:
                    r = bytes(64)
                elif case == 3:
                    i = index + (1 << d)
                ok = i < 1 << d and verify_(r, i, p, hashlib.blake2b(str(value).encode()).digest())
                roots.append(r)
                leaves.append(value)
                idx.append(i)
                depth.append(d)
                poff.append(len(digests))
                digests += p
                want.append(0 if ok else 1)
    assert want.count(0) == len(want) // 4
    n = len(want)
    flags = np.zeros(n, np.uint32)
    lib.emu_merkle_verify(ptr(flags), ptr(b"".join(roots)), ptr(fe_bytes(leaves)),
                          ptr(np.array(idx, np.uint64)), ptr(np.array(depth, np.uint32)), ptr(b"".join(digests)),
                          ptr(np.array(poff, np.uint64)), ctypes.c_longlong(n))
    assert flags.tolist() == want


def interpolate_degree(xs, ys):
    """Polynomial.interpolate_domain(...).degree() restated with lists of ints: products of (X - x_j) times
    inverse(x_i - x_j), inverse(0) = 0"""
    acc = [0, 0, 0]
    for i in range(3):
        prod = [ys[i] % P]
        for j in range(3):
            if j == i:
                continue
            inv = pow((xs[i] - xs[j]) % P, P - 2, P)
            nxt = [0] * (len(prod) + 1)
            for t, c in enumerate(prod):
                nxt[t + 1] = (nxt[t + 1] + c) % P
                nxt[t] = (nxt[t] - xs[j] * c) % P
            prod = [c * inv % P for c in nxt]
        acc = [(a + b) % P for a, b in zip(acc, prod)]
    return max([t for t, c in enumerate(acc) if c], default=-1)


def test_colinearity(lib):
    rng = random.Random(2)
    triples = []
    for _ in range(200):
        triples.append(([rng.randrange(P) for _ in range(3)], [rng.randrange(P) for _ in range(3)]))
        xs = [rng.randrange(P) for _ in range(3)]
        a, b = rng.randrange(P), rng.randrange(P)
        triples.append((xs, [(a * x + b) % P for x in xs]))              # collinear
        triples.append((xs, [b] * 3))                                     # a constant line: degree 0
        ax = rng.randrange(1, P)
        line = [(a * x + b) % P for x in (ax, P - ax)]
        for alpha in (ax, P - ax):                                        # alpha = ax, alpha = bx
            triples.append(([ax, P - ax, alpha], line + [(a * alpha + b) % P]))
            triples.append(([ax, P - ax, alpha], line + [rng.randrange(P)]))
        triples.append(([ax, ax, ax], [1, 2, 3]))                         # every difference zero
    want = [0 if interpolate_degree(xs, ys) == 1 else 1 for xs, ys in triples]
    assert 0 < want.count(0) < len(want)
    flags = np.zeros(len(triples), np.uint32)
    lib.emu_colinear(ptr(flags), ptr(fe_bytes(x for xs, _ in triples for x in xs)),
                     ptr(fe_bytes(y for _, ys in triples for y in ys)), ctypes.c_longlong(len(triples)))
    assert flags.tolist() == want


def test_fri_colinearity_rounds(lib):
    rng = random.Random(3)
    offset, n = C.T.field.generator().value, 1 << 12
    omega = C.T.field.primitive_nth_root(n).value
    ay, by, cy, aidx, alpha, rnd, want = [], [], [], [], [], [], []
    for r in range(6):
        for _ in range(20):
            a = rng.randrange(n >> (r + 1))
            ax = pow(offset, 1 << r, P) * pow(omega, (1 << r) * a, P) % P
            bx = pow(offset, 1 << r, P) * pow(omega, (1 << r) * (a + (n >> (r + 1))), P) % P
            assert bx == P - ax
            s, t = rng.randrange(P), rng.randrange(P)
            al = rng.choice([rng.randrange(P), ax, bx])
            c = (s * al + t) % P if rng.random() < 0.5 else rng.randrange(P)
            ys = [(s * ax + t) % P, (s * bx + t) % P, c]
            ay.append(ys[0]), by.append(ys[1]), cy.append(ys[2]), aidx.append(a), alpha.append(al), rnd.append(r)
            want.append(0 if interpolate_degree([ax, bx, al], ys) == 1 else 1)
    flags = np.zeros(len(want), np.uint32)
    lib.emu_fri_colinear(ptr(flags), ptr(fe_bytes(ay)), ptr(fe_bytes(by)), ptr(fe_bytes(cy)),
                         ptr(np.array(aidx, np.uint64)), ptr(fe_bytes(alpha)), ptr(np.array(rnd, np.uint32)),
                         limbs(offset), limbs(omega), ctypes.c_longlong(len(want)))
    assert flags.tolist() == want


class _Terms:
    def __init__(self, constraints):
        self.terms = [sorted(c.items()) for c in constraints]


def random_air(rng, nregs, ncons):
    nvars = 1 + 2 * nregs
    return [{tuple(rng.randrange(3) if rng.random() < 0.5 else 0 for _ in range(nvars)): rng.randrange(P)
             for _ in range(rng.randrange(1, 6))} for _ in range(ncons)]


def air_points(lib, constraints, nregs, points):
    coeffs, exps, starts = _air_arrays(constraints, nregs)
    ncons = len(constraints)
    out = np.zeros((len(points), ncons, 2), np.uint64)
    rc = lib.emu_air_point(ptr(out), (ctypes.c_uint64 * max(len(coeffs), 1))(*coeffs),
                           (ctypes.c_uint32 * max(len(exps), 1))(*exps), (ctypes.c_size_t * (ncons + 1))(*starts),
                           ctypes.c_size_t(ncons), ctypes.c_size_t(nregs),
                           ptr(fe_bytes(v for p in points for v in p)), ctypes.c_longlong(len(points)))
    assert rc == 0
    return [[int(lo) | int(hi) << 64 for lo, hi in row] for row in out]


@pytest.mark.parametrize("nregs", [1, 2, 3, 5])
def test_air_point_random(lib, nregs):
    rng = random.Random(nregs)
    cons = random_air(rng, nregs, 4)
    points = [[rng.randrange(P) for _ in range(1 + 2 * nregs)] for _ in range(30)] + [[0] * (1 + 2 * nregs)]
    assert air_points(lib, cons, nregs, points) == [SV.Statement.constraint_values(_Terms(cons), p) for p in points]


def test_air_point_fixture(lib):
    rec = A.golden()["faststark"]
    cons = A.golden_air(rec)
    nregs = (len(next(iter(cons[0]))) - 1) // 2
    rng = random.Random(9)
    points = [[rng.randrange(P) for _ in range(1 + 2 * nregs)] for _ in range(8)]
    assert air_points(lib, cons, nregs, points) == [SV.Statement.constraint_values(_Terms(cons), p) for p in points]


def test_combination_against_combination_at(lib):
    import sa_stark
    rec = C.golden()["three_register"]
    stark = C.params(rec)
    cons = C.air(rec)
    boundary = C.inputs(rec)[1]
    st = SV.Statement(stark, cons, boundary)
    nregs, ncons, n = stark.num_registers, len(cons), stark.fri_domain_length
    rng = random.Random(5)
    W = st.num_weights
    weights = [rng.randrange(P) for _ in range(W)]
    zs = [z for z in st.zerofiers]
    its = [i for i in st.interpolants]
    blen = max(len(z) for z in zs)
    pdata = weights + st.transition_shifts + st.boundary_shifts
    for z, i in zip(zs, its):
        pdata += z + [0] * (blen - len(z)) + i + [0] * (blen - len(i))
    items, want = [], []
    for q in range(24):
        i = rng.randrange(n)
        cur, nxt = [rng.randrange(P) for _ in range(nregs)], [rng.randrange(P) for _ in range(nregs)]
        rand, zero = rng.randrange(P), (0 if q == 5 else rng.randrange(1, P))
        if zero == 0:
            value, flag = 0, 2
        else:
            value = SV.combination_at(st, i, cur, nxt, rand, zero, weights)
            flag = q % 3 == 1
            value = (value + flag) % P
        items += [i, value] + cur + nxt + [rand, zero]
        want.append(int(flag))
    coeffs, exps, starts = _air_arrays(cons, nregs)
    flags = np.zeros(len(want), np.uint32)
    rc = lib.emu_verify_combination(
        ptr(flags), ptr(fe_bytes(items)), ptr(fe_bytes(pdata)), ctypes.c_size_t(len(want)), ctypes.c_size_t(1),
        (ctypes.c_uint64 * len(coeffs))(*coeffs), (ctypes.c_uint32 * len(exps))(*exps),
        (ctypes.c_size_t * (ncons + 1))(*starts), ctypes.c_size_t(ncons), ctypes.c_size_t(nregs),
        ctypes.c_size_t(blen), None, ctypes.c_size_t(0), limbs(st.generator), limbs(st.omega),
        ctypes.c_int(n.bit_length() - 1), ctypes.c_size_t(st.expansion_factor))
    assert rc == 0 and flags.tolist() == want
    assert sa_stark.VerifierPlan  # the plan packs this layout (test_verify_cpu.py drives it)


def test_combination_checks(lib):
    z = ctypes.c_size_t(0)
    bad = [(1, 1, 1, 0, 1, 4, 1), (1, 1, 1, 17, 1, 4, 1), (1, 1, 0, 1, 1, 4, 1), (1, 1, 1, 1, 0, 4, 1),
           (1, 1, 1, 1, 1, 31, 1), (1, 1, 1, 1, 1, 4, 16), (1 << 58, 4, 1, 1, 1, 4, 1)]
    for k, nproofs, ncons, nregs, blen, log_n, ef in bad:
        rc = lib.emu_verify_combination(None, None, None, ctypes.c_size_t(k), ctypes.c_size_t(nproofs), None, None,
                                        None, ctypes.c_size_t(ncons), ctypes.c_size_t(nregs), ctypes.c_size_t(blen),
                                        None, z, limbs(0), limbs(0), ctypes.c_int(log_n), ctypes.c_size_t(ef))
        assert rc == -6, (k, nproofs, ncons, nregs, blen, log_n, ef)
