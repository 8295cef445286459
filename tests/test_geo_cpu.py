"""CPU emulation of geometric interpolation plans and zerofiers (tests/emu/emu_geo.cpp over csrc/geo.cuh): the
library's own checks and schedules of the plan build, the batched apply, the zerofier and the prefix-product scan,
with every kernel replaced by a loop over its element function, against Lagrange interpolation and the expanded
product prod (x - step^i) in Python integers."""
import ctypes
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O

P = O.P
SA_EDIVZERO, SA_ESIZE = -4, -6
_vp, _sz, _ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int
STALE = 0x5A5A5A5A


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu_geo())
    for name, res, args in [("emu_geo_plan_bytes", _sz, [_sz]), ("emu_geo_batch_max", _sz, [_sz]),
                            ("emu_geo_plan", _ci, [_vp, _vp, _sz]),
                            ("emu_geo_interp_batch", _ci, [_vp, _vp, _vp, _sz, _sz, _sz]),
                            ("emu_geo_zerofier", _ci, [_vp, _vp, _sz]), ("emu_geo_scan", None, [_vp, _sz]),
                            ("emu_geo_scan_elems", _sz, [_sz])]:
        getattr(lib, name).restype = res
        getattr(lib, name).argtypes = args
    return lib


def root(order):
    return O.primitive_nth_root(order)


def lagrange(xs, ys):
    """the interpolant's coefficients: sum_i y_i / Z'(x_i) * Z / (x - x_i), Z = prod (x - x_i)"""
    k = len(xs)
    z = expanded(xs)
    f = [0] * k
    for xi, yi in zip(xs, ys):
        q = [0] * k  # Z / (x - xi) by synthetic division
        carry = 0
        for m in range(k, 0, -1):
            carry = (z[m] + carry * xi) % P
            q[m - 1] = carry
        d = 0
        for c in reversed(q):
            d = (d * xi + c) % P
        s = yi * pow(d, P - 2, P) % P
        for m in range(k):
            f[m] = (f[m] + s * q[m]) % P
    return f


def expanded(xs):
    z = [1]
    for x in xs:
        z = [((z[t - 1] if t else 0) - x * (z[t] if t < len(z) else 0)) % P for t in range(len(z) + 1)]
    return z


def interpolant(xs, ys):
    """Lagrange in Python ints at small k; the oracle's compiled fast_interpolate above"""
    if len(xs) <= 70:
        return lagrange(xs, ys)
    return O.from_np(O.interpolate_np(O.to_np(xs), O.to_np(ys)))


def plan(E, step, k):
    p = np.full(max(E.emu_geo_plan_bytes(k), 16) // 8, STALE, dtype=np.uint64)
    return E.emu_geo_plan(O._ptr(p), O._ptr(O._fe(step)), k), p


def interp(E, p, values, k, chunk=0):
    out = np.full(values.shape, STALE, dtype=np.uint64)
    rc = E.emu_geo_interp_batch(O._ptr(out), O._ptr(p), O._ptr(values), k, values.shape[0], chunk)
    return rc, out


def zerofier(E, step, k):
    out = np.full((k + 1, 2), STALE, dtype=np.uint64)
    return E.emu_geo_zerofier(O._ptr(out), O._ptr(O._fe(step)), k), out


def rows(rng, batch, k):
    """batch value vectors: random, with a zero row and two equal rows from batch 5 on"""
    v = [[rng.randrange(P) for _ in range(k)] for _ in range(batch)]
    if batch >= 5:
        v[1] = [0] * k
        v[3] = list(v[2])
    return v


EDGES = sorted({e for j in range(7, 11) for e in (2 ** j - 1, 2 ** j, 2 ** j + 1)} | {1100})
SIZES = list(range(1, 71)) + EDGES


def steps(k, rng):
    """roots of orders 2k (the smallest power of two above) up to 2^20 and a random element"""
    lo = max(1, (2 * k - 1).bit_length())
    out = [("order_2^%d" % lo, root(1 << lo)), ("order_2^20", root(1 << 20)), ("random", rng.randrange(2, P - 1))]
    if lo + 1 < 20:
        out.append(("order_2^%d" % (lo + 1), root(1 << (lo + 1))))
    return out


@pytest.mark.parametrize("k", SIZES)
def test_interpolation_and_zerofier_match_python_ints(E, k):
    rng = random.Random(k)
    for name, q in steps(k, rng):
        rc, p = plan(E, q, k)
        assert rc == 0, (name, rc)
        xs = [pow(q, i, P) for i in range(k)]
        for batch in ((1, 2, 5) if k <= 70 or name == "random" else (2,)):
            vals = rows(rng, batch, k)
            rc, out = interp(E, p, np.stack([O.to_np(v) for v in vals]), k)
            assert rc == 0
            for b, v in enumerate(vals):
                assert O.from_np(out[b]) == interpolant(xs, v), (name, batch, b)
        rc, z = zerofier(E, q, k)
        assert rc == 0 and O.from_np(z) == expanded(xs), name


@pytest.mark.parametrize("k", [1, 2, 3, 16, 17, 70, 1024, 1025, 1 << 20, (1 << 26) - 1, 1 << 26, (1 << 26) + 1])
def test_plan_bytes_match_the_library(E, k):
    G.build_cuda()
    G._paths()
    import sa_engine
    lib = sa_engine.load_library()
    K = 1 << (2 * k - 1).bit_length()
    want = 16 * (2 * (-(-k // 16) * 16) + 2 * K) if k <= 1 << 26 else 0
    assert E.emu_geo_plan_bytes(k) == lib.sa_geo_plan_bytes(k) == want
    assert E.emu_geo_batch_max(k) == lib.sa_geo_batch_max(k) == (max(1, (1 << 30) // (48 * K)) if want else 0)
    assert lib.sa_geo_plan_bytes(1 << 20) == 96 << 20


def test_zero_size_and_above_the_cap_are_refused(E):
    for k in (0, (1 << 26) + 1):
        assert E.emu_geo_plan_bytes(k) == 0 and E.emu_geo_batch_max(k) == 0
        p = np.full(2, STALE, dtype=np.uint64)
        assert E.emu_geo_plan(O._ptr(p), O._ptr(O._fe(3)), k) == SA_ESIZE
        out = np.full((2, 2), STALE, dtype=np.uint64)
        assert E.emu_geo_zerofier(O._ptr(out), O._ptr(O._fe(3)), k) == SA_ESIZE
        assert E.emu_geo_interp_batch(O._ptr(out), O._ptr(p), O._ptr(out), k, 1, 0) == SA_ESIZE
        assert (p == STALE).all() and (out == STALE).all()


@pytest.mark.parametrize("k", [2, 3, 4, 5, 8, 11, 16, 17, 64])
def test_steps_with_a_small_order_are_refused(E, k):
    """step^d = 1 for some 1 <= d <= k: 1, p - 1 and roots of every order up to k (k itself included, whose domain
    is a whole subgroup); step = 0 before any work.  The zerofier leaves its output untouched."""
    bad = [1, P - 1, 0] + [root(1 << j) for j in range(1, 20) if 1 << j <= k]
    if k >= 11:  # an odd order: p - 1 = 2^119 * 11 * 37
        bad.append(next(w for w in (pow(x, (P - 1) // 11, P) for x in range(2, 50)) if w != 1))
    for q in bad:
        rc, p = plan(E, q, k)
        assert rc == SA_EDIVZERO, (q, rc)
        rc, z = zerofier(E, q, k)
        assert rc == SA_EDIVZERO and (z == STALE).all(), q
    if k & (k - 1) == 0:
        assert plan(E, root(k), k)[0] == SA_EDIVZERO  # order exactly k
        assert plan(E, root(2 * k), k)[0] == 0        # order 2k: accepted


def test_single_point_is_never_refused(E):
    for q in (0, 1, P - 1, 5):
        rc, p = plan(E, q, 1)
        assert rc == 0
        rc, out = interp(E, p, np.stack([O.to_np([7]), O.to_np([0])]), 1)
        assert rc == 0 and O.from_np(out[0]) == [7] and O.from_np(out[1]) == [0]
        rc, z = zerofier(E, q, 1)
        assert rc == 0 and O.from_np(z) == [P - 1, 1]


@pytest.mark.parametrize("k,batch,chunk", [(5, 5, 2), (33, 7, 3), (64, 4, 1), (100, 3, 2)])
def test_batch_across_chunks_equals_one_chunk(E, k, batch, chunk):
    rng = random.Random(k * batch)
    q = rng.randrange(2, P)
    rc, p = plan(E, q, k)
    assert rc == 0
    vals = np.stack([O.to_np(v) for v in rows(rng, batch, k)])
    rc, whole = interp(E, p, vals, k)
    assert rc == 0
    rc, chunked = interp(E, p, vals, k, chunk)
    assert rc == 0 and (whole == chunked).all()
    rc, none = interp(E, p, vals[:0], k)
    assert rc == 0


def scan_sizes():
    out = set(range(1, 40))
    for j in (1, 2, 3, 4):  # the boundaries of runs at every level: RUN^j - 1, RUN^j, RUN^j + 1 and a run past them
        b = 16 ** j
        out |= {b - 1, b, b + 1, b + 15, b + 16, b + 17, 2 * b - 1, 2 * b, 2 * b + 1}
    return sorted(out)


@pytest.mark.parametrize("n", scan_sizes())
def test_scan_is_the_prefix_products(E, n):
    rng = random.Random(n)
    xs = [rng.randrange(P) for _ in range(n)]
    if n > 3:
        xs[n // 2] = 1
        xs[-1] = P - 1
    a = O.to_np(xs)
    E.emu_geo_scan(O._ptr(a), n)
    acc, want = 1, []
    for x in xs:
        acc = acc * x % P
        want.append(acc)
    assert O.from_np(a) == want
    levels, m = 0, n
    while m > 1:
        m = -(-m // 16)
        levels += m
    assert E.emu_geo_scan_elems(n) == levels
