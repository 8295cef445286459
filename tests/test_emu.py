"""CPU emulation of the kernels' phase functions (tests/emu/emu.cpp) against the oracle:
checks the index maps, twiddle tables, portable field arithmetic, decimal/blake2b leaf
encoding, chunked Merkle reduction and the fused FRI round without a GPU."""
import ctypes
import hashlib
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O

P = O.P


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu())
    lib.emu_ntt.restype = ctypes.c_int
    lib.emu_decimal.restype = ctypes.c_uint32
    return lib


def _call3(fn, a, b):
    out = np.zeros(2, dtype=np.uint64)
    fn(O._ptr(out), O._ptr(O._fe(a)), O._ptr(O._fe(b)))
    return int(out[0]) | (int(out[1]) << 64)


def test_portable_field(E):
    rng = random.Random(5)
    rinv = pow(1 << 128, -1, P)
    edge = [0, 1, 2, P - 1, P - 2, (1 << 64) - 1, 1 << 64, 1 << 127, 407 << 119, (1 << 96) - 1, 1 << 96]
    pairs = [(a, b) for a in edge for b in edge] + [(rng.randrange(P), rng.randrange(P)) for _ in range(5000)]
    for a, b in pairs:
        assert _call3(E.emu_montmul, a, b) == a * b * rinv % P
        assert _call3(E.emu_mul, a, b) == a * b % P
        assert _call3(E.emu_add, a, b) == (a + b) % P
        assert _call3(E.emu_sub, a, b) == (a - b) % P
    for a in edge + [rng.randrange(P) for _ in range(20)]:
        out = np.zeros(2, dtype=np.uint64)
        E.emu_inv(O._ptr(out), O._ptr(O._fe(a)))
        assert (int(out[0]) | (int(out[1]) << 64)) == O.inverse(a)


@pytest.mark.parametrize("shape", [(4, 8), (4, 4), (4, 2), (3, 8), (3, 4), (3, 2), (4, 7), (4, 3)])
@pytest.mark.parametrize("logn", list(range(0, 14)))
def test_tile_ntt_all_sizes(E, logn, shape):
    E.emu_set_shape(*shape)
    rng = random.Random(100 + logn)
    n = 1 << logn
    w = O.primitive_nth_root(n)
    for inverse in (0, 1):
        for batch in (1, 3, 9):
            if logn >= 12 and batch > 1:
                continue
            x = O.to_np([rng.randrange(P) for _ in range(n * batch)])
            out = np.zeros_like(x)
            assert E.emu_ntt(O._ptr(out), O._ptr(x), logn, O._ptr(O._fe(w)), inverse, ctypes.c_size_t(batch)) == 0
            for b in range(batch):
                xb = x[b * n:(b + 1) * n]
                want = xb if n == 1 else (O.intt_np(w, xb) if inverse else O.ntt_np(w, xb))
                assert (out[b * n:(b + 1) * n] == want).all(), (logn, inverse, batch, b)


@pytest.mark.parametrize("shape", [(4, 8), (3, 4)])
@pytest.mark.parametrize("logn", [3, 4, 6, 9, 12, 15])
def test_three_pass_split_small(E, logn, shape):
    """the n = n1*n2*n3 plan used above 2^20, forced at small sizes"""
    E.emu_set_shape(*shape)
    E.emu_ntt_ex.restype = ctypes.c_int
    rng = random.Random(300 + logn)
    n = 1 << logn
    w = O.primitive_nth_root(n)
    for inverse in (0, 1):
        for batch in (1, 3):
            x = O.to_np([rng.randrange(P) for _ in range(n * batch)])
            out = np.zeros_like(x)
            assert E.emu_ntt_ex(O._ptr(out), O._ptr(x), logn, O._ptr(O._fe(w)), inverse, ctypes.c_size_t(batch), 1) == 0
            for b in range(batch):
                xb = x[b * n:(b + 1) * n]
                want = O.intt_np(w, xb) if inverse else O.ntt_np(w, xb)
                assert (out[b * n:(b + 1) * n] == want).all(), (logn, inverse, batch, b)
            # in place
            y = x.copy()
            assert E.emu_ntt_ex(O._ptr(y), O._ptr(y), logn, O._ptr(O._fe(w)), inverse, ctypes.c_size_t(batch), 1) == 0
            assert (y == out).all()


def test_tile_ntt_2_16_and_nonstandard_root(E):
    E.emu_set_shape(4, 8)
    rng = random.Random(9)
    n = 1 << 16
    w = pow(O.primitive_nth_root(n), 12345, P)  # another primitive root
    x = O.to_np([rng.randrange(P) for _ in range(n)])
    out = np.zeros_like(x)
    assert E.emu_ntt(O._ptr(out), O._ptr(x), 16, O._ptr(O._fe(w)), 0, ctypes.c_size_t(1)) == 0
    assert (out == O.ntt_np(w, x)).all()
    assert E.emu_ntt(O._ptr(out), O._ptr(x), 16, O._ptr(O._fe(O.primitive_nth_root(8))), 0, ctypes.c_size_t(1)) == -3
    assert E.emu_ntt(O._ptr(out), O._ptr(x), 4, O._ptr(O._fe(O.primitive_nth_root(64))), 0, ctypes.c_size_t(1)) == -2


def test_decimal_and_leaf(E):
    rng = random.Random(6)
    vals = [0, 1, 9, 10, 99, 100, 10**9 - 1, 10**9, 10**18, 10**19 - 1, 10**19, 10**27, 10**36, 10**38 - 1,
            10**38, P - 1, P - 2, 2**32 - 1, 2**32, 2**64 - 1, 2**64, 2**96 - 1, 2**96, 2**127, 10**9 * (2**32 - 1),
            (10**9 - 1) * 10**27 + 5, 2**128 - 1, 340 * 10**36] + [rng.randrange(P) for _ in range(500)] + \
           [rng.randrange(10**k) for k in range(1, 39) for _ in range(10)]
    # base-1e8 limb boundaries (the quotient estimate of the long division is repaired by one compare: values
    # whose limbs are 0, 1, 1e8 - 1 and whose partial quotients sit next to a multiple of 1e8), 2^32 - 1 quotients
    edge = [0, 1, 10**8 - 1]
    vals += [a + b * 10**8 + c * 10**16 + d * 10**24 + e * 10**32
             for a in edge for b in edge for c in edge for d in edge for e in (0, 1, 3402822)]
    vals += [m * 10**8 * 2**(32 * j) + off for m in (1, 2**32 - 1, 99999999) for j in (0, 1, 2)
             for off in (-1, 0, 1) if 0 <= m * 10**8 * 2**(32 * j) + off < 2**128]
    vals += [rng.randrange(2**128) for _ in range(3000)] + [rng.randrange(2**(8 * k)) for k in range(1, 17) for _ in range(50)]
    for v in vals:
        buf = np.zeros(40, dtype=np.uint8)
        n = E.emu_decimal(O._ptr(buf), O._ptr(O._fe(v)))
        s = str(v).encode()
        assert n == len(s) and buf[:n].tobytes() == s and not buf[n:].any()
        d = np.zeros(64, dtype=np.uint8)
        E.emu_leaf_digest(O._ptr(d), O._ptr(O._fe(v)))
        assert d.tobytes() == hashlib.blake2b(s).digest()
    for _ in range(100):
        l = bytes(rng.randrange(256) for _ in range(64))
        r = bytes(rng.randrange(256) for _ in range(64))
        d = np.zeros(64, dtype=np.uint8)
        E.emu_node_digest(O._ptr(d), O._ptr(np.frombuffer(l, dtype=np.uint8)), O._ptr(np.frombuffer(r, dtype=np.uint8)))
        assert d.tobytes() == hashlib.blake2b(l + r).digest()
        E.emu_node_digest_coop4(O._ptr(d), O._ptr(np.frombuffer(l, dtype=np.uint8)), O._ptr(np.frombuffer(r, dtype=np.uint8)))
        assert d.tobytes() == hashlib.blake2b(l + r).digest()  # four-lanes-per-node schedule


@pytest.mark.parametrize("logn", [0, 1, 2, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17])
def test_merkle_and_fri_round(E, logn):
    rng = random.Random(40 + logn)
    n = 1 << logn
    x = O.to_np([rng.randrange(P) for _ in range(n)])
    tree = np.zeros((2 * n, 64), dtype=np.uint8)
    E.emu_merkle_tree(O._ptr(tree), O._ptr(x), ctypes.c_size_t(n))
    assert (tree[1:] == O.merkle_tree_np(x)[1:]).all()
    if n >= 2:
        alpha, omega, off = rng.randrange(P), O.primitive_nth_root(n), O.GENERATOR
        nxt = np.zeros((n // 2, 2), dtype=np.uint64)
        ntree = np.zeros((n, 64), dtype=np.uint8)
        E.emu_fri_round(O._ptr(nxt), O._ptr(ntree), O._ptr(x), ctypes.c_size_t(n), O._ptr(O._fe(alpha)),
                        O._ptr(O._fe(off)), O._ptr(O._fe(omega)))
        want = O.fri_fold_np(x, alpha, off, omega)
        assert (nxt == want).all()
        assert (ntree[1:] == O.merkle_tree_np(want)[1:]).all()


@pytest.mark.parametrize("rows", [
    [(10, 2, 10, 0, 64)],                    # barrier-free bottom launch, the rest by the default shape
    [(8, 2, 10, 3, 0), (0, 0, 3, 1, 64)],    # partial in-CTA reduction; tiny launches of 8-node CTAs one level each
    [(12, 3, 11, 2, 16), (6, 1, 6, 0, 0)],  # eight bottom nodes per thread; two per thread without shared phase
])
def test_merkle_other_launch_shapes(E, rows):
    """the generalised launch shape (ipt_log, chunk, red_log) builds the same tree whatever the split"""
    spec = ",".join(":".join(str(v) for v in r) for r in rows).encode()  # SA_MK_SHAPE form
    rng = random.Random(77)
    try:
        E.emu_set_merkle_shape(spec)
        for logn in (3, 6, 10, 13):
            n = 1 << logn
            x = O.to_np([rng.randrange(P) for _ in range(n)])
            tree = np.zeros((2 * n, 64), dtype=np.uint8)
            E.emu_merkle_tree(O._ptr(tree), O._ptr(x), ctypes.c_size_t(n))
            assert (tree[1:] == O.merkle_tree_np(x)[1:]).all()
    finally:
        E.emu_set_merkle_shape(b"")
