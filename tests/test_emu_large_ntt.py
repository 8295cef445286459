"""The NTT plan above 2^26 on the CPU: the factored pass-1 twiddles (ntt_plan.cuh) run through the emulated
tile kernels at small forced sizes, and the tables of the real 2^27 ... 2^30 plans, built by the library's own
table code, are checked entry by entry against Python ints."""
import ctypes
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O

P = O.P
FORCE_THREE_PASS_FACTORED = 2  # emu_ntt_plan: three passes, pass-1 twiddles as A (n1 x n2) * B (n1 x n3)


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu_large())
    lib.emu_ntt_plan.restype = ctypes.c_int
    lib.emu_ntt_pass1_twiddles.restype = ctypes.c_int
    return lib


def _int(row):
    return int(row[0]) | (int(row[1]) << 64)


@pytest.mark.parametrize("shape", [(4, 8), (3, 4)])
@pytest.mark.parametrize("logn", [3, 4, 6, 9, 12, 15])
def test_factored_three_pass_small(E, logn, shape):
    """the plan used above 2^26, forced at small sizes: bit for bit with the oracle, also in place"""
    E.emu_set_shape(*shape)
    rng = random.Random(700 + logn)
    n = 1 << logn
    w = O.primitive_nth_root(n)
    for inverse in (0, 1):
        for batch in (1, 3):
            x = O.to_np([rng.randrange(P) for _ in range(n * batch)])
            out = np.zeros_like(x)
            assert E.emu_ntt_plan(O._ptr(out), O._ptr(x), logn, O._ptr(O._fe(w)), inverse, ctypes.c_size_t(batch),
                                  FORCE_THREE_PASS_FACTORED) == 0
            for b in range(batch):
                xb = x[b * n:(b + 1) * n]
                want = O.intt_np(w, xb) if inverse else O.ntt_np(w, xb)
                assert (out[b * n:(b + 1) * n] == want).all(), (logn, inverse, batch, b)
            y = x.copy()
            assert E.emu_ntt_plan(O._ptr(y), O._ptr(y), logn, O._ptr(O._fe(w)), inverse, ctypes.c_size_t(batch),
                                  FORCE_THREE_PASS_FACTORED) == 0
            assert (y == out).all(), (logn, inverse, batch)


def test_factored_matches_full_matrix_plan(E):
    """a non-standard primitive root: the factored and the full-matrix three-pass plans agree"""
    E.emu_set_shape(4, 8)
    rng = random.Random(11)
    logn = 13
    n = 1 << logn
    w = pow(O.primitive_nth_root(n), 4321, P)
    x = O.to_np([rng.randrange(P) for _ in range(n)])
    for inverse in (0, 1):
        full, split = np.zeros_like(x), np.zeros_like(x)
        assert E.emu_ntt_plan(O._ptr(full), O._ptr(x), logn, O._ptr(O._fe(w)), inverse, ctypes.c_size_t(1), 1) == 0
        assert E.emu_ntt_plan(O._ptr(split), O._ptr(x), logn, O._ptr(O._fe(w)), inverse, ctypes.c_size_t(1),
                              FORCE_THREE_PASS_FACTORED) == 0
        assert (full == split).all()
        assert (split == (O.intt_np(w, x) if inverse else O.ntt_np(w, x))).all()


@pytest.mark.parametrize("logn,digits", [(27, (9, 9, 9)), (28, (10, 9, 9)), (29, (10, 10, 9)), (30, (10, 10, 10))])
def test_real_plan_pass1_factors(E, logn, digits):
    """A[k1][m >> l3] * B[k1][m & (n3 - 1)] == w^(k1*m) * scale for the real shapes, at the corners and at
    sampled (k1, m); forward (scale 1) and inverse (w^-1, scale n^-1)"""
    n = 1 << logn
    root = O.primitive_nth_root(n)
    rng = random.Random(logn)
    l1, l2, l3 = digits
    n1, m_count = 1 << l1, 1 << (l2 + l3)
    corners = [(k, m) for k in (0, 1, n1 - 1) for m in (0, 1, (1 << l3) - 1, 1 << l3, m_count - 1)]
    samples = corners + [(rng.randrange(n1), rng.randrange(m_count)) for _ in range(400)]
    k1 = (ctypes.c_longlong * len(samples))(*[k for k, _ in samples])
    m = (ctypes.c_longlong * len(samples))(*[j for _, j in samples])
    for inverse in (0, 1):
        shape = (ctypes.c_int * 4)()
        a = np.zeros((len(samples), 2), dtype=np.uint64)
        b = np.zeros_like(a)
        assert E.emu_ntt_pass1_twiddles(shape, O._ptr(a), O._ptr(b), logn, O._ptr(O._fe(root)), inverse, k1, m,
                                        ctypes.c_size_t(len(samples))) == 0
        assert tuple(shape) == digits + (1,)
        w = pow(root, -1, P) if inverse else root
        scale = pow(n, -1, P) if inverse else 1
        for i, (kk, mm) in enumerate(samples):
            assert _int(a[i]) * _int(b[i]) % P == pow(w, kk * mm, P) * scale % P, (logn, inverse, kk, mm)


def test_plans_up_to_2_26_keep_the_full_matrix(E):
    """sizes the full matrix served before keep it: 2^21 has three passes and no factored tables"""
    n = 1 << 21
    root = O.primitive_nth_root(n)
    samples = [(0, 0), (1, 1), (127, (1 << 14) - 1), (5, 77)]
    k1 = (ctypes.c_longlong * 4)(*[k for k, _ in samples])
    m = (ctypes.c_longlong * 4)(*[j for _, j in samples])
    shape = (ctypes.c_int * 4)()
    a = np.zeros((4, 2), dtype=np.uint64)
    b = np.zeros_like(a)
    assert E.emu_ntt_pass1_twiddles(shape, O._ptr(a), O._ptr(b), 21, O._ptr(O._fe(root)), 0, k1, m,
                                    ctypes.c_size_t(4)) == 0
    assert tuple(shape) == (7, 7, 7, 0)
    for i, (kk, mm) in enumerate(samples):
        assert _int(b[i]) == 1 and _int(a[i]) == pow(root, kk * mm, P)
