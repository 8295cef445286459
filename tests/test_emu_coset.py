"""CPU emulation of coset division plans and batched coset evaluation (tests/emu/emu_coset.cpp over csrc/coset.cuh): the
library's own checks and schedules of the plan build, the batched apply and the batched evaluation, with every
kernel replaced by a loop over its element function, against the oracle (tests/coset_cases.py)."""
import ctypes
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O
from coset_cases import Case, P, formula, rand_poly

SA_EROOTORDER, SA_ENOTPRIM, SA_EDIVZERO, SA_ESIZE = -2, -3, -4, -6
_u64p = ctypes.c_void_p


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu_coset())
    sz, ci = ctypes.c_size_t, ctypes.c_int
    lib.emu_coset_div_plan_bytes.restype = sz
    lib.emu_coset_div_plan_bytes.argtypes = [ci]
    lib.emu_coset_div_plan.restype = ci
    lib.emu_coset_div_plan.argtypes = [_u64p, _u64p, sz, ci, _u64p, _u64p]
    lib.emu_coset_div_apply_batch.restype = ci
    lib.emu_coset_div_apply_batch.argtypes = [_u64p, _u64p, _u64p, sz, sz, ci, _u64p, sz]
    lib.emu_coset_evaluate_batch.restype = ci
    lib.emu_coset_evaluate_batch.argtypes = [_u64p, _u64p, sz, ci, _u64p, _u64p, sz]
    return lib


def fe(x):
    return O._fe(x % P)


def plan(E, divisor, log_n, root, offset):
    d = O.to_np(divisor) if len(divisor) else np.zeros((1, 2), np.uint64)
    p = np.zeros(max(E.emu_coset_div_plan_bytes(log_n), 16), dtype=np.uint8)
    r, o = fe(root), fe(offset)
    rc = E.emu_coset_div_plan(O._ptr(p), O._ptr(d), len(divisor), log_n, O._ptr(r), O._ptr(o))
    return rc, p


def apply(E, p, lhs, qlen, log_n, root):
    batch, ncoef = lhs.shape[0], lhs.shape[1]
    out = np.zeros((batch, qlen, 2), np.uint64)
    r = fe(root)
    rc = E.emu_coset_div_apply_batch(O._ptr(out), O._ptr(p), O._ptr(lhs), ncoef, qlen, log_n, O._ptr(r), batch)
    return rc, out


@pytest.mark.parametrize("full", [True, False], ids=["n", "below_n"])
@pytest.mark.parametrize("batch", [1, 2, 5])
@pytest.mark.parametrize("log_n", list(range(1, 11)))
def test_apply_matches_oracle(E, log_n, batch, full):
    c = Case(log_n, batch, full, seed=100 * log_n + 10 * batch + full)
    rc, p = plan(E, c.divisor, log_n, c.root, c.offset)
    assert rc == 0
    before = p.copy()
    rc, out = apply(E, p, c.lhs_np(), c.qlen, log_n, c.root)
    assert rc == 0
    c.check(out)
    assert (p == before).all()
    for b in range(batch):  # each row alone gives the same
        rc, one = apply(E, p, c.lhs_np()[b:b + 1], c.qlen, log_n, c.root)
        assert rc == 0 and (one[0] == out[b]).all(), b


@pytest.mark.parametrize("batch", [1, 2, 5])
@pytest.mark.parametrize("log_n", list(range(1, 11)))
def test_evaluate_matches_oracle(E, log_n, batch):
    rng = random.Random(5000 + 10 * log_n + batch)
    n = 1 << log_n
    root, offset = O.primitive_nth_root(n), rng.randrange(P)
    for ncoef in sorted({n, max(1, n - 1), max(1, n // 2 + 1), 1}):
        rows = [rand_poly(rng, ncoef - 1) for _ in range(batch)]
        coeffs = np.stack([O.to_np(r) for r in rows])
        out = np.full((batch, n, 2), 0x5A5A, np.uint64)  # whatever the buffer held: every element is written
        r, o = fe(root), fe(offset)
        assert E.emu_coset_evaluate_batch(O._ptr(out), O._ptr(coeffs), ncoef, log_n, O._ptr(r), O._ptr(o), batch) == 0
        for b in range(batch):
            assert O.from_np(out[b]) == O.fast_coset_evaluate(rows[b], offset, root, n), (ncoef, b)


@pytest.mark.parametrize("log_n", list(range(1, 11)))
def test_divisors_that_vanish_and_offset_zero(E, log_n):
    """X - offset * root^3 vanishes at a coset point, the zero polynomial everywhere; on the coset of offset 0 every
    R_i is r_0, so only a divisor with r_0 == 0 vanishes there, and an apply gives the formula's [l0 / r0, 0, ...]"""
    rng = random.Random(6000 + log_n)
    n = 1 << log_n
    root, offset = O.primitive_nth_root(n), rng.randrange(1, P)
    point = offset * pow(root, 3, P) % P
    assert plan(E, [P - point, 1], log_n, root, offset)[0] == SA_EDIVZERO
    assert plan(E, [0] * min(n, 3), log_n, root, offset)[0] == SA_EDIVZERO
    assert plan(E, [0, 1], log_n, root, 0)[0] == SA_EDIVZERO
    assert plan(E, rand_poly(rng, min(n - 1, 2)), log_n, root, offset)[0] == 0
    d = [rng.randrange(1, P)] + rand_poly(rng, min(n - 1, 2))[1:]
    rc, p = plan(E, d, log_n, root, 0)
    assert rc == 0
    lhs = rand_poly(rng, n - 1)
    rc, out = apply(E, p, O.to_np(lhs)[None], n, log_n, root)
    assert rc == 0
    assert O.from_np(out[0]) == formula(lhs, d, 0, root, n, n) == [lhs[0] * O.inverse(d[0]) % P] + [0] * (n - 1)


@pytest.mark.parametrize("log_n", [1, 2, 5, 10])
def test_sizes_outside_1_30_and_roots_are_checked(E, log_n):
    n = 1 << log_n
    root, offset = O.primitive_nth_root(n), 7
    d = rand_poly(random.Random(log_n), 0)
    assert plan(E, [], log_n, root, offset)[0] == SA_ESIZE
    assert plan(E, [1] * (n + 1), log_n, root, offset)[0] == SA_ESIZE
    assert plan(E, d, log_n, O.primitive_nth_root(2 * n), offset)[0] == SA_EROOTORDER
    if log_n > 1:
        assert plan(E, d, log_n, O.primitive_nth_root(n // 2), offset)[0] == SA_ENOTPRIM
    rc, p = plan(E, d, log_n, root, offset)
    assert rc == 0
    lhs = np.zeros((2, n, 2), np.uint64)
    assert apply(E, p, lhs, 0, log_n, root)[0] == SA_ESIZE
    assert apply(E, p, lhs, n + 1, log_n, root)[0] == SA_ESIZE
    assert apply(E, p, np.zeros((2, n + 1, 2), np.uint64), n, log_n, root)[0] == SA_ESIZE
    assert apply(E, p, lhs, n, log_n, O.primitive_nth_root(2 * n))[0] == SA_EROOTORDER
    assert apply(E, p, lhs[:0], n, log_n, root)[0] == 0
    for bad in (0, 31):
        assert plan(E, d, bad, root, offset)[0] == SA_ESIZE
