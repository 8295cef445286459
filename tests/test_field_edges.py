"""The field's carry boundaries (tests/field_edges.py) through the two CPU implementations every GPU
parity test trusts: the C oracle (so_fe_*) and the portable field of field.cuh (tests/emu, the code
sa_selftest_field compares the device against).  Expected values are Python ints."""
import ctypes

import numpy as np
import pytest

import __graft_entry__ as G
import field_edges as FE
import oracle as O

P = O.P
RINV = pow(1 << 128, -1, P)


@pytest.fixture(scope="module")
def vectors():
    return FE.build()


@pytest.fixture(scope="module")
def E():
    return ctypes.CDLL(G.build_emu())


def _val(out):
    return int(out[0]) | (int(out[1]) << 64)


def _binary(fn):
    out = np.zeros(2, dtype=np.uint64)

    def call(a, b):
        fn(O._ptr(out), O._ptr(O._fe(a)), O._ptr(O._fe(b)))
        return _val(out)
    return call


def _unary(fn):
    out = np.zeros(2, dtype=np.uint64)

    def call(a):
        fn(O._ptr(out), O._ptr(O._fe(a)))
        return _val(out)
    return call


def test_generator_covers_every_class(vectors):
    muls, addsubs, invs, counts = vectors
    assert len(muls) >= 2000 and len(addsubs) >= 100 and len(invs) >= 64
    # every (e0, e1, e2) pattern twice with e3 == x; e3 == x - 1 borrows unless x == 0 (e0 in {0, 2^31})
    assert counts["e3==x"] >= 2 * 6 ** 3 and counts["e3==x-1"] >= 6 ** 3
    assert FE.build()[:3] == (muls, addsubs, invs)  # deterministic


def test_reduction_model_matches_montgomery(vectors):
    """the class counts rest on device_reduction; it must reproduce a * b * 2^-128 mod p in (-p, p)"""
    for a, b, _ in vectors[0]:
        r = FE.device_reduction(a, b)["r"]
        assert -P < r < P and r % P == a * b * RINV % P


def test_oracle_field_on_boundaries(vectors):
    muls, addsubs, invs, _ = vectors
    L = O.lib()
    mul, add, sub, inv = _binary(L.so_fe_mul), _binary(L.so_fe_add), _binary(L.so_fe_sub), _unary(L.so_fe_inv)
    for a, b, tag in muls:
        assert mul(a, b) == a * b % P, tag
    for a, b, tag in muls + addsubs:
        assert add(a, b) == (a + b) % P, tag
        assert sub(a, b) == (a - b) % P, tag
        assert sub(b, a) == (b - a) % P, tag
    for a in invs + [b for _, b, _ in muls[::16]]:
        assert inv(a) == pow(a, P - 2, P), a
    assert inv(0) == 0


def test_portable_field_on_boundaries(E, vectors):
    muls, addsubs, invs, _ = vectors
    montmul, mul = _binary(E.emu_montmul), _binary(E.emu_mul)
    add, sub, inv = _binary(E.emu_add), _binary(E.emu_sub), _unary(E.emu_inv)
    for a, b, tag in muls:
        assert montmul(a, b) == a * b * RINV % P, tag
        assert mul(a, b) == a * b % P, tag
    for a, b, tag in muls + addsubs:
        assert add(a, b) == (a + b) % P, tag
        assert sub(a, b) == (a - b) % P, tag
        assert sub(b, a) == (b - a) % P, tag
    for a in invs + [b for _, b, _ in muls[::16]]:
        assert inv(a) == pow(a, P - 2, P), a
