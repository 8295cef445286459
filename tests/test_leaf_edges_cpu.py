"""The leaf-encoding edge corpus (tests/leaf_edges.py) on the CPU: its classes are populated, the division
schedule it is built from matches the long division it restates, and the C oracle's decimal encoding and
blake2b, the emulator's run of hash.cuh, and sa_marshal's pack / unpack all agree with str(v).encode() and
hashlib at every corpus value."""
import ctypes
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O
import leaf_edges as LE

P = LE.P


@pytest.fixture(scope="module")
def corpus():
    values, counts, top_q = LE.build()
    return values, counts, top_q


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu())
    lib.emu_decimal.restype = ctypes.c_uint32
    return lib


def test_classes_are_populated(corpus):
    values, counts, top_q = corpus
    assert LE.build()[0] == values  # seeded: the same corpus every time
    assert len(values) == len(set(values)) and values == sorted(values) and 0 <= values[0] and values[-1] < P
    for name in ("lengths", "limbs", "div", "words"):
        assert counts[name] >= LE.MIN_PER_CLASS, name
    for k, i in LE.DIV_POSITIONS:
        for fname, r in LE.FLAVOURS.items():
            key = "div:%d,%d:%s" % (k, i, fname)
            assert counts[key + ":qmax"] >= LE.MIN_PER_CLASS, key
            assert top_q[key] == LE.qmax(k, i, r), key
    # the largest partial quotient is 2^32 - 1 wherever the bound on Q_k leaves a whole word free
    assert [LE.qmax(k, i, 1) == (1 << 32) - 1 for k, i in LE.DIV_POSITIONS] == \
        [True, True, True, False, True, True, False, True, False]
    # the estimate is repaired often, and a plain 1e-8 factor would round some estimates up to q + 1
    assert counts["repair"] >= LE.MIN_PER_CLASS and counts["k=1e-8:q+1"] >= LE.MIN_PER_CLASS
    assert set(len(str(v)) for v in values) == set(range(1, 40))


def test_division_schedule_restatement(corpus):
    """division_visits against the closed form cur = floor(Q_k / 2^(32 i)) mod (1e8 2^32), Q_k = floor(v /
    1e8^k), at the nine positions in the device's order, and its limbs rebuild the value"""
    values = corpus[0]
    for v in values:
        visits = LE.division_visits(v)
        assert [(k, i) for k, i, _ in visits] == LE.DIV_POSITIONS
        for k, i, cur in visits:
            assert cur == ((v // LE.E8**k) >> (32 * i)) % (LE.E8 << 32), (v, k, i)
        # the remainder of each stage's last word is that stage's limb
        limbs = [cur % LE.E8 for k, i, cur in visits if i == 0] + [v // LE.E8**4]
        assert sum(c * LE.E8**j for j, c in enumerate(limbs)) == v


def test_oracle_decimal_and_blake2b(corpus):
    for v in corpus[0]:
        s = str(v).encode()
        assert O.decimal(v) == s, v
        assert O.blake2b(s) == LE.leaf(v), v


def test_emulator_decimal_and_leaf(E, corpus):
    buf = np.zeros(40, dtype=np.uint8)
    d = np.zeros(64, dtype=np.uint8)
    for v in corpus[0]:
        buf[:] = 0xAA  # the encoding must zero the tail itself
        n = E.emu_decimal(O._ptr(buf), O._ptr(O._fe(v)))
        s = str(v).encode()
        assert n == len(s) and buf[:n].tobytes() == s and not buf[n:].any(), v
        E.emu_leaf_digest(O._ptr(d), O._ptr(O._fe(v)))
        assert d.tobytes() == LE.leaf(v), v


def test_marshal_round_trips(corpus):
    G.build_marshal()
    G._paths()
    import sa_marshal
    from hostmirror_loader import load_host_types
    T = load_host_types()
    values = corpus[0]
    want = b"".join(v.to_bytes(16, "little") for v in values)
    fes = [T.fe(v) for v in values]
    for seq in (values, fes):
        buf = sa_marshal.pack(seq)
        assert bytes(buf) == want
        assert sa_marshal.unpack_ints(buf) == values
        ys = sa_marshal.unpack(buf, T.field, T.FieldElement)
        assert [y.value for y in ys] == values
        assert all(type(y) is T.FieldElement and y.field is T.field for y in ys)
        assert [bytes(y) for y in ys] == [str(v).encode() for v in values]
    assert sa_marshal.unpack_ints(bytes(want)) == values


def test_oracle_tree_on_the_corpus(corpus):
    n = 1 << 12
    xs = LE.tile(corpus[0], n, seed=12)
    got = O.merkle_tree_np(O.to_np(xs))
    want = LE.tree(xs)
    assert [bytes(got[i]) for i in range(1, 2 * n)] == want[1:]
    for i in random.Random(1).sample(range(n), 32) + [0, n - 1]:
        path = O.merkle_open(got, i)
        assert LE.climb(xs[i], i, path) == want[1]


@pytest.mark.parametrize("log_h", [0, 1, 3, 6])
def test_fold_preimage(log_h):
    rng = random.Random(log_h)
    h = 1 << log_h
    target = [rng.randrange(P) for _ in range(h)]
    n = 2 * h
    omega, offset, alpha = O.primitive_nth_root(n), O.GENERATOR, rng.randrange(P)
    cw = LE.fold_preimage(target, alpha, offset, omega)
    assert len(cw) == n
    assert LE.fold(cw, alpha, offset, omega) == target
    assert O.from_np(O.fri_fold_np(O.to_np(cw), alpha, offset, omega)) == target
