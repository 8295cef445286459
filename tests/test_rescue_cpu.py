"""The Rescue-Prime kernel's code without a GPU (tests/emu/emu_rescue.cpp runs csrc/rescue.cuh's element functions,
checks and grid-stride index map on the CPU): every recorded hash and trace row; the independent oracle
(tests/emu/rescue_oracle.cpp) pinned to the fixture; the emulation against the oracle at 1, 2, 27 and the cap's
rounds with random constants, and at the exponents' edge values; the index map at the prover's shapes and with
lane_stride 1, hash-only and trace-only, with every untouched element left stale; and each refusal."""
import random

import numpy as np
import pytest

import rescue_cases as R

P = R.P
STALE = np.uint64(0x5A5A5A5A5A5A5A5A)


def golden_inputs():
    g = R.golden()
    return [int(c["input"]) for c in g["cases"]]


def test_fixture_covers_the_named_inputs():
    g = R.golden()
    assert (g["m"], g["N"], len(g["mds"]), len(g["round_constants"])) == (2, 27, 4, 4 * 27)
    xs = golden_inputs()
    for x in (0, 1, 2, P - 2, P - 1, (1 << 64) - 1, 1 << 64, 1 << 119, 1 << 127,
              57322816861100832358702415967512842988):
        assert x in xs
    assert sum(c["kind"] == "signature_key" for c in g["cases"]) == 4
    assert sum(c["kind"] == "random" for c in g["cases"]) == 16


def test_python_restatement_matches_the_fixture():
    g = R.golden()
    a, ainv = R.exponents()
    for c in g["cases"][:12]:
        h, rows = R.python_rescue(int(c["input"]), R.constants(), 27, a, ainv)
        assert str(h) == c["hash"] and [[str(v) for v in row] for row in rows] == c["trace"]


def test_oracle_matches_the_fixture():
    g = R.golden()
    a, ainv = R.exponents()
    hashes, traces = R.oracle(R.to_np(golden_inputs()), R.to_np(R.constants()), 27, a, ainv)
    got = R.dense_trace(traces)
    for c, h, t in zip(g["cases"], R.from_np(hashes), got):
        assert str(h) == c["hash"]
        assert [[str(v) for v in row] for row in t] == c["trace"]


@pytest.mark.parametrize("threads", [1, 7, 64])
def test_emulation_matches_every_golden_hash_and_row(threads):
    g = R.golden()
    a, ainv = R.exponents()
    xs = golden_inputs()
    n = len(xs)
    hashes = np.zeros((n, 2), np.uint64)
    trace = np.zeros((n * 2 * 28, 2), np.uint64)
    assert R.emu(hashes, trace, R.to_np(xs), R.to_np(R.constants()), 27, a, ainv, 56, 28, threads) == 0
    got = R.dense_trace(trace.reshape(n, 2, 28, 2))
    for c, h, t in zip(g["cases"], R.from_np(hashes), got):
        assert str(h) == c["hash"]
        assert [[str(v) for v in row] for row in t] == c["trace"]


@pytest.mark.parametrize("rounds", [1, 2, 27, R.MAX_ROUNDS])
def test_emulation_equals_the_oracle_with_random_constants(rounds):
    rng = random.Random(rounds)
    consts = [rng.randrange(P) for _ in range(4 + 4 * rounds)]
    a, ainv = R.exponents()
    xs = [rng.randrange(P) for _ in range(5 if rounds == R.MAX_ROUNDS else 21)] + [0, P - 1]
    hashes = np.zeros((len(xs), 2), np.uint64)
    trace = np.zeros((len(xs) * 2 * (rounds + 1), 2), np.uint64)
    assert R.emu(hashes, trace, R.to_np(xs), R.to_np(consts), rounds, a, ainv, 2 * (rounds + 1), rounds + 1) == 0
    want_h, want_t = R.oracle(R.to_np(xs), R.to_np(consts), rounds, a, ainv)
    assert np.array_equal(hashes, want_h) and np.array_equal(trace, want_t.reshape(-1, 2))
    if rounds <= 2:
        for i, x in enumerate(xs[:3]):
            h, rows = R.python_rescue(x, consts, rounds, a, ainv)
            assert R.from_np(hashes[i])[0] == h
            assert R.dense_trace(want_t[i:i + 1])[0] == rows


EXPONENTS = [0, 1, 2, 3, 5, 180331931428153586757283157844700080811, P - 2, (1 << 128) - 1]


@pytest.mark.parametrize("e", EXPONENTS, ids=lambda e: "e%d" % e.bit_length())
def test_exponents(e):
    rng = random.Random(e % 1000)
    assert all(R.oracle_pow(x, e) == pow(x, e, P) for x in [0, 1, P - 1, 2, rng.randrange(P)])
    consts = [rng.randrange(P) for _ in range(4 + 4 * 2)]
    xs = [0, 1, P - 1] + [rng.randrange(P) for _ in range(6)]
    for alpha, alphainv in ((e, 3), (3, e), (e, e)):
        hashes = np.zeros((len(xs), 2), np.uint64)
        trace = np.zeros((len(xs) * 6, 2), np.uint64)
        assert R.emu(hashes, trace, R.to_np(xs), R.to_np(consts), 2, alpha, alphainv, 6, 3) == 0
        for i, x in enumerate(xs):
            h, rows = R.python_rescue(x, consts, 2, alpha, alphainv)
            assert R.from_np(hashes[i])[0] == h
            assert R.dense_trace(trace[6 * i:6 * i + 6].reshape(1, 2, 3, 2))[0] == rows


def _index_map(count, inst_stride, lane_stride, with_hashes, with_trace, rounds=27):
    rng = random.Random(count * 31 + lane_stride)
    xs = [rng.randrange(P) for _ in range(count)]
    a, ainv = R.exponents()
    size = (count - 1) * inst_stride + lane_stride + rounds + 1 + 9
    hashes = np.full((count + 3, 2), STALE) if with_hashes else None
    trace = np.full((size, 2), STALE) if with_trace else None
    assert R.emu(hashes, trace, R.to_np(xs), R.to_np(R.constants()), rounds, a, ainv, inst_stride, lane_stride, 7) == 0
    want_h, want_t = R.oracle(R.to_np(xs), R.to_np(R.constants()), rounds, a, ainv)
    if with_hashes:
        assert np.array_equal(hashes[:count], want_h) and (hashes[count:] == STALE).all()
    if with_trace:
        expect = np.full((size, 2), STALE)
        for b in range(count):
            for s in range(2):
                at = b * inst_stride + s * lane_stride
                expect[at:at + rounds + 1] = want_t[b, s]
        assert np.array_equal(trace, expect)


@pytest.mark.parametrize("count", [1, 3, 17])
@pytest.mark.parametrize("outputs", ["both", "hash", "trace"])
def test_index_map_at_the_prover_shapes(count, outputs):
    T = 28 + 256  # a signature's randomized trace length
    _index_map(count, 2 * T, T, outputs != "trace", outputs != "hash")


@pytest.mark.parametrize("count", [1, 3, 17])
def test_index_map_with_interleaved_registers(count):
    # lane_stride 1: register 1's row r lands on register 0's row r + 1.  One thread writes an input's rows in
    # order, register 0 before register 1, so register 0's rows 0 .. N stay and register 1's row N follows them; a
    # wide inst_stride leaves stale elements between inputs
    rng = random.Random(count)
    xs = [rng.randrange(P) for _ in range(count)]
    a, ainv = R.exponents()
    trace = np.full((count * 40 + 40, 2), STALE)
    assert R.emu(None, trace, R.to_np(xs), R.to_np(R.constants()), 27, a, ainv, 40, 1, 7) == 0
    _, want_t = R.oracle(R.to_np(xs), R.to_np(R.constants()), 27, a, ainv)
    expect = np.full((count * 40 + 40, 2), STALE)
    for b in range(count):
        expect[b * 40 + 1:b * 40 + 29] = want_t[b, 1]
        expect[b * 40:b * 40 + 28] = want_t[b, 0]
    assert np.array_equal(trace, expect)


def test_refusals():
    a, ainv = R.exponents()
    xs = R.to_np([1, 2])
    kc = R.to_np(R.constants() + [0] * (4 * (R.MAX_ROUNDS + 1) - 4 * 27))
    h = np.full((2, 2), STALE)
    t = np.full((2 * 2 * (R.MAX_ROUNDS + 2), 2), STALE)
    ESIZE = -6
    assert R.emu(None, None, xs, kc, 27, a, ainv, 56, 28) == ESIZE
    assert R.emu(h, None, xs, kc, 0, a, ainv, 56, 28) == ESIZE
    assert R.emu(h, None, xs, kc, R.MAX_ROUNDS + 1, a, ainv, 56, 28) == ESIZE
    assert R.emu(h, t, xs, kc, R.MAX_ROUNDS + 1, a, ainv, 2 * (R.MAX_ROUNDS + 2), R.MAX_ROUNDS + 2) == ESIZE
    assert (h == STALE).all() and (t == STALE).all()
    # a largest offset (count - 1) inst_stride + lane_stride + rounds of exactly 2^59 is refused, and so is a stride
    # whose product overflows
    assert R.emu(None, t, xs, kc, 27, a, ainv, (1 << 59) - 27, 0) == ESIZE
    assert R.emu(None, t, xs, kc, 27, a, ainv, 1 << 63, 0) == ESIZE
    assert R.emu(None, t, xs, kc, 27, a, ainv, 1 << 59, 0) == ESIZE
    assert R.emu(None, t, xs[:1], kc, 27, a, ainv, 0, (1 << 59) - 27) == ESIZE
    assert R.emu(None, t, xs[:1], kc, 27, a, ainv, 0, 1 << 62) == ESIZE
    assert R.emu(h, None, np.zeros((0, 2), np.uint64), kc, R.MAX_ROUNDS + 1, a, ainv, 0, 0) == ESIZE
    assert (t == STALE).all()
    # count 0: SA_OK, nothing written, even with out-of-range strides; the cap itself is taken
    assert R.emu(h, t, xs[:0], kc, 27, a, ainv, 1 << 62, 1 << 62) == 0
    assert (h == STALE).all() and (t == STALE).all()
    assert R.emu(h, t, xs, kc, R.MAX_ROUNDS, a, ainv, R.MAX_ROUNDS + 1 + 1, 0) == 0
    want_h, _ = R.oracle(xs, kc, R.MAX_ROUNDS, a, ainv, trace=False)
    assert np.array_equal(h, want_h)
