"""CPU emulation of seeded randomizer draws (tests/emu/emu_sample.cpp over csrc/sample.cuh): the element functions
the kernel runs against hashlib and Python ints, the reduction of 17 bytes mod p at every multiple of p below 2^136
and at the 2^128 boundary, and sa_sample_seeded's checks and index map run thread by thread over a small grid."""
import ctypes
import hashlib
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O
from hostmirror_loader import load_host_types

load_host_types()  # puts the package on sys.path
import sa_stark  # noqa: E402

P = O.P
SA_ESIZE = -6
_vp, _sz, _ci, _u64 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_uint64
STALE = 0x5A5A5A5A5A5A5A5A
SEEDS = [bytes(32), b"\xff" * 32, bytes(random.Random(1).randrange(256) for _ in range(32))]


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu_sample())
    for name, res, args in [("emu_sample_reduce", None, [_vp, ctypes.c_uint32, _u64, _u64]),
                            ("emu_seeded_element", None, [_vp, ctypes.c_char_p, _u64]),
                            ("emu_sample_seeded", _ci, [_vp, ctypes.c_char_p, _sz, _sz, _u64, _sz, _sz, _sz,
                                                        ctypes.c_longlong])]:
        getattr(lib, name).restype = res
        getattr(lib, name).argtypes = args
    return lib


def value(buf):
    return int(buf[0]) | int(buf[1]) << 64


def reduce(E, x):
    out = (ctypes.c_uint64 * 2)()
    E.emu_sample_reduce(out, x >> 128, (x >> 64) & (2**64 - 1), x & (2**64 - 1))
    return value(out)


def element(E, seed, j):
    out = (ctypes.c_uint64 * 2)()
    E.emu_seeded_element(out, seed, j)
    return value(out)


def want(seed, j):
    return int.from_bytes(hashlib.blake2b(seed + j.to_bytes(8, "little")).digest()[:17], "big") % P


def test_seeded_urandom_is_the_contract():
    """the host expansion is blake2b(seed || j as 8 little-endian bytes)[:17], call by call"""
    urandom = sa_stark.seeded_urandom(SEEDS[2])
    for j in range(5):
        assert urandom(17) == hashlib.blake2b(SEEDS[2] + j.to_bytes(8, "little")).digest()[:17]
    for bad in (0, 16, 18, 32):
        with pytest.raises(AssertionError):
            urandom(bad)
    for seed in (b"", bytes(31), bytes(33), "x" * 32, bytearray(32), None):
        with pytest.raises(AssertionError):
            sa_stark.seeded_urandom(seed)


@pytest.mark.parametrize("seed", SEEDS, ids=["zero", "ff", "random"])
def test_elements(E, seed):
    js = list(range(4096)) + [2**32 - 1, 2**32, 2**63, 2**64 - 1]
    for j in js:
        assert element(E, seed, j) == want(seed, j), j


def test_reduction(E):
    """0, 1, p - 1, p, p + 1; k p - 1, k p and k p + 1 for every k up to floor((2^136 - 1) / p); the 2^128 boundary,
    the 2^119 split, the largest 17-byte value and random ones"""
    top = (2**136 - 1) // P
    assert top == 322
    xs = [0, 1, P - 1, P, P + 1, 2**128 - 1, 2**128, 2**128 + 1, 2**136 - 1, 2**119 - 1, 2**119, 407 * 2**119]
    for k in range(2, top + 1):
        xs += [k * P - 1, k * P, k * P + 1]
    rng = random.Random(2)
    xs += [rng.randrange(2**136) for _ in range(2000)]
    for x in xs:
        assert x < 2**136
        assert reduce(E, x) == x % P, x


def run(E, nseeds, seed_stride, first, count, width, lane_stride, n, threads=7, seeds=None):
    seeds = seeds or [bytes(random.Random(100 + b).randrange(256) for _ in range(32)) for b in range(nseeds)]
    out = np.full((n, 2), STALE, dtype=np.uint64)
    rc = E.emu_sample_seeded(out.ctypes.data, b"".join(seeds), nseeds, seed_stride, first, count, width, lane_stride,
                             threads)
    return rc, out, seeds


@pytest.mark.parametrize("width", [1, 2, 3, 5])
@pytest.mark.parametrize("count", [1, 7, 30, 31])
def test_index_map(E, width, count):
    """seed b's draw first + j lands at b seed_stride + (j % width) lane_stride + j // width, every other element
    keeps its stale value; 7 threads loop past their first sweep"""
    nseeds, first = 3, 12345
    lanes = -(-count // width)
    lane_stride = lanes + 2  # a gap after each lane
    seed_stride = width * lane_stride + 3
    n = nseeds * seed_stride + 5
    rc, out, seeds = run(E, nseeds, seed_stride, first, count, width, lane_stride, n)
    assert rc == 0
    expect = {}
    for b in range(nseeds):
        for j in range(count):
            expect[b * seed_stride + (j % width) * lane_stride + j // width] = want(seeds[b], first + j)
    assert len(expect) == nseeds * count
    for i in range(n):
        if i in expect:
            assert value(out[i]) == expect[i], i
        else:
            assert (out[i] == STALE).all(), i


def test_trace_layout(E):
    """width = nregs, lane_stride = T, out at column ncycles of the (B nregs, T) buffer: register-major randomizer
    rows, draw k nregs + s at row k of register s"""
    B, nregs, ncycles, R = 3, 2, 5, 4
    T = ncycles + R
    buf = np.full((B * nregs * T, 2), STALE, dtype=np.uint64)
    seeds = SEEDS
    rc = E.emu_sample_seeded(buf[ncycles:].ctypes.data, b"".join(seeds), B, nregs * T, 0, R * nregs, nregs, T, 5)
    assert rc == 0
    cols = buf.reshape(B, nregs, T, 2)
    for b in range(B):
        for s in range(nregs):
            assert (cols[b, s, :ncycles] == STALE).all()
            for k in range(R):
                assert value(cols[b, s, ncycles + k]) == want(seeds[b], k * nregs + s)


def test_refusals_and_empty_calls(E):
    rc, out, _ = run(E, 2, 10, 0, 5, 0, 1, 20)
    assert rc == SA_ESIZE and (out == STALE).all()
    for nseeds, count in ((0, 5), (2, 0)):
        rc, out, _ = run(E, nseeds, 10, 0, count, 1, 1, 20, seeds=[bytes(32)] * 2)
        assert rc == 0 and (out == STALE).all()
    seeds = [bytes(32)] * 2
    for args in [(2, 10, 2**64 - 4, 5, 1, 1),          # draw index past 2^64 - 1
                 (2, 1 << 59, 0, 5, 1, 1),              # (nseeds - 1) seed_stride
                 (1, 0, 0, 3, 3, 1 << 58),              # (width - 1) lane_stride
                 (2, 2**63, 0, 5, 1, 1),
                 (1, 0, 0, 1 << 59, 1, 1)]:             # item count
        out = np.full((4, 2), STALE, dtype=np.uint64)
        assert E.emu_sample_seeded(out.ctypes.data, b"".join(seeds), *args, 3) == SA_ESIZE, args
        assert (out == STALE).all()
    # the last draw index 2^64 - 1 itself is taken
    rc, out, s = run(E, 1, 4, 2**64 - 4, 4, 1, 1, 4)
    assert rc == 0 and [value(v) for v in out] == [want(s[0], 2**64 - 4 + j) for j in range(4)]
