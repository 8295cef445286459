"""The NTT tile's own product and butterfly (tile_mul / tile_bfly in csrc/ntt_tile.cuh) against the portable
field, on the H100 (``pytest -m gpu``): the carry-boundary operand pairs of tests/field_edges.py, their
Montgomery-shifted twins, and sa_selftest_tile's random and edge draws."""
import os
import sys

import numpy as np
import pytest

import field_edges as FE

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "stark-anatomy_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)
import sa_engine  # noqa: E402

pytestmark = pytest.mark.gpu
P = FE.P
RINV = pow(1 << 128, -1, P)
M64 = (1 << 64) - 1
SA_ESIZE = -6


@pytest.fixture(scope="module")
def lib():
    sa_engine.set_engine(None)
    e = sa_engine.get_engine()  # raises without CUDA / without the built library
    assert e.name == "cuda"
    return e.lib


def _pairs(pairs):
    words = np.array([w for a, b in pairs for v in (a, b) for w in (v & M64, v >> 64)], dtype=np.uint64)
    return words, words.ctypes.data_as(sa_engine._u64p)


def test_tile_bfly_on_carry_boundaries(lib):
    """the product pairs of field_edges drive every borrow and add-back of the reduction; with the first
    operand times 2^-128 the same pairs also meet the product the way a twiddle in Montgomery form does"""
    muls = FE.build()[0]
    pairs = [(a, b) for a, b, _ in muls] + [(b, a) for a, b, _ in muls] + [(a * RINV % P, b) for a, b, _ in muls]
    words, ptr = _pairs(pairs)
    assert lib.sa_selftest_tile(0, 11, ptr, len(pairs)) == 0
    assert lib.sa_selftest_tile(1 << 16, 12, ptr, len(pairs)) == 0


def test_tile_bfly_random_and_edges(lib):
    assert lib.sa_selftest_tile(1 << 22, 2026, None, 0) == 0


def test_tile_selftest_refuses_non_elements(lib):
    """an operand at or above p, or a missing list, is SA_ESIZE before any launch"""
    for pair in [(1, P), (P + (1 << 64), 1), ((1 << 128) - 1, 1)]:
        words, ptr = _pairs([pair])
        assert lib.sa_selftest_tile(16, 1, ptr, 1) == SA_ESIZE
    assert lib.sa_selftest_tile(16, 1, None, 1) == SA_ESIZE
