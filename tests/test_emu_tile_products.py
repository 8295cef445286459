"""Field products the NTT tile issues (tests/emu/emu_tile_count.cpp), per thread and phase, for the launched tile
shapes with a middle stage: the middle stage parks its outputs unmultiplied and the last stage applies those
twiddles on load except on its m = 0 rows, every thread of a phase issues the same number of products, and the
outputs are the oracle's."""
import ctypes
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O

P = O.P
E_PTS = 16                    # elements per thread (16-point register transforms)
DFT = {16: 17, 4: 1, 2: 0}    # products of an R-point register transform (the k = 0 butterflies are add/sub only)


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu_tile_count())
    lib.emu_tile_products.restype = ctypes.c_int
    return lib


@pytest.mark.parametrize("logl,c", [(10, 4), (9, 4), (10, 8), (9, 8)])
def test_tile_products_per_phase(E, logl, c):
    L = 1 << logl
    units = L // E_PTS                  # 16-point units per column in each full stage
    tpt = units * c                     # threads per tile
    r_last = 1 << (logl - 8)            # 16 * 16 * 4 at 2^10, 16 * 16 * 2 at 2^9
    rng = random.Random(900 + 10 * logl + c)
    x = O.to_np([rng.randrange(P) for _ in range(L * c)])
    out = np.zeros_like(x)
    counts = np.zeros(3 * tpt, dtype=np.int64)
    w = O.primitive_nth_root(L)
    assert E.emu_tile_products(O._ptr(out), O._ptr(x), logl, c, O._ptr(O._fe(w)), O._ptr(counts)) == 0
    for j in range(c):
        assert (out[j * L:(j + 1) * L] == O.ntt_np(w, x[j * L:(j + 1) * L])).all(), j

    first, middle, last = counts.reshape(3, tpt)
    # first stage: the 16-point transform and 15 inter-stage twiddles
    assert (first == DFT[16] + E_PTS - 1).all()
    # middle stage: the 16-point transform only
    assert (middle == DFT[16]).all()
    # last stage: per radix-r_last unit its transform and the r_last - 1 twiddles of the rows with m != 0
    assert (last == (E_PTS // r_last) * (DFT[r_last] + r_last - 1)).all()

    # per column: 4352 -> 4160 products at 2^10 (4.25 -> 4.06 per point), 2048 -> 1824 at 2^9 (4.0 -> 3.56);
    # the saving is the middle stage's m = 0 twiddles (all w^0) less the last stage's k = 0 rows, which still multiply
    per_col = counts.sum() // c
    assert counts.sum() == c * per_col
    before = 2 * units * (DFT[16] + E_PTS - 1) + (L // r_last) * DFT[r_last]
    m_values = r_last                   # M of the middle stage
    skipped = (units // m_values) * (E_PTS - 1) - (units // m_values) * (m_values - 1)
    assert per_col == before - skipped
    assert (before, per_col) == {10: (4352, 4160), 9: (2048, 1824)}[logl]
