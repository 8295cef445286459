"""CPU emulation of coset combinations (tests/emu/emu_combine.cpp over csrc/coset.cuh): the library's own check and
schedule of sa_coset_combine_evaluate, with every kernel replaced by a loop over its element function, against the
combination restated with Python ints and the oracle's fast_coset_evaluate (tests/combine_cases.py).  The emulation
starts `out` from a stale pattern, so an element the first group fails to write shows up."""
import ctypes
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O
from combine_cases import P, codeword, make_terms

SA_EROOTORDER, SA_ENOTPRIM, SA_ESIZE = -2, -3, -6


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu_combine())
    sz, vp = ctypes.c_size_t, ctypes.c_void_p
    lib.emu_coset_combine_evaluate.restype = ctypes.c_int
    lib.emu_coset_combine_evaluate.argtypes = [vp, ctypes.c_int, vp, vp, ctypes.POINTER(vp), ctypes.POINTER(sz),
                                               ctypes.POINTER(sz), ctypes.POINTER(ctypes.c_uint64), sz]
    return lib


def run(E, out, log_n, root, offset, rows, terms):
    """emu_coset_combine_evaluate over host copies of the rows; returns the code"""
    arrs = [O.to_np(r) if r else np.zeros((0, 2), np.uint64) for r in rows]
    t = len(terms)
    srcs = (ctypes.c_void_p * t)(*[arrs[r].ctypes.data for r, _, _ in terms])
    lens = (ctypes.c_size_t * t)(*[len(rows[r]) for r, _, _ in terms])
    shifts = (ctypes.c_size_t * t)(*[s for _, s, _ in terms])
    ws = []
    for _, _, w in terms:
        ws += [w & 0xFFFFFFFFFFFFFFFF, w >> 64]
    weights = (ctypes.c_uint64 * (2 * t))(*ws)
    return E.emu_coset_combine_evaluate(O._ptr(out), log_n, O._ptr(O._fe(root)), O._ptr(O._fe(offset)), srcs, lens,
                                        shifts, weights, t)


@pytest.mark.parametrize("offset_kind", ["random", "zero", "one"])
@pytest.mark.parametrize("T", [0, 1, 9, 64, 65, 129])
@pytest.mark.parametrize("log_n", list(range(1, 11)))
def test_combination_matches_oracle(E, log_n, T, offset_kind):
    n = 1 << log_n
    seed = 1000 * log_n + T
    rows, terms = make_terms(seed, n, T)
    root = O.primitive_nth_root(n)
    offset = {"random": random.Random(seed).randrange(2, P), "zero": 0, "one": 1}[offset_kind]
    out = np.zeros((n, 2), np.uint64)
    assert run(E, out, log_n, root, offset, rows, terms) == 0
    assert O.from_np(out) == codeword(rows, terms, n, root, offset)


@pytest.mark.parametrize("log_n", [1, 2, 5, 10])
def test_errors_leave_out_untouched(E, log_n):
    """each refused call returns its code and writes nothing"""
    n = 1 << log_n
    root = O.primitive_nth_root(n)
    rows, terms = make_terms(log_n, n, 9)
    pattern = np.full((n, 2), 0x1234, np.uint64)
    bad_rows = rows + [[1] * (n // 2 + 1)]
    cases = [
        (log_n, root, bad_rows, terms + [(len(rows), n // 2, 5)], SA_ESIZE),  # shift + len = n + 1
        (log_n, root, rows, [(0, n - len(rows[0]) + 1, 1)] + terms, SA_ESIZE),
        (0, root, rows, terms, SA_ESIZE),
        (31, root, rows, terms, SA_ESIZE),
        (log_n, O.primitive_nth_root(2 * n), rows, terms, SA_EROOTORDER),
    ]
    if log_n > 1:
        cases.append((log_n, O.primitive_nth_root(n // 2), rows, terms, SA_ENOTPRIM))
    for lg, r, rs, ts, code in cases:
        out = pattern.copy()
        assert run(E, out, lg, r, 7, rs, ts) == code, (lg, code)
        assert (out == pattern).all(), (lg, code)
