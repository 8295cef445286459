"""Batched Merkle trees (sa_merkle_tree_batch) through the CPU emulation (tests/emu/emu_merkle.cpp): the library's
batch loop, per-tree views
and launch schedule (csrc/fri_merkle.cuh) over emulated CTAs, checked tree by tree against the oracle.  The fused
top, which needs the device's arrival counters, is checked on the GPU (test_gpu_merkle_batch.py)."""
import ctypes
import hashlib
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O

P = O.P
MK_MAX_TREES = 65535  # trees per launch (csrc/fri_merkle.cuh)


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu_merkle())
    lib.emu_merkle_tree_batch.restype = ctypes.c_int
    return lib


def rows(seed, batch, n):
    rng = random.Random(seed)
    x = np.stack([O.to_np([rng.randrange(P) for _ in range(n)]) for _ in range(batch)])
    x[:, 0] = 0
    if n > 4:  # the edge values of test_gpu.py::test_merkle_tree_and_open
        x[:, 1] = (7, 0)
        x[:, 2] = O._fe(10**19)
        x[:, 3] = O._fe(P - 1)
    return x


def trees_of(E, x):
    batch, n = x.shape[0], x.shape[1]
    trees = np.full((batch, 2 * n, 64), 0xA5, dtype=np.uint8)  # node 0 must be written, not found zero
    x = np.ascontiguousarray(x)
    assert E.emu_merkle_tree_batch(O._ptr(trees), O._ptr(x), ctypes.c_size_t(n), ctypes.c_size_t(batch)) == 0
    return trees


def check(trees, x):
    for b in range(x.shape[0]):
        assert (trees[b, 0] == 0).all(), b
        assert (trees[b, 1:] == O.merkle_tree_np(x[b])[1:]).all(), b


@pytest.mark.parametrize("batch", [1, 2, 3, 5])
@pytest.mark.parametrize("logn", range(14))
def test_batch_matches_oracle(E, logn, batch):
    x = rows(100 * logn + batch, batch, 1 << logn)
    check(trees_of(E, x), x)


@pytest.mark.parametrize("rows_spec", [
    [(8, 2, 10, 3, 0), (0, 0, 3, 1, 64)],    # partial in-CTA reduction; tiny launches of 8-node CTAs one level each
    [(12, 3, 11, 2, 16), (6, 1, 6, 0, 0)],  # eight bottom nodes per thread; two per thread without shared phase
])
def test_batch_other_launch_shapes(E, rows_spec):
    spec = ",".join(":".join(str(v) for v in r) for r in rows_spec).encode()  # SA_MK_SHAPE form
    try:
        E.emu_set_merkle_shape(spec)
        for logn in (3, 6, 10, 13):
            for batch in (1, 3):
                x = rows(7 * logn + batch, batch, 1 << logn)
                check(trees_of(E, x), x)
    finally:
        E.emu_set_merkle_shape(b"")


@pytest.mark.parametrize("logn", [0, 6, 12])
def test_equal_rows_and_zero_row(E, logn):
    n = 1 << logn
    x = rows(9 + logn, 4, n)
    x[2] = x[0]
    x[3] = 0
    trees = trees_of(E, x)
    check(trees, x)
    assert (trees[0] == trees[2]).all()
    assert (trees[3, 1:] == O.merkle_tree_np(np.zeros((n, 2), dtype=np.uint64))[1:]).all()


def test_batch_past_one_launch(E):
    """more trees than one launch takes: the second group starts at tree MK_MAX_TREES, with its own rows"""
    batch = MK_MAX_TREES + 2
    x = np.zeros((batch, 1, 2), dtype=np.uint64)
    x[:, 0, 0] = np.arange(batch, dtype=np.uint64)
    trees = trees_of(E, x)
    assert (trees[:, 0] == 0).all()
    for b in list(range(3)) + list(range(MK_MAX_TREES - 2, batch)):
        assert trees[b, 1].tobytes() == hashlib.blake2b(str(b).encode()).digest(), b  # merkle.py:13, one leaf
