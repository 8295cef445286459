"""CPU emulation of the subproduct tree (tests/emu/emu.cpp over csrc/poly_tree.cuh) against the oracle: the
library's own schedule of the tree zerofier, the walk down the tree (sa_poly_eval_mode 2), the interpolation plan
build and the batched apply, with every kernel replaced by a loop over its element function.  The emulation takes
the tree at any k >= 1, so full and ragged trees of a few points are checked without a GPU."""
import ctypes
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O

P = O.P
SA_EDIVZERO = -4
FE = 16  # bytes per field element


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu())
    for fn in ("emu_zerofier", "emu_poly_eval_walk", "emu_interp_plan", "emu_interp_apply_batch"):
        getattr(lib, fn).restype = ctypes.c_int
    lib.emu_interp_plan_bytes.restype = ctypes.c_size_t
    lib.emu_interp_plan_bytes.argtypes = [ctypes.c_size_t]
    return lib


def _rand(rng, n):
    return O.to_np([rng.randrange(P) for _ in range(n)])


def _distinct(rng, k):
    pts = set()
    while len(pts) < k:
        pts.add(rng.randrange(P))
    return O.to_np(sorted(pts, key=lambda _: rng.random()))


def _plan(E, domain, walk):
    k = domain.shape[0]
    plan = np.zeros(E.emu_interp_plan_bytes(k), dtype=np.uint8)
    rc = E.emu_interp_plan(O._ptr(plan), O._ptr(domain), ctypes.c_size_t(k), int(walk))
    return rc, plan


def _apply(E, plan, values):
    batch, k = values.shape[0], values.shape[1]
    out = np.zeros_like(values)
    assert E.emu_interp_apply_batch(O._ptr(out), O._ptr(plan), O._ptr(values), ctypes.c_size_t(k),
                                    ctypes.c_size_t(batch)) == 0
    return out


@pytest.mark.parametrize("k", list(range(1, 71)) + [127, 128, 129, 300, 513])
def test_tree_zerofier(E, k):
    d = _rand(random.Random(1000 + k), k)
    out = np.zeros((k + 1, 2), dtype=np.uint64)
    assert E.emu_zerofier(O._ptr(out), O._ptr(d), ctypes.c_size_t(k)) == 0
    assert (out == O.zerofier_np(d)).all()


@pytest.mark.parametrize("k", list(range(1, 34)))
def test_walk_matches_horner(E, k):
    rng = random.Random(2000 + k)
    pts = _rand(rng, k)
    pts[k // 2] = pts[0]  # a repeated point
    for ncoef in sorted({1, max(k - 1, 1), k, k + 1, 3 * k + 1}):
        for f in (_rand(rng, ncoef), np.zeros((ncoef, 2), dtype=np.uint64)):  # and the zero polynomial
            out = np.zeros_like(pts)
            assert E.emu_poly_eval_walk(O._ptr(out), O._ptr(f), ctypes.c_size_t(ncoef), O._ptr(pts),
                                        ctypes.c_size_t(k)) == 0
            assert (out == O.poly_eval_np(f, pts)).all(), (k, ncoef)


@pytest.mark.parametrize("k", list(range(1, 41)) + [100, 257])
def test_plan_and_batched_apply(E, k):
    rng = random.Random(3000 + k)
    d = _distinct(rng, k)
    rc, plan = _plan(E, d, walk=False)
    assert rc == 0
    rc, plan_walk = _plan(E, d, walk=True)
    assert rc == 0
    assert plan_walk.tobytes() == plan.tobytes()  # M'(d_i) by the walk == by Horner
    for batch in (1, 2, 5):
        v = _rand(rng, batch * k).reshape(batch, k, 2)
        if batch > 1:
            v[-1] = v[0]  # two equal rows
            v[1] = 0  # a zero row (at B = 2 it replaces the copy)
        out = _apply(E, plan, v)
        for b in range(batch):
            assert (out[b] == O.interpolate_np(d, v[b])).all(), (k, batch, b)


@pytest.mark.parametrize("k", [2, 5, 33])
def test_coincident_points(E, k):
    d = _distinct(random.Random(4000 + k), k)
    d[k - 1] = d[0]
    for walk in (False, True):
        assert _plan(E, d, walk)[0] == SA_EDIVZERO


@pytest.fixture(scope="module")
def lib():
    G.build_cuda()
    G._paths()
    import sa_engine
    return sa_engine.load_library()


@pytest.mark.parametrize("k", [1025, 2048, 4097, 5000, 1 << 16, (1 << 16) + 1, 1 << 20])
def test_plan_layout_is_the_library_s(E, lib, k):
    """above 1024 points the library builds the tree plan the emulation builds"""
    assert E.emu_interp_plan_bytes(k) == lib.sa_interp_plan_bytes(k)


def test_small_tree_plan_layout(E):
    for k in (1, 2, 3, 16, 17, 1024):
        log_k = (k - 1).bit_length()
        sec = lambda n: (n + 15) // 16 * 16  # noqa: E731
        assert E.emu_interp_plan_bytes(k) == FE * (sec(log_k * 2 * (1 << log_k)) + sec(1 << log_k))
    assert E.emu_interp_plan_bytes(0) == 0 and E.emu_interp_plan_bytes((1 << 20) + 1) == 0
