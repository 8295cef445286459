"""CPU emulation of what proving many statements of one AIR at once adds (tests/emu/emu_batch.cpp): the batched
applies of csrc/air.cuh give every trace the rows (and exact-division flags) of the single apply on that trace alone,
across chunks of traces and of rows; the combination into many rows gives each row the single combination of its own
terms; the gathers and Merkle paths with an index set per group read each group's own indices; and every error
leaves the outputs untouched."""
import ctypes
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O
from test_air_cpu import plan
from test_air_exact_cpu import exact_case

SA_EINDEX, SA_ESIZE = -5, -6


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu_batch())
    sz, vp, ci = ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int
    lib.emu_air_plan_bytes.restype = sz
    lib.emu_air_plan_bytes.argtypes = [ci, sz, sz, sz]
    lib.emu_air_plan.restype = ci
    lib.emu_air_plan.argtypes = [vp, vp, vp, vp, sz, sz, sz, vp, sz, ci, vp, vp, vp]
    lib.emu_air_quotients.argtypes = [vp, vp, vp, sz, sz, sz, sz, ci, vp]
    lib.emu_air_quotients_exact.argtypes = [vp, vp, vp, vp, sz, sz, sz, sz, sz, ci, vp]
    lib.emu_air_quotients_batch.argtypes = [vp, vp, vp, sz, sz, sz, sz, sz, ci, vp, sz, sz]
    lib.emu_air_quotients_exact_batch.argtypes = [vp, vp, vp, vp, sz, sz, sz, sz, sz, sz, ci, vp, sz, sz]
    lib.emu_air_batch_max.restype = sz
    lib.emu_air_batch_max.argtypes = [sz, sz, ci]
    lib.emu_coset_combine_evaluate_batch.argtypes = [vp, sz, ci, vp, vp, vp, vp, vp, vp, vp, sz]
    lib.emu_gather_batch_sets.argtypes = [vp, vp, sz, sz, sz, vp, sz]
    lib.emu_merkle_open_batch_sets.argtypes = [vp, vp, sz, sz, sz, vp, sz]
    return lib


def traces_of(seed, batch, nregs, ncoef):
    rng = random.Random(seed)
    return [[[rng.randrange(O.P) for _ in range(ncoef)] for _ in range(nregs)] for _ in range(batch)]


def singles(E, buf, traces, ncons, qlen, tail, log_n, root):
    """each trace's exact apply alone: (rows (B, ncons * qlen, 2), flags (B, ncons))"""
    rows, flags = [], []
    for tr in traces:
        out = np.zeros((ncons * qlen, 2), np.uint64)
        f = np.zeros(ncons, np.uint32)
        t = O.to_np([v for row in tr for v in row])
        assert E.emu_air_quotients_exact(O._ptr(out), O._ptr(f), O._ptr(buf), O._ptr(t), len(tr), len(tr[0]), qlen,
                                         ncons, tail, log_n, O._ptr(O._fe(root))) == 0
        rows.append(out)
        flags.append(f)
    return np.stack(rows), np.stack(flags)


def batched(E, buf, traces, ncons, qlen, tail, log_n, root, chunk=(0, 0)):
    """(rc, plain rows, exact rows, flags) of the batched applies"""
    B, nregs, ncoef = len(traces), len(traces[0]), len(traces[0][0])
    t = O.to_np([v for tr in traces for row in tr for v in row])
    plain = np.zeros((B, ncons * qlen, 2), np.uint64)
    rc = E.emu_air_quotients_batch(O._ptr(plain), O._ptr(buf), O._ptr(t), nregs, ncoef, qlen, ncons, B, log_n,
                                   O._ptr(O._fe(root)), *chunk)
    assert rc == 0
    out = np.zeros_like(plain)
    flags = np.zeros((B, ncons), np.uint32)
    rc = E.emu_air_quotients_exact_batch(O._ptr(out), O._ptr(flags), O._ptr(buf), O._ptr(t), nregs, ncoef, qlen,
                                         ncons, B, tail, log_n, O._ptr(O._fe(root)), *chunk)
    return rc, plain, out, flags


def check(E, seed, log_n, nregs, batch, ncons=3, chunk=(0, 0)):
    n = 1 << log_n
    air, trace, z, max_ncoef, root, offset, step, qlen = exact_case(seed, log_n, nregs, ncons)
    rc, buf = plan(E, air, nregs, max_ncoef, z, log_n, root, offset, step)
    assert rc == 0
    traces = [trace] + traces_of(seed, batch - 1, nregs, len(trace[0]))
    tail = n - (len(z) - 1)
    want_rows, want_flags = singles(E, buf, traces, ncons, qlen, tail, log_n, root)
    rc, plain, out, flags = batched(E, buf, traces, ncons, qlen, tail, log_n, root, chunk)
    assert rc == 0
    assert np.array_equal(out, want_rows) and np.array_equal(plain, want_rows)
    assert np.array_equal(flags, want_flags)


@pytest.mark.parametrize("batch", [1, 2, 5])
@pytest.mark.parametrize("nregs", [1, 2, 3])
@pytest.mark.parametrize("log_n", list(range(1, 11)))
def test_batched_apply_is_each_traces_apply(E, log_n, nregs, batch):
    check(E, 100 * log_n + 10 * nregs + batch, log_n, nregs, batch)


@pytest.mark.parametrize("chunk", [(1, 1), (2, 1), (2, 4), (3, 2), (4, 5), (1, 2)])
def test_batched_apply_across_chunks(E, chunk):
    """chunks of traces and of rows that do not divide the batch's or one trace's rows"""
    for log_n in (3, 6):
        check(E, 7 + log_n, log_n, 2, 5, ncons=3, chunk=chunk)


def test_batch_max_rule(E):
    for log_n in (1, 10, 16, 20, 26, 30):
        cap = max(1, (1 << 30) // (32 << log_n))
        for nregs, ncons in ((2, 4), (1, 1), (9, 9), (1, 10 ** 6)):
            assert E.emu_air_batch_max(nregs, ncons, log_n) == max(1, cap // (2 * nregs + ncons))
    assert E.emu_air_batch_max(2, 4, 31) == 0 and E.emu_air_batch_max(2, 4, 16) == 64


def test_batched_apply_errors_leave_outputs_untouched(E):
    log_n, nregs, ncons, batch = 4, 2, 2, 3
    n = 1 << log_n
    air, trace, z, max_ncoef, root, offset, step, qlen = exact_case(3, log_n, nregs, ncons)
    rc, buf = plan(E, air, nregs, max_ncoef, z, log_n, root, offset, step)
    assert rc == 0
    t = O.to_np([v for tr in [trace] * batch for row in tr for v in row])
    good = dict(nregs=nregs, ncoef=len(trace[0]), qlen=qlen, ncons=ncons, tail=n - (len(z) - 1), log_n=log_n,
                root=root)
    bad = [dict(tail=n + 1), dict(qlen=0), dict(qlen=n + 1), dict(ncons=0), dict(nregs=0), dict(ncoef=0),
           dict(ncoef=n + 1), dict(log_n=31), dict(root=O.primitive_nth_root(n * 2))]
    for change in bad:
        a = dict(good, **change)
        out = np.full((batch * max(1, a["ncons"]) * max(1, a["qlen"]), 2), 0x1234, np.uint64)
        flags = np.full(batch * 2, 0x77, np.uint32)
        args = (O._ptr(buf), O._ptr(t), a["nregs"], a["ncoef"], a["qlen"], a["ncons"], batch)
        assert E.emu_air_quotients_exact_batch(O._ptr(out), O._ptr(flags), *args, a["tail"], a["log_n"],
                                               O._ptr(O._fe(a["root"])), 0, 0) != 0, change
        if "tail" not in change:
            assert E.emu_air_quotients_batch(O._ptr(out), *args, a["log_n"], O._ptr(O._fe(a["root"])), 0, 0) != 0
        assert (out == 0x1234).all() and (flags == 0x77).all(), change
    out = np.full((4, 2), 0x1234, np.uint64)  # an empty batch writes nothing
    assert E.emu_air_quotients_batch(O._ptr(out), O._ptr(buf), O._ptr(t), nregs, len(trace[0]), qlen, ncons, 0, log_n,
                                     O._ptr(O._fe(root)), 0, 0) == 0 and (out == 0x1234).all()


# ---- combinations into many rows ----
def combine(E, log_n, root, offset, srcs, terms, nrows):
    """terms (src index, shift, weight, row): (rc, out (nrows, n, 2))"""
    n = 1 << log_n
    out = np.zeros((max(nrows, 1), n, 2), np.uint64)
    arrs = [O.to_np(s) for s in srcs]
    T = len(terms)
    ptrs = (ctypes.c_void_p * max(T, 1))(*[O._ptr(arrs[i]) for i, _, _, _ in terms])
    lens = np.array([len(srcs[i]) for i, _, _, _ in terms] or [0], np.uintp)
    shifts = np.array([s for _, s, _, _ in terms] or [0], np.uintp)
    rows = np.array([r for _, _, _, r in terms] or [0], np.uintp)
    w = np.array([x for _, _, wt, _ in terms for x in (wt & (2 ** 64 - 1), wt >> 64)] or [0], np.uint64)
    rc = E.emu_coset_combine_evaluate_batch(O._ptr(out), nrows, log_n, O._ptr(O._fe(root)), O._ptr(O._fe(offset)),
                                            ptrs, O._ptr(lens), O._ptr(shifts), O._ptr(rows), O._ptr(w), T)
    return rc, out


@pytest.mark.parametrize("nrows,T", [(1, 3), (3, 7), (5, 130), (4, 0), (6, 65)])
@pytest.mark.parametrize("log_n", [3, 7])
def test_combination_rows_are_single_combinations(E, log_n, nrows, T):
    n = 1 << log_n
    rng = random.Random(31 * log_n + nrows + T)
    root, offset = O.primitive_nth_root(n), rng.randrange(1, O.P)
    srcs = [[rng.randrange(O.P) for _ in range(rng.randrange(0, n // 2 + 1))] for _ in range(5)]
    terms = []
    for _ in range(T):
        i = rng.randrange(5)
        terms.append((i, rng.randrange(n - len(srcs[i]) + 1), rng.randrange(O.P), rng.randrange(nrows)))
    rc, out = combine(E, log_n, root, offset, srcs, terms, nrows)
    assert rc == 0
    for r in range(nrows):
        c = [0] * n
        for i, s, w, row in terms:
            if row == r:
                for j, v in enumerate(srcs[i]):
                    c[s + j] = (c[s + j] + w * v) % O.P
        want = O.fast_coset_evaluate(c, offset, root, n) if any(s + len(srcs[i]) for i, s, _, _ in terms) else [0] * n
        assert O.from_np(out[r]) == want, r


def test_combination_errors_leave_out_untouched(E):
    log_n, n = 4, 16
    root = O.primitive_nth_root(n)
    srcs = [[1, 2, 3]]
    for terms, nrows in (([(0, 0, 5, 2)], 2), ([(0, 14, 5, 0)], 1), ([(0, 0, 5, 0)], 0)):
        out = np.full((max(nrows, 1), n, 2), 0x1234, np.uint64)
        arr = O.to_np(srcs[0])
        ptrs = (ctypes.c_void_p * 1)(O._ptr(arr))
        rc = E.emu_coset_combine_evaluate_batch(
            O._ptr(out), nrows, log_n, O._ptr(O._fe(root)), O._ptr(O._fe(3)), ptrs,
            O._ptr(np.array([3], np.uintp)), O._ptr(np.array([terms[0][1]], np.uintp)),
            O._ptr(np.array([terms[0][3]], np.uintp)), O._ptr(np.array([5, 0], np.uint64)), 1)
        assert rc == SA_ESIZE and (out == 0x1234).all()


# ---- openings with an index set per group ----
@pytest.mark.parametrize("batch,group", [(1, 1), (6, 3), (7, 3), (4, 4), (5, 1)])
def test_gather_and_paths_read_each_groups_set(E, batch, group):
    log_n, k = 5, 6
    n = 1 << log_n
    rng = random.Random(batch * 10 + group)
    vals = O.to_np([rng.randrange(O.P) for _ in range(batch * n)]).reshape(batch, n, 2)
    trees = np.stack([O.merkle_tree_np(v) for v in vals])
    nsets = -(-batch // group)
    sets = [[rng.randrange(n) for _ in range(k)] for _ in range(nsets)]
    idx = np.array([i for s in sets for i in s], np.uint64)
    out = np.zeros((batch, k, 2), np.uint64)
    assert E.emu_gather_batch_sets(O._ptr(out), O._ptr(vals), n, batch, group, O._ptr(idx), k) == 0
    paths = np.zeros((batch, k, log_n, 64), np.uint8)
    assert E.emu_merkle_open_batch_sets(O._ptr(paths), O._ptr(trees), n, batch, group, O._ptr(idx), k) == 0
    for b in range(batch):
        s = sets[b // group]
        assert np.array_equal(out[b], vals[b][s])
        for q, i in enumerate(s):
            assert [bytes(p) for p in paths[b, q]] == O.merkle_open(trees[b], i)


def test_openings_errors_leave_outputs_untouched(E):
    n, batch, k = 8, 4, 2
    vals = np.zeros((batch * n, 2), np.uint64)
    trees = np.zeros((batch, 2 * n, 64), np.uint8)
    for group, idx, code in ((0, [1, 2, 3, 4], SA_ESIZE), (2, [1, 2, 3, n], SA_EINDEX), (4, [n, 0], SA_EINDEX)):
        i = np.array(idx, np.uint64)
        out = np.full((batch, k, 2), 0x1234, np.uint64)
        paths = np.full((batch, k, 3, 64), 0x12, np.uint8)
        assert E.emu_gather_batch_sets(O._ptr(out), O._ptr(vals), n, batch, group, O._ptr(i), k) == code
        assert E.emu_merkle_open_batch_sets(O._ptr(paths), O._ptr(trees), n, batch, group, O._ptr(i), k) == code
        assert (out == 0x1234).all() and (paths == 0x12).all()
