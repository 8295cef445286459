"""CPU emulation of transition quotients (tests/emu/emu_air.cpp over csrc/air.cuh): the library's own checks,
compilation and schedules of sa_air_plan / sa_air_quotients, with every kernel replaced by a loop over its element
function, against the quotients restated with Python ints (tests/air_cases.py) and the reference's own quotients in
tests/golden/air.json.  The emulation starts its workspaces and `out` from a stale pattern, so an element the
schedule fails to write shows up."""
import ctypes

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O
from air_cases import (P, flatten, golden, golden_air, ints, make_case, plan_bytes_rule, quotients)

SA_EROOTORDER, SA_ENOTPRIM, SA_EDIVZERO, SA_ESIZE = -2, -3, -4, -6


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu_air())
    sz, vp, ci = ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int
    lib.emu_air_plan_bytes.restype = sz
    lib.emu_air_plan_bytes.argtypes = [ci, sz, sz, sz]
    lib.emu_air_plan.restype = ci
    lib.emu_air_plan.argtypes = [vp, vp, vp, vp, sz, sz, sz, vp, sz, ci, vp, vp, vp]
    lib.emu_air_quotients.restype = ci
    lib.emu_air_quotients.argtypes = [vp, vp, vp, sz, sz, sz, sz, ci, vp]
    return lib


def plan(E, air, nregs, max_ncoef, zerofier, log_n, root, offset, step):
    """(code, plan array)"""
    coeffs, exps, starts = flatten(air, nregs)
    nbytes = E.emu_air_plan_bytes(log_n, max_ncoef, nregs, starts[-1])
    buf = np.zeros((max(nbytes, 16) // 16, 2), np.uint64)
    c = np.array(coeffs or [0], np.uint64)
    e = np.array(exps or [0], np.uint32)
    s = np.array(starts, np.uintp)
    z = O.to_np(zerofier) if zerofier else np.zeros((1, 2), np.uint64)
    rc = E.emu_air_plan(O._ptr(buf), O._ptr(c), O._ptr(e), O._ptr(s), len(air), nregs, max_ncoef, O._ptr(z),
                        len(zerofier), log_n, O._ptr(O._fe(root)), O._ptr(O._fe(offset)), O._ptr(O._fe(step)))
    return rc, buf


def apply(E, out, buf, trace, nregs, qlen, ncons, log_n, root):
    t = O.to_np([v for row in trace for v in row])
    return E.emu_air_quotients(O._ptr(out), O._ptr(buf), O._ptr(t), nregs, len(trace[0]), qlen, ncons, log_n,
                               O._ptr(O._fe(root)))


def run(E, air, trace, zerofier, max_ncoef, root, offset, step, qlen, log_n):
    nregs = len(trace)
    rc, buf = plan(E, air, nregs, max_ncoef, zerofier, log_n, root, offset, step)
    assert rc == 0
    out = np.zeros((len(air) * qlen, 2), np.uint64)
    assert apply(E, out, buf, trace, nregs, qlen, len(air), log_n, root) == 0
    got = O.from_np(out)
    return [got[c * qlen:(c + 1) * qlen] for c in range(len(air))]


def check(E, seed, log_n, nregs, ncons, **kw):
    air, trace, zerofier, max_ncoef, root, offset, step, qlen = make_case(seed, log_n, nregs, ncons, **kw)
    got = run(E, air, trace, zerofier, max_ncoef, root, offset, step, qlen, log_n)
    want = quotients(air, trace, zerofier, 1 << log_n, root, offset, step)
    assert got == [w[:qlen] for w in want]


@pytest.mark.parametrize("ncons", [1, 2, 7])
@pytest.mark.parametrize("nregs", [1, 2, 3, 5])
@pytest.mark.parametrize("log_n", list(range(1, 11)))
def test_matches_restatement(E, log_n, nregs, ncons):
    check(E, 100 * log_n + 10 * nregs + ncons, log_n, nregs, ncons)


@pytest.mark.parametrize("log_n", [1, 3, 6, 9])
@pytest.mark.parametrize("offset_kind, step_kind", [("zero", "root"), ("one", "outside"), ("random", "outside"),
                                                    ("random", "power"), ("zero", "outside")])
def test_offsets_and_steps(E, log_n, offset_kind, step_kind):
    """offset 0 and 1, step = root, a power of root, and a step outside <root>"""
    check(E, 7 * log_n + len(offset_kind + step_kind), log_n, 2, 7, offset_kind=offset_kind, step_kind=step_kind)


@pytest.mark.parametrize("log_n", [2, 5, 8, 10])
@pytest.mark.parametrize("nregs", [1, 3])
def test_short_trace_and_qlen(E, log_n, nregs):
    """ncoef below the plan's max_ncoef, and a truncated qlen"""
    n = 1 << log_n
    check(E, 31 * log_n + nregs, log_n, nregs, 7, short=True, qlen=max(1, n - n // 3))


def test_x_steps_are_not_consecutive(E):
    """one group of sparse, unsorted x exponents 0, 5, 6, 13, 40 and a duplicate trace vector in another order"""
    log_n, nregs = 6, 2
    n = 1 << log_n
    rng_vals = [3, 5, 7, 11, 13, 17, 19]
    air = [{(40, 1, 0, 0, 0): rng_vals[0], (5, 1, 0, 0, 0): rng_vals[1], (13, 1, 0, 0, 0): rng_vals[2],
            (0, 1, 0, 0, 0): rng_vals[3], (6, 1, 0, 0, 0): rng_vals[4], (7, 0, 0, 0, 1): rng_vals[5],
            (2, 0, 0, 0, 1): rng_vals[6]}]
    root = O.primitive_nth_root(n)
    trace = [[(i * 7919 + r) % P for i in range(10)] for r in range(nregs)]
    z = [5, 1]
    got = run(E, air, trace, z, 10, root, 3, root, n, log_n)
    assert got == quotients(air, trace, z, n, root, 3, root)


@pytest.mark.parametrize("rec_name", ["faststark", "false_witness", "config5"])
def test_golden(E, rec_name):
    """the reference's quotients (fast_coset_divide of evaluate_symbolic) bit for bit"""
    rec = golden()[rec_name]
    air, trace = golden_air(rec), [ints(r) for r in rec["trace"]]
    got = run(E, air, trace, ints(rec["zerofier"]), len(trace[0]), int(rec["root"]), int(rec["offset"]),
              int(rec["step"]), rec["qlen"], rec["log_n"])
    assert got == [ints(q) for q in rec["quotients"]]


@pytest.mark.parametrize("nregs", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("log_n", [0, 1, 2, 4, 5, 10, 30, 31])
def test_plan_bytes_rule(E, log_n, nregs):
    for max_ncoef in (0, 1, 2, 17, 1 << 10, (1 << 10) + 1):
        for nterms in (0, 1, 7, 1000, (1 << 32) - 1, 1 << 32):
            assert E.emu_air_plan_bytes(log_n, max_ncoef, nregs, nterms) == \
                plan_bytes_rule(log_n, max_ncoef, nregs, nterms), (max_ncoef, nterms)
    assert E.emu_air_plan_bytes(log_n, 1, 0, 1) == 0


@pytest.mark.parametrize("log_n", [1, 2, 5, 10])
def test_errors_leave_out_untouched(E, log_n):
    """each refused build or apply returns its code and writes nothing"""
    n = 1 << log_n
    nregs = 2
    air, trace, zerofier, max_ncoef, root, offset, step, _ = make_case(log_n, log_n, nregs, 3)
    pattern = np.full((16, 2), 0x1234, np.uint64)
    span = max_ncoef - 1

    def build_code(**kw):
        a = dict(air=air, nregs=nregs, max_ncoef=max_ncoef, zerofier=zerofier, log_n=log_n, root=root,
                 offset=offset, step=step)
        a.update(kw)
        return plan(E, **a)

    # a term whose degree bound is exactly n, and one just below
    x_at = n - span
    assert build_code(air=[{(x_at, 1) + (0,) * (2 * nregs - 1): 1}])[0] == SA_ESIZE
    below = [{(x_at - 1, 1) + (0,) * (2 * nregs - 1): 1}] if x_at >= 1 else [{(0,) * (1 + 2 * nregs): 1}]
    assert build_code(air=below)[0] == 0
    builds = [dict(log_n=0), dict(log_n=31), dict(nregs=0), dict(air=[]), dict(max_ncoef=0),
              dict(max_ncoef=n + 1), dict(zerofier=[]), dict(zerofier=[1] * (n + 1)),
              dict(air=[{(n,) + (0,) * (2 * nregs): 1}]),
              dict(root=O.primitive_nth_root(2 * n), code=SA_EROOTORDER)]
    if log_n > 1:
        builds.append(dict(root=O.primitive_nth_root(n // 2), code=SA_ENOTPRIM))
    for kw in builds:
        code = kw.pop("code", SA_ESIZE)
        assert build_code(**kw)[0] == code, kw
    assert build_code(zerofier=[0, 0])[0] == SA_EDIVZERO
    # applies
    rc, buf = build_code()
    assert rc == 0
    applies = [dict(log_n=0), dict(log_n=31), dict(qlen=0), dict(qlen=n + 1), dict(ncons=0), dict(nregs=0),
               dict(root=O.primitive_nth_root(2 * n), code=SA_EROOTORDER)]
    if log_n > 1:
        applies.append(dict(root=O.primitive_nth_root(n // 2), code=SA_ENOTPRIM))
    for kw in applies:
        code = kw.pop("code", SA_ESIZE)
        a = dict(nregs=nregs, qlen=n, ncons=len(air), log_n=log_n, root=root)
        a.update(kw)
        out = pattern.copy()
        assert apply(E, out, buf, trace, a["nregs"], a["qlen"], a["ncons"], a["log_n"], a["root"]) == code, kw
        assert (out == pattern).all(), kw
    out = pattern.copy()
    t = O.to_np([1] * (n + 1))
    assert E.emu_air_quotients(O._ptr(out), O._ptr(buf), O._ptr(t), 1, n + 1, 1, 1, log_n, O._ptr(O._fe(root))) \
        == SA_ESIZE
    assert (out == pattern).all()
