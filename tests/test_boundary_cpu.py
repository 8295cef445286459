"""CPU emulation of boundary quotients (tests/emu/emu_boundary.cpp over csrc/boundary.cuh): the library's own checks
and schedules of sa_boundary_plan / sa_boundary_quotients, with every kernel replaced by a loop over its element
function (the store by warps of 32 lanes, their ballot and the leader that raises a row's flag), against the outputs
restated with Python ints (tests/boundary_cases.py) and the reference's own quotients and codewords in
tests/golden/boundary.json.  The emulation starts its workspace, outputs and flags from a stale pattern, so an
element the schedule fails to write, or a flag it fails to clear, shows up."""
import ctypes

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O
from boundary_cases import (P, digest, expected, golden, golden_boundary, ints, make_case, plan_bytes_rule,
                            reference)

SA_EROOTORDER, SA_ENOTPRIM, SA_EDIVZERO, SA_ESIZE = -2, -3, -4, -6


@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu_boundary())
    sz, vp, ci = ctypes.c_size_t, ctypes.c_void_p, ctypes.c_int
    lib.emu_boundary_plan_bytes.restype = sz
    lib.emu_boundary_plan_bytes.argtypes = [ci, sz]
    lib.emu_boundary_plan.restype = ci
    lib.emu_boundary_plan.argtypes = [vp, vp, vp, vp, vp, sz, ci, vp, vp]
    lib.emu_boundary_quotients.restype = ci
    lib.emu_boundary_quotients.argtypes = [vp, vp, vp, vp, vp, sz, sz, ci, vp]
    lib.emu_boundary_store_atomics.restype = ctypes.c_longlong
    return lib


def plan(E, rows, log_n, root, offset, nregs=None, zlens=None, ilens=None):
    """(code, plan array) for per-register (zerofier, interpolant) rows of ints"""
    nregs = len(rows) if nregs is None else nregs
    zs = [O.to_np(z or [0]) for z, _ in rows]
    its = [O.to_np(i or [0]) for _, i in rows]
    ptrs = lambda arrs: (ctypes.c_void_p * max(1, len(arrs)))(*[a.ctypes.data for a in arrs])  # noqa: E731
    zl = zlens if zlens is not None else [len(z) for z, _ in rows]
    il = ilens if ilens is not None else [len(i) for _, i in rows]
    nbytes = E.emu_boundary_plan_bytes(log_n, nregs)
    buf = np.zeros((max(nbytes, 16) // 16, 2), np.uint64)
    rc = E.emu_boundary_plan(O._ptr(buf), ptrs(zs), (ctypes.c_size_t * max(1, len(zl)))(*zl), ptrs(its),
                             (ctypes.c_size_t * max(1, len(il)))(*il), nregs, log_n, O._ptr(O._fe(root)),
                             O._ptr(O._fe(offset)))
    return rc, buf


def apply(E, buf, trace, log_n, root, nregs=None, ncoef=None, outs=None):
    """(code, quot rows, codewords, flags)"""
    nregs = len(trace) if nregs is None else nregs
    ncoef = len(trace[0]) if ncoef is None else ncoef
    n = 1 << log_n
    t = O.to_np([v for row in trace for v in row])
    quot, cw, flags = outs or (np.zeros((max(1, nregs * ncoef), 2), np.uint64),
                               np.zeros((max(1, nregs * n), 2), np.uint64), np.zeros(max(1, nregs), np.uint32))
    rc = E.emu_boundary_quotients(O._ptr(quot), O._ptr(cw), O._ptr(flags), O._ptr(buf), O._ptr(t), nregs, ncoef,
                                  log_n, O._ptr(O._fe(root)))
    q, c = O.from_np(quot), O.from_np(cw)
    return rc, [q[s * ncoef:(s + 1) * ncoef] for s in range(nregs)], [c[s * n:(s + 1) * n] for s in range(nregs)], \
        [int(f) for f in flags[:nregs]]


def run(E, rows, trace, log_n, root, offset):
    rc, buf = plan(E, rows, log_n, root, offset)
    assert rc == 0
    rc, quot, cw, flags = apply(E, buf, trace, log_n, root)
    assert rc == 0
    return quot, cw, flags


def check(E, trace, rows, log_n, root, offset, false_regs=None):
    """every register against the restatement, and the clean ones against the reference's division"""
    n = 1 << log_n
    quot, cw, flags = run(E, rows, trace, log_n, root, offset)
    for s, (t, (z, i)) in enumerate(zip(trace, rows)):
        q_want, cw_want, flag_want = expected(t, z, i, n, root, offset)
        ref = reference(t, z, i, n, root, offset)
        assert flag_want == (ref is None), s
        assert (quot[s], cw[s], bool(flags[s])) == (q_want, cw_want, flag_want), s
        if ref is not None:
            assert quot[s] == ref[0] + [0] * (len(t) - len(ref[0])) and cw[s] == ref[1], s
        if false_regs is not None:
            assert bool(flags[s]) == (s in false_regs), s
    return flags


GRID = [(lg, r, k) for lg in range(1, 11) for r in (1, 2, 3, 5) for k in range(1, 6) if k < 1 << lg]


@pytest.mark.parametrize("log_n, nregs, k", GRID)
def test_matches_restatement(E, log_n, nregs, k):
    """clean registers and, from two registers on, one false one; k, k-1, ... points per register"""
    seed = 100 * log_n + 10 * nregs + k
    npoints = [max(1, k - s % 2) for s in range(nregs)]
    false_regs = (seed % nregs,) if nregs > 1 else ()
    _, _, trace, rows, _, root, offset = make_case(seed, log_n, nregs, npoints, false_regs=false_regs)
    check(E, trace, rows, log_n, root, offset, false_regs)


@pytest.mark.parametrize("log_n", [2, 3, 5, 8, 10])
@pytest.mark.parametrize("offset_kind", ["one", "generator"])
def test_offsets(E, log_n, offset_kind):
    k = min(3, (1 << log_n) - 1)
    _, _, trace, rows, _, root, offset = make_case(7 * log_n, log_n, 3, [k, 1, k], offset_kind=offset_kind,
                                                   false_regs=(1,))
    check(E, trace, rows, log_n, root, offset, (1,))


@pytest.mark.parametrize("log_n", [1, 2, 4, 7, 10])
def test_ncoef_equal_to_n(E, log_n):
    n = 1 << log_n
    k = min(5, n - 1)
    _, _, trace, rows, _, root, offset = make_case(log_n, log_n, 2, [k, 1], ncoef=n)
    check(E, trace, rows, log_n, root, offset, ())


@pytest.mark.parametrize("log_n", [3, 4, 6, 9])
@pytest.mark.parametrize("const_values", [True, False])
def test_ncoef_below_deg_z(E, log_n, const_values):
    """ncoef < deg Z: clean exactly when T = I (a constant I here), every tail coefficient checked"""
    _, _, trace, rows, _, root, offset = make_case(log_n + 50, log_n, 2, [5, 4], ncoef=2, const_values=const_values)
    flags = check(E, trace, rows, log_n, root, offset)
    assert [bool(f) for f in flags] == [not const_values] * 2


def test_false_boundaries_flag_exactly_their_registers(E):
    """5 registers at 2^6 with every subset of false registers of one seed: the flags name exactly those"""
    log_n = 6
    for false_regs in ((), (0,), (4,), (1, 3), (0, 2, 4), (0, 1, 2, 3, 4)):
        _, _, trace, rows, _, root, offset = make_case(61, log_n, 5, [1, 2, 3, 4, 5], false_regs=false_regs)
        check(E, trace, rows, log_n, root, offset, false_regs)


@pytest.mark.parametrize("log_n", [1, 2, 3, 4, 5, 6, 8])
def test_one_atomic_per_flagged_row_a_warp_touches(E, log_n):
    """below n = 32 a warp spans 32 / n rows; each flagged row costs one atomicOr per warp that sees its tail"""
    n = 1 << log_n
    nregs = 5
    k = min(2, n - 1)
    false_regs = (0, 3, 4)
    _, _, trace, rows, _, root, offset = make_case(log_n + 80, log_n, nregs, [k] * nregs, false_regs=false_regs)
    check(E, trace, rows, log_n, root, offset, false_regs)
    want = 0
    for s in false_regs:
        _, cw_s, _ = expected(trace[s], rows[s][0], rows[s][1], n, root, offset)
        u = O.intt(root, cw_s)
        bad = [s * n + j for j in range(max(0, len(trace[s]) - k), n) if u[j]]
        want += len({i // 32 for i in bad})
    assert E.emu_boundary_store_atomics() == want


@pytest.mark.parametrize("name", ["faststark", "false_boundary", "multi", "short", "config5"])
def test_golden(E, name):
    """the reference's (T - I) / Z and fast_coset_evaluate of it, bit for bit; a raising division is flagged"""
    rec = golden()[name]
    rows = [(ints(z), ints(i)) for z, i in zip(rec["zerofiers"], rec["interpolants"])]
    trace = [ints(t) for t in rec["trace"]]
    quot, cw, flags = run(E, rows, trace, rec["log_n"], int(rec["root"]), int(rec["offset"]))
    for s in range(rec["nregs"]):
        q = rec["quotients"][s]
        assert bool(flags[s]) == (q is None), s
        if q is not None:
            assert quot[s] == ints(q) + [0] * (len(trace[s]) - len(q)), s
            assert digest(cw[s]) == rec["codeword_digests"][s], s
    assert golden_boundary(rec)  # the boundary is recorded too


@pytest.mark.parametrize("nregs", [0, 1, 2, 3, 5, 16, 17, 1 << 40, 1 << 59, (1 << 64) - 1])
@pytest.mark.parametrize("log_n", [0, 1, 2, 4, 5, 10, 30, 31])
def test_plan_bytes_rule(E, log_n, nregs):
    assert E.emu_boundary_plan_bytes(log_n, nregs) == plan_bytes_rule(log_n, nregs)


@pytest.mark.parametrize("log_n", [1, 2, 5, 10])
def test_errors_leave_outputs_untouched(E, log_n):
    """each refused build or apply returns its code and writes nothing"""
    n = 1 << log_n
    _, _, trace, rows, _, root, offset = make_case(log_n, log_n, 2, [1, 1])
    builds = [dict(log_n=0), dict(log_n=31), dict(nregs=0), dict(zlens=[0, 2]), dict(zlens=[2, n + 1]),
              dict(ilens=[0, 1]), dict(ilens=[1, n + 1]), dict(offset=0), dict(offset=P),
              dict(root=O.primitive_nth_root(2 * n), code=SA_EROOTORDER)]
    if log_n > 1:
        builds.append(dict(root=O.primitive_nth_root(n // 2), code=SA_ENOTPRIM))
    for kw in builds:
        code = kw.pop("code", SA_ESIZE)
        a = dict(rows=rows, log_n=log_n, root=root, offset=offset)
        a.update(kw)
        assert plan(E, **a)[0] == code, kw
    # errors after the build's work: a zerofier that vanishes on the coset, a zero top coefficient
    on_coset = [offset * root % P, P - 1]  # x_1 - X
    assert plan(E, [(on_coset, [1]), rows[1]], log_n, root, offset)[0] == SA_EDIVZERO
    assert plan(E, [rows[0], (rows[1][0] + [0], rows[1][1])], log_n, root, offset)[0] == SA_ESIZE
    rc, buf = plan(E, rows, log_n, root, offset)
    assert rc == 0
    pattern = (np.full((2 * n, 2), 0x1234, np.uint64), np.full((2 * n, 2), 0x1234, np.uint64),
               np.full(2, 0x1234, np.uint32))
    applies = [dict(log_n=0), dict(log_n=31), dict(nregs=0), dict(ncoef=0), dict(ncoef=n + 1),
               dict(root=O.primitive_nth_root(2 * n), code=SA_EROOTORDER)]
    if log_n > 1:
        applies.append(dict(root=O.primitive_nth_root(n // 2), code=SA_ENOTPRIM))
    padded = [r + [0] * (n + 1 - len(r)) for r in trace]
    for kw in applies:
        code = kw.pop("code", SA_ESIZE)
        a = dict(log_n=log_n, root=root)
        a.update(kw)
        outs = tuple(p.copy() for p in pattern)
        assert apply(E, buf, padded, a["log_n"], a["root"], nregs=a.get("nregs"), ncoef=a.get("ncoef", len(trace[0])),
                     outs=outs)[0] == code, kw
        assert all((o == p).all() for o, p in zip(outs, pattern)), kw
