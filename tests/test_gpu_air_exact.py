"""Exact transition quotients on the device (sa_air_quotients_exact through CudaEngine.air_quotients_exact): rows
bit for bit the unchecked apply's and flags exactly the reference's remainder test (the cases and restatement of
tests/test_air_exact_cpu.py), large sizes by property, several chunks of constraints, the kernel launches (the
unchecked apply's), errors before any launch, a CUDA graph whose replay clears the flags again, and the store's
registers."""
import os
import random
import re
import subprocess
import tempfile

import pytest

import oracle as O
from air_cases import P, make_air, numerator, pmul, quotients
from test_air_exact_cpu import divides, exact_case, x_constraint
from test_gpu_air import PKG, down, need_device, release, rows, up
import sa_engine

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    sa_engine.set_engine(None)
    e = sa_engine.get_engine()
    assert e.name == "cuda"
    return e


@pytest.fixture(autouse=True)
def _cuda_engine(eng):
    sa_engine.set_engine(eng)
    yield
    release(eng)


def both(eng, air, trace, z, max_ncoef, root, offset, step, qlen, log_n):
    plan = eng.air_plan(air, len(trace), up(eng, z), max_ncoef, log_n, root, offset, step)
    assert plan.zdeg == len(z) - 1
    t = rows(eng, trace)
    plain = eng.air_quotients(plan, t, qlen)
    out, flags = eng.air_quotients_exact(plan, t, qlen, check=False)
    return plan, t, plain, out, flags


CASES = [(lg, r, c) for lg in list(range(1, 13)) + [16] for r in (1, 2, 3) for c in (1, 2, 7)]


@pytest.mark.parametrize("log_n, nregs, ncons", CASES)
def test_matches_restatement(eng, log_n, nregs, ncons):
    """flags == the restated coset row's tail, and == the long division of the numerator up to 2^10"""
    n = 1 << log_n
    air, trace, z, max_ncoef, root, offset, step, qlen = exact_case(1000 * log_n + 10 * nregs + ncons, log_n, nregs,
                                                                    ncons)
    _, _, plain, out, flags = both(eng, air, trace, z, max_ncoef, root, offset, step, qlen, log_n)
    assert bool((out == plain).all())
    tail = n - (len(z) - 1)
    want = [int(any(r[tail:])) for r in quotients(air, trace, z, n, root, offset, step)]
    if log_n <= 10:
        assert want == [0 if divides(numerator(a, trace, step), z) else 1 for a in air]
    assert [int(bool(f)) for f in flags.tolist()] == want


def check_large(eng, log_n, ncons, nregs=2, max_ncoef=4097):
    """exact numerators Q Z (flag clear, row Q) and Q Z + x^k (flag set) among seeded trace constraints whose flags
    are set; rows equal the unchecked apply's"""
    rng = random.Random(log_n + ncons)
    z = [rng.randrange(P) for _ in range(29)] + [1]
    q = [rng.randrange(P) for _ in range(1000)]
    qz = pmul(q, z)
    air = make_air(log_n, log_n, nregs, ncons, max_ncoef)
    air = [a if a else {(3,) + (1,) * (2 * nregs): c + 1} for c, a in enumerate(air)]
    air[0] = x_constraint(qz, nregs)
    air[-1] = x_constraint(qz[:7] + [(qz[7] + 1) % P] + qz[8:], nregs)
    trace = [[rng.randrange(P) for _ in range(max_ncoef)] for _ in range(nregs)]
    root, offset, step = O.primitive_nth_root(1 << log_n), rng.randrange(2, P), O.primitive_nth_root(1 << log_n - 2)
    _, _, plain, out, flags = both(eng, air, trace, z, max_ncoef, root, offset, step, len(q) + 2, log_n)
    assert bool((out == plain).all()) and down(out[0]) == q + [0, 0]
    # the seeded constraints' numerators are trace polynomials of this size: none divides by this Z
    assert [int(bool(v)) for v in flags.tolist()] == [0] + [1] * (ncons - 1)


@pytest.mark.parametrize("log_n", [20, 22])
def test_large_sizes_by_property(eng, log_n):
    need_device(eng, log_n, 24)
    check_large(eng, log_n, 7)


def test_constraints_past_one_chunk(eng):
    """2 chunk + 1 constraints at 2^21: the first and the last chunk's flags land on their own constraints"""
    log_n = 21
    ncons = 2 * eng.lib.sa_coset_batch_max(log_n) + 1
    need_device(eng, log_n, 2 * ncons + 8)
    check_large(eng, log_n, ncons, nregs=1, max_ncoef=65)


def launches(eng, fn):
    before = eng.launch_count()
    fn()
    return eng.launch_count() - before


@pytest.mark.parametrize("log_n", [10, 16])
def test_kernel_launches_are_the_unchecked_applys(eng, log_n):
    """the exact store replaces the plain one, so the kernel launches are the unchecked apply's; the one memset that
    clears the flags is not a kernel launch (test_graph_replay_clears_the_flags shows it runs in stream order)"""
    for nregs, ncons in ((1, 1), (2, 7)):
        air, trace, z, max_ncoef, root, offset, step, qlen = exact_case(nregs * ncons, log_n, nregs, ncons)
        plan, t, _, _, _ = both(eng, air, trace, z, max_ncoef, root, offset, step, qlen, log_n)
        plain = launches(eng, lambda: eng.air_quotients(plan, t, qlen))
        exact = launches(eng, lambda: eng.air_quotients_exact(plan, t, qlen, check=False))
        assert exact == plain, (plain, exact)


def test_errors_before_any_launch(eng):
    import torch
    log_n = 8
    n = 1 << log_n
    air, trace, z, max_ncoef, root, offset, step, qlen = exact_case(5, log_n, 2, 3)
    plan, t, _, _, _ = both(eng, air, trace, z, max_ncoef, root, offset, step, qlen, log_n)
    torch.cuda.synchronize()
    out = torch.full((3, qlen, 2), 0x0A5A5A5A, dtype=torch.int64, device=eng.device)
    flags = torch.full((3,), 0x77, dtype=torch.int32, device=eng.device)
    fp = sa_engine.ctypes.cast(flags.data_ptr(), sa_engine.ctypes.POINTER(sa_engine.ctypes.c_uint32))
    r = sa_engine._limbs(root)
    before = eng.launch_count()
    tail = n - (len(z) - 1)
    for args, code in (((2, max_ncoef, qlen, 3, n + 1, log_n), -6), ((2, max_ncoef, 0, 3, tail, log_n), -6),
                       ((2, 0, qlen, 3, tail, log_n), -6), ((0, max_ncoef, qlen, 3, tail, log_n), -6),
                       ((2, max_ncoef, qlen, 0, tail, log_n), -6), ((2, max_ncoef, qlen, 3, tail, 31), -6)):
        assert eng.lib.sa_air_quotients_exact(out.data_ptr(), fp, plan.plan.data_ptr(), t.data_ptr(), *args, r,
                                              eng._stream()) == code, args
    assert eng.lib.sa_air_quotients_exact(out.data_ptr(), fp, plan.plan.data_ptr(), t.data_ptr(), 2, max_ncoef, qlen,
                                          3, tail, log_n, sa_engine._limbs(O.primitive_nth_root(2 * n)),
                                          eng._stream()) == -2
    for q in (0, n + 1):
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.air_quotients_exact(plan, t, q)
    assert eng.launch_count() == before
    assert bool((out == 0x0A5A5A5A).all()) and bool((flags == 0x77).all())


@pytest.mark.parametrize("log_n", [10, 16])
def test_graph_replay_clears_the_flags(eng, log_n):
    """captured after a warm call: a replay over an unclean division sets the flag, and a replay after a clean
    numerator is copied into the captured trace clears it again"""
    import torch
    rng = random.Random(log_n)
    z = [rng.randrange(P) for _ in range(9)] + [1]
    root, ncoef = O.primitive_nth_root(1 << log_n), 64
    # N = T_0: exact when the trace row is a multiple of Z
    plan = eng.air_plan([{(0, 1, 0): 1}], 1, up(eng, z), ncoef, log_n, root, rng.randrange(2, P), root)
    clean = pmul([rng.randrange(P) for _ in range(ncoef - len(z) + 1)], z)
    dirty = clean[:3] + [(clean[3] + 1) % P] + clean[4:]
    t = rows(eng, [dirty])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.air_quotients_exact(plan, t, ncoef, check=False)
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out, flags = eng.air_quotients_exact(plan, t, ncoef, check=False)
    g.replay()
    torch.cuda.synchronize()
    assert flags.tolist() != [0]
    t.copy_(rows(eng, [clean]))
    g.replay()
    torch.cuda.synchronize()
    assert flags.tolist() == [0]
    assert pmul(down(out[0])[:ncoef - len(z) + 1], z) == clean


def test_store_has_no_spills():
    """ptxas's report for k_air_store_exact: no spill stores or loads"""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress",
                              "550", "-c", "-Xptxas", "-v", "-o", os.path.join(tmp, "poly.o"),
                              os.path.join(PKG, "csrc", "poly.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = res.stderr.splitlines()
    at = [i for i, line in enumerate(lines) if "Compiling entry function" in line and "k_air_store_exact" in line]
    assert len(at) == 1
    report = " ".join(lines[at[0]:at[0] + 4])
    spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert spills and spills.groups() == ("0", "0"), report
