"""Coset division plans and batched coset evaluation on the device (sa_coset_div_plan, sa_coset_div_apply_batch and
sa_coset_evaluate_batch through CudaEngine.coset_div_plan / coset_div_apply / coset_evaluate, the route of the drop-in's
fast_coset_divide and fast_coset_evaluate): every row against the oracle (tests/coset_cases.py) and against a single
apply, large sizes by exact properties, batches across chunks, the launches of a chunk, errors before any launch, two
streams sharing one plan and an apply captured in a CUDA graph."""
import os
import random
import sys

import numpy as np
import pytest

import oracle as O
from coset_cases import Case, formula

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "stark-anatomy_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)
import sa_engine  # noqa: E402

pytestmark = pytest.mark.gpu
GIB = 1 << 30
MARGIN = 2 * GIB
P = O.P


@pytest.fixture(scope="module")
def eng():
    sa_engine.set_engine(None)
    e = sa_engine.get_engine()
    assert e.name == "cuda"
    return e


def release(eng):
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert eng.lib.sa_release_workspaces() == 0


@pytest.fixture(autouse=True)
def _cuda_engine(eng):
    sa_engine.set_engine(eng)
    yield
    release(eng)


def up(eng, arr):
    return eng.upload(np.ascontiguousarray(arr).reshape(-1, 2).view(np.int64)).reshape(arr.shape)


def down(vec):
    return vec.cpu().numpy().view(np.uint64)


def rand_dev(eng, shape, seed):
    """random canonical elements (< 2^125 < p) on the device"""
    import torch
    g = torch.Generator(device=eng.device)
    g.manual_seed(seed)
    x = torch.randint(0, 1 << 62, tuple(shape) + (2,), dtype=torch.int64, device=eng.device, generator=g)
    x[..., 1] &= (1 << 61) - 1
    return x


def need_device(eng, log_n, batch, vectors=8):
    """skip unless the plan, a chunk's workspaces, the batch's rows in and out and `vectors` more n-element vectors
    fit in free memory"""
    import torch
    release(eng)
    free, _ = torch.cuda.mem_get_info(eng.device)
    n = 1 << log_n
    chunk = min(batch, eng.lib.sa_coset_batch_max(log_n))
    want = eng.lib.sa_coset_div_plan_bytes(log_n) + 32 * n * chunk + 32 * n * batch + 16 * n * vectors + MARGIN
    if free < want:
        pytest.skip("2^%d, B = %d needs %.1f GiB free on the device, %.1f GiB are" % (log_n, batch, want / GIB, free / GIB))


def cyclic_product(eng, a, b, log_n, root):
    """a * b at order n (exact when deg a + deg b < n)"""
    n = 1 << log_n
    fa, fb = eng.ntt(eng.pad(a, n), log_n, root), eng.ntt(eng.pad(b, n), log_n, root)
    return eng.ntt(eng.pointwise_mul(fa, fb), log_n, root, inverse=True)


@pytest.mark.parametrize("full", [True, False], ids=["n", "below_n"])
@pytest.mark.parametrize("batch", [1, 2, 5])
@pytest.mark.parametrize("log_n", list(range(1, 13)) + [16])
def test_apply_matches_oracle_and_single_applies(eng, log_n, batch, full):
    """every row: the documented formula, the exact quotient of a clean division, the reference's fast_coset_divide
    on numerators of degree n/2 .. n - 1, zero for a zero row and equal rows for equal numerators; every row equals
    the same numerator applied alone, and the plan's bytes are unchanged"""
    c = Case(log_n, batch, full, seed=100 * log_n + 10 * batch + full)
    plan = eng.coset_div_plan(up(eng, O.to_np(c.divisor)), log_n, c.root, c.offset)
    before = plan.plan.clone()
    lhs = up(eng, c.lhs_np())
    out = eng.coset_div_apply(plan, lhs, c.qlen)
    assert tuple(out.shape) == (batch, c.qlen, 2)
    got = down(out)
    c.check(got)
    for b in range(batch):
        one = eng.coset_div_apply(plan, lhs[b], c.qlen)
        assert tuple(one.shape) == (c.qlen, 2)
        assert (down(one) == got[b]).all(), b
    assert bool((plan.plan == before).all())


@pytest.mark.parametrize("log_n, batch", [(20, 3), (22, 3), (24, 1), (26, 1)])
def test_large_sizes_by_coset_property(eng, log_n, batch):
    """sizes the oracle cannot reach: every row of n coefficients U * offset^-j evaluates on the coset to L / R
    (coset_evaluate(out) * coset_evaluate(r) == coset_evaluate(lhs)), and a clean division q * r returns q followed
    by zeros"""
    need_device(eng, log_n, batch + 1, vectors=10)
    n = 1 << log_n
    rng = random.Random(log_n)
    root, offset = O.primitive_nth_root(n), rng.randrange(1, P)
    dr = n // 4
    r = rand_dev(eng, (dr + 1,), 10 + log_n)
    lhs = rand_dev(eng, (batch, n), 20 + log_n)
    plan = eng.coset_div_plan(r, log_n, root, offset)
    out = eng.coset_div_apply(plan, lhs, n)
    R = eng.coset_evaluate(r, log_n, root, offset)
    for b in range(batch):
        got = eng.pointwise_mul(eng.coset_evaluate(out[b], log_n, root, offset), R)
        assert bool((got == eng.coset_evaluate(lhs[b], log_n, root, offset)).all()), b
    del lhs, out, got, R
    q = rand_dev(eng, (n - dr - 1,), 30 + log_n)
    clean = cyclic_product(eng, q, r, log_n, root)
    got = eng.coset_div_apply(plan, clean, n)
    assert bool((got[:q.shape[0]] == q).all())
    assert not bool(got[q.shape[0]:].any())


def test_batch_across_chunks(eng):
    """two full chunks and one more row at 2^21: every row, the last chunk's single row included, equals a single
    apply"""
    log_n = 21
    n, chunk = 1 << log_n, eng.lib.sa_coset_batch_max(log_n)
    batch = 2 * chunk + 1
    need_device(eng, log_n, batch)
    root = O.primitive_nth_root(n)
    plan = eng.coset_div_plan(rand_dev(eng, (n // 2,), 1), log_n, root, 3)
    lhs = rand_dev(eng, (batch, n - 5), 2)
    out = eng.coset_div_apply(plan, lhs, n // 2 + 3)
    for b in range(batch):
        assert bool((out[b] == eng.coset_div_apply(plan, lhs[b], n // 2 + 3)).all()), b


@pytest.mark.parametrize("log_n", [4, 12, 16])
def test_a_chunk_launches_what_one_row_does(eng, log_n):
    """after a warm-up, one chunk of rows issues the launches of a single row (and so does a chunk of evaluations)"""
    n, chunk = 1 << log_n, eng.lib.sa_coset_batch_max(log_n)
    chunk = min(chunk, 4096)
    root = O.primitive_nth_root(n)
    plan = eng.coset_div_plan(rand_dev(eng, (n // 2 + 1,), 3), log_n, root, 5)
    lhs = rand_dev(eng, (chunk, n), 4)
    for fn in (lambda x: eng.coset_div_apply(plan, x, n), lambda x: eng.coset_evaluate(x, log_n, root, 5)):
        fn(lhs)
        fn(lhs[0])
        before = eng.launch_count()
        fn(lhs[0])
        single = eng.launch_count() - before
        before = eng.launch_count()
        fn(lhs)
        assert eng.launch_count() - before == single


@pytest.mark.parametrize("log_n", [3, 12])
def test_divisors_that_vanish_and_offset_zero(eng, log_n):
    """a divisor with a zero on the coset (X - offset * root^3), the zero divisor and, on the coset of offset 0, a
    divisor with r_0 == 0 raise "divide by zero" at plan time; offset 0 with r_0 != 0 gives the formula's row"""
    n = 1 << log_n
    root, offset = O.primitive_nth_root(n), 11
    point = offset * pow(root, 3, P) % P
    for d, off in (([P - point, 1], offset), ([0, 0, 0], offset), ([0, 2, 3], 0)):
        with pytest.raises(AssertionError, match="divide by zero"):
            eng.coset_div_plan(up(eng, O.to_np(d)), log_n, root, off)
    lhs = [random.Random(log_n).randrange(P) for _ in range(n)]
    plan = eng.coset_div_plan(up(eng, O.to_np([1, 2, 3])), log_n, root, 0)
    got = O.from_np(down(eng.coset_div_apply(plan, up(eng, O.to_np(lhs)), n)))
    assert got == formula(lhs, [1, 2, 3], 0, root, n, n) == [lhs[0]] + [0] * (n - 1)


@pytest.mark.parametrize("log_n", [3, 12])
def test_bad_roots_and_sizes_outside_1_30_are_refused_before_any_launch(eng, log_n):
    import torch
    n = 1 << log_n
    root = O.primitive_nth_root(n)
    d = up(eng, O.to_np([1, 2, 3]))
    plan = eng.coset_div_plan(d, log_n, root, 7)
    lhs = rand_dev(eng, (3, n), 5)
    eng.coset_div_apply(plan, lhs, n)
    for bad, msg in ((O.primitive_nth_root(2 * n), "must be nth root"), (O.primitive_nth_root(n // 2), "is not primitive")):
        before = eng.launch_count()
        with pytest.raises(AssertionError, match=msg):
            eng.coset_div_plan(d, log_n, bad, 7)
        with pytest.raises(AssertionError, match=msg):
            eng.coset_div_apply(sa_engine.CosetDivPlan(plan.plan, log_n, bad, 7), lhs, n)
        with pytest.raises(AssertionError, match=msg):
            eng.coset_evaluate(lhs, log_n, bad, 7)
        assert eng.launch_count() == before
    before = eng.launch_count()
    for shape in ((3, n + 1, 2), (3, n, 3), (3, 0, 2), (2 * n,), (1, 3, n, 2)):
        x = torch.zeros(shape, dtype=torch.int64, device=eng.device)
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.coset_div_apply(plan, x, n)
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.coset_evaluate(x, log_n, root, 7)
    for qlen in (0, n + 1):
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.coset_div_apply(plan, lhs, qlen)
    for divisor, lg in ((torch.zeros((n + 1, 2), dtype=torch.int64, device=eng.device), log_n),
                        (torch.zeros((0, 2), dtype=torch.int64, device=eng.device), log_n), (d, 0), (d, 31)):
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.coset_div_plan(divisor, lg, root, 7)
    out = eng.coset_div_apply(plan, lhs[:0], n // 2)
    assert tuple(out.shape) == (0, n // 2, 2)
    assert tuple(eng.coset_evaluate(lhs[:0], log_n, root, 7).shape) == (0, n, 2)
    assert eng.launch_count() == before


@pytest.mark.parametrize("log_n", [10, 16])
def test_one_plan_on_two_streams(eng, log_n):
    """the plan is only read: two streams apply it at the same time to different batches"""
    import torch
    n = 1 << log_n
    root = O.primitive_nth_root(n)
    plan = eng.coset_div_plan(rand_dev(eng, (n // 2,), 6), log_n, root, 9)
    lhss = [rand_dev(eng, (3 + i, n), 7 + i) for i in range(2)]
    want = [down(torch.stack([eng.coset_div_apply(plan, row, n) for row in x])) for x in lhss]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for rnd in range(2):  # the first round grows each stream's workspaces, the second runs without any allocation
        outs = []
        for s, x in zip(streams, lhss):
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                outs.append(eng.coset_div_apply(plan, x, n))
        torch.cuda.synchronize()
        for got, w in zip(outs, want):
            assert (down(got) == w).all(), rnd


@pytest.mark.parametrize("log_n", [10, 16])
def test_apply_in_a_cuda_graph(eng, log_n):
    """an apply captured in a CUDA graph (any host synchronisation would end the capture) replays exactly on new
    numerators copied into the captured input"""
    import torch
    n, batch = 1 << log_n, 4
    root = O.primitive_nth_root(n)
    plan = eng.coset_div_plan(rand_dev(eng, (n // 2,), 8), log_n, root, 13)
    lin = rand_dev(eng, (batch, n), 9)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.coset_div_apply(plan, lin, n)  # grows s's workspaces and caches the transforms' plans outside the capture
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out = eng.coset_div_apply(plan, lin, n)
    for i in range(2):
        fresh = rand_dev(eng, (batch, n), 100 + i)
        lin.copy_(fresh)
        g.replay()
        torch.cuda.synchronize()
        want = torch.stack([eng.coset_div_apply(plan, row, n) for row in fresh])
        assert bool((out == want).all()), i


@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("log_n", list(range(1, 13)))
def test_evaluate_matches_oracle(eng, log_n, batch):
    rng = random.Random(9000 + 10 * log_n + batch)
    n = 1 << log_n
    root, offset = O.primitive_nth_root(n), rng.randrange(P)
    for ncoef in sorted({1, max(1, n // 2 + 1), n}):
        rows = [[rng.randrange(P) for _ in range(ncoef)] for _ in range(batch)]
        out = eng.coset_evaluate(up(eng, np.stack([O.to_np(r) for r in rows])), log_n, root, offset)
        assert tuple(out.shape) == (batch, n, 2)
        got = down(out)
        for b in range(batch):
            assert O.from_np(got[b]) == O.fast_coset_evaluate(rows[b], offset, root, n), (ncoef, b)
        one = eng.coset_evaluate(up(eng, O.to_np(rows[0])), log_n, root, offset)
        assert tuple(one.shape) == (n, 2) and (down(one) == got[0]).all()


def test_evaluate_2_20_matches_oracle(eng):
    """at 2^20, every row equals the oracle's fast_coset_evaluate"""
    log_n, batch = 20, 3
    need_device(eng, log_n, batch)
    n = 1 << log_n
    root, offset = O.primitive_nth_root(n), 85408008396924667383611388730472331217
    coeffs = rand_dev(eng, (batch, n // 4 + 3), 11)
    got = down(eng.coset_evaluate(coeffs, log_n, root, offset))
    for b, row in enumerate(down(coeffs)):
        assert O.from_np(got[b]) == O.fast_coset_evaluate(O.from_np(row), offset, root, n), b


@pytest.mark.parametrize("log_n", [27, 28])
def test_sizes_past_2_26(eng, log_n):
    """2^27 and 2^28: a clean division q * r returns q followed by zeros, and an evaluation equals Horner
    (poly_eval) at sampled coset points"""
    need_device(eng, log_n, 1, vectors=8)
    n = 1 << log_n
    rng = random.Random(log_n)
    root, offset = O.primitive_nth_root(n), rng.randrange(1, P)
    dr = n // 4
    r = rand_dev(eng, (dr + 1,), 10 + log_n)
    q = rand_dev(eng, (n - dr - 1,), 30 + log_n)
    clean = cyclic_product(eng, q, r, log_n, root)
    plan = eng.coset_div_plan(r, log_n, root, offset)
    got = eng.coset_div_apply(plan, clean, n)
    assert bool((got[:q.shape[0]] == q).all())
    assert not bool(got[q.shape[0]:].any())
    del clean, plan, got
    f = q[:n // 64 + 3]  # Horner's work is coefficients x points
    idx = sorted({0, 1, n // 2, n - 1} | {rng.randrange(n) for _ in range(60)})
    points = up(eng, O.to_np([offset * pow(root, i, P) % P for i in idx]))
    ev = eng.coset_evaluate(f, log_n, root, offset)
    assert bool((ev[idx] == eng.poly_eval(f, points, mode=1)).all())
