"""Geometric interpolation plans and zerofiers on the device (sa_geo_plan, sa_geo_interp_batch and sa_geo_zerofier
through CudaEngine): byte equality with the subproduct tree's apply and zerofier over the explicit domain step^i up to
the tree's 2^20 points, values and roots at sampled domain points above it, batches across chunks, the launches of a
batch, errors before any launch, one plan on two streams, graph replay and the new kernels' spills."""
import os
import random
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import oracle as O

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "stark-anatomy_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)
import sa_engine  # noqa: E402

pytestmark = pytest.mark.gpu
P = O.P
GIB = 1 << 30


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


def rand_np(seed, n):
    rng = np.random.default_rng(seed)
    lo = rng.integers(0, 1 << 64, size=n, dtype=np.uint64)
    hi = rng.integers(0, 0xCB80000000000000, size=n, dtype=np.uint64)  # < p's top limb => < p
    return np.stack([lo, hi], axis=1)


def rows_np(seed, batch, k):
    """batch value vectors; from two rows on, row 1 is all zero, and from five rows on row 4 repeats row 2"""
    v = np.stack([rand_np(seed + b, k) for b in range(batch)])
    if batch >= 2:
        v[1] = 0
    if batch >= 5:
        v[4] = v[2]
    return v


def up(eng, arr):
    return eng.upload(np.ascontiguousarray(arr).reshape(-1, 2).view(np.int64)).reshape(arr.shape)


def down(vec):
    return vec.cpu().numpy().view(np.uint64)


def domain(step, k):
    x, out = 1, []
    for _ in range(k):
        out.append(x)
        x = x * step % P
    return out


def need_device(eng, k, batch):
    import torch
    release(eng)
    free, _ = torch.cuda.mem_get_info(eng.device)
    K = 1 << (2 * k - 1).bit_length()
    want = 2 * eng.lib.sa_geo_plan_bytes(k) + 48 * K * min(batch, eng.lib.sa_geo_batch_max(k)) + 64 * k * batch + \
        2 * GIB
    if free < want:
        pytest.skip("k = %d, B = %d needs %.1f GiB free on the device, %.1f GiB are"
                    % (k, batch, want / GIB, free / GIB))


def step_for(k, kind, seed):
    """a root of unity of order 2^(ceil(log2 k) + 1), or a seeded random element"""
    if kind == "root":
        return O.primitive_nth_root(1 << (max(1, (2 * k - 1).bit_length())))
    return random.Random(seed).randrange(2, P - 1)


SMALL = [1, 2, 3, 5, 17, 64, 100, 284, 1000, 1023, 1024, 1025, 1500, 2047, 2048, 2049, 4096, 5000]


@pytest.mark.parametrize("kind", ["root", "random"])
@pytest.mark.parametrize("k", SMALL)
def test_equals_the_tree_on_the_explicit_domain(eng, k, kind):
    """batches of 1, 2 and 5 rows (a zero row, two equal rows) and the zerofier: the tree's bytes"""
    q = step_for(k, kind, k)
    dom = up(eng, O.to_np(domain(q, k)))
    tree = eng.interp_plan(dom)
    plan = eng.geo_interp_plan(q, k)
    before = plan.plan.clone()
    for batch in (1, 2, 5):
        vv = up(eng, rows_np(100 * k + batch, batch, k))
        got = eng.geo_interp_apply(plan, vv)
        assert bool((got == eng.interp_apply(tree, vv)).all()), batch
        assert bool((eng.geo_interp_apply(plan, vv[0]) == got[0]).all())
    assert bool((plan.plan == before).all())
    assert bool((eng.geo_zerofier(q, k) == eng.zerofier(dom)).all())


@pytest.mark.parametrize("k", [1 << 16, (1 << 16) + 12345, 1 << 20])
def test_equals_the_tree_at_large_sizes(eng, k):
    need_device(eng, k, 2)
    q = step_for(k, "root", 0)
    dom = up(eng, O.to_np(domain(q, k)))
    vv = up(eng, rows_np(7 + k % 97, 2, k))
    want = eng.interp_apply(eng.interp_plan(dom), vv)
    assert bool((eng.geo_interp_apply(eng.geo_interp_plan(q, k), vv) == want).all())
    assert bool((eng.geo_zerofier(q, k) == eng.zerofier(dom)).all())


ABOVE = [(1 << 20) + 1, 1 << 22, pytest.param(1 << 24, marks=pytest.mark.slow)]


@pytest.mark.parametrize("k", ABOVE)
def test_above_the_tree(eng, k):
    """the interpolant takes the values at 64 sampled domain points (Horner); the zerofier vanishes there and equals
    the product of the linear factors in Python ints at two points outside the domain"""
    need_device(eng, k, 1)
    assert not eng.tree_fits(k)
    q = step_for(k, "root", 0)
    vals = rand_np(k % 1009, k)
    f = eng.geo_interp_apply(eng.geo_interp_plan(q, k), up(eng, vals))
    rng = random.Random(k)
    idx = sorted(rng.sample(range(k), 62) + [0, k - 1])
    pts = up(eng, O.to_np([pow(q, i, P) for i in idx]))
    assert (down(eng.poly_eval(f, pts, mode=1)) == vals[idx]).all()
    z = eng.geo_zerofier(q, k)
    assert not down(eng.poly_eval(z, pts, mode=1)).any()
    outside = [3, rng.randrange(2, P)]
    got = O.from_np(down(eng.poly_eval(z, up(eng, O.to_np(outside)), mode=1)))
    for x, g in zip(outside, got):
        want, d = 1, 1
        for _ in range(k):
            want = want * (x - d) % P
            d = d * q % P
        assert g == want


def test_batch_across_chunks(eng):
    """two full chunks and one more vector: every row equals a single apply"""
    k = (1 << 18) + 1
    chunk = eng.lib.sa_geo_batch_max(k)
    batch = 2 * chunk + 1
    need_device(eng, k, batch)
    plan = eng.geo_interp_plan(step_for(k, "random", 1), k)
    vv = up(eng, rows_np(11, batch, k))
    out = eng.geo_interp_apply(plan, vv)
    for b in range(batch):
        assert bool((out[b] == eng.geo_interp_apply(plan, vv[b])).all()), b


@pytest.mark.parametrize("k", [1, 1000, (1 << 16) + 1])
def test_a_batch_launches_what_one_vector_does(eng, k):
    """after a warm-up, a batch up to the chunk size issues one vector's launches: four kernels and four transforms'
    passes (the strided copy is no launch)"""
    batch = min(5, eng.lib.sa_geo_batch_max(k))
    plan = eng.geo_interp_plan(step_for(k, "random", 2), k)
    vv = up(eng, rows_np(13, batch, k))
    eng.geo_interp_apply(plan, vv)
    eng.geo_interp_apply(plan, vv[0])
    before = eng.launch_count()
    eng.geo_interp_apply(plan, vv[0])
    single = eng.launch_count() - before
    before = eng.launch_count()
    eng.geo_interp_apply(plan, vv)
    assert eng.launch_count() - before == single
    assert single >= 8


def test_errors_before_any_launch(eng):
    import torch
    k = 1000
    plan = eng.geo_interp_plan(step_for(k, "random", 3), k)
    for shape in [(3, k - 1, 2), (3, k + 1, 2), (3, k, 3), (k * 2,), (1, 3, k, 2)]:
        vv = torch.zeros(shape, dtype=torch.int64, device=eng.device)
        before = eng.launch_count()
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.geo_interp_apply(plan, vv)
        assert eng.launch_count() == before, shape
    before = eng.launch_count()
    assert tuple(eng.geo_interp_apply(plan, torch.zeros((0, k, 2), dtype=torch.int64, device=eng.device)).shape) == \
        (0, k, 2)
    assert eng.lib.sa_geo_interp_batch(None, plan.plan.data_ptr(), None, k, 0, eng._stream()) == 0
    for bad_k in (0, (1 << 26) + 1):
        assert eng.lib.sa_geo_plan_bytes(bad_k) == 0 and eng.lib.sa_geo_batch_max(bad_k) == 0
        assert eng.lib.sa_geo_interp_batch(None, None, None, bad_k, 1, eng._stream()) == -6
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.geo_interp_plan(5, bad_k)
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.geo_zerofier(5, bad_k)
    with pytest.raises(AssertionError, match="divide by zero"):
        eng.geo_interp_plan(0, 2)
    assert eng.launch_count() == before
    # a refused step leaves the zerofier's output untouched
    out = torch.full((9, 2), 7, dtype=torch.int64, device=eng.device)
    rc = eng.lib.sa_geo_zerofier(out.data_ptr(), sa_engine._limbs(O.primitive_nth_root(8)), 8, eng._stream())
    assert rc == -4 and bool((out == 7).all())
    with pytest.raises(AssertionError, match="divide by zero"):
        eng.geo_interp_plan(O.primitive_nth_root(1024), 1024)  # order exactly k
    eng.geo_interp_plan(O.primitive_nth_root(2048), 1024)


@pytest.mark.parametrize("k", [1000, 5000])
def test_one_plan_on_two_streams(eng, k):
    import torch
    plan = eng.geo_interp_plan(step_for(k, "random", 4), k)
    vvs = [up(eng, rows_np(17 + 10 * i, 3 + i, k)) for i in range(2)]
    want = [down(eng.geo_interp_apply(plan, vv)) for vv in vvs]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for rnd in range(2):
        outs = []
        for s, vv in zip(streams, vvs):
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                outs.append(eng.geo_interp_apply(plan, vv))
        torch.cuda.synchronize()
        for got, w in zip(outs, want):
            assert (down(got) == w).all(), rnd


@pytest.mark.parametrize("k", [1000, 5000])
def test_batch_in_a_cuda_graph(eng, k):
    import torch
    batch = 4
    q = step_for(k, "random", 5)
    plan = eng.geo_interp_plan(q, k)
    tree = eng.interp_plan(up(eng, O.to_np(domain(q, k))))
    vin = up(eng, rows_np(19, batch, k))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.geo_interp_apply(plan, vin)
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out = eng.geo_interp_apply(plan, vin)
    for i in range(2):
        vals = up(eng, rows_np(23 + 10 * i, batch, k))
        vin.copy_(vals)
        g.replay()
        torch.cuda.synchronize()
        assert bool((out == eng.interp_apply(tree, vals)).all()), i


def test_geo_kernels_have_no_spills():
    """ptxas's report for every k_geo_ kernel: no spill stores or loads"""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress",
                              "550", "-c", "-Xptxas", "-v", "-o", os.path.join(tmp, "poly.o"),
                              os.path.join(PKG, "csrc", "poly.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = res.stderr.splitlines()
    at = [i for i, line in enumerate(lines) if "Compiling entry function" in line and "k_geo_" in line]
    assert len(at) == 8
    for i in at:
        report = " ".join(lines[i:i + 4])
        spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
        assert spills and spills.groups() == ("0", "0"), report
