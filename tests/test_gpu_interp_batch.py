"""Batched interpolation applies (sa_interp_apply_batch through CudaEngine.interp_apply on a (B, k, 2) tensor): every
row equals the oracle and the same vector applied alone, rows do not leak into each other, batches larger than one
chunk, the launches of a batch, errors before any launch, two streams sharing one plan and a batch captured in a CUDA
graph."""
import os
import sys

import numpy as np
import pytest

import oracle as O

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "stark-anatomy_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)
import sa_engine  # noqa: E402

pytestmark = pytest.mark.gpu
GIB = 1 << 30
MARGIN = 2 * GIB


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


def down(eng, vec):
    return vec.cpu().numpy().view(np.uint64)


def need_device(eng, k, batch):
    """skip unless the plan, its build workspace, a chunk's workspaces and the batch's values fit in free memory"""
    import torch
    release(eng)
    free, _ = torch.cuda.mem_get_info(eng.device)
    big_k = 1 << (k - 1).bit_length()
    chunk = min(batch, eng.lib.sa_interp_batch_max(k))
    want = eng.lib.sa_interp_plan_bytes(k) + 16 * (big_k.bit_length() + 24) * big_k + 96 * big_k * chunk + \
        16 * 4 * k * batch + MARGIN
    if free < want:
        pytest.skip("k = %d, B = %d needs %.1f GiB free on the device, %.1f GiB are" % (k, batch, want / GIB, free / GIB))


@pytest.mark.parametrize("batch", [1, 2, 5])
@pytest.mark.parametrize("k", [1, 2, 3, 17, 284, 1000, 1024, 1025, 1500, 4096, 5000])
def test_batch_matches_oracle_and_single_applies(eng, k, batch):
    """every row: the oracle's coefficients (k <= 1500) and the same vector through a single apply; a zero row gives
    the zero polynomial, identical rows identical ones; the plan's bytes are the same afterwards"""
    dom = rand_np(100 + k, k)
    plan = eng.interp_plan(up(eng, dom))
    before = plan.plan.clone()
    vals = rows_np(1000 + 11 * k + batch, batch, k)
    vv = up(eng, vals)
    out = eng.interp_apply(plan, vv)
    assert tuple(out.shape) == (batch, k, 2)
    got = down(eng, out)
    for b in range(batch):
        if k <= 1500:
            assert (got[b] == O.interpolate_np(dom, vals[b])).all(), (k, b)
        assert (got[b] == down(eng, eng.interp_apply(plan, vv[b]))).all(), (k, b)
    if batch >= 2:
        assert not got[1].any()
    if batch >= 5:
        assert (got[4] == got[2]).all()
    assert bool((plan.plan == before).all())


@pytest.mark.parametrize("k", [1 << 16, (1 << 16) + 12345, 1 << 20])
def test_batch_large(eng, k):
    """sizes the oracle cannot reach: every row equals a single apply, and the Horner kernel on a sample of the
    points gives each row's values back"""
    batch = 3
    need_device(eng, k, batch)
    dom, vals = rand_np(2000 + k % 101, k), rows_np(3000 + k % 101, batch, k)
    vd, vv = up(eng, dom), up(eng, vals)
    plan = eng.interp_plan(vd)
    out = eng.interp_apply(plan, vv)
    step = 257
    sample = vd[::step].contiguous()
    for b in range(batch):
        assert bool((out[b] == eng.interp_apply(plan, vv[b])).all()), b
        assert (down(eng, eng.poly_eval(out[b].contiguous(), sample, mode=1)) == vals[b, ::step]).all(), b


def test_batch_across_chunks(eng):
    """a batch of two full chunks and one more vector at a ragged tree size: every row, the last chunk's single row
    included, equals a single apply"""
    k = (1 << 16) + 1
    chunk = eng.lib.sa_interp_batch_max(k)
    batch = 2 * chunk + 1
    need_device(eng, k, batch)
    plan = eng.interp_plan(up(eng, rand_np(4000, k)))
    vv = up(eng, rows_np(4001, batch, k))
    out = eng.interp_apply(plan, vv)
    for b in range(batch):
        assert bool((out[b] == eng.interp_apply(plan, vv[b])).all()), b


@pytest.mark.parametrize("k", [1000, 1025, 5000, (1 << 16) + 1])
def test_a_batch_launches_what_one_apply_does(eng, k):
    """after a warm-up, a batch up to the chunk size issues the launches of a single apply: 2 for the Lagrange
    kernels, one ladder over the tree above them"""
    batch = min(5, eng.lib.sa_interp_batch_max(k))
    plan = eng.interp_plan(up(eng, rand_np(5000 + k, k)))
    vv = up(eng, rows_np(5001 + k, batch, k))
    eng.interp_apply(plan, vv)
    eng.interp_apply(plan, vv[0])
    before = eng.launch_count()
    eng.interp_apply(plan, vv[0])
    single = eng.launch_count() - before
    before = eng.launch_count()
    eng.interp_apply(plan, vv)
    assert eng.launch_count() - before == single
    if k <= 1024:
        assert single == 2


@pytest.mark.parametrize("k", [1000, 2048])
def test_bad_shapes_are_refused_before_any_launch(eng, k):
    import torch
    plan = eng.interp_plan(up(eng, rand_np(6000 + k, k)))
    bad = [(3, k - 1, 2), (3, k + 1, 2), (3, k, 3), (3, k, 1), (k * 2,), (1, 3, k, 2), (k, 2, 2)]
    for shape in bad:
        vv = torch.zeros(shape, dtype=torch.int64, device=eng.device)
        before = eng.launch_count()
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.interp_apply(plan, vv)
        assert eng.launch_count() == before, shape
    before = eng.launch_count()
    out = eng.interp_apply(plan, torch.zeros((0, k, 2), dtype=torch.int64, device=eng.device))
    assert tuple(out.shape) == (0, k, 2)
    assert eng.launch_count() == before
    assert eng.lib.sa_interp_apply_batch(None, plan.plan.data_ptr(), None, k, 0, eng._stream()) == 0
    assert eng.launch_count() == before


@pytest.mark.parametrize("k", [1000, 5000])
def test_one_plan_batches_on_two_streams(eng, k):
    """the plan is only read: two streams apply it at the same time to different batches"""
    import torch
    plan = eng.interp_plan(up(eng, rand_np(7000 + k, k)))
    vvs = [up(eng, rows_np(7001 + k + 10 * i, 3 + i, k)) for i in range(2)]
    want = [down(eng, torch.stack([eng.interp_apply(plan, row) for row in vv])) for vv in vvs]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for rnd in range(2):  # the first round grows each stream's workspace, the second runs without any allocation
        outs = []
        for s, vv in zip(streams, vvs):
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                outs.append(eng.interp_apply(plan, vv))
        torch.cuda.synchronize()
        for got, w in zip(outs, want):
            assert (down(eng, got) == w).all(), rnd


@pytest.mark.parametrize("k", [1000, 5000])
def test_batch_in_a_cuda_graph(eng, k):
    """a batch captured in a CUDA graph (any host synchronisation would end the capture) replays exactly on new
    values copied into the captured input"""
    import torch
    batch = 4
    dom = rand_np(8000 + k, k)
    plan = eng.interp_plan(up(eng, dom))
    vin = up(eng, rows_np(8001 + k, batch, k))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.interp_apply(plan, vin)  # grows s's workspaces outside the capture
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out = eng.interp_apply(plan, vin)
    for i in range(2):
        vals = rows_np(8100 + k + 10 * i, batch, k)
        vin.copy_(up(eng, vals))
        g.replay()
        torch.cuda.synchronize()
        got = down(eng, out)
        for b in range(batch):
            assert (got[b] == O.interpolate_np(dom, vals[b])).all(), (i, b)
