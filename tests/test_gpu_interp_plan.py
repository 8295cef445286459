"""Interpolation plans (sa_interp_plan / sa_interp_apply through CudaEngine.interp_plan / interp_apply) on the
device: the same coefficients as sa_interpolate and the oracle, a plan that applies leave untouched, errors before
any launch, two streams sharing one plan, and an apply captured in a CUDA graph (no host synchronisation)."""
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


def up(eng, arr):
    return eng.upload(np.ascontiguousarray(arr).view(np.int64))


def down(eng, vec):
    return eng.download(vec).view(np.uint64)


def need_device(eng, k):
    """skip unless the plan, sa_interpolate's own plan and build workspace and a few vectors fit in free memory"""
    import torch
    release(eng)
    free, _ = torch.cuda.mem_get_info(eng.device)
    big_k = 1 << (k - 1).bit_length()
    want = 2 * eng.lib.sa_interp_plan_bytes(k) + 16 * (big_k.bit_length() + 24) * big_k + MARGIN
    if free < want:
        pytest.skip("k = %d needs %.1f GiB free on the device, %.1f GiB are" % (k, want / GIB, free / GIB))


@pytest.mark.parametrize("k", [1, 2, 3, 17, 284, 512, 513, 1000, 1024, 1025, 1500, 2048, 4096, 5000])
def test_apply_matches_oracle_and_interpolate(eng, k):
    """three value vectors through one plan: the oracle's coefficients (k <= 1500) and sa_interpolate's (every k),
    and the plan's bytes are the same afterwards"""
    dom = rand_np(900 + k, k)
    vd = up(eng, dom)
    plan = eng.interp_plan(vd)
    assert plan.k == k and plan.plan.numel() == eng.lib.sa_interp_plan_bytes(k)
    before = plan.plan.clone()
    for s in range(3):
        vals = rand_np(1900 + 7 * k + s, k)
        vv = up(eng, vals)
        got = down(eng, eng.interp_apply(plan, vv))
        assert got.shape[0] == k
        if k <= 1500:
            assert (got == O.interpolate_np(dom, vals)).all(), (k, s)
        assert (got == down(eng, eng.interpolate(vd, vv))).all(), (k, s)
    assert bool((plan.plan == before).all())


@pytest.mark.parametrize("k", [1 << 16, (1 << 16) + 12345, 1 << 18, 1 << 20])
def test_apply_large(eng, k):
    """sizes the oracle cannot reach (M'(d_i) by the walk down the tree): apply == sa_interpolate, and the Horner
    kernel on a sample of the points gives the values back"""
    need_device(eng, k)
    dom, vals = rand_np(2900 + k % 101, k), rand_np(2901 + k % 101, k)
    vd, vv = up(eng, dom), up(eng, vals)
    plan = eng.interp_plan(vd)
    poly = eng.interp_apply(plan, vv)
    assert eng.length(poly) == k
    assert bool((poly == eng.interpolate(vd, vv)).all())
    step = 257
    assert (down(eng, eng.poly_eval(poly, vd[::step].contiguous(), mode=1)) == vals[::step]).all()


@pytest.mark.parametrize("k", [3, 1500, 5000, (1 << 16) + 1])
def test_coincident_points(eng, k):
    """the Lagrange kernels (3), Horner for M'(d_i) (1500, 5000) and the walk (2^16 + 1) all report the repeated
    point while the plan is built"""
    dom = rand_np(3900 + k, k)
    dom[k - 1] = dom[0]
    with pytest.raises(AssertionError, match="divide by zero"):
        eng.interp_plan(up(eng, dom))


@pytest.mark.parametrize("k", [1000, 2048])
def test_wrong_length_is_refused_before_any_launch(eng, k):
    plan = eng.interp_plan(up(eng, rand_np(4900 + k, k)))
    for n in (k - 1, k + 1, 0):
        vv = up(eng, rand_np(4901 + n, n))
        before = eng.launch_count()
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.interp_apply(plan, vv)
        assert eng.launch_count() == before


@pytest.mark.parametrize("k", [1000, 5000])
def test_one_plan_on_two_streams(eng, k):
    """the plan is only read: two streams apply it at the same time to different values"""
    import torch
    dom = rand_np(5900 + k, k)
    vd = up(eng, dom)
    plan = eng.interp_plan(vd)
    vals = [rand_np(5901 + k + i, k) for i in range(2)]
    vvs = [up(eng, v) for v in vals]
    want = [down(eng, eng.interpolate(vd, v)) for v in vvs]
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


@pytest.mark.parametrize("k", [1000, 5000, 1 << 16])
def test_apply_in_a_cuda_graph(eng, k):
    """an apply captured in a CUDA graph (any host synchronisation would end the capture) replays exactly on new
    values copied into the captured input"""
    import torch
    dom = rand_np(6900 + k, k)
    vd = up(eng, dom)
    plan = eng.interp_plan(vd)
    vin = up(eng, rand_np(6901 + k, k))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.interp_apply(plan, vin)  # grows s's workspaces outside the capture
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out = eng.interp_apply(plan, vin)
    for i in range(2):
        vals = rand_np(6902 + k + i, k)
        vin.copy_(up(eng, vals))
        g.replay()
        torch.cuda.synchronize()
        assert (down(eng, out) == down(eng, eng.interpolate(vd, up(eng, vals)))).all(), i
