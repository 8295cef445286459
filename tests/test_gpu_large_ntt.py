"""Transforms of 2^27 ... 2^30 points on the H100 (``pytest -m gpu``): the three-pass plan with factored pass-1
twiddles (ntt_plan.cuh), through sa_ntt, sa_ntt_multi, sa_ntt_host and the drop-in ntt module.

2^27 is checked against the OpenMP oracle.  2^28 ... 2^30 (16 GiB per vector at 2^30) are checked like the 2^26
case of test_gpu.py: an impulse against host pow at sampled indices, all-ones against n * e_0 and a random round
trip, all in place.  A size is skipped when the device has not got the memory free; nothing larger than what is
free is ever allocated, and every size releases its workspaces when it is done."""
import os
import random
import sys

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
MARGIN = 2 * GIB  # plan tables, gather buffers, torch's own reserve


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


def release(eng):
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert eng.lib.sa_release_workspaces() == 0


def need_device(eng, vectors, log_n):
    """skip unless `vectors` n-element vectors (the transform's own workspace counted) fit in free memory"""
    import torch
    release(eng)
    free, _ = torch.cuda.mem_get_info(eng.device)
    want = vectors * (16 << log_n) + MARGIN
    if free < want:
        pytest.skip("2^%d needs %.1f GiB free on the device, %.1f GiB are" % (log_n, want / GIB, free / GIB))


def need_host(nbytes):
    avail = os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    if avail < nbytes + 4 * GIB:
        pytest.skip("needs %.1f GiB of free host memory, %.1f GiB are" % (nbytes / GIB, avail / GIB))


def rand_np(seed, n):
    rng = np.random.default_rng(seed)
    lo = rng.integers(0, 1 << 64, size=n, dtype=np.uint64)
    hi = rng.integers(0, 0xCB80000000000000, size=n, dtype=np.uint64)  # < p's top limb => < p
    return np.stack([lo, hi], axis=1)


def up(eng, arr):
    return eng.upload(np.ascontiguousarray(arr).view(np.int64))


def down(eng, vec):
    return eng.download(vec).view(np.uint64)


def random_root(log_n, seed):
    n = 1 << log_n
    return pow(O.primitive_nth_root(n), 2 * random.Random(seed).randrange(n // 2) + 1, P)  # odd power: primitive


def sa_ntt(eng, out, vec, log_n, w, inverse=0, batch=1):
    return eng.lib.sa_ntt(out.data_ptr(), vec.data_ptr(), log_n, sa_engine._limbs(w), inverse, batch, eng._stream())


def test_ntt_2_27_against_oracle(eng):
    """forward and inverse with a random primitive root, out of place and in place, bit for bit"""
    log_n = 27
    n = 1 << log_n
    need_device(eng, 3, log_n)
    need_host(5 * 16 * n)
    w = random_root(log_n, 27)
    x = rand_np(27, n)
    vx = up(eng, x)
    want = O.ntt_np(w, x, parallel=True)
    assert (down(eng, eng.ntt(vx, log_n, w)) == want).all()
    want_inv = O.intt_np(w, x, parallel=True)
    assert (down(eng, eng.ntt(vx, log_n, w, inverse=True)) == want_inv).all()
    del want_inv
    assert sa_ntt(eng, vx, vx, log_n, w) == 0
    assert (down(eng, vx) == want).all()
    assert sa_ntt(eng, vx, vx, log_n, w, inverse=1) == 0
    assert (down(eng, vx) == x).all()


@pytest.mark.parametrize("log_n", [pytest.param(28, marks=pytest.mark.slow),
                                   pytest.param(29, marks=pytest.mark.slow),
                                   pytest.param(30, marks=pytest.mark.slow)])
def test_ntt_largest_sizes_in_place(eng, log_n):
    """an impulse at a random j comes out as c * w^(i*j) (sampled indices, host pow), all-ones as n * e_0, and
    a random vector survives the round trip; one vector plus the transform's workspace"""
    import torch
    n = 1 << log_n
    need_device(eng, 2, log_n)
    w = random_root(log_n, log_n)
    rng = random.Random(log_n)
    j, c = rng.randrange(n), rng.randrange(1, P)
    v = eng.zeros(n)
    s64 = lambda u: u - (1 << 64) if u >= (1 << 63) else u  # limb as the int64 torch stores
    v[j, 0] = s64(c & 0xFFFFFFFFFFFFFFFF)
    v[j, 1] = s64(c >> 64)
    assert sa_ntt(eng, v, v, log_n, w) == 0
    idx = [0, 1, n - 1, n // 2] + [rng.randrange(n) for _ in range(500)]
    got = eng.gather(v, idx).view(np.uint64)
    for k, i in enumerate(idx):
        assert int(got[k][0]) | (int(got[k][1]) << 64) == c * pow(w, (i * j) % n, P) % P, i
    v.zero_()
    v[:, 0] = 1
    assert sa_ntt(eng, v, v, log_n, w) == 0
    assert int(v[0, 0]) == n and int(v[0, 1]) == 0 and not bool(v[1:].any())
    # random values regenerated chunk by chunk from seeded generators, so no second 16 GiB copy is kept
    chunk = 1 << 24
    gen = torch.Generator(device=eng.device)

    def chunk_values(ci):
        gen.manual_seed(1000 * log_n + ci)
        x = torch.randint(0, 1 << 62, (chunk, 2), dtype=torch.int64, device=eng.device, generator=gen)
        x[:, 1] &= (1 << 61) - 1
        return x

    for ci in range(n // chunk):
        v[ci * chunk:(ci + 1) * chunk] = chunk_values(ci)
    assert sa_ntt(eng, v, v, log_n, w) == 0
    assert sa_ntt(eng, v, v, log_n, w, inverse=1) == 0
    for ci in range(n // chunk):
        assert bool((v[ci * chunk:(ci + 1) * chunk] == chunk_values(ci)).all()), ci


def test_ntt_multi_2_27(eng):
    """sa_ntt_multi into two local buffers stores what sa_ntt computes, in both"""
    log_n = 27
    n = 1 << log_n
    need_device(eng, 5, log_n)
    w = random_root(log_n, 271)
    vx = up(eng, rand_np(271, n))
    ref = eng.ntt(vx, log_n, w)
    outs = [eng.zeros(n), eng.zeros(n)]
    eng.ntt_multi(outs, 0, vx, log_n, w)
    assert bool((outs[0] == ref).all()) and bool((outs[1] == ref).all())


def test_ntt_host_2_27_batch_2(eng):
    """sa_ntt_host above 2^26 (one transform at a time through one staging buffer) equals the device result,
    and its inverse, in place on the host buffer, returns the input"""
    log_n, batch = 27, 2
    n = 1 << log_n
    need_device(eng, 5, log_n)  # staging buffer, then input, output and workspace of the device transform
    need_host(3 * batch * 16 * n)
    w = random_root(log_n, 272)
    x = rand_np(272, batch * n)
    y = np.empty_like(x)
    root = sa_engine._limbs(w)
    assert eng.lib.sa_ntt_host(y.ctypes.data, x.ctypes.data, log_n, root, 0, batch, eng._stream()) == 0
    for b in range(batch):
        assert bool((eng.ntt(up(eng, x[b * n:(b + 1) * n]), log_n, w) == up(eng, y[b * n:(b + 1) * n])).all()), b
    assert eng.lib.sa_ntt_host(y.ctypes.data, y.ctypes.data, log_n, root, 1, batch, eng._stream()) == 0
    assert np.array_equal(y, x)


def test_dropin_coset_evaluate_2_27(eng):
    """fast_coset_evaluate of a 1000-coefficient polynomial on a 2^27 coset: sampled values equal Horner at
    g * w^i, and intt gives back the coefficients times g^i followed by zeros"""
    import sa_host
    import ntt as N
    log_n = 27
    n = 1 << log_n
    need_device(eng, 5, log_n)
    field = sa_host.algebra.Field.main()
    FE = sa_host.algebra.FieldElement
    rng = random.Random(273)
    coeffs = [rng.randrange(P) for _ in range(1000)]
    g, w = field.generator(), field.primitive_nth_root(n)
    cw = N.fast_coset_evaluate(N.Polynomial([FE(c, field) for c in coeffs]), g, w, n)
    assert len(cw) == n and not isinstance(cw, list)
    idx = [0, 1, n - 1, n // 2] + [rng.randrange(n) for _ in range(300)]
    got = eng.gather(N.sa_devlist.to_device(cw), idx).view(np.uint64)
    for k, i in enumerate(idx):
        x = g.value * pow(w.value, i, P) % P
        acc = 0
        for c in reversed(coeffs):
            acc = (acc * x + c) % P
        assert int(got[k][0]) | (int(got[k][1]) << 64) == acc, i
    back = N.sa_devlist.to_device(N.intt(w, cw))
    scaled = [c * pow(g.value, i, P) % P for i, c in enumerate(coeffs)]
    assert bool((back[:1000] == up(eng, O.to_np(scaled))).all())
    assert not bool(back[1000:].any())


def test_short_vector_is_refused_before_any_launch(eng):
    """at log_n 27 (a valid 2^27 root) a vector shorter than batch << log_n raises "unsupported size" in every
    sa_engine entry point, and no kernel is launched"""
    log_n = 27
    n = 1 << log_n
    need_device(eng, 2, log_n)
    w = O.primitive_nth_root(n)
    short = eng.empty(n - 1)
    full = eng.empty(n)
    before = eng.launch_count()
    calls = [lambda: eng.ntt(short, log_n, w),
             lambda: eng.ntt(full, log_n, w, batch=2),
             lambda: eng.ntt(eng.empty(16), log_n, w, inverse=True),
             lambda: eng.ntt_into(short, short, log_n, w),
             lambda: eng.ntt_multi([short], 0, short, log_n, w),
             lambda: eng.ntt_mcast(0, full, 0, full, log_n, w, batch=2)]
    for call in calls:
        with pytest.raises(AssertionError, match="unsupported size"):
            call()
    assert eng.launch_count() == before
