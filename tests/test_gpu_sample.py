"""Seeded randomizer draws on the device (sa_sample_seeded through CudaEngine.sample_seeded): every element against
hashlib and Python ints for three seeds and 2^20 draws each, the index map at the provers' own shapes, a grid past
its wrap, one launch per call, errors before any launch, graph replay, and no spills."""
import hashlib
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import oracle as O
import stark_seeded_cases as SS
from test_gpu_air import PKG, release

import sa_engine  # noqa: E402  (on sys.path through test_gpu_air)

pytestmark = pytest.mark.gpu
P = O.P
STALE = 0x5A5A5A5A5A5A5A5A  # each 64-bit limb of an untouched element
STALE_V = STALE | STALE << 64  # its value
SEEDS = [bytes(32), b"\xff" * 32, SS.seed("gpu")]


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


def want(seed, j):
    return int.from_bytes(hashlib.blake2b(seed + j.to_bytes(8, "little")).digest()[:17], "big") % P


def stale(eng, n):
    return eng.upload(np.full((n, 2), STALE, dtype=np.uint64).view(np.int64))


def values(eng, vec):
    return O.from_np(eng.download(vec).reshape(-1, 2).view(np.uint64))


@pytest.mark.parametrize("s", range(3), ids=["zero", "ff", "random"])
def test_every_element_against_hashlib(eng, s):
    n = 1 << 20
    first = [0, (1 << 32) - 1000, (1 << 64) - n][s]  # across 2^32 and up to 2^64 - 1
    out = eng.sample_seeded(stale(eng, n), [SEEDS[s]], first, n)
    assert values(eng, out) == [want(SEEDS[s], first + j) for j in range(n)]


@pytest.mark.parametrize("B", [1, 3, 17])
def test_index_map_at_the_provers_shapes(eng, B):
    """the trace randomizers into (B nregs, T) columns at row ncycles, and the randomizer coefficients into
    (B, max_degree + 1): every drawn element in its place, every other element untouched"""
    nregs, ncycles, R, width = 3, 1000, 8, 1024
    T = ncycles + R
    seeds = [SS.seed("map", B, b) for b in range(B)]
    dev = eng.upload_seeds(seeds)
    cols = eng.sample_seeded(stale(eng, B * nregs * T), dev, 0, R * nregs, width=nregs, lane_stride=T,
                             seed_stride=nregs * T, offset=ncycles)
    got = values(eng, cols)
    for b in range(B):
        for s in range(nregs):
            row = got[(b * nregs + s) * T:(b * nregs + s + 1) * T]
            assert row[:ncycles] == [STALE_V] * ncycles
            assert row[ncycles:] == [want(seeds[b], k * nregs + s) for k in range(R)]
    rvec = eng.sample_seeded(stale(eng, B * width + 5), dev, R * nregs, width)
    got = values(eng, rvec)
    for b in range(B):
        assert got[b * width:(b + 1) * width] == [want(seeds[b], R * nregs + i) for i in range(width)]
    assert got[B * width:] == [STALE_V] * 5


def test_grid_past_its_wrap(eng):
    """grid_for caps the grid at 16 SMs of 256-thread blocks: two and a half sweeps plus a ragged tail, width 5"""
    import torch
    sms = torch.cuda.get_device_properties(eng.device).multi_processor_count
    per_sweep = 16 * sms * 256
    count = 2 * per_sweep + per_sweep // 2 + 37
    width, lane = 5, -(-count // 5)
    out = eng.sample_seeded(stale(eng, 2 * width * lane + 3), SEEDS[1:], 7, count, width=width, lane_stride=lane,
                            seed_stride=width * lane)
    got = values(eng, out)
    for b in range(2):
        expect = [STALE_V] * (width * lane)
        for j in range(count):
            expect[(j % width) * lane + j // width] = want(SEEDS[1 + b], 7 + j)
        assert got[b * width * lane:(b + 1) * width * lane] == expect, b
    assert got[2 * width * lane:] == [STALE_V] * 3


def test_one_launch_and_errors_before_any_launch(eng):
    dev = eng.upload_seeds(SEEDS)
    out = stale(eng, 3 * 102)
    before = eng.launch_count()
    eng.sample_seeded(out, dev, 0, 100, width=3, lane_stride=34, seed_stride=102)
    assert eng.launch_count() - before == 1
    expect = [STALE_V] * (3 * 102)
    for b in range(3):
        for j in range(100):
            expect[b * 102 + (j % 3) * 34 + j // 3] = want(SEEDS[b], j)
    assert values(eng, out) == expect
    st = eng._stream()
    lib = eng.lib
    before = eng.launch_count()
    assert lib.sa_sample_seeded(out.data_ptr(), dev.data_ptr(), 3, 100, 0, 100, 0, 1, st) == -6  # width 0
    assert lib.sa_sample_seeded(out.data_ptr(), dev.data_ptr(), 0, 100, 0, 100, 1, 1, st) == 0
    assert lib.sa_sample_seeded(out.data_ptr(), dev.data_ptr(), 3, 100, 0, 0, 1, 1, st) == 0
    assert lib.sa_sample_seeded(None, None, 3, 100, (1 << 64) - 5, 6, 1, 1, st) == -6  # draw index past 2^64 - 1
    assert lib.sa_sample_seeded(None, None, 3, 1 << 59, 0, 6, 1, 1, st) == -6  # the seeds' offsets
    assert lib.sa_sample_seeded(None, None, 1, 0, 0, 4, 4, 1 << 58, st) == -6  # the lanes' offsets
    assert lib.sa_sample_seeded(None, None, 1 << 40, 1, 0, 1 << 20, 1, 1, st) == -6  # the item count
    for kw in ({"width": 0}, {"count": 107}, {"offset": 7}, {"seed_stride": 104}):
        args = dict(first=0, count=100, seed_stride=100)  # last offset 299 of 306: each change reaches 306
        args.update(kw)
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.sample_seeded(out, dev, **args)
    with pytest.raises(AssertionError, match="unsupported size"):
        eng.sample_seeded(out, [bytes(31)], 0, 1)
    with pytest.raises(AssertionError, match="unsupported size"):
        eng.sample_seeded(out, dev, (1 << 64) - 5, 6)
    assert eng.launch_count() == before
    assert values(eng, out) == expect


def test_graph_replay(eng):
    import torch
    n = 5000
    dev = eng.upload_seeds(SEEDS[:2])
    out = stale(eng, 2 * n)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.sample_seeded(out, dev, 11, n)
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        eng.sample_seeded(out, dev, 11, n)
    for r in range(2):
        seeds = [SS.seed("graph", r, b) for b in range(2)]
        dev.copy_(eng.upload_seeds(seeds))
        out.fill_(0)
        g.replay()
        torch.cuda.synchronize()
        assert values(eng, out) == [want(sd, 11 + j) for sd in seeds for j in range(n)], r


def test_kernel_has_no_spills():
    """ptxas's report for k_sample_seeded: no spill stores or loads"""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress",
                              "550", "-c", "-Xptxas", "-v", "-o", os.path.join(tmp, "sample.o"),
                              os.path.join(PKG, "csrc", "sample.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = res.stderr.splitlines()
    at = [i for i, line in enumerate(lines) if "Compiling entry function" in line and "k_sample_seeded" in line]
    assert len(at) == 1
    report = " ".join(lines[at[0]:at[0] + 4])
    spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert spills and spills.groups() == ("0", "0"), report
