"""The Rescue-Prime kernel on the device (sa_rescue through CudaEngine.rescue and sa_rescue.hash_batch /
trace_batch): every recorded hash and trace; 2^16 random inputs in full and 2^24 inputs by samples against the
independent oracle, with every hash-only output equal to its trace's row N, register 0; the prover's index map with
stale elements; a grid past its wrap; one launch per call and errors before any launch; graph replay; no spills."""
import os
import random
import re
import subprocess
import tempfile

import numpy as np
import pytest

import rescue_cases as R
import stark_rescue_cases as SR
from test_gpu_air import PKG, release

import sa_engine  # noqa: E402  (on sys.path through test_gpu_air)
import sa_rescue  # noqa: E402

pytestmark = pytest.mark.gpu
P = R.P
STALE = 0x5A5A5A5A5A5A5A5A
A, AINV = R.exponents()


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


def dev(eng, values):
    return eng.upload(R.to_np(values).view(np.int64))


def stale(eng, n):
    return eng.upload(np.full((n, 2), STALE, dtype=np.uint64).view(np.int64))


def host(eng, vec):
    return eng.download(vec).reshape(-1, 2).view(np.uint64)


def random_inputs(n, seed):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 1 << 64, size=(n, 2), dtype=np.uint64)
    a[:, 1] %= np.uint64(407 << 55)  # below 407 * 2^119 < p
    return a


def test_every_golden_case(eng):
    g = R.golden()
    rp = SR.RescuePrime()
    xs = [int(c["input"]) for c in g["cases"]]
    assert [str(h.value) for h in sa_rescue.hash_batch(rp, xs)] == [c["hash"] for c in g["cases"]]
    traces = sa_rescue.trace_batch(rp, xs)
    assert [[[str(v.value) for v in row] for row in t] for t in traces] == [c["trace"] for c in g["cases"]]


def test_2_16_inputs_in_full(eng):
    n = 1 << 16
    xs = random_inputs(n, 16)
    kc = dev(eng, R.constants())
    inputs = eng.upload(xs.view(np.int64))
    hashes, trace = eng.empty(n), eng.empty(n * 56)
    eng.rescue(inputs, kc, 27, A, AINV, hashes=hashes, trace=trace)
    want_h, want_t = R.oracle(xs, R.to_np(R.constants()), 27, A, AINV)
    assert np.array_equal(host(eng, hashes), want_h)
    assert np.array_equal(host(eng, trace), want_t.reshape(-1, 2))


@pytest.mark.slow
def test_2_24_inputs_sampled(eng):
    import torch
    n = 1 << 24
    xs = random_inputs(n, 24)
    xs[0], xs[1], xs[-1] = (0, 0), ((1 << 64) - 1, 0), (0, 407 << 55)  # 0, 2^64 - 1, p - 1
    kc = dev(eng, R.constants())
    inputs = eng.upload(xs.view(np.int64))
    hashes, trace = eng.empty(n), eng.empty(n * 56)
    eng.rescue(inputs, kc, 27, A, AINV, hashes=hashes)
    eng.rescue(inputs, kc, 27, A, AINV, trace=trace)
    # every hash-only output is its trace's row N, register 0 (compared on the device)
    assert torch.equal(hashes, trace.reshape(n, 2, 28, 2)[:, 0, 27])
    idx = np.unique(np.concatenate([np.arange(1024), np.arange(n - 1024, n), np.arange(4096) * (n // 4096) + 777]))
    want_h, want_t = R.oracle(xs[idx], R.to_np(R.constants()), 27, A, AINV)
    sel = torch.from_numpy(idx).to(trace.device)
    assert np.array_equal(host(eng, hashes.index_select(0, sel)), want_h)
    got_t = trace.reshape(n, 56, 2).index_select(0, sel)
    assert np.array_equal(host(eng, got_t), want_t.reshape(-1, 2))


@pytest.mark.parametrize("B", [1, 3, 17])
def test_prover_index_map_with_stale_elements(eng, B):
    T = 28 + 256
    rng = random.Random(B)
    xs = [rng.randrange(P) for _ in range(B)]
    out = stale(eng, B * 2 * T + 5)
    hashes = stale(eng, B + 2)
    eng.rescue(dev(eng, xs), dev(eng, R.constants()), 27, A, AINV, hashes=hashes, trace=out, inst_stride=2 * T,
               lane_stride=T)
    want_h, want_t = R.oracle(R.to_np(xs), R.to_np(R.constants()), 27, A, AINV)
    expect = np.full((B * 2 * T + 5, 2), STALE, np.uint64)
    for b in range(B):
        for s in range(2):
            expect[(2 * b + s) * T:(2 * b + s) * T + 28] = want_t[b, s]
    assert np.array_equal(host(eng, out), expect)
    got_h = host(eng, hashes)
    assert np.array_equal(got_h[:B], want_h) and (got_h[B:] == STALE).all()


def test_grid_past_its_wrap(eng):
    """grid_for caps the grid at 16 blocks of 128 threads per SM: two and a half sweeps plus a ragged tail"""
    import torch
    sms = torch.cuda.get_device_properties(eng.device).multi_processor_count
    per_sweep = 16 * sms * 128
    n = 2 * per_sweep + per_sweep // 2 + 37
    xs = random_inputs(n, 5)
    kc = dev(eng, R.constants())
    inputs = eng.upload(xs.view(np.int64))
    hashes, trace = stale(eng, n + 1), stale(eng, n * 56 + 1)
    eng.rescue(inputs, kc, 27, A, AINV, hashes=hashes, trace=trace)
    assert torch.equal(hashes[:n], trace[:n * 56].reshape(n, 2, 28, 2)[:, 0, 27])
    idx = np.unique(np.concatenate([np.arange(64), per_sweep - 1 + np.arange(3), 2 * per_sweep + np.arange(3),
                                    np.arange(n - 200, n)]))
    want_h, want_t = R.oracle(xs[idx], R.to_np(R.constants()), 27, A, AINV)
    sel = torch.from_numpy(idx).to(trace.device)
    assert np.array_equal(host(eng, hashes.index_select(0, sel)), want_h)
    assert np.array_equal(host(eng, trace[:n * 56].reshape(n, 56, 2).index_select(0, sel)), want_t.reshape(-1, 2))
    assert (host(eng, hashes[n:]) == STALE).all() and (host(eng, trace[n * 56:]) == STALE).all()


def test_one_launch_and_errors_before_any_launch(eng):
    kc = dev(eng, R.constants())
    xs = dev(eng, [1, 2, 3])
    hashes = stale(eng, 3)
    before = eng.launch_count()
    eng.rescue(xs, kc, 27, A, AINV, hashes=hashes)
    assert eng.launch_count() - before == 1
    want_h, _ = R.oracle(R.to_np([1, 2, 3]), R.to_np(R.constants()), 27, A, AINV, trace=False)
    assert np.array_equal(host(eng, hashes), want_h)
    lib, st = eng.lib, eng._stream()
    e = (R._u128(A), R._u128(AINV))
    t = stale(eng, 3 * 56)
    before = eng.launch_count()
    assert lib.sa_rescue(None, None, xs.data_ptr(), 3, kc.data_ptr(), 27, *e, 56, 28, st) == -6
    assert lib.sa_rescue(hashes.data_ptr(), None, xs.data_ptr(), 3, kc.data_ptr(), 0, *e, 56, 28, st) == -6
    assert lib.sa_rescue(hashes.data_ptr(), None, xs.data_ptr(), 3, kc.data_ptr(), 513, *e, 56, 28, st) == -6
    assert lib.sa_rescue(None, t.data_ptr(), xs.data_ptr(), 3, kc.data_ptr(), 27, *e, (1 << 58) - 13, 0, st) == -6
    assert lib.sa_rescue(None, t.data_ptr(), xs.data_ptr(), 1, kc.data_ptr(), 27, *e, 0, (1 << 59) - 27, st) == -6
    assert lib.sa_rescue(hashes.data_ptr(), None, xs.data_ptr(), 1 << 59, kc.data_ptr(), 27, *e, 0, 0, st) == -6
    assert lib.sa_rescue(hashes.data_ptr(), t.data_ptr(), xs.data_ptr(), 0, kc.data_ptr(), 27, *e, 56, 28, st) == 0
    for kw in ({"rounds": 0}, {"rounds": 513}, {"alpha": 1 << 128}, {"alphainv": -1}, {"hashes": None},
               {"trace": stale(eng, 3 * 56 - 1)}, {"hashes": stale(eng, 2)}, {"rounds": 28}):
        args = dict(rounds=27, alpha=A, alphainv=AINV, hashes=hashes, trace=None)
        args.update(kw)
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.rescue(xs, kc, **args)
    assert eng.launch_count() == before
    assert np.array_equal(host(eng, hashes), want_h) and (host(eng, t) == STALE).all()


def test_graph_replay(eng):
    import torch
    n = 3000
    kc = dev(eng, R.constants())
    inputs = eng.upload(random_inputs(n, 0).view(np.int64))
    hashes, trace = eng.empty(n), eng.empty(n * 56)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eng.rescue(inputs, kc, 27, A, AINV, hashes=hashes, trace=trace)
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        eng.rescue(inputs, kc, 27, A, AINV, hashes=hashes, trace=trace)
    for r in range(2):
        xs = random_inputs(n, 100 + r)
        inputs.copy_(eng.upload(xs.view(np.int64)))
        hashes.fill_(0)
        trace.fill_(0)
        g.replay()
        torch.cuda.synchronize()
        want_h, want_t = R.oracle(xs, R.to_np(R.constants()), 27, A, AINV)
        assert np.array_equal(host(eng, hashes), want_h), r
        assert np.array_equal(host(eng, trace), want_t.reshape(-1, 2)), r


def test_kernel_has_no_spills():
    """ptxas's report for k_rescue: no spill stores or loads"""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress",
                              "550", "-c", "-Xptxas", "-v", "-o", os.path.join(tmp, "rescue.o"),
                              os.path.join(PKG, "csrc", "rescue.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = res.stderr.splitlines()
    at = [i for i, line in enumerate(lines) if "Compiling entry function" in line and "k_rescue" in line]
    assert len(at) == 1
    report = " ".join(lines[at[0]:at[0] + 4])
    spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert spills and spills.groups() == ("0", "0"), report
