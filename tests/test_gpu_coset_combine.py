"""Coset combinations on the device (sa_coset_combine_evaluate through the C ABI and CudaEngine.coset_combine_evaluate):
every case against the combination restated with Python ints and the oracle's fast_coset_evaluate
(tests/combine_cases.py), the prover's chain from coset division through the combination to the FRI commit and
Fri.prove, large sizes by an exact property, the launches of a call, errors before any launch, two streams sharing
sources, a call captured in a CUDA graph, and the kernel's registers."""
import ctypes
import os
import pickle
import random
import re
import subprocess
import sys
import tempfile

import numpy as np
import pytest

import oracle as O
from combine_cases import P, codeword, make_terms, ncomb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "stark-anatomy_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)
import sa_engine  # noqa: E402

pytestmark = pytest.mark.gpu
GIB = 1 << 30
PATTERN = 0x0A5A5A5A5A5A5A5A  # a non-zero fill: an element the call fails to write shows up


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


def up(eng, values):
    if not values:
        return eng.empty(0)
    return eng.upload(O.to_np(values).view(np.int64))


def down(vec):
    return O.from_np(vec.cpu().numpy().view(np.uint64))


def rand_dev(eng, shape, seed):
    """random canonical elements (< 2^125 < p) on the device"""
    import torch
    g = torch.Generator(device=eng.device)
    g.manual_seed(seed)
    x = torch.randint(0, 1 << 62, tuple(shape) + (2,), dtype=torch.int64, device=eng.device, generator=g)
    x[..., 1] &= (1 << 61) - 1
    return x


def filled(eng, n):
    import torch
    return torch.full((n, 2), PATTERN, dtype=torch.int64, device=eng.device)


def abi(eng, out, log_n, root, offset, vecs, terms):
    """sa_coset_combine_evaluate into `out` (any contents) over device rows vecs[r] for terms (r, shift, weight)"""
    t = len(terms)
    ws = []
    for _, _, w in terms:
        ws += [w & 0xFFFFFFFFFFFFFFFF, w >> 64]
    return eng.lib.sa_coset_combine_evaluate(
        out.data_ptr(), log_n, sa_engine._limbs(root), sa_engine._limbs(offset),
        (ctypes.c_void_p * t)(*[vecs[r].data_ptr() for r, _, _ in terms]),
        (ctypes.c_size_t * t)(*[vecs[r].shape[0] for r, _, _ in terms]),
        (ctypes.c_size_t * t)(*[s for _, s, _ in terms]), (ctypes.c_uint64 * (2 * t))(*ws), t, eng._stream())


def eng_terms(vecs, terms):
    return [(vecs[r], s, w) for r, s, w in terms]


def need_device(eng, log_n, vectors):
    import torch
    release(eng)
    free, _ = torch.cuda.mem_get_info(eng.device)
    want = (16 << log_n) * vectors + 2 * GIB
    if free < want:
        pytest.skip("2^%d needs %.1f GiB free on the device, %.1f GiB are" % (log_n, want / GIB, free / GIB))


CASES = [(lg, T, k) for lg in range(1, 13) for T in (0, 1, 9, 64, 65, 129) for k in ("random", "zero", "one")] + \
        [(16, T, "random") for T in (0, 1, 9, 64, 65, 129)] + [(20, T, "random") for T in (1, 9, 65, 129)]


@pytest.mark.parametrize("log_n, T, offset_kind", CASES)
def test_matches_oracle(eng, log_n, T, offset_kind):
    """out, filled with a non-zero pattern first, is the reference's combined_codeword; the engine call agrees"""
    n = 1 << log_n
    seed = 1000 * log_n + T
    rows, terms = make_terms(seed, n, T, max_len=None if log_n <= 12 else 1 << 12)
    root = O.primitive_nth_root(n)
    offset = {"random": random.Random(seed).randrange(2, P), "zero": 0, "one": 1}[offset_kind]
    vecs = [up(eng, r) for r in rows]
    out = filled(eng, n)
    assert abi(eng, out, log_n, root, offset, vecs, terms) == 0
    want = codeword(rows, terms, n, root, offset)
    assert down(out) == want
    got = eng.coset_combine_evaluate(eng_terms(vecs, terms), log_n, root, offset)
    assert tuple(got.shape) == (n, 2) and bool((got == out).all())


def faststark_terms(eng, log_n, seed):
    """FastStark-shaped terms for a FRI domain of n = 2^log_n (expansion factor 4, max_degree = n/4 - 1): two
    transition quotients from one coset_div_apply batch (rows of one tensor), two boundary-quotient-like rows of other
    lengths from separate tensors, a randomizer; FastStark's shifts max_degree - deg q and seeded weights"""
    n, m = 1 << log_n, 1 << (log_n - 2)
    rng = random.Random(seed)
    omicron = O.primitive_nth_root(m)
    plan = eng.coset_div_plan(rand_dev(eng, (m // 4 + 1,), seed), log_n - 2, omicron, O.GENERATOR)
    qlen = m - m // 4
    quotients = eng.coset_div_apply(plan, rand_dev(eng, (2, m), seed + 1), qlen)
    rows = [rand_dev(eng, (m,), seed + 2)] + [quotients[0], quotients[1]] + \
        [rand_dev(eng, (m - 5,), seed + 3), rand_dev(eng, (m // 2 + 3,), seed + 4)]
    terms = [(rows[0], 0, rng.randrange(P))]
    for q in rows[1:]:
        terms += [(q, 0, rng.randrange(P)), (q, m - q.shape[0], rng.randrange(P))]
    return terms


def oracle_codeword(terms, n, root, offset):
    c = [0] * n
    for vec, shift, w in terms:
        for j, v in enumerate(down(vec)):
            c[shift + j] = (c[shift + j] + w * v) % P
    return O.fast_coset_evaluate(c, offset, root, n)


@pytest.mark.parametrize("log_n", [12, 16])
def test_prover_chain_into_fri(eng, log_n):
    """quotients from coset_div_apply and other rows -> coset_combine_evaluate -> fri_commit: every round root and the
    last codeword equal the oracle's FRI commit of the oracle's codeword; Fri.prove gives the same pickled transcript
    on the device codeword (wrapped as a DeviceCodeword) as on the plain list"""
    from hostmirror_loader import load_host_types
    T = load_host_types()
    import fri as F
    import sa_devlist
    n = 1 << log_n
    omega = O.primitive_nth_root(n)
    terms = faststark_terms(eng, log_n, 50 + log_n)
    cw = eng.coset_combine_evaluate(terms, log_n, omega, O.GENERATOR)
    want = oracle_codeword(terms, n, omega, O.GENERATOR)
    assert down(cw) == want
    ncol = 16
    roots, alphas, layers = O.fri_commit_np(O.to_np(want), O.GENERATOR, omega, 4, ncol)
    got_roots = []
    got_layers, _ = eng.fri_commit(cw, len(roots), O.GENERATOR, omega,
                                   lambda r, root, wanted: (got_roots.append(root), alphas[r] if wanted else 0)[1])
    assert got_roots == roots
    assert down(got_layers[-1]) == O.from_np(layers[-1])
    fri = F.Fri(T.field.generator(), T.field.primitive_nth_root(n), n, 4, ncol)
    ps_list, ps_dev = F.ProofStream(), F.ProofStream()
    idx_list = fri.prove([T.fe(v) for v in want], ps_list)
    idx_dev = fri.prove(sa_devlist.DeviceCodeword(cw, None, T.field, n), ps_dev)
    assert idx_dev == idx_list
    assert pickle.dumps(ps_dev.objects) == pickle.dumps(ps_list.objects)


@pytest.mark.parametrize("log_n", [22, 24, 26])
def test_large_sizes_by_property(eng, log_n):
    """intt(out) * offset^-i is the combination: checked on sampled indices with Python ints, and zero from ncomb on"""
    need_device(eng, log_n, 8)
    n = 1 << log_n
    rng = random.Random(log_n)
    root, offset = O.primitive_nth_root(n), rng.randrange(2, P)
    q = rand_dev(eng, (2, n // 4), log_n)
    terms = [(rand_dev(eng, (n // 4,), log_n + 1), 0, rng.randrange(P))]
    for k, length in enumerate((n // 4, n // 4, n // 8 + 3)):
        row = q[k] if k < 2 else rand_dev(eng, (length,), log_n + 2)
        terms += [(row, 0, rng.randrange(P)), (row, n // 4 - row.shape[0] + 17 * k, rng.randrange(P))]
    m = max(s + v.shape[0] for v, s, _ in terms)
    out = eng.coset_combine_evaluate(terms, log_n, root, offset)
    coeffs = eng.ntt(out, log_n, root, inverse=True)
    del out
    assert not bool(coeffs[m:].any())
    idx = sorted({0, 1, m - 1, n // 4 - 1, n // 8} | {rng.randrange(m) for _ in range(4096)})
    got = O.from_np(coeffs[idx].cpu().numpy().view(np.uint64))
    c = dict.fromkeys(idx, 0)
    for v, s, w in terms:  # each term's elements at the sampled indices it covers
        sel = [i for i in idx if s <= i < s + v.shape[0]]
        for i, x in zip(sel, down(v[[i - s for i in sel]])):
            c[i] += w * x
    inv = O.inverse(offset)
    for i, g in zip(idx, got):
        assert g * pow(inv, i, P) % P == c[i] % P, i


@pytest.mark.parametrize("log_n", [12, 20])
@pytest.mark.parametrize("T", [1, 64, 65, 129])
def test_launch_count(eng, log_n, T):
    """after a warm call, exactly 1 + ceil(T / 64) launches plus those of one sa_ntt at that size"""
    n = 1 << log_n
    root = O.primitive_nth_root(n)
    rows = [rand_dev(eng, (n // 2,), 3), rand_dev(eng, (n // 4,), 4)]
    terms = [(rows[t % 2], t % 7, t + 1) for t in range(T)]
    eng.coset_combine_evaluate(terms, log_n, root, 3)
    x = rand_dev(eng, (n,), 5)
    eng.ntt_into(x, x, log_n, root)
    before = eng.launch_count()
    eng.ntt_into(x, x, log_n, root)
    per_ntt = eng.launch_count() - before
    before = eng.launch_count()
    eng.coset_combine_evaluate(terms, log_n, root, 3)
    assert eng.launch_count() - before == 1 + (T + 63) // 64 + per_ntt


@pytest.mark.parametrize("log_n", [3, 12])
def test_errors_before_any_launch(eng, log_n):
    """every refused call leaves the launch count and out as they were"""
    import torch
    n = 1 << log_n
    root = O.primitive_nth_root(n)
    vecs = [rand_dev(eng, (n // 2,), 1), rand_dev(eng, (n // 2 + 1,), 2)]
    good = [(0, 0, 5), (0, n // 2, 6)]
    out = filled(eng, n)
    abi(eng, out, log_n, root, 7, vecs, good)  # warm
    out.fill_(PATTERN)
    before = eng.launch_count()
    for lg, r, terms, code in ((log_n, root, good + [(1, n // 2, 9)], -6),  # shift + len = n + 1
                               (0, root, good, -6), (31, root, good, -6),
                               (log_n, O.primitive_nth_root(2 * n), good, -2),
                               (log_n, O.primitive_nth_root(n // 2), good, -3)):
        assert abi(eng, out, lg, r, 7, vecs, terms) == code, (lg, code)
    msg = "unsupported size"
    bad_terms = [[(vecs[1], n // 2, 1)], [(vecs[0], -1, 1)], [(vecs[0].to(torch.int32), 0, 1)],
                 [(vecs[0].reshape(-1), 0, 1)], [(vecs[0].cpu(), 0, 1)], [(vecs[0][::2], 0, 1)],
                 [(torch.zeros((4, 3), dtype=torch.int64, device=eng.device), 0, 1)]]
    for terms in bad_terms:
        with pytest.raises(AssertionError, match=msg):
            eng.coset_combine_evaluate(terms, log_n, root, 7)
    for lg in (0, 31):
        with pytest.raises(AssertionError, match=msg):
            eng.coset_combine_evaluate([(vecs[0], 0, 1)], lg, root, 7)
    with pytest.raises(AssertionError, match="must be nth root"):
        eng.coset_combine_evaluate([(vecs[0], 0, 1)], log_n, O.primitive_nth_root(2 * n), 7)
    assert eng.launch_count() == before
    assert bool((out == PATTERN).all())
    assert not bool(eng.coset_combine_evaluate([], log_n, root, 7).any())  # the empty combination


@pytest.mark.parametrize("log_n", [10, 16])
def test_two_streams_sharing_sources(eng, log_n):
    """two calls at once on two streams, over the same source rows with different weights and shifts"""
    import torch
    n = 1 << log_n
    root = O.primitive_nth_root(n)
    rows = [rand_dev(eng, (n // 2,), 11), rand_dev(eng, (n // 4,), 12)]
    sets = [[(rows[t % 2], (3 * t + i) % (n // 4), 100 * i + t) for t in range(70)] for i in range(2)]
    want = [eng.coset_combine_evaluate(s, log_n, root, 5 + i) for i, s in enumerate(sets)]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for rnd in range(2):  # the first round grows each stream's workspaces, the second runs without any allocation
        outs = []
        for i, (s, terms) in enumerate(zip(streams, sets)):
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                outs.append(eng.coset_combine_evaluate(terms, log_n, root, 5 + i))
        torch.cuda.synchronize()
        for got, w in zip(outs, want):
            assert bool((got == w).all()), rnd


@pytest.mark.parametrize("log_n", [10, 16])
def test_in_a_cuda_graph(eng, log_n):
    """a call captured after one warm call replays to the same output, and to the new codeword after new values are
    copied into the captured rows (a replay uses the terms it was captured with)"""
    import torch
    n = 1 << log_n
    root = O.primitive_nth_root(n)
    rows = [rand_dev(eng, (n // 2,), 21), rand_dev(eng, (n // 4 + 1,), 22)]
    terms = [(rows[t % 2], t, 7 * t + 1) for t in range(66)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        want = eng.coset_combine_evaluate(terms, log_n, root, 9)
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out = eng.coset_combine_evaluate(terms, log_n, root, 9)
    g.replay()
    torch.cuda.synchronize()
    assert bool((out == want).all())
    rows[0].copy_(rand_dev(eng, (n // 2,), 23))
    g.replay()
    torch.cuda.synchronize()
    assert bool((out == eng.coset_combine_evaluate(terms, log_n, root, 9)).all())


def test_kernel_has_no_spills():
    """ptxas's report for k_coset_combine: no spill stores or loads"""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress",
                              "550", "-c", "-Xptxas", "-v", "-o", os.path.join(tmp, "poly.o"),
                              os.path.join(PKG, "csrc", "poly.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = res.stderr.splitlines()
    at = [i for i, line in enumerate(lines) if "Compiling entry function" in line and "k_coset_combine" in line]
    assert len(at) == 1
    report = " ".join(lines[at[0]:at[0] + 4])
    spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert spills and spills.groups() == ("0", "0"), report
