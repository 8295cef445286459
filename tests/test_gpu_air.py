"""Transition quotients on the device (sa_air_plan / sa_air_quotients through CudaEngine.air_plan / air_quotients):
every case against the quotients restated with Python ints (tests/air_cases.py), the reference's quotients of
tests/golden/air.json bit for bit, the prover's chain from the recorded trace polynomials through the combination to
the recorded FRI codeword and transcript, large sizes by an exact property, several chunks of constraints, the
launches of an apply, errors before any launch, one plan on two streams, an apply captured in a CUDA graph, and the
kernel's registers."""
import hashlib
import json
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
from air_cases import (P, evaluate, golden, golden_air, ints, make_air, make_case, quotients)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "stark-anatomy_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)
import sa_engine  # noqa: E402

pytestmark = pytest.mark.gpu
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


def up(eng, values):
    return eng.upload(O.to_np(values).view(np.int64))


def down(vec):
    return O.from_np(vec.contiguous().cpu().numpy().view(np.uint64).reshape(-1, 2))


def rows(eng, trace):
    return up(eng, [v for r in trace for v in r]).reshape(len(trace), len(trace[0]), 2)


def run(eng, air, trace, zerofier, max_ncoef, root, offset, step, qlen, log_n):
    plan = eng.air_plan(air, len(trace), up(eng, zerofier), max_ncoef, log_n, root, offset, step)
    out = eng.air_quotients(plan, rows(eng, trace), qlen)
    assert tuple(out.shape) == (len(air), qlen, 2)
    return [down(out[c]) for c in range(len(air))]


CASES = [(lg, r, c, "random", "root") for lg in range(1, 13) for r in (1, 2, 3, 5) for c in (1, 2, 7)] + \
        [(lg, 2, 7, o, s) for lg in (1, 6, 12) for o, s in (("zero", "root"), ("one", "outside"),
                                                              ("random", "outside"))] + \
        [(16, r, 7, "random", s) for r, s in ((1, "root"), (2, "outside"))]


@pytest.mark.parametrize("log_n, nregs, ncons, offset_kind, step_kind", CASES)
def test_matches_restatement(eng, log_n, nregs, ncons, offset_kind, step_kind):
    seed = 100 * log_n + 10 * nregs + ncons
    air, trace, z, max_ncoef, root, offset, step, qlen = make_case(seed, log_n, nregs, ncons, offset_kind=offset_kind,
                                                                   step_kind=step_kind)
    want = quotients(air, trace, z, 1 << log_n, root, offset, step)
    assert run(eng, air, trace, z, max_ncoef, root, offset, step, qlen, log_n) == want


@pytest.mark.parametrize("log_n", [4, 10, 12])
def test_short_trace_and_qlen(eng, log_n):
    n = 1 << log_n
    qlen = n - n // 3
    air, trace, z, max_ncoef, root, offset, step, _ = make_case(log_n, log_n, 3, 7, short=True)
    want = quotients(air, trace, z, n, root, offset, step)
    assert run(eng, air, trace, z, max_ncoef, root, offset, step, qlen, log_n) == [w[:qlen] for w in want]


@pytest.mark.parametrize("rec_name", ["faststark", "false_witness", "config5"])
def test_golden(eng, rec_name):
    """the reference's fast_coset_divide(evaluate_symbolic(...)) bit for bit"""
    rec = golden()[rec_name]
    trace = [ints(r) for r in rec["trace"]]
    got = run(eng, golden_air(rec), trace, ints(rec["zerofier"]), len(trace[0]), int(rec["root"]),
              int(rec["offset"]), int(rec["step"]), rec["qlen"], rec["log_n"])
    assert got == [ints(q) for q in rec["quotients"]]


def test_engine_takes_mpolynomial_shapes(eng):
    """objects with a .dictionary and values with .value, short tuples zero-padded and merged where they meet"""
    class V:
        def __init__(self, v):
            self.value = v

    class M:
        def __init__(self, d):
            self.dictionary = d
    rec = golden()["faststark"]
    air = golden_air(rec)
    trace = [ints(r) for r in rec["trace"]]
    wrapped = [M({k: V(v) for k, v in a.items()}) for a in air]
    wrapped[0].dictionary[(0,)] = V(5)  # (0,) and (0, 0, 0, 0, 0) meet: the constant term grows by 5
    wrapped[0].dictionary[(0, 0, 0, 0, 0)] = V(P - 5 + air[0].get((0, 0, 0, 0, 0), 0))
    got = run(eng, wrapped, trace, ints(rec["zerofier"]), len(trace[0]), int(rec["root"]), int(rec["offset"]),
              int(rec["step"]), rec["qlen"], rec["log_n"])
    assert got == [ints(q) for q in rec["quotients"]]


def test_prover_chain_into_fri(eng):
    """the recorded trace polynomials -> air_quotients -> coset_combine_evaluate with the recorded boundary quotients,
    randomizer and the weights sample_weights derives from the recorded transcript: the recorded combined codeword,
    element for element, and the drop-in Fri.prove on it reproduces the recorded transcript"""
    from hostmirror_loader import load_host_types
    T = load_host_types()
    import fri as F
    import sa_devlist
    rec = golden()["faststark"]
    with open(os.path.join(ROOT, "tests", "golden", "faststark_trace.json")) as f:
        g = json.load(f)
    calls, p, fp = g["calls"], g["params"], g["fri_prove"][0]
    trace = [ints(r) for r in rec["trace"]]
    assert trace == [ints(c["out"]["poly"]) for c in calls if c["fn"] == "fast_interpolate"]
    plan = eng.air_plan(golden_air(rec), 2, up(eng, ints(rec["zerofier"])), len(trace[0]), rec["log_n"],
                        int(rec["root"]), int(rec["offset"]), int(rec["step"]))
    tq = eng.air_quotients(plan, rows(eng, trace), rec["qlen"])
    evals = [ints(c["args"][0]["poly"]) for c in calls if c["fn"] == "fast_coset_evaluate"]
    boundary, randomizer = evals[1:3], evals[3]
    n = p["fri_domain_length"]
    max_degree = len(randomizer) - 1
    objects = [T.dec_obj(o) for o in fp["prior_objects"]]
    seed = O.fiat_shamir(objects)
    weights = [O.sample(hashlib.blake2b(seed + bytes(i)).digest()) for i in range(9)]
    terms = [(up(eng, randomizer), 0, weights[0])]
    for i in range(2):
        q = tq[i]
        terms += [(q, 0, weights[1 + 2 * i]), (q, max_degree - (q.shape[0] - 1), weights[2 + 2 * i])]
    for i, b in enumerate(boundary):
        v = up(eng, b)
        terms += [(v, 0, weights[5 + 2 * i]), (v, max_degree - (len(b) - 1), weights[6 + 2 * i])]
    omega = O.primitive_nth_root(n)
    cw = eng.coset_combine_evaluate(terms, n.bit_length() - 1, omega, O.GENERATOR)
    assert down(cw) == ints(fp["codeword"])
    fri = F.Fri(T.field.generator(), T.field.primitive_nth_root(n), n, p["expansion_factor"],
                p["num_colinearity_checks"])
    ps = F.ProofStream()
    ps.objects = objects
    idx = fri.prove(sa_devlist.DeviceCodeword(cw, None, T.field, n), ps)
    assert idx == fp["indices"]
    assert hashlib.sha256(pickle.dumps(ps.objects)).hexdigest() == fp["after_sha256"]


def need_device(eng, log_n, vectors):
    import torch
    release(eng)
    free, _ = torch.cuda.mem_get_info(eng.device)
    want = (16 << log_n) * vectors + 2 * GIB
    if free < want:
        pytest.skip("2^%d needs %.1f GiB free on the device, %.1f GiB are" % (log_n, want / GIB, free / GIB))


def check_by_property(eng, out, air, trace, z, root, offset, step, log_n, rng, npts=6):
    """q(x) Z(x) = N(x) at sampled coset points x = offset root^k: q from the device (poly_eval of a whole row), Z and
    N with Python ints"""
    n = 1 << log_n
    ks = [0, n - 1] + [rng.randrange(n) for _ in range(npts - 2)]
    xs = [offset * pow(root, k, P) % P for k in ks]
    pts = up(eng, xs)
    for c, a in enumerate(air):
        qv = down(eng.poly_eval(out[c], pts))
        for x, q in zip(xs, qv):
            zx = sum(v * pow(x, i, P) for i, v in enumerate(z)) % P
            assert q * zx % P == evaluate(a, trace, step, x), (c, x)


@pytest.mark.parametrize("log_n", [20, 22])
def test_large_sizes_by_property(eng, log_n):
    need_device(eng, log_n, 24)
    n = 1 << log_n
    rng = random.Random(log_n)
    nregs, max_ncoef = 2, 4097
    air = make_air(log_n, log_n, nregs, 7, max_ncoef)
    trace = [[rng.randrange(P) for _ in range(max_ncoef)] for _ in range(nregs)]
    z = [rng.randrange(P) for _ in range(29)]
    root, offset, step = O.primitive_nth_root(n), rng.randrange(2, P), O.primitive_nth_root(n // 4)
    plan = eng.air_plan(air, nregs, up(eng, z), max_ncoef, log_n, root, offset, step)
    out = eng.air_quotients(plan, rows(eng, trace), n)
    check_by_property(eng, out, air, trace, z, root, offset, step, log_n, rng)


def test_constraints_past_one_chunk(eng):
    """2 chunk + 1 constraints at 2^21: three chunks, the last of one constraint"""
    log_n = 21
    n = 1 << log_n
    chunk = eng.lib.sa_coset_batch_max(log_n)
    ncons = 2 * chunk + 1
    need_device(eng, log_n, 2 * ncons + 8)
    rng = random.Random(21)
    air = make_air(21, log_n, 1, ncons, 65)
    air = [a if a else {(3, 1, 1): c + 1} for c, a in enumerate(air)]  # every row non-zero
    trace = [[rng.randrange(P) for _ in range(65)]]
    z = [rng.randrange(P) for _ in range(9)]
    root, offset = O.primitive_nth_root(n), rng.randrange(2, P)
    plan = eng.air_plan(air, 1, up(eng, z), 65, log_n, root, offset, root)
    out = eng.air_quotients(plan, rows(eng, trace), n)
    check_by_property(eng, out, air, trace, z, root, offset, root, log_n, rng, npts=3)


def launches(eng, fn):
    before = eng.launch_count()
    fn()
    return eng.launch_count() - before


@pytest.mark.parametrize("log_n", [10, 16])
def test_launch_count_fixed_within_a_chunk(eng, log_n):
    """after a warm call, an apply's launches do not depend on nregs or ncons within a chunk"""
    counts = set()
    for nregs, ncons in ((1, 1), (2, 3), (5, 7), (3, 20)):
        air, trace, z, max_ncoef, root, offset, step, qlen = make_case(nregs * ncons, log_n, nregs, ncons)
        plan = eng.air_plan(air, nregs, up(eng, z), max_ncoef, log_n, root, offset, step)
        t = rows(eng, trace)
        eng.air_quotients(plan, t, qlen)
        counts.add(launches(eng, lambda: eng.air_quotients(plan, t, qlen)))
    assert len(counts) == 1, counts


@pytest.mark.parametrize("log_n", [3, 12])
def test_errors_before_any_launch(eng, log_n):
    """refused builds and applies leave the launch count (and out) as they were"""
    import torch
    n = 1 << log_n
    air, trace, z, max_ncoef, root, offset, step, qlen = make_case(log_n, log_n, 2, 3)
    zd = up(eng, z)
    plan = eng.air_plan(air, 2, zd, max_ncoef, log_n, root, offset, step)
    t = rows(eng, trace)
    eng.air_quotients(plan, t, qlen)
    msg = "unsupported size"
    before = eng.launch_count()
    span = max_ncoef - 1
    bad_builds = [dict(air=[{(n - span, 1, 0, 0, 0): 1}]), dict(air=[{(0,) * 6: 1}]), dict(air=[]),
                  dict(nregs=0), dict(max_ncoef=0), dict(max_ncoef=n + 1), dict(log_n=0), dict(log_n=31),
                  dict(z=up(eng, [1] * (n + 1)))]
    for kw in bad_builds:
        a = dict(air=air, nregs=2, z=zd, max_ncoef=max_ncoef, log_n=log_n)
        a.update(kw)
        with pytest.raises(AssertionError, match=msg):
            eng.air_plan(a["air"], a["nregs"], a["z"], a["max_ncoef"], a["log_n"], root, offset, step)
    with pytest.raises(AssertionError, match="must be nth root"):
        eng.air_plan(air, 2, zd, max_ncoef, log_n, O.primitive_nth_root(2 * n), offset, step)
    bad_traces = [t[:1], t.to(torch.int32), t.cpu(), t.reshape(2, -1), t[:, :0],
                  torch.zeros((2, max_ncoef + 1, 2), dtype=torch.int64, device=eng.device)]
    for bt in bad_traces:
        with pytest.raises(AssertionError, match=msg):
            eng.air_quotients(plan, bt, qlen)
    for q in (0, n + 1):
        with pytest.raises(AssertionError, match=msg):
            eng.air_quotients(plan, t, q)
    out = torch.full((3, qlen, 2), 0x0A5A5A5A, dtype=torch.int64, device=eng.device)
    r = sa_engine._limbs(root)
    for args in ((2, max_ncoef, 0, 3, log_n), (2, 0, qlen, 3, log_n), (0, max_ncoef, qlen, 3, log_n),
                 (2, max_ncoef, qlen, 0, log_n), (2, max_ncoef, qlen, 3, 31)):
        assert eng.lib.sa_air_quotients(out.data_ptr(), plan.plan.data_ptr(), t.data_ptr(), *args, r,
                                        eng._stream()) == -6, args
    assert eng.lib.sa_air_quotients(out.data_ptr(), plan.plan.data_ptr(), t.data_ptr(), 2, max_ncoef, qlen, 3, log_n,
                                    sa_engine._limbs(O.primitive_nth_root(2 * n)), eng._stream()) == -2
    assert eng.launch_count() == before
    assert bool((out == 0x0A5A5A5A).all())
    with pytest.raises(AssertionError, match="divide by zero"):
        eng.air_plan(air, 2, up(eng, [0, 0]), max_ncoef, log_n, root, offset, step)


@pytest.mark.parametrize("log_n", [10, 16])
def test_one_plan_on_two_streams(eng, log_n):
    import torch
    air, trace, z, max_ncoef, root, offset, step, qlen = make_case(log_n + 1, log_n, 2, 7)
    plan = eng.air_plan(air, 2, up(eng, z), max_ncoef, log_n, root, offset, step)
    traces = [rows(eng, trace), rows(eng, [[(v + 1) % P for v in r] for r in trace])]
    want = [eng.air_quotients(plan, t, qlen) for t in traces]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for rnd in range(2):
        outs = []
        for s, t in zip(streams, traces):
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                outs.append(eng.air_quotients(plan, t, qlen))
        torch.cuda.synchronize()
        for got, w in zip(outs, want):
            assert bool((got == w).all()), rnd


@pytest.mark.parametrize("log_n", [10, 16])
def test_in_a_cuda_graph(eng, log_n):
    """an apply captured after one warm call replays to the same rows, and to new rows after new coefficients are
    copied into the captured trace"""
    import torch
    air, trace, z, max_ncoef, root, offset, step, qlen = make_case(log_n + 2, log_n, 2, 7)
    plan = eng.air_plan(air, 2, up(eng, z), max_ncoef, log_n, root, offset, step)
    t = rows(eng, trace)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        want = eng.air_quotients(plan, t, qlen)
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out = eng.air_quotients(plan, t, qlen)
    g.replay()
    torch.cuda.synchronize()
    assert bool((out == want).all())
    t2 = [[(3 * v + 1) % P for v in r] for r in trace]
    t.copy_(rows(eng, t2))
    g.replay()
    torch.cuda.synchronize()
    assert [down(out[c]) for c in range(len(air))] == quotients(air, t2, z, 1 << log_n, root, offset, step)


def test_kernel_has_no_spills():
    """ptxas's report for k_air_eval: no spill stores or loads"""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress",
                              "550", "-c", "-Xptxas", "-v", "-o", os.path.join(tmp, "poly.o"),
                              os.path.join(PKG, "csrc", "poly.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = res.stderr.splitlines()
    at = [i for i, line in enumerate(lines) if "Compiling entry function" in line and "k_air_eval" in line]
    assert len(at) == 1
    report = " ".join(lines[at[0]:at[0] + 4])
    spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
    assert spills and spills.groups() == ("0", "0"), report
