"""Boundary quotients on the device (sa_boundary_plan / sa_boundary_quotients through CudaEngine.boundary_plan /
boundary_quotients): every case against the outputs restated with Python ints (tests/boundary_cases.py), the
reference's quotients and codewords of tests/golden/boundary.json bit for bit, the prover's chain from the recorded
trace polynomials to the recorded Merkle roots, combined codeword and FRI transcript with nothing recorded in
between, large sizes by an exact property, several chunks of registers, the launches of an apply, errors before any
launch, one plan on two streams, an apply captured in a CUDA graph, and the kernels' registers."""
import ctypes
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
from boundary_cases import (P, digest, expected, golden, golden_boundary, ints, make_case, reference)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "stark-anatomy_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)
import sa_engine  # noqa: E402

pytestmark = pytest.mark.gpu
GIB = 1 << 30
REMAINDER = "cannot perform polynomial division because remainder is not zero"


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


def run(eng, boundary, nregs, omicron, trace, log_n, root, offset):
    plan = eng.boundary_plan(boundary, nregs, omicron, log_n, root, offset)
    quot, cw, flags = eng.boundary_quotients(plan, rows(eng, trace), check=False)
    assert tuple(quot.shape) == (nregs, len(trace[0]), 2) and tuple(cw.shape) == (nregs, 1 << log_n, 2)
    return [down(quot[s]) for s in range(nregs)], [down(cw[s]) for s in range(nregs)], flags.tolist()


def check(eng, seed, log_n, nregs, npoints, false_regs=(), full=True, **kw):
    """the device against the restatement (full) or, for large n, the reference's division of the clean registers,
    and the flags against false_regs"""
    n = 1 << log_n
    boundary, omicron, trace, brows, _, root, offset = make_case(seed, log_n, nregs, npoints, false_regs=false_regs,
                                                                 **kw)
    quot, cw, flags = run(eng, boundary, nregs, omicron, trace, log_n, root, offset)
    assert [bool(f) for f in flags] == [s in false_regs for s in range(nregs)]
    for s, (t, (z, i)) in enumerate(zip(trace, brows)):
        if full:
            assert (quot[s], cw[s]) == expected(t, z, i, n, root, offset)[:2], s
        if s not in false_regs:
            q, c = reference(t, z, i, n, root, offset)
            assert quot[s] == q + [0] * (len(t) - len(q)) and cw[s] == c, s


CASES = [(lg, r, k) for lg in range(1, 13) for r in (1, 2, 3, 5) for k in (1, 3, 5) if k < 1 << lg]


@pytest.mark.parametrize("log_n, nregs, k", CASES)
def test_matches_restatement(eng, log_n, nregs, k):
    seed = 100 * log_n + 10 * nregs + k
    npoints = [max(1, k - s % 3) for s in range(nregs)]
    check(eng, seed, log_n, nregs, npoints, (seed % nregs,) if nregs > 1 else ())


@pytest.mark.parametrize("log_n", [2, 6, 12])
@pytest.mark.parametrize("kw", [dict(offset_kind="one"), dict(offset_kind="generator"), dict(ncoef="n"),
                                dict(ncoef=2, const_values=True), dict(ncoef=2)])
def test_offsets_and_lengths(eng, log_n, kw):
    """offset 1 and the generator, ncoef = n, and ncoef < deg Z (clean only when T = I)"""
    kw = dict(kw)
    if kw.get("ncoef") == "n":
        kw["ncoef"] = 1 << log_n
    k = min(3, (1 << log_n) - 1)
    if kw.get("ncoef") == 2:  # below deg Z = 3
        false_regs = () if kw.get("const_values") else (0, 1)
    else:
        false_regs = (1,)
    check(eng, log_n + 7, log_n, 2, [k, k], false_regs, **kw)


@pytest.mark.parametrize("log_n, k", [(16, 1), (16, 5), (20, 3)])
def test_large_against_the_reference(eng, log_n, k):
    check(eng, log_n, log_n, 2, [k, 1], (1,), full=log_n <= 16)


@pytest.mark.parametrize("name", ["faststark", "false_boundary", "multi", "short", "config5"])
def test_golden(eng, name):
    """the reference's (T - I) / Z and fast_coset_evaluate of it, bit for bit, through the engine's own zerofiers and
    interpolants; a raising division is flagged, and check=True raises the reference's message for it"""
    rec = golden()[name]
    nregs, trace = rec["nregs"], [ints(t) for t in rec["trace"]]
    args = (golden_boundary(rec), nregs, int(rec["omicron"]), rec["log_n"], int(rec["root"]), int(rec["offset"]))
    quot, cw, flags = run(eng, *args[:3], trace, *args[3:])
    for s in range(nregs):
        q = rec["quotients"][s]
        assert bool(flags[s]) == (q is None), s
        if q is not None:
            assert quot[s] == ints(q) + [0] * (len(trace[s]) - len(q)), s
            assert digest(cw[s]) == rec["codeword_digests"][s], s
    plan = eng.boundary_plan(*args)
    bad = [s for s in range(nregs) if rec["quotients"][s] is None]
    if bad:
        with pytest.raises(AssertionError, match=re.escape("%s (registers %s)" % (REMAINDER, bad))):
            eng.boundary_quotients(plan, rows(eng, trace))
    else:
        eng.boundary_quotients(plan, rows(eng, trace))


def test_engine_takes_field_elements(eng):
    """values and omicron with .value, as FastStark's boundary carries them; the plan's degree bounds"""
    class V:
        def __init__(self, v):
            self.value = v
    rec = golden()["multi"]
    boundary = [(c, r, V(v)) for c, r, v in golden_boundary(rec)]
    trace = [ints(t) for t in rec["trace"]]
    plan = eng.boundary_plan(boundary, 3, V(int(rec["omicron"])), rec["log_n"], int(rec["root"]), int(rec["offset"]))
    assert plan.degrees == [1, 3, 5]
    assert plan.degree_bounds(len(trace[0])) == [len(trace[0]) - 1 - d for d in (1, 3, 5)]
    quot, cw, _ = eng.boundary_quotients(plan, rows(eng, trace))
    assert [digest(down(cw[s])) for s in range(3)] == rec["codeword_digests"]


def test_prover_chain(eng):
    """the recorded trace polynomials -> boundary_quotients -> merkle_trees: the recorded proof's first two objects;
    then air_quotients -> coset_combine_evaluate with the device's boundary rows: the recorded combined codeword; and
    the drop-in Fri.prove on it reproduces the recorded transcript"""
    from hostmirror_loader import load_host_types
    from air_cases import golden as air_golden, golden_air
    T = load_host_types()
    import fri as F
    import sa_devlist
    with open(os.path.join(ROOT, "tests", "golden", "faststark_trace.json")) as f:
        g = json.load(f)
    calls, p, fp = g["calls"], g["params"], g["fri_prove"][0]
    n = p["fri_domain_length"]
    log_n = n.bit_length() - 1
    omega = O.primitive_nth_root(n)
    trace = [ints(c["out"]["poly"]) for c in calls if c["fn"] == "fast_interpolate"]
    omicron = int([c for c in calls if c["fn"] == "fast_zerofier"][0]["args"][1]["f"])
    brec = golden()["faststark"]
    t = rows(eng, trace)
    bplan = eng.boundary_plan(golden_boundary(brec), 2, omicron, log_n, omega, O.GENERATOR)
    bq, bcw, _ = eng.boundary_quotients(bplan, t)
    roots = eng.tree_roots(eng.merkle_trees(bcw))
    assert roots == [T.dec_obj(o) for o in fp["prior_objects"][:2]]

    arec = air_golden()["faststark"]
    aplan = eng.air_plan(golden_air(arec), 2, up(eng, ints(arec["zerofier"])), len(trace[0]), arec["log_n"],
                         int(arec["root"]), int(arec["offset"]), int(arec["step"]))
    tq = eng.air_quotients(aplan, t, arec["qlen"])
    randomizer = [ints(c["args"][0]["poly"]) for c in calls if c["fn"] == "fast_coset_evaluate"][3]
    max_degree = len(randomizer) - 1
    objects = [T.dec_obj(o) for o in fp["prior_objects"]]
    seed = O.fiat_shamir(objects)
    weights = [O.sample(hashlib.blake2b(seed + bytes(i)).digest()) for i in range(9)]
    terms = [(up(eng, randomizer), 0, weights[0])]
    for i in range(2):
        q = tq[i]
        terms += [(q, 0, weights[1 + 2 * i]), (q, max_degree - (q.shape[0] - 1), weights[2 + 2 * i])]
    for i, bound in enumerate(bplan.degree_bounds(len(trace[0]))):
        v = bq[i][:bound + 1]
        terms += [(v, 0, weights[5 + 2 * i]), (v, max_degree - bound, weights[6 + 2 * i])]
    cw = eng.coset_combine_evaluate(terms, log_n, omega, O.GENERATOR)
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


def random_rows(eng, nrows, ncoef, seed):
    """canonical random elements on the device, (nrows, ncoef, 2): high limbs below 2^55, so values below 2^119 < p"""
    import torch
    g = torch.Generator(device=eng.device).manual_seed(seed)
    r = torch.randint(-(1 << 63), (1 << 63) - 1, (nrows, ncoef, 2), dtype=torch.int64, device=eng.device, generator=g)
    r[..., 1] &= (1 << 55) - 1
    return r


def clean_trace(eng, z, i, r, log_n):
    """I + Z R on the device for a short Z and I: Z R by transforms of order 2^log_n, then I added on the host"""
    n = 1 << log_n
    root = O.primitive_nth_root(n)
    prod = eng.ntt(eng.pointwise_mul(eng.ntt(eng.pad(up(eng, z), n), log_n, root),
                                     eng.ntt(eng.pad(r, n), log_n, root)), log_n, root, inverse=True)
    ncoef = r.shape[0] + len(z) - 1
    head = down(prod[:len(i)])
    prod[:len(i)] = up(eng, [(a + b) % P for a, b in zip(head, i)])
    return prod[:ncoef]


@pytest.mark.parametrize("log_n", [22, 24])
def test_large_sizes_by_property(eng, log_n):
    """clean divisions I + Z R at n / 4 coefficients: quot == R followed by zeros, no flag, and the codewords equal
    R's values (Horner) at sampled coset points"""
    import torch
    n = 1 << log_n
    need_device(eng, log_n, 12)
    rng = random.Random(log_n)
    nregs, ncoef = 2, n // 4
    boundary, omicron, _, brows, _, _, offset = make_case(log_n, 4, nregs, [3, 1])  # points of order 64
    root = O.primitive_nth_root(n)
    trace = torch.empty((nregs, ncoef, 2), dtype=torch.int64, device=eng.device)
    rs = random_rows(eng, nregs, ncoef, log_n)
    for s, (z, i) in enumerate(brows):
        rs[s, ncoef - (len(z) - 1):] = 0
        trace[s] = clean_trace(eng, z, i, rs[s, :ncoef - (len(z) - 1)], log_n - 1)
    plan = eng.boundary_plan(boundary, nregs, omicron, log_n, root, offset)
    quot, cw, flags = eng.boundary_quotients(plan, trace)
    assert flags.tolist() == [0, 0]
    assert bool((quot == rs).all())
    ks = [0, n - 1] + [rng.randrange(n) for _ in range(4)]
    pts = up(eng, [offset * pow(root, k, P) % P for k in ks])
    for s in range(nregs):
        want = down(eng.poly_eval(rs[s], pts, mode=1))
        assert [down(cw[s, k:k + 1])[0] for k in ks] == want, s


def test_registers_past_one_chunk(eng):
    """2 chunk + 1 registers at 2^21: three chunks, the last of one register, a false register in each"""
    log_n = 21
    chunk = eng.lib.sa_coset_batch_max(log_n)
    nregs = 2 * chunk + 1
    need_device(eng, log_n, nregs + chunk + 8)
    false_regs = (3, chunk + 5, 2 * chunk)
    boundary, omicron, trace, brows, rs, root, offset = make_case(21, log_n, nregs, [1 + s % 3 for s in range(nregs)],
                                                                  ncoef=65, false_regs=false_regs)
    plan = eng.boundary_plan(boundary, nregs, omicron, log_n, root, offset)
    quot, cw, flags = eng.boundary_quotients(plan, rows(eng, trace), check=False)
    assert [bool(f) for f in flags.tolist()] == [s in false_regs for s in range(nregs)]
    n = 1 << log_n
    rng = random.Random(21)
    ks = [0, n - 1, rng.randrange(n)]
    for s in range(nregs):
        if s in false_regs:
            continue
        assert down(quot[s]) == rs[s] + [0] * (65 - len(rs[s])), s
        got = down(cw[s][ks])
        xs = [offset * pow(root, k, P) % P for k in ks]
        assert got == [sum(c * pow(x, j, P) for j, c in enumerate(rs[s])) % P for x in xs], s


def launches(eng, fn):
    before = eng.launch_count()
    fn()
    return eng.launch_count() - before


@pytest.mark.parametrize("log_n", [10, 16])
def test_launch_count_fixed_within_a_chunk(eng, log_n):
    """after a warm call, an apply's launches do not depend on nregs within a chunk"""
    counts = set()
    for nregs in (1, 2, 5, 9):
        boundary, omicron, trace, _, _, root, offset = make_case(nregs, log_n, nregs, [2] * nregs)
        plan = eng.boundary_plan(boundary, nregs, omicron, log_n, root, offset)
        t = rows(eng, trace)
        eng.boundary_quotients(plan, t, check=False)
        counts.add(launches(eng, lambda: eng.boundary_quotients(plan, t, check=False)))
    assert len(counts) == 1, counts


@pytest.mark.parametrize("log_n", [3, 12])
def test_errors_before_any_launch(eng, log_n):
    """refused builds and applies leave the launch count, the plan and the outputs as they were"""
    import torch
    n = 1 << log_n
    boundary, omicron, trace, brows, _, root, offset = make_case(log_n, log_n, 2, [2, 1])
    plan = eng.boundary_plan(boundary, 2, omicron, log_n, root, offset)
    t = rows(eng, trace)
    eng.boundary_quotients(plan, t)
    zs = [up(eng, z) for z, _ in brows]
    its = [up(eng, i) for _, i in brows]
    msg = "unsupported size"
    torch.cuda.synchronize()
    before = eng.launch_count()
    bad_builds = [dict(boundary=boundary + [(1, 2, 5)]), dict(boundary=[b for b in boundary if b[1] == 0]),
                  dict(boundary=boundary + [(c, 1, 1) for c in range(3, 2 * n + 3, 2)]), dict(nregs=0),
                  dict(log_n=0), dict(log_n=31), dict(offset=0), dict(offset=P)]
    for kw in bad_builds:
        a = dict(boundary=boundary, nregs=2, log_n=log_n, offset=offset)
        a.update(kw)
        with pytest.raises(AssertionError, match=msg):
            eng.boundary_plan(a["boundary"], a["nregs"], omicron, a["log_n"], root, a["offset"])
    bad_traces = [t[:1], t.to(torch.int32), t.cpu(), t.reshape(2, -1), t[:, :0],
                  torch.zeros((2, n + 1, 2), dtype=torch.int64, device=eng.device)]
    for bt in bad_traces:
        with pytest.raises(AssertionError, match=msg):
            eng.boundary_quotients(plan, bt)
    # the C ABI's own checks
    vp, sz = ctypes.c_void_p * 2, ctypes.c_size_t * 2
    r, o = sa_engine._limbs(root), sa_engine._limbs(offset)
    saved = plan.plan.clone()

    def build(nregs=2, zl=None, il=None, lg=log_n, rt=r, of=o):
        zl = zl or [z.shape[0] for z in zs]
        il = il or [i.shape[0] for i in its]
        return eng.lib.sa_boundary_plan(plan.plan.data_ptr(), vp(*[z.data_ptr() for z in zs]), sz(*zl),
                                        vp(*[i.data_ptr() for i in its]), sz(*il), nregs, lg, rt, of, eng._stream())
    for kw in (dict(nregs=0), dict(zl=[0, 2]), dict(zl=[3, n + 1]), dict(il=[0, 1]), dict(il=[2, n + 1]),
               dict(lg=0), dict(lg=31), dict(of=sa_engine._limbs(0))):
        assert build(**kw) == -6, kw
    assert build(rt=sa_engine._limbs(O.primitive_nth_root(2 * n))) == -2
    assert build(rt=sa_engine._limbs(O.primitive_nth_root(n // 2))) == -3
    quot = torch.full((2, len(trace[0]), 2), 0x0A5A5A5A, dtype=torch.int64, device=eng.device)
    cw = torch.full((2, n, 2), 0x0A5A5A5A, dtype=torch.int64, device=eng.device)
    flags = torch.full((2,), 0x0A5A5A5A, dtype=torch.int32, device=eng.device)
    fp = ctypes.cast(flags.data_ptr(), ctypes.POINTER(ctypes.c_uint32))
    for args in ((0, len(trace[0]), log_n, r), (2, 0, log_n, r), (2, n + 1, log_n, r), (2, 1, 31, r),
                 (2, 1, 0, r)):
        assert eng.lib.sa_boundary_quotients(quot.data_ptr(), cw.data_ptr(), fp, plan.plan.data_ptr(), t.data_ptr(),
                                             *args, eng._stream()) == -6, args
    assert eng.lib.sa_boundary_quotients(quot.data_ptr(), cw.data_ptr(), fp, plan.plan.data_ptr(), t.data_ptr(), 2,
                                         len(trace[0]), log_n, sa_engine._limbs(O.primitive_nth_root(2 * n)),
                                         eng._stream()) == -2
    assert eng.launch_count() == before
    assert bool((quot == 0x0A5A5A5A).all()) and bool((cw == 0x0A5A5A5A).all()) and bool((flags == 0x0A5A5A5A).all())
    assert bool((plan.plan == saved).all())
    # after the build's synchronisation: two cycles at one point, a zerofier that vanishes on the coset (offset 1 and
    # a point of <root>), a zero top coefficient
    with pytest.raises(AssertionError, match="divide by zero"):
        eng.boundary_plan(boundary + [(boundary[0][0] + 4 * n, boundary[0][1], 1)], 2, omicron, log_n, root, offset)
    with pytest.raises(AssertionError, match="divide by zero"):
        eng.boundary_plan([(0, 0, 1), (4, 1, 2)], 2, omicron, log_n, root, 1)
    zs[1] = up(eng, down(zs[1]) + [0])
    assert build() == -6


@pytest.mark.parametrize("log_n", [10, 16])
def test_one_plan_on_two_streams(eng, log_n):
    import torch
    boundary, omicron, trace, _, _, root, offset = make_case(log_n + 1, log_n, 3, [3, 1, 2])
    plan = eng.boundary_plan(boundary, 3, omicron, log_n, root, offset)
    traces = [rows(eng, trace), rows(eng, [[(v + 1) % P for v in r] for r in trace])]
    want = [eng.boundary_quotients(plan, t, check=False) for t in traces]
    assert want[0][2].tolist() == [0, 0, 0] and all(want[1][2].tolist())
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for rnd in range(2):
        outs = []
        for s, t in zip(streams, traces):
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                outs.append(eng.boundary_quotients(plan, t, check=False))
        torch.cuda.synchronize()
        for got, w in zip(outs, want):
            assert all(bool((a == b).all()) for a, b in zip(got, w)), rnd


@pytest.mark.parametrize("log_n", [10, 16])
def test_in_a_cuda_graph(eng, log_n):
    """an apply captured after one warm call replays to the same outputs; after a false trace is copied in, the
    replay flags its register, and after the clean trace is copied back the next replay clears the flag again"""
    import torch
    n = 1 << log_n
    boundary, omicron, trace, brows, _, root, offset = make_case(log_n + 2, log_n, 2, [3, 2])
    plan = eng.boundary_plan(boundary, 2, omicron, log_n, root, offset)
    t = rows(eng, trace)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        want = eng.boundary_quotients(plan, t, check=False)
    s.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        out = eng.boundary_quotients(plan, t, check=False)
    g.replay()
    torch.cuda.synchronize()
    assert all(bool((a == b).all()) for a, b in zip(out, want)) and out[2].tolist() == [0, 0]
    bad = [list(trace[0]), [(v + (j == 0)) % P for j, v in enumerate(trace[1])]]
    t.copy_(rows(eng, bad))
    g.replay()
    torch.cuda.synchronize()
    assert out[2].tolist()[0] == 0 and out[2].tolist()[1] != 0
    assert (down(out[0][1]), down(out[1][1])) == expected(bad[1], *brows[1], n, root, offset)[:2]
    t.copy_(rows(eng, trace))
    g.replay()
    torch.cuda.synchronize()
    assert all(bool((a == b).all()) for a, b in zip(out, want)) and out[2].tolist() == [0, 0]


def test_kernels_have_no_spills():
    """ptxas's report for k_boundary_point and k_boundary_store: no spill stores or loads"""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        res = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-diag-suppress",
                              "550", "-c", "-Xptxas", "-v", "-o", os.path.join(tmp, "poly.o"),
                              os.path.join(PKG, "csrc", "poly.cu")], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    lines = res.stderr.splitlines()
    for kernel in ("k_boundary_point", "k_boundary_store"):
        at = [i for i, line in enumerate(lines) if "Compiling entry function" in line and kernel in line]
        assert len(at) == 1, kernel
        report = " ".join(lines[at[0]:at[0] + 4])
        spills = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", report)
        assert spills and spills.groups() == ("0", "0"), report
