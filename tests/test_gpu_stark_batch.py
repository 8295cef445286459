"""Batched proofs on the H100 (StarkPlan.prove_batch, PlainStarkPlan.prove_batch, sign_batch through CudaEngine):
the fixture's two signatures as one batch give the recorded bytes; synthetic batches equal sequential proofs and the
test-side verifier accepts them; the plain batch is its FastStark twin minus the zerofier openings; the batched
kernels match the single calls across chunks; a chunk of a batch issues the launches of one proof; errors come before
any launch; each new call replays from a CUDA graph; and the changed kernels do not spill."""
import os
import pickle
import random
import re
import subprocess
import tempfile

import numpy as np
import pytest

import oracle as O
import stark_batch_cases as SB
import stark_cases as C
import stark_plain_cases as S
import stark_verify as V
import sa_engine
import sa_stark
from air_cases import make_case
from test_gpu_air import PKG, release, rows, up

pytestmark = pytest.mark.gpu
P = C.P


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


@pytest.mark.parametrize("fast", [True, False])
def test_fixture_signatures_as_one_batch(eng, fast):
    import test_stark_batch_cpu as T
    T.test_fixture_signatures_as_one_batch(fast)


def batch_case(log_fri, B, seed):
    st, cons, trace, boundary = C.synthetic(seed, log_fri)
    traces = [trace]
    for k in range(1, B):  # further statements of the same AIR: broken at a middle row, still proofs
        t = [list(r) for r in trace]
        t[len(t) // 2 + k][0] = C.T.fe((t[len(t) // 2 + k][0].value + k) % P)
        traces.append(t)
    return st, cons, traces, boundary


@pytest.mark.parametrize("log_fri,B", [(12, 16), (16, 4), (20, 2)])
def test_synthetic_batch_equals_sequential_and_verifies(eng, log_fri, B):
    st, cons, traces, boundary = batch_case(log_fri, B, log_fri)
    zpoly, zvals = C.zerofier(st)
    zcw = C.zerofier_codeword(zvals, True)
    plan = sa_stark.StarkPlan(st, cons, zpoly)
    nt = st.num_registers * st.num_randomizers
    rng = random.Random(B)
    per = [[rng.randrange(P) for _ in range(nt + plan.max_degree + 1)] for _ in range(B)]
    got = SB.run_batch(plan, traces, [boundary] * B, C.Urandom(SB.batch_draws(per, nt)), None, zcw)
    assert isinstance(got, list), got
    zroot = O.merkle_root_np(O.to_np(zvals))
    for b in (0, B - 1):
        want, _ = C.run(st, traces[b], None, boundary, zpoly, zcw, C.Urandom(per[b]), plan=plan)
        assert got[b] == want, b
    assert V.verify(st, got[0], cons, boundary, zroot) is True
    if B > 1:
        assert V.verify(st, got[1], cons, boundary, zroot) is False  # the broken witness


def test_plain_batch_is_faststark_twin_at_2_16(eng):
    st, cons, trace, boundary = C.synthetic(3, 16)
    B = 3
    zpoly, zvals = C.zerofier(st)
    zcw = C.zerofier_codeword(zvals, True)
    fast = sa_stark.StarkPlan(st, cons, zpoly)
    plain = sa_stark.PlainStarkPlan(S.plain_stark(st), cons)
    nt = st.num_registers * st.num_randomizers
    rng = random.Random(3)
    per = [[rng.randrange(P) for _ in range(nt + fast.max_degree + 1)] for _ in range(B)]
    a = SB.run_batch(fast, [trace] * B, [boundary] * B, C.Urandom(SB.batch_draws(per, nt)), None, zcw)
    b = SB.run_batch(plain, [trace] * B, [boundary] * B, C.Urandom(SB.batch_draws(per, nt)))
    for f, p in zip(a, b):
        assert pickle.loads(p) == S.without_zerofier_openings(f, st.num_colinearity_checks)


def air_setup(eng, log_n, nregs, ncons, B, seed=1):
    air, trace, z, max_ncoef, root, offset, step, qlen = make_case(seed, log_n, nregs, ncons)
    plan = eng.air_plan(air, nregs, up(eng, z), max_ncoef, log_n, root, offset, step)
    torch = eng.torch
    first = rows(eng, trace)
    g = torch.Generator(device=eng.device).manual_seed(seed)
    # canonical residues: both limbs below 2^62, and p > 2^126
    more = torch.randint(0, 1 << 62, (B - 1,) + tuple(first.shape), generator=g, device=eng.device)
    return plan, torch.cat([first[None], more]), qlen


@pytest.mark.parametrize("log_n,nregs,ncons,B", [(20, 2, 4, 9), (20, 1, 40, 2), (12, 1, 2, 64)])
def test_air_batch_matches_single_across_chunks(eng, log_n, nregs, ncons, B):
    """chunks of 4 traces at 2^20 (9 traces), of one trace in two row chunks (40 rows, 32 per chunk), one chunk of 64"""
    assert B > eng.lib.sa_air_batch_max(nregs, ncons, log_n) or ncons > eng.lib.sa_coset_batch_max(log_n) or B == 64
    plan, t, qlen = air_setup(eng, log_n, nregs, ncons, B)
    out = eng.air_quotients(plan, t, qlen)
    ex, flags = eng.air_quotients_exact(plan, t, qlen, check=False)
    for b in range(B):
        one = eng.air_quotients(plan, t[b], qlen)
        o2, f2 = eng.air_quotients_exact(plan, t[b], qlen, check=False)
        assert bool((out[b] == one).all()) and bool((ex[b] == o2).all()) and bool((flags[b] == f2).all()), b


def combine_terms(eng, log_n, nrows, T, seed):
    rng = random.Random(seed)
    n = 1 << log_n
    srcs = [up(eng, [rng.randrange(P) for _ in range(rng.randrange(1, n // 2))]) for _ in range(4)]
    terms = []
    for _ in range(T):
        v = srcs[rng.randrange(4)]
        terms.append((v, rng.randrange(n - v.shape[0] + 1), rng.randrange(P), rng.randrange(nrows)))
    return terms


def test_combination_batch_matches_single(eng):
    log_n, nrows = 16, 5
    root, off = O.primitive_nth_root(1 << log_n), 7
    terms = combine_terms(eng, log_n, nrows, 150, 1)
    out = eng.coset_combine_evaluate_batch(terms, nrows, log_n, root, off)
    for r in range(nrows):
        one = eng.coset_combine_evaluate([t[:3] for t in terms if t[3] == r], log_n, root, off)
        assert bool((out[r] == one).all()), r


def test_openings_with_sets_match_single(eng):
    n, B, group, k = 1 << 12, 6, 3, 9
    rng = random.Random(2)
    vals = up(eng, [rng.randrange(P) for _ in range(B * n)]).reshape(B, n, 2)
    trees = eng.merkle_trees(vals)
    sets = [[rng.randrange(n) for _ in range(k)] for _ in range(B // group)]
    g = eng.gather_batch(vals, sets, group=group)
    paths = eng.merkle_open_batch(trees, sets, group=group)
    for b in range(B):
        s = sets[b // group]
        assert np.array_equal(g[b], eng.gather_batch(vals[b:b + 1], s)[0])
        assert paths[b] == eng.merkle_open_batch(trees[b:b + 1], s)[0]


def launches(eng, fn):
    eng.synchronize()
    before = eng.launch_count()
    fn()
    eng.synchronize()
    return eng.launch_count() - before


def test_a_chunk_of_a_batch_issues_one_proofs_launches(eng):
    """the transition applies, the combination, the randomizer evaluation and the trees issue B = 1's launches at
    B = 4 within one chunk (the batched interpolation and boundary applies have their own tests)"""
    log_n, nregs, ncons, B = 14, 2, 3, 4
    assert B <= eng.lib.sa_air_batch_max(nregs, ncons, log_n)
    plan, t, qlen = air_setup(eng, log_n, nregs, ncons, B)
    eng.air_quotients(plan, t, qlen)  # grow the workspaces first
    eng.air_quotients_exact(plan, t, qlen, check=False)
    assert launches(eng, lambda: eng.air_quotients(plan, t[0], qlen)) == \
        launches(eng, lambda: eng.air_quotients(plan, t, qlen))
    assert launches(eng, lambda: eng.air_quotients_exact(plan, t[0], qlen, check=False)) == \
        launches(eng, lambda: eng.air_quotients_exact(plan, t, qlen, check=False))
    root = O.primitive_nth_root(1 << log_n)
    terms = combine_terms(eng, log_n, B, 70, 3)
    eng.coset_combine_evaluate_batch(terms, B, log_n, root, 5)
    assert launches(eng, lambda: eng.coset_combine_evaluate([t[:3] for t in terms], log_n, root, 5)) == \
        launches(eng, lambda: eng.coset_combine_evaluate_batch(terms, B, log_n, root, 5))
    coeffs = t.reshape(B * nregs, -1, 2)
    eng.coset_evaluate(coeffs, log_n, root, 5)
    assert launches(eng, lambda: eng.coset_evaluate(coeffs[0], log_n, root, 5)) == \
        launches(eng, lambda: eng.coset_evaluate(coeffs[:B], log_n, root, 5))
    cw = eng.coset_evaluate(coeffs, log_n, root, 5)
    eng.merkle_trees(cw)
    assert launches(eng, lambda: eng.merkle_trees(cw[:1])) == launches(eng, lambda: eng.merkle_trees(cw))


def test_prove_batch_pre_fri_launches_are_one_proofs(eng):
    """a whole batch of 4 synthetic proofs at 2^12 against one proof, FRI and the zerofier openings excluded"""
    st, cons, traces, boundary = batch_case(12, 4, 4)
    zpoly, zvals = C.zerofier(st)
    zcw = C.zerofier_codeword(zvals, True)
    plan = sa_stark.StarkPlan(st, cons, zpoly)
    counts, per_b = {}, {}
    fri_prove = plan.fri.prove

    def counted(codeword, ps):
        if "start" in counts:
            counts.setdefault("pre", eng.launch_count() - counts["start"])
        return fri_prove(codeword, ps)
    plan.fri.prove = counted
    try:
        for B in (1, 4, 1):
            SB.run_batch(plan, traces[:B], [boundary] * B, C.Urandom([7] * 100000), None, zcw)  # warm
            counts.clear()
            eng.synchronize()
            counts["start"] = eng.launch_count()
            got = SB.run_batch(plan, traces[:B], [boundary] * B, C.Urandom([7] * 100000), None, zcw)
            assert isinstance(got, list), got
            per_b[B] = counts.pop("pre")
    finally:
        del plan.fri.prove
    # the boundary plan build is the only stage that grows with B nregs: one zerofier and interpolation per register
    assert per_b[4] - per_b[1] <= 3 * st.num_registers * 3 * 4, per_b


def test_errors_before_any_launch(eng):
    log_n = 10
    plan, t, qlen = air_setup(eng, log_n, 2, 2, 3)
    root = O.primitive_nth_root(1 << log_n)
    terms = combine_terms(eng, log_n, 2, 4, 5)
    n = 1 << log_n
    vals = up(eng, [1] * (4 * n)).reshape(4, n, 2)
    trees = eng.merkle_trees(vals)
    bad = [lambda: eng.air_quotients(plan, t, n + 1),
           lambda: eng.coset_combine_evaluate_batch(terms, 1, log_n, root, 3),
           lambda: eng.gather_batch(vals, [[0], [n]], group=2),
           lambda: eng.merkle_open_batch(trees, [[0], [1], [2]], group=2),
           lambda: eng.gather_batch(vals, [[0]], group=0)]
    for call in bad:
        before = eng.launch_count()
        with pytest.raises(sa_engine.SaError):
            call()
        assert eng.launch_count() == before
    # and in the library itself, below the binding's checks
    import ctypes
    out = eng.torch.full((4, 1, 2), 7, dtype=eng.torch.int64, device=eng.device)
    idx = (ctypes.c_uint64 * 2)(0, n)
    before = eng.launch_count()
    assert eng.lib.sa_gather_batch_sets(out.data_ptr(), vals.data_ptr(), n, 4, 2, idx, 1, eng._stream()) == -5
    assert eng.lib.sa_gather_batch_sets(out.data_ptr(), vals.data_ptr(), n, 4, 0, idx, 1, eng._stream()) == -6
    assert eng.launch_count() == before and bool((out == 7).all())


def test_graph_replay_of_each_new_call(eng):
    import torch
    log_n = 12
    plan, t, qlen = air_setup(eng, log_n, 2, 3, 4)
    root = O.primitive_nth_root(1 << log_n)
    terms = combine_terms(eng, log_n, 3, 10, 6)
    calls = [lambda: eng.air_quotients(plan, t, qlen),
             lambda: eng.air_quotients_exact(plan, t, qlen, check=False)[0],
             lambda: eng.coset_combine_evaluate_batch(terms, 3, log_n, root, 11)]
    for call in calls:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            want = call().clone()
        s.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            out = call()
        out.fill_(0)
        g.replay()
        torch.cuda.synchronize()
        assert bool((out == want).all())


def test_changed_kernels_have_no_spills():
    with tempfile.TemporaryDirectory() as tmp:
        reports = ""
        for src in ("poly.cu", "merkle_fri.cu"):
            reports += subprocess.run(
                ["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                 "-diag-suppress", "550", "-c", "-Xptxas", "-v", "-o", os.path.join(tmp, src + ".o"),
                 os.path.join(PKG, "csrc", src)], capture_output=True, text=True, check=True).stderr
    for kernel in ("k_air_eval", "k_air_store_exact", "k_coset_combine", "k_gather", "k_merkle_paths"):
        m = re.search(r"Compiling entry function '(_Z\d+%s[^']*)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads"
                      % kernel, reports, re.S)
        assert m and m.groups()[1:] == ("0", "0"), kernel
