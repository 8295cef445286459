"""Batched FRI on the H100 (sa_fri_commit_batch through CudaEngine.fri_commit_batch, Fri.commit_batch and
Fri.prove_batch): batched commits equal one sa_fri_commit per row (layers, trees, roots) at n = 2^1 .. 2^12 for batches
of 1, 2, 5 and 16, at 2^16 x 4, 2^20 x 2 and at n = 2 past one launch group; Fri.prove_batch pushes, as pickled bytes,
what Fri.prove pushes; a batched commit issues the launches of one commit, calls back once per round, and its query
phase issues as many calls for 16 proofs as for one; an aborting callback stops the launches; errors come before any
launch; and k_merkle_chunk does not spill."""
import hashlib
import os
import pickle
import re
import subprocess
import tempfile

import numpy as np
import pytest

import oracle as O
import stark_cases as C
import sa_devlist
import sa_engine
import sa_host
import fri as dropin_fri
from sa_engine import FRI_CHALLENGE_FN, SaError
from test_gpu_air import PKG, release

pytestmark = pytest.mark.gpu
P = O.P
MK_MAX_TREES = 65535


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


def rand_rows(seed, batch, n):
    rng = np.random.default_rng(seed)
    lo = rng.integers(0, 1 << 64, size=(batch, n), dtype=np.uint64)
    hi = rng.integers(0, 0xCB80000000000000, size=(batch, n), dtype=np.uint64)  # < p's top limb => < p
    x = np.stack([lo, hi], axis=2)
    if n > 2:
        x[:, 0] = 0
        x[:, 1] = O._fe(P - 1)
    if batch > 2:
        x[2] = x[0]
    return x


def up(eng, x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).to(eng.device)


def alpha_of(r, root):
    """a challenge that depends on the round's root, as Fiat-Shamir's does"""
    return int.from_bytes(hashlib.blake2b(root + bytes([r])).digest()[:17], "big") % P


def batched(eng, vecs, rounds, offset, omega, pick=None):
    calls = []

    def on_roots(r, roots, want):
        calls.append((r, roots, want))
        return [alpha_of(r, root) if pick is None else pick(r, b) for b, root in enumerate(roots)] if want else None
    layers, trees = eng.fri_commit_batch(vecs, rounds, offset, omega, on_roots)
    return calls, layers, trees


def single(eng, vec, rounds, offset, omega, b=0, pick=None):
    roots = []

    def on_root(r, root, want):
        roots.append(root)
        return (alpha_of(r, root) if pick is None else pick(r, b)) if want else None
    layers, trees = eng.fri_commit(vec, rounds, offset, omega, on_root)
    return roots, layers, trees


def check_rows(eng, vecs, rounds, offset, omega, rows, pick=None):
    calls, layers, trees = batched(eng, vecs, rounds, offset, omega, pick)
    assert [(r, w) for r, _, w in calls] == [(r, r != rounds - 1) for r in range(rounds)]
    for b in rows:
        roots, sl, st = single(eng, vecs[b], rounds, offset, omega, b, pick)
        assert [c[1][b] for c in calls] == roots, b
        for r in range(rounds):
            assert bool((layers[r][b] == sl[r]).all()), (b, r)
            assert bool((trees[r][b, 1:] == st[r][1:]).all()), (b, r)
    return calls, layers, trees


@pytest.mark.parametrize("batch", [1, 2, 5, 16])
@pytest.mark.parametrize("log_n", range(1, 13))
def test_commit_batch_equals_single_commits(eng, log_n, batch):
    n = 1 << log_n
    x = rand_rows(100 * log_n + batch, batch, n)
    omega = O.primitive_nth_root(n)
    calls, layers, trees = check_rows(eng, up(eng, x), log_n + 1, O.GENERATOR, omega, range(batch))
    assert calls[0][1] == [O.merkle_root_np(x[b]) for b in range(batch)]


@pytest.mark.parametrize("log_n,batch", [(16, 4), (20, 2)])
def test_commit_batch_large(eng, log_n, batch):
    n = 1 << log_n
    x = rand_rows(log_n, batch, n)
    check_rows(eng, up(eng, x), log_n - 6, 7, O.primitive_nth_root(n), range(batch))


def test_forced_challenges(eng):
    """alpha 0, 1 and p - 1, and row 3 of zeros"""
    x = rand_rows(5, 5, 1024)
    x[3] = 0
    choices = [0, 1, P - 1]
    check_rows(eng, up(eng, x), 11, O.GENERATOR, O.primitive_nth_root(1024), range(5),
               pick=lambda r, b: choices[(r + b) % 3])


def test_batch_past_one_launch_group(eng):
    batch, n = MK_MAX_TREES + 2, 2
    x = rand_rows(7, batch, n)
    calls, layers, trees = check_rows(eng, up(eng, x), 2, O.GENERATOR, P - 1,
                                      [0, 1, MK_MAX_TREES - 1, MK_MAX_TREES, MK_MAX_TREES + 1])
    roots = [hashlib.blake2b(str(v).encode()).digest() for v in O.from_np(layers[1].cpu().numpy().view(np.uint64)
                                                                          .reshape(-1, 2))]
    assert calls[1][1] == roots


def launches(eng, fn):
    eng.synchronize()
    before = eng.launch_count()
    fn()
    eng.synchronize()
    return eng.launch_count() - before


@pytest.mark.parametrize("log_n,rounds", [(12, 4), (16, 8)])
def test_launches_and_waits_of_one_commit(eng, log_n, rounds):
    n = 1 << log_n
    x = up(eng, rand_rows(1, 16, n))
    omega = O.primitive_nth_root(n)
    one = launches(eng, lambda: single(eng, x[0], rounds, 7, omega))
    assert launches(eng, lambda: batched(eng, x[:1], rounds, 7, omega)) == one
    got = []
    assert launches(eng, lambda: got.append(batched(eng, x, rounds, 7, omega))) == one
    assert len(got[0][0]) == rounds  # one host wait and one callback per round for the whole batch


def fri_case(log_n, k):
    n = 1 << log_n
    return dropin_fri.Fri(C.T.field.generator(), C.T.field.primitive_nth_root(n), n, 4, k)


def prove_pair(eng, f, x, form, prefixed):
    B, n = x.shape[0], x.shape[1]
    field = C.T.field

    def streams():
        out = [C.SignatureProofStream(b"doc %d" % b) if prefixed else sa_host.ip.ProofStream() for b in range(B)]
        for ps in out:
            ps.push(b"prefix")
        return out
    want_s, got_s = streams(), streams()
    want = [f.prove(sa_devlist.DeviceCodeword(up(eng, x[b]), None, field, n), ps) for b, ps in enumerate(want_s)]
    if form == "tensor":
        arg = up(eng, x)
    elif form == "device":
        arg = [sa_devlist.DeviceCodeword(up(eng, x[b]), None, field, n) for b in range(B)]
    else:
        arg = [C.T.elems(O.from_np(x[b])) for b in range(B)]
    got = f.prove_batch(arg, got_s)
    assert got == want
    for g, w in zip(got_s, want_s):
        assert pickle.dumps(g.objects) == pickle.dumps(w.objects)


@pytest.mark.parametrize("form", ["tensor", "device", "lists"])
def test_prove_batch_is_prove(eng, form):
    prove_pair(eng, fri_case(12, 64), rand_rows(3, 16, 1 << 12), form, True)


@pytest.mark.parametrize("log_n,batch", [(16, 4), (20, 2)])
def test_prove_batch_is_prove_large(eng, log_n, batch):
    prove_pair(eng, fri_case(log_n, 32), rand_rows(log_n, batch, 1 << log_n), "tensor", False)


def test_query_calls_do_not_grow_with_the_batch(eng):
    f = fri_case(12, 64)
    x = rand_rows(9, 16, 1 << 12)
    counts = []
    for B in (1, 16):
        v = up(eng, x[:B])
        streams = [sa_host.ip.ProofStream() for _ in range(B)]
        d2h = eng.stats["d2h_calls"]
        n = launches(eng, lambda: f.prove_batch(v, streams))
        counts.append((n, eng.stats["d2h_calls"] - d2h))
    rounds = f.num_rounds()
    assert counts[0] == counts[1]
    # the roots of each round, the last codewords, one gather per layer but the last, one path read per layer
    assert counts[0][1] == rounds + 1 + (rounds - 1) + rounds


def test_callback_abort_stops_the_launches(eng):
    n = 1 << 12
    x = up(eng, rand_rows(2, 4, n))
    omega = O.primitive_nth_root(n)

    def fail(r):
        def on(r_, roots, want):
            if r_ == r:
                raise KeyError("stop")
            return [5] * len(roots) if want else None
        return on

    def single_fail(r):
        def on(r_, root, want):
            if r_ == r:
                raise KeyError("stop")
            return 5 if want else None
        return on
    for r in (0, 2):
        def run_batch():
            with pytest.raises(KeyError):
                eng.fri_commit_batch(x, 5, 7, omega, fail(r))

        def run_single():
            with pytest.raises(KeyError):
                eng.fri_commit(x[0], 5, 7, omega, single_fail(r))
        assert launches(eng, run_batch) == launches(eng, run_single)
    check_rows(eng, x, 5, 7, omega, [3])  # and the next call works


def test_errors_before_any_launch(eng):
    import torch
    x = up(eng, rand_rows(1, 2, 8))
    omega = O.primitive_nth_root(8)
    lib = eng.lib
    st = eng._stream()
    cb = FRI_CHALLENGE_FN(lambda *a: 1)
    buf = torch.empty((4096, 64), dtype=torch.uint8, device=eng.device)
    one = sa_engine._limbs(1)
    before = eng.launch_count()
    for n, rounds in ((6, 1), (0, 1), (8, 0), (8, 5), (1, 2)):
        assert lib.sa_fri_commit_batch(buf.data_ptr(), buf.data_ptr(), x.data_ptr(), n, 2, rounds, one, one, cb,
                                       None, st) == -6
    for layers, trees, cws in ((None, buf.data_ptr(), x.data_ptr()), (buf.data_ptr(), None, x.data_ptr()),
                               (buf.data_ptr(), buf.data_ptr(), None)):
        assert lib.sa_fri_commit_batch(layers, trees, cws, 8, 2, 3, one, one, cb, None, st) == -6
    assert lib.sa_fri_commit_batch(buf.data_ptr(), buf.data_ptr(), x.data_ptr(), 8, 2, 3, one, one, None, None,
                                   st) == -6
    assert lib.sa_fri_commit_batch(None, None, None, 8, 0, 3, one, one, None, None, st) == 0
    for bad in (x.reshape(16, 2), x[:, :6].contiguous()):
        with pytest.raises(SaError):
            eng.fri_commit_batch(bad, 2, 7, omega, lambda *a: [1, 1])
    with pytest.raises(SaError):
        eng.fri_commit_batch(x, 5, 7, omega, lambda *a: [1, 1])
    assert eng.launch_count() == before


def test_merkle_chunk_has_no_spills():
    with tempfile.TemporaryDirectory() as tmp:
        report = subprocess.run(
            ["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
             "-diag-suppress", "550", "-c", "-Xptxas", "-v", "-o", os.path.join(tmp, "merkle_fri.o"),
             os.path.join(PKG, "csrc", "merkle_fri.cu")], capture_output=True, text=True, check=True).stderr
    m = re.search(r"Compiling entry function '(_Z\d+k_merkle_chunk[^']*)'.*?(\d+) bytes spill stores, (\d+) bytes "
                  r"spill loads.*?Used (\d+) registers", report, re.S)
    assert m and m.group(2) == m.group(3) == "0" and int(m.group(4)) <= 128, m and m.groups()
