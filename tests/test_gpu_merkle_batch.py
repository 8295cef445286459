"""Batched Merkle trees, openings and gathers on the GPU (sa_merkle_tree_batch, sa_merkle_open_batch,
sa_gather_batch through sa_engine): every tree against the oracle and against single-tree calls, the 2^20 golden
root, batches past the initial arrival counters and past one launch, launch counts, errors before any launch, and
batches on one stream beside FRI commits on another."""
import ctypes
import random
import threading

import numpy as np
import pytest

import oracle as O
import dropin_cases as C
import sa_engine

pytestmark = pytest.mark.gpu
P = O.P
MK_MAX_TREES = 65535  # trees per launch (csrc/fri_merkle.cuh)


@pytest.fixture(scope="module")
def eng():
    sa_engine.set_engine(None)
    e = sa_engine.get_engine()  # raises without CUDA / without the built library
    assert e.name == "cuda"
    return e


@pytest.fixture(autouse=True)
def _cuda_engine(eng):
    sa_engine.set_engine(eng)
    yield


def rand_rows(seed, batch, n):
    rng = np.random.default_rng(seed)
    lo = rng.integers(0, 1 << 64, size=(batch, n), dtype=np.uint64)
    hi = rng.integers(0, 0xCB80000000000000, size=(batch, n), dtype=np.uint64)  # < p's top limb => < p
    x = np.stack([lo, hi], axis=2)
    x[:, 0] = 0
    if n > 4:  # the edge values of test_gpu.py::test_merkle_tree_and_open
        x[:, 1] = (7, 0)
        x[:, 2] = O._fe(10**19)
        x[:, 3] = O._fe(P - 1)
    return x


def up(eng, x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).to(eng.device)


@pytest.mark.parametrize("batch", [1, 2, 5])
@pytest.mark.parametrize("log_n", [0, 1, 5, 6, 7, 10, 12, 13, 14, 15, 16, 17, 18])
def test_batch_matches_oracle_and_single_calls(eng, log_n, batch):
    n = 1 << log_n
    x = rand_rows(1000 * log_n + batch, batch, n)
    vecs = up(eng, x)
    trees = eng.merkle_trees(vecs)
    assert tuple(trees.shape) == (batch, 2 * n, 64)
    got = trees.cpu().numpy()
    want = [O.merkle_tree_np(x[b]) for b in range(batch)]
    for b in range(batch):
        assert (got[b, 0] == 0).all(), b
        assert (got[b, 1:] == want[b][1:]).all(), b
        assert (got[b] == eng.merkle_tree(vecs[b]).cpu().numpy()).all(), b
    assert eng.tree_roots(trees) == [w[1].tobytes() for w in want]
    idx = sorted({0, 1 % n, n // 2, n - 1, random.Random(log_n).randrange(n)})
    paths = eng.merkle_open_batch(trees, idx)
    assert len(paths) == batch
    for b in range(batch):
        assert paths[b] == eng.merkle_open(trees[b], idx) == [O.merkle_open(want[b], i) for i in idx], b
    assert (eng.gather_batch(vecs, idx).view(np.uint64) == x[:, idx]).all()


def test_batch_2_20_golden_root(eng):
    from conftest import load_golden
    import sa_marshal
    c = [m for m in load_golden("merkle.json")["commit"] if m["n"] == 1 << 20][0]
    n = 1 << 20
    x = rand_rows(2020, 3, n)
    x[1] = np.frombuffer(bytes(sa_marshal.pack(C.seeded(1, n))), dtype=np.uint64).reshape(n, 2)
    vecs = up(eng, x)
    trees = eng.merkle_trees(vecs)
    assert eng.tree_roots(trees)[1].hex() == c["root"]
    for b in (0, 2):
        assert bool((trees[b] == eng.merkle_tree(vecs[b])).all()), b


def test_batch_past_the_initial_counters(eng):
    """100 trees of 2^10 leaves (16 CTAs each, fused top): more trees than the 64 counters a stream starts with"""
    n = 1 << 10
    vecs = up(eng, rand_rows(100, 100, n))
    trees = eng.merkle_trees(vecs)
    for b in range(100):
        assert bool((trees[b] == eng.merkle_tree(vecs[b])).all()), b


def test_batch_past_one_launch(eng):
    """MK_MAX_TREES + 2 trees of 128 leaves (two CTAs per tree and the fused top: one launch per tree): two
    groups, each issuing the launches of one tree, the second with its own rows, trees and counters"""
    import torch
    n, batch = 128, MK_MAX_TREES + 2
    vecs = torch.randint(0, 1 << 62, (batch, n, 2), dtype=torch.int64, device=eng.device)
    vecs[..., 1] &= (1 << 61) - 1
    eng.synchronize()
    c0 = eng.launch_count()
    eng.merkle_tree(vecs[0])
    single = eng.launch_count() - c0
    c0 = eng.launch_count()
    trees = eng.merkle_trees(vecs)
    assert eng.launch_count() - c0 == 2 * single
    for b in [0, 1, MK_MAX_TREES - 1, MK_MAX_TREES, batch - 1] + random.Random(3).sample(range(batch), 20):
        assert bool((trees[b] == eng.merkle_tree(vecs[b])).all()), b


@pytest.mark.parametrize("log_n", [0, 1, 6, 7, 10, 12, 14, 16, 18, 20])
def test_batch_issues_the_launches_of_one_tree(eng, log_n):
    import torch
    n = 1 << log_n
    vecs = torch.randint(0, 1 << 62, (8, n, 2), dtype=torch.int64, device=eng.device)
    vecs[..., 1] &= (1 << 61) - 1
    eng.merkle_trees(vecs)  # counters grown for 8 trees
    eng.synchronize()
    c0 = eng.launch_count()
    eng.merkle_tree(vecs[0])
    single = eng.launch_count() - c0
    assert single >= 1
    for batch in (1, 2, 5, 8):
        c0 = eng.launch_count()
        eng.merkle_trees(vecs[:batch])
        assert eng.launch_count() - c0 == single, batch
    trees = eng.merkle_trees(vecs)
    idx = [0, n - 1, n // 2]
    c0 = eng.launch_count()
    eng.merkle_open_batch(trees, idx)
    eng.gather_batch(vecs, idx)
    assert eng.launch_count() - c0 == (2 if log_n else 1)  # a one-leaf tree has no siblings to open


def test_errors_before_any_launch(eng):
    import torch
    lib = eng.lib
    n = 1 << 8
    vecs = torch.zeros((3, n, 2), dtype=torch.int64, device=eng.device)
    trees = eng.merkle_trees(vecs)
    eng.synchronize()
    c0 = eng.launch_count()
    with pytest.raises(AssertionError, match="cannot open invalid index"):
        eng.merkle_open_batch(trees, [0, n])
    st = eng._stream()
    out = torch.empty(3 * 2 * 8 * 64, dtype=torch.uint8, device=eng.device)
    bad = (ctypes.c_uint64 * 2)(0, n)
    assert lib.sa_merkle_open_batch(out.data_ptr(), trees.data_ptr(), n, 3, bad, 2, st) == -5
    assert lib.sa_gather_batch(out.data_ptr(), vecs.data_ptr(), n, 3, bad, 2, st) == -5
    assert lib.sa_merkle_open_batch(out.data_ptr(), trees.data_ptr(), n, 0, bad, 2, st) == -5
    with pytest.raises(AssertionError, match="cannot open invalid index"):
        eng.gather_batch(vecs, [n])
    with pytest.raises(AssertionError, match="non-power-of-two"):
        eng.merkle_trees(torch.zeros((2, 3, 2), dtype=torch.int64, device=eng.device))
    assert lib.sa_merkle_tree_batch(out.data_ptr(), vecs.data_ptr(), 12, 3, st) == -1
    assert lib.sa_merkle_open_batch(out.data_ptr(), trees.data_ptr(), 12, 3, bad, 1, st) == -1
    for bad_shape in ((n, 2), (3, n, 3), (3, n, 2, 1)):
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.merkle_trees(torch.zeros(bad_shape, dtype=torch.int64, device=eng.device))
        with pytest.raises(AssertionError, match="unsupported size"):
            eng.gather_batch(torch.zeros(bad_shape, dtype=torch.int64, device=eng.device), [0])
    with pytest.raises(AssertionError, match="unsupported size"):
        eng.merkle_open_batch(trees[0], [0])
    with pytest.raises(AssertionError, match="unsupported size"):
        eng.tree_roots(trees[:, :3])
    # nothing to do: no launch
    assert tuple(eng.merkle_trees(vecs[:0]).shape) == (0, 2 * n, 64)
    assert eng.merkle_open_batch(trees[:0], [0, 1]) == []
    assert eng.merkle_open_batch(trees, []) == [[], [], []]
    assert eng.gather_batch(vecs[:0], [0, 1]).shape == (0, 2, 2)
    assert eng.gather_batch(vecs, []).shape == (3, 0, 2)
    good = (ctypes.c_uint64 * 1)(1)
    assert lib.sa_merkle_tree_batch(out.data_ptr(), vecs.data_ptr(), n, 0, st) == 0
    assert lib.sa_merkle_open_batch(out.data_ptr(), trees.data_ptr(), n, 0, good, 1, st) == 0
    assert lib.sa_gather_batch(out.data_ptr(), vecs.data_ptr(), n, 0, good, 1, st) == 0
    assert eng.launch_count() == c0


def test_batches_and_fri_commits_on_two_streams(eng):
    """batched trees from one host thread on one stream and whole FRI commits from another on a second stream:
    the arrival counters are per stream (and grow on the first stream meanwhile), so neither may leak into the
    other's results"""
    import torch
    log_n = 13
    n = 1 << log_n
    omega, off = O.primitive_nth_root(n), O.GENERATOR
    xb = rand_rows(800, 5, n)
    xw = rand_rows(801, 70, 1 << 10)
    cw = rand_rows(802, 1, n)[0]
    alphas = [random.Random(803).randrange(P) for _ in range(8)]
    got = {"trees": [], "wide": [], "roots": []}
    errs = []

    def batches():
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                vb, vw = up(eng, xb), up(eng, xw)
                for rep in range(10):
                    got["trees"].append(eng.merkle_trees(vb).cpu().numpy())
                    got["wide"].append(eng.tree_roots(eng.merkle_trees(vw)))
            st.synchronize()
        except BaseException as exc:  # surfaces in the main thread
            errs.append(exc)

    def commits():
        try:
            st = torch.cuda.Stream()
            with torch.cuda.stream(st):
                v = up(eng, cw)
                for rep in range(10):
                    roots = []
                    eng.fri_commit(v, 8, off, omega, lambda r, root, want: (roots.append(root), alphas[r])[1])
                    got["roots"].append(roots)
            st.synchronize()
        except BaseException as exc:
            errs.append(exc)
    ts = [threading.Thread(target=batches), threading.Thread(target=commits)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errs, errs
    want_trees = [O.merkle_tree_np(xb[b]) for b in range(5)]
    want_wide = [O.merkle_tree_np(xw[b])[1].tobytes() for b in range(70)]
    c, o, w, want_roots = cw, off, omega, []
    for r in range(8):
        want_roots.append(O.merkle_tree_np(c)[1].tobytes())
        if r < 7:
            c = O.fri_fold_np(c, alphas[r], o, w)
            o, w = o * o % P, w * w % P
    for rep in range(10):
        for b in range(5):
            assert (got["trees"][rep][b, 1:] == want_trees[b][1:]).all(), (rep, b)
        assert got["wide"][rep] == want_wide, rep
        assert got["roots"][rep] == want_roots, rep
