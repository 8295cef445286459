"""Merkle leaves, FRI layers and openings on the GPU over the leaf-encoding edge corpus (tests/leaf_edges.py):
values of every decimal length 1..39, zero and full base-1e8 limbs, and the partial dividends where the long
division's FP64 quotient estimate is closest to rounding up or has to be repaired.  Each width tiles the corpus
in a seeded permutation.  Every leaf digest is checked against hashlib.blake2b(str(v).encode()), every inner
node against a hashlib-only tree (up to 2^16 leaves) or the C oracle's tree, and every opened path by climbing
to the root with hashlib.  The four routes a leaf takes are covered: sa_merkle_tree / sa_merkle_tree_batch
(values read from a codeword row), sa_fri_round and sa_fri_commit (values folded on the fly), and the drop-in
fri.Merkle / DeviceCodeword route."""
import functools
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O
import leaf_edges as LE

G._paths()
import sa_engine  # noqa: E402

pytestmark = pytest.mark.gpu
P = O.P
HASHLIB_TREE_MAX = 1 << 16  # up to this width the whole tree is checked against LE.tree


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


@functools.lru_cache(maxsize=None)
def corpus():
    """(values, limbs uint64[m, 2], leaf digests uint8[m, 64])"""
    values = LE.build()[0]
    digests = np.frombuffer(b"".join(LE.leaf(v) for v in values), dtype=np.uint8).reshape(-1, 64)
    return values, O.to_np(values), digests


def tile_idx(n, seed):
    """corpus indices for a width n: the corpus repeated, each copy in its own seeded permutation, cut to n"""
    m = len(corpus()[0])
    rng = np.random.default_rng(seed)
    return np.concatenate([rng.permutation(m) for _ in range(-(-n // m))])[:n]


def up(eng, x):
    """uint64[n, 2] -> device vector; uint64[B, n, 2] -> device batch of B rows"""
    import torch
    return torch.from_numpy(np.ascontiguousarray(x).view(np.int64)).to(eng.device)


def first_bad(got, want):
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = np.nonzero((got != want).reshape(len(got), -1).any(axis=1))[0] if len(got) else []
    return int(bad[0]) if len(bad) else None


def check_tree(got, idx, what, node0=True):
    """a device tree (uint8[2n, 64]) of the corpus values at idx: leaves against hashlib, inner nodes against
    the hashlib tree (n <= 2^16) or the oracle's"""
    values, limbs, digests = corpus()
    n = len(idx)
    assert got.shape == (2 * n, 64), what
    if node0:
        assert not got[0].any(), what
    i = first_bad(got[n:], digests[idx])
    assert i is None, "%s: leaf %d (value %d) differs from blake2b(str(v))" % (what, i, values[idx[i]])
    if n <= HASHLIB_TREE_MAX:
        want = np.frombuffer(b"".join(LE.tree([values[j] for j in idx])[1:n]), dtype=np.uint8).reshape(-1, 64)
    else:
        want = O.merkle_tree_np(limbs[idx])[1:n]
    i = first_bad(got[1:n], want)
    assert i is None, "%s: inner node %d differs" % (what, i + 1)


def check_paths(paths, vals, idx, root, what):
    assert len(paths) == len(idx), what
    for path, v, i in zip(paths, vals, idx):
        assert LE.climb(v, i, path) == root, (what, i, v)


@pytest.mark.parametrize("log_n", [0, 1, 6, 7, 10, 14, 15, 16, 18, 20])
def test_merkle_tree_widths(eng, log_n):
    """one CTA (<= 64), chunk 64 with the fused top, chunk 128, chunk 256, ipt_log 1 and the throughput shape"""
    n = 1 << log_n
    idx = tile_idx(n, 100 + log_n)
    got = eng.merkle_tree(up(eng, corpus()[1][idx])).cpu().numpy()
    check_tree(got, idx, "merkle_tree 2^%d" % log_n)


@pytest.mark.parametrize("batch,log_n", [(5, 12), (3, 18)])
def test_merkle_tree_batch_rows(eng, batch, log_n):
    """every row its own permutation: a row read at the wrong stride hashes another row's values"""
    n = 1 << log_n
    idx = [tile_idx(n, 200 + 10 * log_n + b) for b in range(batch)]
    trees = eng.merkle_trees(up(eng, np.stack([corpus()[1][i] for i in idx])))
    got = trees.cpu().numpy()
    for b in range(batch):
        check_tree(got[b], idx[b], "merkle_trees row %d of %d x 2^%d" % (b, batch, log_n))
    assert eng.tree_roots(trees) == [bytes(got[b, 1]) for b in range(batch)]


@functools.lru_cache(maxsize=None)
def preimage(log_n):
    """(codeword limbs, corpus indices of its fold, alpha, offset, omega): a codeword of 2^log_n points whose
    fold with alpha is the corpus tiled to 2^(log_n - 1)"""
    values = corpus()[0]
    idx = tile_idx(1 << (log_n - 1), 300 + log_n)
    omega, offset = O.primitive_nth_root(1 << log_n), O.GENERATOR
    alpha = random.Random(log_n).randrange(P)
    cw = LE.fold_preimage([values[j] for j in idx], alpha, offset, omega, random.Random(400 + log_n))
    return O.to_np(cw), idx, alpha, offset, omega


@pytest.mark.parametrize("log_n", [11, 17, 21])
def test_fri_round_folds_to_the_corpus(eng, log_n):
    cw, idx, alpha, offset, omega = preimage(log_n)
    out, tree = eng.fri_round(up(eng, cw), alpha, offset, omega)
    got = eng.download(out).view(np.uint64)
    assert first_bad(got, corpus()[1][idx]) is None, "the folded layer is not the corpus"
    check_tree(tree.cpu().numpy(), idx, "fri_round 2^%d" % log_n, node0=False)


@pytest.mark.parametrize("log_n", [17, 21])
def test_fri_commit_layer_one_is_the_corpus(eng, log_n):
    cw, idx, alpha, offset, omega = preimage(log_n)
    rounds = 6
    alphas = [alpha] + [random.Random(500 + r).randrange(P) for r in range(1, rounds)]
    roots = []
    layers, trees = eng.fri_commit(up(eng, cw), rounds, offset, omega,
                                   lambda r, root, want: (roots.append(root), alphas[r] if want else 0)[1])
    assert first_bad(eng.download(layers[1]).view(np.uint64), corpus()[1][idx]) is None
    t1 = trees[1].cpu().numpy()
    n1 = len(idx)
    i = first_bad(t1[n1:], corpus()[2][idx])
    assert i is None, "layer 1 leaf %d (value %d)" % (i, corpus()[0][idx[i]])
    c, o, w = cw, offset, omega
    for r in range(rounds):
        assert roots[r] == O.merkle_root_np(c), r
        assert eng.tree_root(trees[r]) == roots[r], r
        if r + 1 < rounds:
            c = O.fri_fold_np(c, alphas[r], o, w)
            o, w = o * o % P, w * w % P


def test_openings_every_index_of_2_10(eng):
    values, limbs, _ = corpus()
    n, batch = 1 << 10, 3
    idx = [tile_idx(n, 600 + b) for b in range(batch)]
    vecs = up(eng, np.stack([limbs[i] for i in idx]))
    trees = eng.merkle_trees(vecs)
    opened = list(range(n - 1, -1, -1)) + [0, 0, n - 1, n - 1, 517, 517, 3]
    want = [LE.tree([values[j] for j in i]) for i in idx]
    batch_paths = eng.merkle_open_batch(trees, opened)
    gathered = eng.gather_batch(vecs, opened).view(np.uint64)
    for b in range(batch):
        vals = [values[idx[b][i]] for i in opened]
        paths = eng.merkle_open(trees[b], opened)
        check_paths(paths, vals, opened, want[b][1], "merkle_open row %d" % b)
        assert batch_paths[b] == paths, b
        for path, i in zip(paths, opened):  # the siblings of the hashlib tree, bottom-up
            assert path == [want[b][((n + i) >> l) ^ 1] for l in range(10)], (b, i)
        assert O.from_np(gathered[b]) == vals, b
        assert O.from_np(eng.gather(vecs[b], opened).view(np.uint64)) == vals, b


def test_openings_of_2_20(eng):
    values, limbs, _ = corpus()
    n, batch = 1 << 20, 2
    idx = [tile_idx(n, 700 + b) for b in range(batch)]
    vecs = up(eng, np.stack([limbs[i] for i in idx]))
    trees = eng.merkle_trees(vecs)
    roots = eng.tree_roots(trees)
    opened = [0, n - 1] + random.Random(20).sample(range(n), 64)
    batch_paths = eng.merkle_open_batch(trees, opened)
    gathered = eng.gather_batch(vecs, opened).view(np.uint64)
    for b in range(batch):
        vals = [values[idx[b][i]] for i in opened]
        assert roots[b] == O.merkle_root_np(limbs[idx[b]]), b
        paths = eng.merkle_open(trees[b], opened)
        check_paths(paths, vals, opened, roots[b], "merkle_open 2^20 row %d" % b)
        assert batch_paths[b] == paths, b
        assert O.from_np(gathered[b]) == vals and O.from_np(eng.gather(vecs[b], opened).view(np.uint64)) == vals


@pytest.mark.parametrize("log_n", [16, 17])
def test_dropin_merkle_on_the_corpus(eng, log_n):
    """fri.Merkle on a host list of FieldElements (sa_marshal.pack, upload) and on a DeviceCodeword with the same
    values; openings through both, in DeviceCodeword.open_paths' host branch (n <= 2^16, at most two indices or
    a downloaded tree) and its device branch"""
    from hostmirror_loader import load_host_types
    T = load_host_types()
    import fri as F
    import sa_devlist
    values, limbs, _ = corpus()
    n = 1 << log_n
    idx = tile_idx(n, 800 + log_n)
    xs = [values[j] for j in idx]
    root = LE.tree(xs)[1]
    fes = [T.fe(v) for v in xs]
    assert F.Merkle.commit(fes) == root
    opened = [0, n - 1] + random.Random(log_n).sample(range(n), 30)
    for i in opened[:8]:
        path = F.Merkle.open(i, fes)
        assert LE.climb(xs[i], i, path) == root and F.Merkle.verify(root, i, path, fes[i]), i

    def resident():
        return sa_devlist.DeviceCodeword(up(eng, limbs[idx]), None, T.field, n)
    dc = resident()
    assert F.Merkle.commit(dc) == root
    for i in opened[:4]:
        path = F.Merkle.open(i, dc)
        assert LE.climb(xs[i], i, path) == root and F.Merkle.verify(root, i, path, fes[i]), i
    assert (dc._host_tree is not None) == (n <= sa_devlist.SMALL_TREE)  # one index at a time: host branch at 2^16
    check_paths(dc.open_paths(opened[:2]), [xs[i] for i in opened[:2]], opened[:2], root, "open_paths, two")
    check_paths(dc.open_paths(opened), [xs[i] for i in opened], opened, root, "open_paths, many")
    dc = resident()  # no tree downloaded yet: more than two indices go to the device
    paths = dc.open_paths(opened)
    assert dc._host_tree is None
    check_paths(paths, [xs[i] for i in opened], opened, root, "open_paths on the device")
    for path, i in zip(paths, opened):
        assert F.Merkle.verify(root, i, path, fes[i]), i
    assert [x.value for x in dc[:4]] == xs[:4]
