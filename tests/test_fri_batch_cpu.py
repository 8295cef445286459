"""Batched FRI without a GPU.

* The emulated commit (tests/emu/emu_fri_batch.cpp): the library's round schedule and per-tree fold views over
  emulated launches, every layer and tree checked against the oracle's fri_commit for n = 2^1 .. 2^12 and batches
  of 1, 2, 3 and 5, with Fiat-Shamir challenges and with forced ones (0, 1, p - 1), equal and zero rows, a batch
  past one launch group, the refusals and an aborting callback.
* Fri.commit_batch / Fri.prove_batch through a test double that adds fri_commit_batch to the batch double of
  tests/stark_batch_cases.py: every stream holds, as pickled bytes, what Fri.prove pushes, for lists, device lists
  and one (B, N, 2) array, plain and prefixed streams, with a number of opening calls independent of B.
* The provers with fri_batch=True: the recorded two-signature fixtures byte for byte, synthetic batches equal to
  the default route, failures with their message and proof_index, and sign_batch.
"""
import ctypes
import hashlib
import pickle
import random

import numpy as np
import pytest

import __graft_entry__ as G
import oracle as O
import stark_batch_cases as SB
import stark_cases as C
import stark_plain_cases as S
import sa_devlist
import sa_engine
import sa_host
import sa_stark
import fri as dropin_fri
from sa_engine import FRI_CHALLENGE_FN

P = O.P
MK_MAX_TREES = 65535  # trees per launch (csrc/fri_merkle.cuh)


# ---------------------------------------------------------------------------------------------- the emulation
@pytest.fixture(scope="module")
def E():
    lib = ctypes.CDLL(G.build_emu_fri_batch())
    lib.emu_fri_commit_batch.restype = ctypes.c_int
    lib.emu_fri_commit_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_size_t,
                                         ctypes.c_size_t, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p,
                                         FRI_CHALLENGE_FN, ctypes.c_void_p]
    return lib


def commit(E, x, rounds, offset, omega, alphas_of, trees_fill=0xA5):
    """emu_fri_commit_batch over the (B, n, 2) rows x: (rc, the callback's calls, layers[r] (B, n >> r, 2) with
    layers[0] = x, trees[r] (B, 2 (n >> r), 64))"""
    B, n = x.shape[0], x.shape[1]
    x = np.ascontiguousarray(x)
    layers = np.full((max(B * (n - (n >> (rounds - 1))), 1), 2), 0x5A, dtype=np.uint64)
    trees = np.full((max(B * (4 * n - ((4 * n) >> rounds)), 1), 64), trees_fill, dtype=np.uint8)
    calls = []

    def cb(_user, r, roots_ptr, alphas_out, want):
        roots = ctypes.string_at(roots_ptr, 64 * B)
        calls.append((r, [roots[64 * b:64 * b + 64] for b in range(B)], want))
        alphas = alphas_of(r, calls[-1][1])
        if alphas is None:
            return 1
        if want:
            for b, a in enumerate(alphas):
                alphas_out[2 * b], alphas_out[2 * b + 1] = a & 0xFFFFFFFFFFFFFFFF, a >> 64
        return 0
    rc = E.emu_fri_commit_batch(O._ptr(layers), O._ptr(trees), O._ptr(x), n, B, rounds, O._ptr(O._fe(offset)),
                                O._ptr(O._fe(omega)), FRI_CHALLENGE_FN(cb), None)
    out_l, out_t, lo, to, ln = [x], [], 0, 0, n
    for r in range(rounds):
        out_t.append(trees[to:to + B * 2 * ln].reshape(B, 2 * ln, 64))
        to += B * 2 * ln
        if r + 1 < rounds:
            out_l.append(layers[lo:lo + B * (ln // 2)].reshape(B, ln // 2, 2))
            lo += B * (ln // 2)
            ln //= 2
    return rc, calls, out_l, out_t


def rows(seed, batch, n):
    rng = random.Random(seed)
    x = np.stack([O.to_np([rng.randrange(P) for _ in range(n)]) for _ in range(batch)])
    x[:, 0] = 0
    if n > 4:
        x[:, 1] = O._fe(P - 1)
    return x


def check_against_chain(x, layers, trees, alphas, offset, omega):
    """every row's layers and trees (node 0 aside, which no round but the first writes) are the single chain's"""
    for b in range(x.shape[0]):
        cur, om, off = x[b], omega, offset
        for r in range(len(trees)):
            assert (layers[r][b] == cur).all(), (b, r)
            assert (trees[r][b, 1:] == O.merkle_tree_np(cur)[1:]).all(), (b, r)
            if r + 1 < len(trees):
                cur = O.fri_fold_np(cur, alphas[r][b], off, om)
                om, off = om * om % P, off * off % P
        assert (trees[0][b, 0] == 0).all()


@pytest.mark.parametrize("batch", [1, 2, 3, 5])
@pytest.mark.parametrize("logn", range(1, 13))
def test_emulated_commit_matches_oracle(E, logn, batch):
    """Fiat-Shamir challenges, each row with its own transcript: roots, alphas and layers are fri_commit_np's"""
    n = 1 << logn
    x = rows(31 * logn + batch, batch, n)
    omega = O.primitive_nth_root(n)
    prior = [[b"row %d" % b] for b in range(batch)]
    objects = [list(p) for p in prior]

    def alphas_of(r, roots):
        out = []
        for b, root in enumerate(roots):
            objects[b].append(root)
            out.append(O.sample(O.fiat_shamir(objects[b])))
        return out
    rounds = O.fri_num_rounds(n, 1, 0)  # down to codewords of two elements
    rc, calls, layers, trees = commit(E, x, rounds, O.GENERATOR, omega, alphas_of)
    assert rc == 0
    assert [(r, w) for r, _, w in calls] == [(r, int(r != rounds - 1)) for r in range(rounds)]
    for b in range(batch):
        roots, alphas, want = O.fri_commit_np(x[b], O.GENERATOR, omega, 1, 0, prior[b])
        assert [c[1][b] for c in calls] == roots, b
        for r in range(rounds):
            assert (layers[r][b] == want[r]).all(), (b, r)
            assert (trees[r][b, 1:] == O.merkle_tree_np(want[r])[1:]).all(), (b, r)


@pytest.mark.parametrize("logn", [1, 2, 5, 9, 12])
def test_forced_alphas_equal_rows_and_zero_row(E, logn):
    """alpha 0, 1 and p - 1, rows 0 and 2 equal, row 3 zero, down to codewords of one element"""
    n = 1 << logn
    x = rows(logn, 5, n)
    x[2] = x[0]
    x[3] = 0
    choices = [0, 1, P - 1, 5, 0]
    alphas = []

    def alphas_of(r, roots):
        a = [choices[(b + r) % 5] for b in range(5)]
        alphas.append(a)
        return a
    rounds = logn + 1
    offset, omega = 7, O.primitive_nth_root(n)
    rc, calls, layers, trees = commit(E, x, rounds, offset, omega, alphas_of)
    assert rc == 0 and len(calls) == rounds
    check_against_chain(x, layers, trees, alphas, offset, omega)
    assert (trees[-1][3, 1:] == O.merkle_tree_np(np.zeros((1, 2), np.uint64))[1:]).all()


def test_batch_past_one_launch_group(E):
    """more trees than one launch takes: the second group starts at tree MK_MAX_TREES with its own rows, scalars and
    roots"""
    batch, n = MK_MAX_TREES + 2, 2
    x = np.zeros((batch, n, 2), dtype=np.uint64)
    x[:, 0, 0] = np.arange(batch, dtype=np.uint64)
    x[:, 1, 0] = 3
    alphas = []

    def alphas_of(r, roots):
        a = [b % 7 for b in range(batch)]
        alphas.append(a)
        return a
    rc, calls, layers, trees = commit(E, x, 2, O.GENERATOR, P - 1, alphas_of)
    assert rc == 0 and len(calls) == 2
    pick = list(range(3)) + list(range(MK_MAX_TREES - 2, batch))
    check_against_chain(x[pick], [layers[0][pick], layers[1][pick]], [trees[0][pick], trees[1][pick]],
                        [[alphas[0][b] for b in pick]], O.GENERATOR, P - 1)
    for b in pick:
        assert calls[0][1][b] == O.merkle_root_np(x[b])
        assert calls[1][1][b] == hashlib.blake2b(str(O.from_np(layers[1][b])[0]).encode()).digest()


def test_refusals_and_empty_batch(E):
    x = np.zeros((2, 8, 2), dtype=np.uint64)
    buf = np.zeros((256, 64), dtype=np.uint8)
    cb = FRI_CHALLENGE_FN(lambda *a: 1)
    one = O._ptr(O._fe(1))
    for n, rounds in ((6, 1), (0, 1), (8, 0), (8, 5), (1, 2)):
        assert E.emu_fri_commit_batch(O._ptr(buf), O._ptr(buf), O._ptr(x), n, 2, rounds, one, one, cb, None) == -6
    for nulls in ((None, O._ptr(buf), O._ptr(x)), (O._ptr(buf), None, O._ptr(x)), (O._ptr(buf), O._ptr(buf), None)):
        assert E.emu_fri_commit_batch(*nulls, 8, 2, 3, one, one, cb, None) == -6
    # a lone round folds nothing: no layer buffer needed
    rc, calls, _, trees = commit(E, x, 1, 1, O.primitive_nth_root(8), lambda r, roots: [])
    assert rc == 0 and len(calls) == 1 and calls[0][2] == 0
    assert E.emu_fri_commit_batch(None, None, None, 8, 0, 3, one, one, FRI_CHALLENGE_FN(lambda *a: 1 / 0), None) == 0


def test_callback_abort(E):
    x = rows(3, 3, 64)
    seen = []

    def alphas_of(r, roots):
        seen.append(r)
        return [1, 2, 3] if r == 0 else None
    rc, calls, layers, trees = commit(E, x, 4, O.GENERATOR, O.primitive_nth_root(64), alphas_of)
    assert rc == -7 and seen == [0, 1]
    assert (trees[2] == 0xA5).all() and (trees[3] == 0xA5).all()  # nothing after the aborted round
    assert (layers[2] == 0x5A).all()


# ------------------------------------------------------------------------------------------- the drop-in Fri
class FriBatchEngine(SB.BatchStarkEngine):
    """the batch double plus fri_commit_batch, restated as fri_commit's chain per row with one callback per round"""
    name = "oracle-test-double-fri-batch"

    def fri_commit_batch(self, vecs, rounds, offset, omega, on_roots):
        self._log("fri_commit_batch", vecs.shape[0], vecs.shape[1], rounds)
        cur = np.ascontiguousarray(vecs)
        layers, trees = [cur], []
        for r in range(rounds):
            t = np.stack([O.merkle_tree_np(row) for row in cur])
            trees.append(t)
            want = r != rounds - 1
            alphas = on_roots(r, [row[1].tobytes() for row in t], want)
            if not want:
                break
            cur = np.stack([O.fri_fold_np(row, a, offset, omega) for row, a in zip(cur, alphas)])
            layers.append(cur)
            omega, offset = omega * omega % P, offset * offset % P
        return layers, trees


@pytest.fixture
def double():
    prev = sa_engine._ENGINE
    eng = FriBatchEngine()
    sa_engine.set_engine(eng)
    yield eng
    sa_engine.set_engine(prev)


def make_fri(logn, k):
    n = 1 << logn
    return dropin_fri.Fri(C.T.field.generator(), C.T.field.primitive_nth_root(n), n, 4, k)


def codewords(seed, batch, n):
    rng = random.Random(seed)
    cws = [[C.T.fe(rng.randrange(P)) for _ in range(n)] for _ in range(batch)]
    if batch > 2:
        cws[2] = list(cws[0])  # equal values, other objects
    return cws


def streams(kind, batch):
    if kind == "plain":
        return [sa_host.ip.ProofStream() for _ in range(batch)]
    return [C.SignatureProofStream(b"document %d" % b) for b in range(batch)]


def as_input(kind, cws):
    if kind == "lists":
        return cws
    if kind == "device":
        return [sa_devlist.DeviceCodeword(sa_devlist.to_device(cw), None, C.T.field, len(cw)) for cw in cws]
    return np.stack([O.to_np([v.value for v in cw]) for cw in cws])


@pytest.mark.parametrize("stream", ["plain", "signature"])
@pytest.mark.parametrize("form", ["lists", "device", "array"])
@pytest.mark.parametrize("logn,k,batch", [(4, 2, 3), (6, 2, 1), (6, 2, 4), (10, 4, 5)])
def test_prove_batch_is_prove(double, form, stream, logn, k, batch):
    f = make_fri(logn, k)
    cws = codewords(logn * 10 + batch, batch, 1 << logn)
    want_streams = streams(stream, batch)
    for ps in want_streams:
        ps.push(b"prefix")
    want = [f.prove(as_input(form, [cw])[0] if form != "array" else as_input("device", [cw])[0], ps)
            for cw, ps in zip(cws, want_streams)]
    got_streams = streams(stream, batch)
    for ps in got_streams:
        ps.push(b"prefix")
    got = f.prove_batch(as_input(form, cws), got_streams)
    assert got == want
    for g, w in zip(got_streams, want_streams):
        assert pickle.dumps(g.objects) == pickle.dumps(w.objects)


def test_identity_within_a_proof(double):
    """a c-value of round r is the a- or b-value object of round r + 1, and the last round's c-values are the pushed
    last codeword's elements"""
    f = make_fri(8, 4)
    ps = sa_host.ip.ProofStream()
    f.prove_batch(as_input("array", codewords(3, 1, 256)), [ps])
    rounds = f.num_rounds()
    last = ps.objects[rounds]
    triples = [o for o in ps.objects if isinstance(o, tuple)]
    k = f.num_colinearity_tests
    by_round = [triples[r * k:(r + 1) * k] for r in range(rounds - 1)]
    for r in range(rounds - 2):
        for s in range(k):
            c = by_round[r][s][2]
            assert any(c is x for x in by_round[r + 1][s][:2])
    assert all(any(t[2] is e for e in last) for t in by_round[-1])


def test_commit_batch_is_commit(double):
    f = make_fri(6, 2)
    cws = codewords(5, 3, 64)
    want = [sa_host.ip.ProofStream() for _ in cws]
    wcw = [f.commit(cw, ps) for cw, ps in zip(cws, want)]
    got = [sa_host.ip.ProofStream() for _ in cws]
    gcw = f.commit_batch(cws, got)
    for g, w, gc, wc in zip(got, want, gcw, wcw):
        assert pickle.dumps(g.objects) == pickle.dumps(w.objects)
        assert len(gc) == len(wc) and [list(c) for c in gc] == [list(c) for c in wc]
        assert gc[-1] is g.objects[-1]


@pytest.mark.parametrize("batch", [1, 6])
def test_opening_calls_do_not_grow_with_the_batch(double, batch):
    f = make_fri(10, 4)
    f.prove_batch(as_input("array", codewords(1, batch, 1024)), streams("plain", batch))
    names = [c[0] for c in double.calls]
    rounds = f.num_rounds()
    assert names.count("fri_commit_batch") == 1
    assert names.count("merkle_open_batch") == rounds and names.count("gather_batch") == rounds - 1
    assert names.count("download") == 1  # the last codewords


def test_prove_batch_refuses_wrong_length(double):
    f = make_fri(6, 2)
    with pytest.raises(AssertionError, match="initial codeword length"):
        f.prove_batch(codewords(1, 2, 32), streams("plain", 2))


# ------------------------------------------------------------------------------------------------ the provers
@pytest.fixture
def batch_double():
    prev = sa_engine._ENGINE
    sa_engine.set_engine(FriBatchEngine())
    yield
    sa_engine.set_engine(prev)


class FriBatched:
    """a plan whose prove_batch takes the batched FRI route"""

    def __init__(self, plan):
        self.plan = plan

    def prove_batch(self, *args):
        return self.plan.prove_batch(*args, fri_batch=True)


@pytest.mark.parametrize("fast", [True, False])
def test_fixture_signatures_with_batched_fri(batch_double, fast):
    g = C.golden() if fast else S.golden()
    first, second = g["rpsss"], g["rpsss_second"]
    st = C.params(first) if fast else S.stark(first)
    recs = (first, second)
    traces, boundaries = zip(*[C.inputs(r) for r in recs])
    draws = C.Urandom(SB.batch_draws([r["draws"] for r in recs], SB.ntrace(first)))
    ss = [C.stream(r) for r in recs]
    if fast:
        zpoly, zvals = C.zerofier(st)
        plan = FriBatched(sa_stark.StarkPlan(st, C.air(first), zpoly))
        proofs = SB.run_batch(plan, list(traces), list(boundaries), draws, ss, C.zerofier_codeword(zvals, True))
    else:
        plan = FriBatched(sa_stark.PlainStarkPlan(st, C.air(first)))
        proofs = SB.run_batch(plan, list(traces), list(boundaries), draws, ss)
    assert isinstance(proofs, list), proofs
    assert draws.count == len(first["draws"]) + len(second["draws"])
    for rec, proof, ps in zip(recs, proofs, ss):
        assert hashlib.sha256(proof).hexdigest() == rec["proof_sha256"]
        assert ps.serialize() == proof


@pytest.mark.parametrize("fast", [True, False])
def test_synthetic_batch_equals_default_route(batch_double, fast):
    st, cons, trace, boundary = C.synthetic(5, 10)
    B = 3
    zpoly, zvals = C.zerofier(st)
    zcw = C.zerofier_codeword(zvals, True)
    plan = sa_stark.StarkPlan(st, cons, zpoly) if fast else sa_stark.PlainStarkPlan(S.plain_stark(st), cons)
    nt = st.num_registers * st.num_randomizers
    rng = random.Random(4)
    per = [[rng.randrange(P) for _ in range(nt + plan.max_degree + 1)] for _ in range(B)]
    got = {}
    for route in (False, True):
        draws = C.Urandom(SB.batch_draws(per, nt))
        target = FriBatched(plan) if route else plan
        got[route] = SB.run_batch(target, [trace] * B, [boundary] * B, draws, None, zcw if fast else None)
        assert draws.count == B * len(per[0])
    assert isinstance(got[True], list) and got[True] == got[False]


FAILING = [(fast, bad) for fast in (True, False) for bad in ("broken_witness", "false_boundary")
           if "raises" in (C.golden() if fast else S.golden())[bad]]


@pytest.mark.parametrize("fast,bad", FAILING)
@pytest.mark.parametrize("at", [0, 2])
def test_failure_keeps_message_and_index(batch_double, fast, bad, at):
    g = C.golden() if fast else S.golden()
    rec, good = g[bad], g["three_register"]
    st = C.params(rec) if fast else S.stark(rec)
    recs = [good] * 3
    recs[at] = rec
    traces, boundaries = zip(*[C.inputs(r) for r in recs])
    zpoly, zvals = C.zerofier(C.params(rec))
    zcw = C.zerofier_codeword(zvals, True)
    plan = sa_stark.StarkPlan(st, C.air(rec), zpoly) if fast else sa_stark.PlainStarkPlan(st, C.air(rec))
    got = SB.run_batch(FriBatched(plan), list(traces), list(boundaries), C.Urandom([7] * 100000), None,
                       zcw if fast else None)
    assert isinstance(got, AssertionError), got
    assert str(got).startswith(rec["raises"]) and got.proof_index == at


@pytest.mark.parametrize("fast", [True, False])
def test_sign_batch_with_batched_fri(batch_double, fast):
    g = C.golden() if fast else S.golden()
    first, second = g["rpsss"], g["rpsss_second"]
    signer = SB.Signer(first, fast)
    docs = [bytes.fromhex(first["document"]), bytes.fromhex(second["document"]), b"third"]
    nt = SB.ntrace(first)
    per = [[str(v) for v in range(s, s + len(first["draws"]))] for s in (11, 5, 3)]
    out = {}
    real = sa_stark.os.urandom
    try:
        for route in (False, True):
            sa_stark.os.urandom = C.Urandom(SB.batch_draws(per, nt))
            out[route] = sa_stark.sign_batch(signer, 1, docs, fri_batch=route)
    finally:
        sa_stark.os.urandom = real
    assert out[True] == out[False] and len(set(out[True])) == 3


def test_empty_batch_does_no_device_work(double):
    f = make_fri(6, 2)
    assert f.commit_batch([], []) == [] and f.prove_batch([], []) == []
    assert f.commit_batch(np.zeros((0, 64, 2), np.uint64), []) == [] and double.calls == []
