"""The device prover at the sizes it is advertised for: synthetic AIRs at FRI domains 2^16 to 2^22, with 1 to 9
registers, expansion factors 4 to 16 and 2 to 8 colinearity checks, proved by sa_stark through CudaEngine and judged
without the test double (too slow above 2^16):

  1. the test-side verifier (tests/stark_verify.py) accepts the proof;
  2. the verifier's per-index equation holds at the first and last 1024 indices, at the expansion_factor indices
     whose neighbour wraps past n, and at one seeded index in every aligned block of 256: no block of the committed
     and combined codewords goes unchecked;
  3. the oracle's inverse transform of the combined codeword is zero from max_degree + 1 on, and each boundary
     codeword and the randomizer codeword is zero past its own bound, with a non-zero coefficient at it;
  4. the proof's Merkle roots are the oracle's roots of the downloaded codewords.

The 2^22 case has 9 registers and 9 constraints, so the prover's batched coset calls cross one chunk of
sa_coset_batch_max (8 rows at 2^22).  A witness broken at one middle row gives a proof the verifier rejects, and a
false boundary value raises the reference's remainder message."""
import contextlib
import functools
import pickle
import random
import time

import numpy as np
import pytest

import oracle as O
import stark_cases as C
import stark_verify as V
import sa_devlist
import sa_engine
import sa_stark

pytestmark = pytest.mark.gpu
P = O.P
GIB = 1 << 30


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
    import torch
    torch.cuda.synchronize()


def need_device(eng, log_n, vectors):
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert eng.lib.sa_release_workspaces() == 0
    free, _ = torch.cuda.mem_get_info(eng.device)
    want = (16 << log_n) * vectors + 2 * GIB
    if free < want:
        pytest.skip("2^%d needs %.1f GiB free on the device, %.1f GiB are" % (log_n, want / GIB, free / GIB))


@functools.lru_cache(maxsize=2)
def synthetic(seed, log_fri, nregs, expansion_factor, colinearity_checks):
    """(Params, constraints as {exponent tuple: int}, trace rows as ints, boundary as ints) of a valid AIR built as
    stark_cases.synthetic builds one -- register i's next value a seeded polynomial in the current row, register 0's
    cubic, register 1's linear with an x term, the others quadratic; boundary points on every register's first row,
    register 0's last row and two seeded rows of register 1 (of register 0 when it is the only one) -- with
    num_cycles solved so that the FRI domain has exactly 2^log_fri points"""
    rng = random.Random(seed)
    n = 1 << log_fri
    odl = n // expansion_factor
    # a randomized trace of odl / 4 rows, times the constraint degree 3, lies in [odl / 2, odl): omicron domain odl
    ncycles = odl // 4 - 4 * colinearity_checks
    stark = sa_stark.Params(C.T.field, expansion_factor, colinearity_checks, 2 * colinearity_checks, nregs, ncycles,
                            transition_constraints_degree=3)
    assert stark.fri_domain_length == n
    nvars = 1 + 2 * nregs
    cons, maps = [], []
    for i in range(nregs):
        degree = 3 if i == 0 else 1 if i == 1 else 2
        terms = {}
        for _ in range(1 + rng.randrange(3)):
            e = [0] * nvars
            for _ in range(rng.randrange(degree + 1)):
                e[1 + rng.randrange(nregs)] += 1
            terms[tuple(e)] = rng.randrange(1, P)
        top = [0] * nvars
        for _ in range(degree):
            top[1 + rng.randrange(nregs)] += 1
        terms[tuple(top)] = rng.randrange(1, P)
        if i == 1:
            terms[tuple([1] + [0] * (nvars - 1))] = rng.randrange(1, P)
        maps.append([(v, k[0], [(j, e) for j, e in enumerate(k[1:1 + nregs]) if e]) for k, v in terms.items()])
        nxt = [0] * nvars
        nxt[1 + nregs + i] = 1
        d = {tuple(nxt): 1}
        for k, v in terms.items():
            d[k] = (d.get(k, 0) - v) % P
        cons.append(d)
    w = stark.omicron.value
    row = [rng.randrange(P) for _ in range(nregs)]
    rows = [row]
    x = 1
    for c in range(ncycles - 1):
        nxt = []
        for terms in maps:
            acc = 0
            for v, xe, vars_ in terms:
                t = v * pow(x, xe, P) if xe else v
                for j, e in vars_:
                    t = t * (row[j] if e == 1 else pow(row[j], e, P)) % P
                acc += t
            nxt.append(acc % P)
        row = nxt
        rows.append(row)
        x = x * w % P
    r1 = min(1, nregs - 1)
    boundary = [(0, s, rows[0][s]) for s in range(nregs)] + [(ncycles - 1, 0, rows[-1][0])]
    boundary += [(c, r1, rows[c][r1]) for c in rng.sample(range(1, ncycles - 1), 2)]
    return stark, cons, rows, boundary


def zerofier(eng, stark):
    """FastStark.preprocess's transition zerofier (of omicron^i, i < num_cycles - 1) built on the device, as int
    coefficients, and its codeword on the FRI domain as a DeviceCodeword; the codeword is checked at two points
    against the product of the linear factors in Python ints"""
    w, m, n = stark.omicron.value, stark.original_trace_length - 1, stark.fri_domain_length
    domain = [pow(w, i, P) for i in range(m)]
    z = eng.zerofier(eng.upload(O.to_np(domain).view(np.int64)))
    cw = eng.coset_evaluate(z, n.bit_length() - 1, stark.omega.value, stark.generator.value)
    for i in (1, n - 3):
        x = stark.generator.value * pow(stark.omega.value, i, P) % P
        want = 1
        for d in domain:
            want = want * (x - d) % P
        assert V.element(eng.download(cw[i:i + 1]).view(np.uint64), 0) == want
    return O.from_np(eng.download(z).view(np.uint64)), sa_devlist.DeviceCodeword(cw, None, C.T.field, n)


def fe(rows):
    return [C.T.elems(r) for r in rows]


def fe_boundary(boundary):
    return [(c, r, C.T.fe(v)) for c, r, v in boundary]


def prove(eng, stark, cons, rows, boundary, zpoly, zcw, seed, recorder=None):
    plan = sa_stark.StarkPlan(stark, cons, zpoly)
    rng = random.Random(seed)
    draws = C.Urandom([rng.randrange(P) for _ in range(stark.num_registers * stark.num_randomizers
                                                       + plan.max_degree + 1)])
    with recorder or contextlib.nullcontext():
        return C.run(stark, fe(rows), None, fe_boundary(boundary), zpoly, zcw, draws, plan=plan)[0], plan


def sweep_indices(n, ef, seed):
    """the first and last 1024 indices, the ef indices whose neighbour i + ef wraps past n, and one seeded index in
    every aligned block of 256"""
    rng = random.Random(seed)
    idx = set(range(min(1024, n))) | set(range(max(0, n - 1024), n)) | set(range(n - ef, n))
    idx |= {b + rng.randrange(256) for b in range(0, n, 256)}
    return sorted(idx)


def coefficients(root, values):
    """the oracle's inverse transform of a coset codeword: coefficient j times generator^j, which is zero exactly
    where coefficient j is (so no rescaling is needed to test zeros)"""
    return O.intt_np(root, values, parallel=True)


def top_and_tail(coeffs, bound):
    """(is coefficient `bound` non-zero, are all coefficients past `bound` zero)"""
    return bool(coeffs[bound].any()), not coeffs[bound + 1:].any()


MATRIX = [  # (log_fri, nregs, expansion_factor, colinearity_checks)
    (16, 1, 4, 2),
    (16, 3, 16, 8),
    (18, 3, 4, 2),
    (18, 8, 8, 4),
    (20, 3, 4, 2),
    pytest.param(22, 9, 4, 2, marks=pytest.mark.slow),
]


@pytest.mark.parametrize("log_fri,nregs,ef,checks", MATRIX)
def test_prover_at_scale(eng, log_fri, nregs, ef, checks):
    n = 1 << log_fri
    need_device(eng, log_fri, 9 * (nregs + 1) + 48)
    times = {}
    t0 = time.perf_counter()
    stark, cons, rows, boundary = synthetic(log_fri, log_fri, nregs, ef, checks)
    zpoly, zcw = zerofier(eng, stark)
    times["inputs"] = time.perf_counter() - t0

    t0 = time.perf_counter()
    rec = V.Recorder(eng)
    proof, plan = prove(eng, stark, cons, rows, boundary, zpoly, zcw, log_fri, rec)
    times["prove"] = time.perf_counter() - t0
    assert isinstance(proof, bytes), proof
    assert rec.trees_calls == [(nregs + 1, n, 2)]
    committed = eng.download(rec.committed).view(np.uint64)
    combined = eng.download(rec.combined).view(np.uint64)
    zvals = eng.download(zcw.device_vector()).view(np.uint64)
    assert committed.shape == (nregs + 1, n, 2) and combined.shape == (n, 2) and zvals.shape == (n, 2)

    # 1. the verifier accepts the proof, with the zerofier root computed by the oracle
    t0 = time.perf_counter()
    assert V.verify(stark, proof, cons, fe_boundary(boundary), O.merkle_root_np(zvals))
    times["verify"] = time.perf_counter() - t0

    # 2. the per-index equation with no 256-block unvisited, with the weights the verifier draws
    t0 = time.perf_counter()
    st = V.Statement(stark, cons, boundary)
    w = V.weights(stark, proof, len(cons))
    assert rec.weights == w
    idx = sweep_indices(n, ef, log_fri)
    assert len(idx) >= n // 256 and {i // 256 for i in idx} == set(range(n // 256))
    assert V.failures(st, idx, committed, combined, zvals, w) == []
    times["sweep"] = time.perf_counter() - t0

    # 3. exact degrees: the combination below max_degree + 1, each committed codeword at its own bound
    t0 = time.perf_counter()
    omega = stark.omega.value
    assert not coefficients(omega, combined)[plan.max_degree + 1:].any()
    bounds = stark.boundary_quotient_degree_bounds(plan.trace_length, fe_boundary(boundary)) + [plan.max_degree]
    for s, bound in enumerate(bounds):
        assert top_and_tail(coefficients(omega, committed[s]), bound) == (True, True), (s, bound)
    times["degrees"] = time.perf_counter() - t0

    # 4. the roots in the proof are the oracle's roots of what was committed and folded
    objects = pickle.loads(proof)
    assert objects[:nregs + 1] == [O.merkle_root_np(committed[s]) for s in range(nregs + 1)]
    assert objects[nregs + 1] == O.merkle_root_np(combined)
    print("2^%d, %d registers, expansion %d, %d checks: %s" % (
        log_fri, nregs, ef, checks, ", ".join("%s %.2f s" % kv for kv in times.items())))


@pytest.fixture(scope="module")
def case20(eng):
    stark, cons, rows, boundary = synthetic(20, 20, 3, 4, 2)
    zpoly, zcw = zerofier(eng, stark)
    return stark, cons, rows, boundary, zpoly, zcw


def test_broken_witness_at_2_20_rejected(eng, case20):
    """register 0 off by one at a middle row (not a boundary row): a proof, and the verifier rejects it"""
    need_device(eng, 20, 9 * 4 + 48)
    stark, cons, rows, boundary, zpoly, zcw = case20
    c = len(rows) // 2
    assert all(bc != c for bc, _, _ in boundary)
    broken = [list(r) for r in rows]
    broken[c][0] = (broken[c][0] + 1) % P
    proof, _ = prove(eng, stark, cons, broken, boundary, zpoly, zcw, 7)
    assert isinstance(proof, bytes), proof
    assert V.verify(stark, proof, cons, fe_boundary(boundary), O.merkle_root_np(
        eng.download(zcw.device_vector()).view(np.uint64))) is False


def test_false_boundary_at_2_20_raises(eng, case20):
    need_device(eng, 20, 9 * 4 + 48)
    stark, cons, rows, boundary, zpoly, zcw = case20
    c, r, v = boundary[-1]
    proof, _ = prove(eng, stark, cons, rows, boundary[:-1] + [(c, r, (v + 1) % P)], zpoly, zcw, 8)
    assert isinstance(proof, AssertionError) and str(proof).startswith(sa_stark.REMAINDER), proof
