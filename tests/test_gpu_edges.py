"""GPU tests at the places random parity campaigns do not reach (run on the H100: ``pytest -m gpu``):

* the device field (field.cuh's PTX carry chains) on the boundary operands of tests/field_edges.py;
* every grid-stride kernel past the end of its first sweep (grid_for caps the grid at per_sm x SMs
  blocks, so larger inputs make each thread loop), sizes derived from this device's SM count;
* the three-pass NTT plan shapes (log_n 23..26) and batches of three-pass transforms in one call;
* the subproduct tree at its largest size (2^20 points) and one point past it.

Every result is compared bit for bit with the CPU oracle, with Python ints, or (where the oracle cannot
reach) through exact algebraic properties."""
import math
import os
import random
import sys

import numpy as np
import pytest

import field_edges as FE
import oracle as O

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "stark-anatomy_b200")
if PKG not in sys.path:
    sys.path.insert(0, PKG)
import sa_engine  # noqa: E402

pytestmark = pytest.mark.gpu
P = O.P
RINV = pow(1 << 128, -1, P)


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


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def vectors():
    return FE.build()


def rand_np(seed, n):
    rng = np.random.default_rng(seed)
    lo = rng.integers(0, 1 << 64, size=n, dtype=np.uint64)
    hi = rng.integers(0, 0xCB80000000000000, size=n, dtype=np.uint64)  # < p's top limb => < p
    return np.stack([lo, hi], axis=1)


def up(eng, arr):
    return eng.upload(np.ascontiguousarray(arr).view(np.int64))


def down(eng, vec):
    return eng.download(vec).view(np.uint64)


def past_wrap(per_sweep):
    """two and a half sweeps plus a ragged tail"""
    return 2 * per_sweep + per_sweep // 2 + 37


# ---- the device field on its carry boundaries ------------------------------------------------------------
def test_device_add_sub_on_boundaries(eng, vectors):
    """a 2-point transform with root p - 1 is (x0 + x1, x0 - x1) (fe_add / fe_sub, no twiddle); its inverse
    halves both.  One operand pair per batch item, both orders."""
    muls, addsubs, _, _ = vectors
    pairs = [(a, b) for a, b, _ in addsubs + muls]
    pairs += [(b, a) for a, b in pairs]
    x = O.to_np([v for ab in pairs for v in ab])
    vx = up(eng, x)
    fwd = O.from_np(down(eng, eng.ntt(vx, 1, P - 1, batch=len(pairs))))
    inv = O.from_np(down(eng, eng.ntt(vx, 1, P - 1, inverse=True, batch=len(pairs))))
    half = (P + 1) // 2
    for i, (a, b) in enumerate(pairs):
        assert fwd[2 * i] == (a + b) % P and fwd[2 * i + 1] == (a - b) % P, (a, b)
        assert inv[2 * i] == (a + b) * half % P and inv[2 * i + 1] == (a - b) * half % P, (a, b)


def test_device_product_on_boundaries(eng, vectors):
    """sa_pointwise_mul computes montmul(to_mont(a), b); with a = A * 2^-128 the second product sees exactly
    the chosen operands (A, B), whose low 128 bits drive the reduction's borrow and add-back"""
    muls = vectors[0]
    a = [A * RINV % P for A, _, _ in muls] + [A for A, _, _ in muls]
    b = [B for _, B, _ in muls] * 2
    got = O.from_np(down(eng, eng.pointwise_mul(up(eng, O.to_np(a)), up(eng, O.to_np(b)))))
    tags = [t for _, _, t in muls] * 2
    for u, v, g, t in zip(a, b, got, tags):
        assert g == u * v % P, t


def plan_sections(plan, n):
    """the offset^i, 1/R_i and offset^-i sections of a coset division plan of n >= 16 elements (Montgomery form)"""
    raw = plan.plan.cpu().numpy().view(np.uint64).reshape(3, n, 2)
    return raw[0], raw[1], raw[2]


def mont(x):
    """the Montgomery form x * 2^128 mod p of uint64[n, 2]"""
    return O.pointwise_mul_np(np.ascontiguousarray(x), np.tile(O._fe((1 << 128) % P), (x.shape[0], 1)))


def test_batch_inverse_on_boundaries(eng, vectors):
    """k_batch_inverse through a coset division plan of order 128 and offset 1 whose divisor is the inverse transform
    of the chosen values, so R_i are those values: one CTA, one divisor per thread's batch inversion, so each entry
    of the plan's 1/R_i section is one fe_mont_inv of a chosen value"""
    muls, _, invs, _ = vectors
    divisors = invs + [b for _, b, _ in muls[::8] if b]
    n = 128
    root = O.primitive_nth_root(n)
    for lo in range(0, len(divisors), n):
        chunk = divisors[lo:lo + n]
        values = chunk + [1] * (n - len(chunk))
        plan = eng.coset_div_plan(up(eng, O.to_np(O.intt(root, values))), 7, root, 1)
        inv = O.from_np(plan_sections(plan, n)[1])
        assert [v * RINV % P for v in inv[:len(chunk)]] == [pow(v, P - 2, P) for v in chunk]


# ---- grid-stride kernels past their first sweep ----------------------------------------------------------
def _element_of_order_dividing(T):
    """an element h != 1 with h^T == 1 (order gcd(T, p - 1); p - 1 = 11 * 37 * 2^119)"""
    g = math.gcd(T, P - 1)
    primes = [q for q in (2, 11, 37) if g % q == 0]
    for c in range(2, 1000):
        h = pow(c, (P - 1) // g, P)
        if all(pow(h, g // q, P) != 1 for q in primes):
            assert pow(h, T, P) == 1 and h != 1
            return h
    raise AssertionError("no element of order %d" % g)


def test_coset_powers_past_wrap(eng, sms):
    """k_coset_load loops past its 8 * SMs * 256 threads: the plan's offset^i and offset^-i
    tables (k_pow_table) equal the oracle's powers, and an evaluation row equals the oracle's fast_coset_evaluate,
    for offsets 0, 1, p - 1, a random one and one whose powers repeat with the load's sweep T"""
    T = 8 * sms * 256
    log_n = T.bit_length()
    n = 1 << log_n
    root = O.primitive_nth_root(n)
    x = rand_np(8100, n)
    x[T] = O._fe(P - 1)
    vx = up(eng, x)
    ones = O.to_np([1] * n)
    rng = random.Random(8101)
    for f in (0, 1, P - 1, rng.randrange(2, P), _element_of_order_dividing(T)):
        pw, _, ipw = plan_sections(eng.coset_div_plan(up(eng, O.to_np([1])), log_n, root, f), n)
        assert (pw == mont(O.scale_np(ones, f))).all(), f
        assert (ipw == mont(O.scale_np(ones, O.inverse(f)))).all(), f
        got = O.from_np(down(eng, eng.coset_evaluate(vx, log_n, root, f)))
        assert got == O.fast_coset_evaluate(O.from_np(x), f, root, n), f


def test_pointwise_mul_past_wrap(eng, sms):
    n = past_wrap(16 * sms * 256)
    a, b = rand_np(8200, n), rand_np(8201, n)
    a[n - 1], b[n - 2] = O._fe(P - 1), O._fe(P - 1)
    assert (down(eng, eng.pointwise_mul(up(eng, a), up(eng, b))) == O.pointwise_mul_np(a, b)).all()


def test_batch_inverse_past_wrap(eng, sms):
    """k_batch_inverse: one sweep is 16 * SMs CTAs of 128 threads, each inverting
    8 strided elements at once.  A coset plan just past one sweep holds 1/R_i with inv_i * R_i == 2^128 at every i
    (R from an evaluation of the divisor); a divisor vanishing at one coset point in the second sweep or in the
    last 8 must be reported."""
    import torch
    S = 16 * sms * 128 * 8
    log_n = S.bit_length()
    n = 1 << log_n
    root, offset = O.primitive_nth_root(n), random.Random(8300).randrange(2, P)
    divisor = up(eng, rand_np(8301, n))
    inv = eng.coset_div_plan(divisor, log_n, root, offset).plan.view(torch.int64).reshape(3, n, 2)[1]
    R = eng.coset_evaluate(divisor, log_n, root, offset)
    assert (down(eng, eng.pointwise_mul(inv, R)) == O._fe((1 << 128) % P)).all()
    for z in (S + 12345, n - 5):  # second sweep, last group of 8
        vanishing = up(eng, O.to_np([P - offset * pow(root, z, P) % P, 1]))
        with pytest.raises(AssertionError, match="divide by zero"):
            eng.coset_div_plan(vanishing, log_n, root, offset)


@pytest.mark.parametrize("log_n", [20, 21])
def test_fri_fold_and_round_past_wrap(eng, sms, log_n):
    """k_fri_fold loops past 16 * SMs * 128 pairs; the fused round (fold + Merkle tree) at the same size.
    Offset and omega are not the defaults (a random offset, an odd power of the primitive root)."""
    n = 1 << log_n
    assert n // 2 > 16 * sms * 128
    rng = random.Random(8400 + log_n)
    x = rand_np(8400 + log_n, n)
    alpha, off = rng.randrange(P), rng.randrange(2, P)
    omega = pow(O.primitive_nth_root(n), 2 * rng.randrange(n // 2) + 1, P)
    want = O.fri_fold_np(x, alpha, off, omega)
    vx = up(eng, x)
    assert (down(eng, eng.fri_fold(vx, alpha, off, omega)) == want).all()
    nxt, tree = eng.fri_round(vx, alpha, off, omega)
    assert (down(eng, nxt) == want).all()
    assert (tree.cpu().numpy()[1:] == O.merkle_tree_np(want)[1:]).all()


# ---- three-pass NTT shapes -------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n", [23, 24, pytest.param(25, marks=pytest.mark.slow),
                                   pytest.param(26, marks=pytest.mark.slow)])
def test_ntt_three_pass_shapes_match_oracle(eng, log_n):
    """(l1, l2, l3) = (8, 8, 7), (8, 8, 8), (9, 8, 8), (9, 9, 8): forward and inverse against the oracle"""
    n = 1 << log_n
    w = pow(O.primitive_nth_root(n), 2 * random.Random(log_n).randrange(n // 2) + 1, P)
    x = rand_np(8500 + log_n, n)
    vx = up(eng, x)
    got = down(eng, eng.ntt(vx, log_n, w))
    assert (got == O.ntt_np(w, x, parallel=True)).all()
    got = down(eng, eng.ntt(vx, log_n, w, inverse=True))
    assert (got == O.intt_np(w, x, parallel=True)).all()


@pytest.mark.parametrize("log_n,batch", [(21, 3), (22, 2), (23, 2)])
def test_ntt_three_pass_batched_matches_oracle(eng, log_n, batch):
    """several three-pass transforms in one sa_ntt call (pass 3 addresses batch item b at (b / n2) * n);
    forward against the oracle, the batched inverse back to the input, and an in-place call"""
    n = 1 << log_n
    w = O.primitive_nth_root(n)
    x = rand_np(8600 + log_n, n * batch)
    want = O.ntt_batch_np(w, x.reshape(batch, n, 2)).reshape(-1, 2)
    vx = up(eng, x)
    y = eng.ntt(vx, log_n, w, batch=batch)
    assert (down(eng, y) == want).all()
    assert bool((eng.ntt(y, log_n, w, inverse=True, batch=batch) == vx).all())
    if log_n == 22:
        assert eng.lib.sa_ntt(vx.data_ptr(), vx.data_ptr(), log_n, sa_engine._limbs(w), 0, batch, eng._stream()) == 0
        assert (down(eng, vx) == want).all()


# ---- the subproduct tree at its limit (TREE_MAX_LOG = 20) ------------------------------------------------
def test_zerofier_2_20_by_property(eng):
    """monic, vanishes on a sample of the domain, equals the product of the two halves' zerofiers"""
    k = 1 << 20
    vd = up(eng, rand_np(8700, k))
    z = eng.zerofier(vd)
    zh = down(eng, z)
    assert zh.shape[0] == k + 1 and (zh[k] == np.array([1, 0], dtype=np.uint64)).all()
    assert (down(eng, eng.poly_eval(z, vd[::257].contiguous(), mode=1)) == 0).all()
    zl, zr = eng.zerofier(vd[:k // 2].contiguous()), eng.zerofier(vd[k // 2:].contiguous())
    log_n = 21  # > deg(zl * zr) = 2^20
    n = 1 << log_n
    w = O.primitive_nth_root(n)
    prod = eng.ntt(eng.pointwise_mul(eng.ntt(eng.pad(zl, n), log_n, w), eng.ntt(eng.pad(zr, n), log_n, w)), log_n, w,
                   inverse=True)
    ph = down(eng, prod)
    assert (ph[:k + 1] == zh).all() and (ph[k + 1:] == 0).all()


def test_poly_eval_tree_walk_2_20(eng):
    """mode 2 at 2^20 points and coefficients (its Newton step runs batched three-pass transforms): equal to
    Horner on a sample of the points and to the oracle on a few"""
    k = 1 << 20
    coeffs, pts = rand_np(8800, k), rand_np(8801, k)
    vc, vp = up(eng, coeffs), up(eng, pts)
    got = down(eng, eng.poly_eval(vc, vp, mode=2))
    step = 257
    assert (got[::step] == down(eng, eng.poly_eval(vc, vp[::step].contiguous(), mode=1))).all()
    few = [0, 1, k // 2, k - 1]
    assert (got[few] == O.poly_eval_np(coeffs, pts[few])).all()


def test_tree_one_past_the_limit(eng):
    """2^20 + 1 points: the tree entry points report "unsupported size", mode 0 falls back to Horner"""
    k = (1 << 20) + 1
    dom, vals = rand_np(8900, k), rand_np(8901, k)
    vd = up(eng, dom)
    with pytest.raises(AssertionError, match="unsupported size"):
        eng.zerofier(vd)
    with pytest.raises(AssertionError, match="unsupported size"):
        eng.interpolate(vd, up(eng, vals))
    coeffs = rand_np(8902, 1024)  # 2^30 coefficient-point products: the walk's range, were the tree big enough
    vc = up(eng, coeffs)
    with pytest.raises(AssertionError, match="unsupported size"):
        eng.poly_eval(vc, vd, mode=2)
    got = down(eng, eng.poly_eval(vc, vd))
    rng = random.Random(8903)
    idx = sorted({0, 1, k // 2, k - 2, k - 1} | {rng.randrange(k) for _ in range(59)})
    assert (got[idx] == O.poly_eval_np(coeffs, dom[idx])).all()
    # as many coefficients past the limit, few points
    pts = dom[:512]
    got = down(eng, eng.poly_eval(vd, up(eng, pts)))
    assert (got[:8] == O.poly_eval_np(dom, pts[:8])).all()
