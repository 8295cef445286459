"""Edge values for the decimal leaf encoding of hash.cuh (plain Python ints, no GPU).

A Merkle leaf is blake2b(str(value).encode()) (merkle.py:13-14, algebra.py:53-57).  The device builds the
decimal string in `fe_decimal_words`: a long division into base-1e8 limbs whose quotient words come from an
FP64 estimate repaired by one compare (`dec_div_1e8`), a digit count from the top non-zero limb, and a shift
that drops the leading zero bytes in three conditional word stages and one byte stage.  Uniform field
elements are almost all 38 or 39 digits long and sit nowhere near the division's rounding boundaries, so
this module builds the values on purpose, in named classes:

* lengths: for every digit count L = 1..39, 10^(L-1), 10^(L-1) + 1, 10^L - 1, 10^L - 2 and random values
  of exactly L digits (every byte shift of the output, and every digit-count threshold of the top limb);
* limbs: c0 + c1 1e8 + c2 1e16 + c3 1e24 + c4 1e32 with every limb in {0, 1, 1e8 - 1} and random limbs
  (zero limbs inside a value and every top-limb choice);
* div: values whose long division meets a chosen partial dividend cur = q 1e8 + r at each of the nine
  estimated positions (stage k, word i), with r in {1e8 - 1, 0, 1} and q at its largest reachable value,
  2^31 and 1.  r = 1e8 - 1 puts the estimate closest to q + 1, r = 0 makes it q - 1 so the repair runs;
* words: 2^32j - 1, 2^32j, 2^32j + 1, p - 1, p - 2, 0, 1 and the fixed values of test_emu.py.

`division_visits` restates the division schedule on Python ints; `build()` uses it to assert that every
class, and every (position, flavour) at the largest q, holds at least MIN_PER_CLASS values.  Expected
digests come from `str(v).encode()` and hashlib only (`leaf`, `tree`).
"""
import hashlib
import random
from collections import Counter

P = 1 + 407 * (1 << 119)
E8 = 10**8
M32 = (1 << 32) - 1
MIN_PER_CLASS = 8
K_EST = 9.999999999999e-9  # dec_div_1e8's 1e-8 (1 - 1e-13)

# (stage k, word i) of every estimated quotient word, in the order the device visits them
DIV_POSITIONS = [(0, 2), (0, 1), (0, 0), (1, 2), (1, 1), (1, 0), (2, 1), (2, 0), (3, 0)]
FLAVOURS = {"r=1e8-1": E8 - 1, "r=0": 0, "r=1": 1}


def _top_word(k):
    return 3 if k <= 1 else (2 if k == 2 else 1)


def division_visits(v):
    """[(k, i, cur)]: the partial dividends cur = rem * 2^32 + word that fe_decimal_words hands to
    dec_div_1e8 for value v, stage by stage (word `top` of each stage is an exact division)"""
    q = [(v >> (32 * j)) & M32 for j in range(4)]
    out = []
    for k in range(4):
        top = _top_word(k)
        rem = q[top] % E8
        q[top] //= E8
        for i in range(top - 1, -1, -1):
            cur = (rem << 32) | q[i]
            out.append((k, i, cur))
            q[i], rem = divmod(cur, E8)
    return out


def estimate(cur, k_est=K_EST):
    """dec_div_1e8's quotient estimate, on IEEE doubles exactly as the device rounds them"""
    return int(float(cur) * k_est)


def qmax(k, i, r):
    """the largest q with a value v < p whose division meets cur = q 1e8 + r at (k, i)"""
    qk_max = (P - 1) // E8**k
    return min(M32, ((qk_max >> (32 * i)) - r) // E8)


def _div_value(k, i, cur, rng, extreme=None):
    """a value v < p whose division meets cur at (k, i): Q_k = M 1e8 2^(32(i+1)) + cur 2^(32i) + low and
    v = Q_k 1e8^k + c.  extreme = 'min' / 'max' takes M, low and c at their ends instead of at random."""
    qk_max = (P - 1) // E8**k
    base = cur << (32 * i)
    step = E8 << (32 * (i + 1))
    m_hi = (qk_max - base) // step
    pick = {"min": lambda hi: 0, "max": lambda hi: hi}.get(extreme, lambda hi: rng.randint(0, hi))
    m = pick(m_hi)
    qk = m * step + base
    qk += pick(min((1 << (32 * i)) - 1, qk_max - qk))
    c_hi = min(E8**k - 1, P - 1 - qk * E8**k)
    return qk * E8**k + pick(c_hi)


def lengths(rng):
    out = []
    for L in range(1, 40):
        lo, hi = 10**(L - 1) if L > 1 else 0, 10**L - 1
        out += [10**(L - 1), 10**(L - 1) + 1, 10**L - 1, 10**L - 2]
        out += [rng.randint(lo, min(hi, P - 1)) for _ in range(MIN_PER_CLASS)]
    return [v for v in out if 0 <= v < P]


def limb_patterns(rng):
    edge = [0, 1, E8 - 1]
    out = []
    for c0 in edge:
        for c1 in edge:
            for c2 in edge:
                for c3 in edge:
                    for c4 in edge:
                        out.append(c0 + c1 * E8 + c2 * E8**2 + c3 * E8**3 + c4 * E8**4)
    for _ in range(256):  # random limbs, each one of 0, 1, 1e8 - 1 or random, the top limb below p's
        limbs = [rng.choice(edge + [rng.randrange(E8)]) for _ in range(4)]
        limbs.append(rng.choice([0, 1, rng.randrange(P // E8**4 + 1)]))
        out.append(sum(c * E8**j for j, c in enumerate(limbs)))
    return [v for v in out if v < P]


def division_boundaries(rng):
    out = []
    for k, i in DIV_POSITIONS:
        for r in FLAVOURS.values():
            for q in sorted({qmax(k, i, r), 1 << 31, 1}):
                if q > qmax(k, i, r):
                    continue
                cur = q * E8 + r
                vals = [_div_value(k, i, cur, rng, "min"), _div_value(k, i, cur, rng, "max")]
                vals += [_div_value(k, i, cur, rng) for _ in range(MIN_PER_CLASS)]
                for v in vals:
                    assert v < P and (k, i, cur) in division_visits(v), (k, i, q, r, v)
                out += vals
    return out


def word_edges():
    out = [0, 1, P - 1, P - 2]
    for j in range(1, 4):
        out += [(1 << (32 * j)) - 1, 1 << (32 * j), (1 << (32 * j)) + 1]
    # the fixed values of test_emu.py::test_decimal_and_leaf
    out += [0, 1, 9, 10, 99, 100, 10**9 - 1, 10**9, 10**18, 10**19 - 1, 10**19, 10**27, 10**36, 10**38 - 1,
            10**38, 2**64 - 1, 2**64, 2**96 - 1, 2**96, 2**127, 10**9 * (2**32 - 1), (10**9 - 1) * 10**27 + 5,
            340 * 10**36]
    out += [m * E8 * 2**(32 * j) + off for m in (1, 2**32 - 1, E8 - 1) for j in (0, 1, 2) for off in (-1, 0, 1)]
    return [v for v in out if 0 <= v < P]


def classify(classes):
    """class counts of the corpus: the named classes' sizes and, from the division schedule, how many values
    meet each (position, flavour) at all and at the largest reachable q ("div:k,i:flavour:qmax"); also the
    largest q met at each position in each flavour, and the count of estimates the division must repair
    ("repair") and of those a plain 1e-8 factor would round up to q + 1 ("k=1e-8:q+1")"""
    c = Counter()
    top_q = {}
    for name, vals in classes.items():
        c[name] = len(vals)
    for v in sorted(set(x for vals in classes.values() for x in vals)):
        for k, i, cur in division_visits(v):
            q, r = divmod(cur, E8)
            d = estimate(cur)
            assert d in (q, q - 1), (v, k, i, cur, d)  # the rounding argument of dec_div_1e8's comment
            c["repair"] += d == q - 1
            c["k=1e-8:q+1"] += estimate(cur, 1e-8) > q
            for fname, fr in FLAVOURS.items():
                if r == fr:
                    key = "div:%d,%d:%s" % (k, i, fname)
                    c[key] += 1
                    top_q[key] = max(top_q.get(key, 0), q)
                    if q == qmax(k, i, fr):
                        c[key + ":qmax"] += 1
    return c, top_q


def _check_coverage(classes):
    c, top_q = classify(classes)
    for name in classes:
        assert c[name] >= MIN_PER_CLASS, (name, c[name])
    for k, i in DIV_POSITIONS:
        for fname, fr in FLAVOURS.items():
            key = "div:%d,%d:%s" % (k, i, fname)
            assert c[key + ":qmax"] >= MIN_PER_CLASS, (key, c[key + ":qmax"])
            assert top_q[key] == qmax(k, i, fr), (key, top_q[key])
    lens = Counter(len(str(v)) for vals in classes.values() for v in vals)
    for L in range(1, 40):
        assert lens[L] >= MIN_PER_CLASS, ("digits", L, lens[L])
    assert c["repair"] >= MIN_PER_CLASS and c["k=1e-8:q+1"] >= MIN_PER_CLASS, c
    return c, top_q


def build(seed=2025):
    """(values, class_counts, top_q): the sorted, de-duplicated corpus in [0, p), the class counts of
    `classify`, and the largest q met at each division position and flavour; the same seed gives the same
    corpus"""
    rng = random.Random(seed)
    classes = {"lengths": lengths(rng), "limbs": limb_patterns(rng), "div": division_boundaries(rng),
               "words": word_edges()}
    counts, top_q = _check_coverage(classes)
    values = sorted(set(v for vals in classes.values() for v in vals))
    assert all(0 <= v < P for v in values)
    return values, counts, top_q


def leaf(v):
    return hashlib.blake2b(str(v).encode()).digest()


def node(left, right):
    return hashlib.blake2b(left + right).digest()


def tree(values):
    """heap-ordered Merkle tree of `values` with hashlib only: list of 2n digests, node 1 the root, node
    n + i leaf i, node i = blake2b(node 2i || node 2i+1); node 0 is 64 zero bytes (the device zeroes it)"""
    n = len(values)
    assert n and n & (n - 1) == 0
    t = [bytes(64)] * n + [leaf(v) for v in values]
    for i in range(n - 1, 0, -1):
        t[i] = node(t[2 * i], t[2 * i + 1])
    return t


def climb(v, index, path):
    """the root an authentication path (siblings bottom-up) leads to from the leaf of value v at index"""
    acc = leaf(v)
    for sib in path:
        acc = node(sib, acc) if index & 1 else node(acc, sib)
        index >>= 1
    return acc


def tile(values, n, seed):
    """n values: the corpus repeated, each copy in its own seeded permutation, cut to n"""
    rng = random.Random(seed)
    out = []
    while len(out) < n:
        block = list(values)
        rng.shuffle(block)
        out += block
    return out[:n]


def fold_preimage(target, alpha, offset, omega, rng=None):
    """a codeword of length 2 len(target) whose split-and-fold (fri.py:85) with alpha, offset and omega is
    exactly `target`: random a_i, and b_i = (2 c_i - (1 + t_i) a_i) / (1 - t_i) with t_i = alpha / (offset
    omega^i).  The inverses are one batch inversion on Python ints."""
    rng = rng or random.Random(len(target))
    h = len(target)
    xs = [0] * h
    x = offset
    for i in range(h):
        xs[i] = x
        x = x * omega % P
    inv_x = _batch_inverse(xs)
    t = [alpha * ix % P for ix in inv_x]
    assert all(ti != 1 for ti in t), "alpha is a point of the domain"
    den_inv = _batch_inverse([(1 - ti) % P for ti in t])
    a = [rng.randrange(P) for _ in range(h)]
    b = [(2 * c - (1 + ti) * ai) * di % P for c, ti, ai, di in zip(target, t, a, den_inv)]
    return a + b


def _batch_inverse(xs):
    """Montgomery's trick: every x^-1 from one Fermat inversion (no x may be 0)"""
    pre = [1] * (len(xs) + 1)
    acc = 1
    for i, x in enumerate(xs):
        assert x % P
        acc = acc * x % P
        pre[i + 1] = acc
    inv = pow(acc, P - 2, P)
    out = [0] * len(xs)
    for i in range(len(xs) - 1, -1, -1):
        out[i] = inv * pre[i] % P
        inv = inv * xs[i] % P
    return out


def fold(cw, alpha, offset, omega):
    """fri.py:85 on Python ints (small codewords; the tests use it to check fold_preimage)"""
    h = len(cw) // 2
    out = []
    x = offset
    two_inv = (P + 1) // 2
    for i in range(h):
        t = alpha * pow(x, P - 2, P) % P
        out.append(((1 + t) * cw[i] + (1 - t) * cw[h + i]) * two_inv % P)
        x = x * omega % P
    return out
