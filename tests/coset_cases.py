"""Cases of the coset division tests, shared by the CPU emulation (tests/test_emu_coset.py) and the GPU suite
(tests/test_gpu_coset_div.py): one divisor on a random coset of order n = 2^log_n and a batch of numerators, with
what each row must come out as.

Row b of an apply is out[b][j] = U[j] * offset^-j, j < qlen, U = intt(ntt(l * offset^i) / ntt(r * offset^i)) at
order n (`formula`).  On top of that:
  * a clean division l = q * r gives q followed by zeros;
  * a numerator of degree in [n/2, n) gives, on its deg l - deg r + 1 first coefficients, the reference's
    fast_coset_divide(l, r, offset, root, n) (the reference keeps order n there);
  * a zero row gives zeros, two equal rows equal quotients."""
import random

import numpy as np

import oracle as O

P = O.P
KINDS = ["clean", "random", "zero", "random", "copy"]  # row b of a batch of B is KINDS[b] (B <= 5)


def rand_poly(rng, deg):
    """deg + 1 coefficients, the leading one non-zero"""
    return [rng.randrange(P) for _ in range(deg)] + [rng.randrange(1, P)]


def pad(coeffs, n):
    return list(coeffs) + [0] * (n - len(coeffs))


def formula(lhs, rhs, offset, root, n, qlen):
    """the documented row: U[j] * offset^-j for j < qlen"""
    a, b = np.zeros((n, 2), np.uint64), np.zeros((n, 2), np.uint64)
    a[:len(lhs)] = O.scale_np(O.to_np(lhs), offset)
    b[:len(rhs)] = O.scale_np(O.to_np(rhs), offset)
    u = O.intt_np(root, O.pointwise_div_np(O.ntt_np(root, a), O.ntt_np(root, b)))
    return O.from_np(O.scale_np(u, O.inverse(offset)))[:qlen]


class Case:
    """full: ncoef = qlen = n and a divisor of deg r + 1 coefficients; otherwise ncoef = n - 1 (at least 1),
    qlen = n / 2 and a divisor zero-padded to n coefficients"""

    def __init__(self, log_n, batch, full, seed):
        rng = random.Random(seed)
        n = self.n = 1 << log_n
        self.log_n, self.batch = log_n, batch
        self.root = O.primitive_nth_root(n)
        self.offset = rng.randrange(1, P)
        self.ncoef = n if full else max(1, n - 1)
        self.qlen = n if full else max(1, n // 2)
        dr = rng.randrange(0, min(n // 2, self.ncoef - 1) + 1)
        self.divisor = rand_poly(rng, dr)
        if not full:
            self.divisor = pad(self.divisor, n)
        self.rows, self.quotients = [], []
        for b in range(batch):
            kind, q = KINDS[b], None
            if kind == "clean":
                q = rand_poly(rng, rng.randrange(0, self.ncoef - dr))
                row = O.fast_multiply(q, self.divisor[:dr + 1], O.primitive_nth_root(2 * n), 2 * n)
            elif kind == "random":
                lo = min(n // 2, self.ncoef - 1)
                row = rand_poly(rng, rng.randrange(lo, self.ncoef))
            elif kind == "zero":
                row = []
            else:
                row, q = self.rows[0], self.quotients[0]
            self.rows.append(pad(row, self.ncoef))
            self.quotients.append(q)

    def lhs_np(self):
        return np.stack([O.to_np(r) for r in self.rows])

    def check(self, out):
        """out: uint64[batch, qlen, 2]"""
        n, qlen, r = self.n, self.qlen, self.divisor
        dr = O.degree(r)
        for b in range(self.batch):
            got, row = O.from_np(out[b]), self.rows[b]
            assert got == formula(row, r, self.offset, self.root, n, qlen), (self.log_n, b)
            if self.quotients[b] is not None:
                assert got == pad(self.quotients[b], n)[:qlen], (self.log_n, b)
            dl = O.degree(row)
            if dl < 0:
                assert not any(got), (self.log_n, b)
            elif n // 2 <= dl and dr <= dl:
                m = min(qlen, dl - dr + 1)
                want = O.fast_coset_divide(row, r, self.offset, self.root, n)
                assert got[:m] == want[:m], (self.log_n, b)
        if self.batch >= 5:
            assert (out[4] == out[0]).all()
